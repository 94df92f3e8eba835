"""GPU: SegDetectorRepresenter end to end on the device (megreader_b200/db_boxes.boxes_from_maps, .SegDetectorRepresenter) against
the oracle's restatement of the reference (oracle/db_boxes_port.py: cv2 for contours, boxes, fill and mean, the unpinned Clipper
offset restatement for the unclip), at the yaml's validation shape and odd sizes, max_candidates 100 and 1000, dest =
'thresh_binary', resize = True with a destination size other than the map's, boxes whose unclip leaves the image; the
reference's return structure; graph capture; and the seg_detector_db model in eval mode plus boxes in one CUDA graph."""
import numpy as np
import pytest
import torch

from tests.db_boxes_cases import prob_maps

pytestmark = pytest.mark.gpu

cv2 = pytest.importorskip("cv2")


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs CUDA")
    return torch.device("cuda:0")


def _oracle(binary, dest, thresh, box_thresh, maxc, sizes=None):
    from oracle.db_boxes_port import SegDetectorRepresenter
    rep = SegDetectorRepresenter(thresh, box_thresh, maxc, resize=sizes is not None)
    N, H, W = binary.shape[0], binary.shape[-2], binary.shape[-1]
    out = []
    for n in range(N):
        h, w = sizes[n] if sizes is not None else (H, W)
        out.append(rep.boxes_from_bitmap(torch.from_numpy(binary[n]), torch.from_numpy(dest[n] > thresh), w, h))
    return out


def _edge_maps(seed, N, H, W):
    """text-like blobs cut by the frame: their unclipped boxes leave the image"""
    rng = np.random.RandomState(seed)
    m = np.full((N, 1, H, W), 0.05, np.float32)
    for n in range(N):
        for _ in range(12):
            y, x = rng.randint(0, H), rng.choice([rng.randint(0, 8), rng.randint(W - 8, W), rng.randint(0, W)])
            h, w = rng.randint(4, 30), rng.randint(10, 120)
            m[n, 0, max(0, y - h // 2):y + h // 2, max(0, x - w // 2):x + w // 2] = rng.uniform(0.75, 1.0)
    return m


def _compare(got, want, n_images, scale=1.0):
    """boxes identical; the calipers' tie class (DESIGN §7) may move a box by one map pixel (scale destination pixels), on
    at most 1 % of the boxes (at least one)"""
    boxes, scores, count = (t.cpu().numpy() for t in got)
    assert count.tolist() == [len(w) for w in want]
    off, total = 0, 0
    for n in range(n_images):
        for c, wb in enumerate(want[n]):
            d = np.abs(boxes[n, c].astype(np.float64) - np.array(wb)).max()
            assert d <= np.ceil(scale), (n, c, boxes[n, c].tolist(), wb)
            off += d > 0
            total += 1
        assert not boxes[n, count[n]:].any() and not scores[n, count[n]:].any()
    assert off <= max(1, 0.01 * total), (off, total)
    return total


CASES = [  # (name, maps, thresh, box_thresh, max_candidates)
    ("val_4x576x1024_c1000", lambda: prob_maps(11, 4, 576, 1024), 0.3, 0.7, 1000),
    ("val_4x576x1024_c100", lambda: prob_maps(11, 4, 576, 1024), 0.3, 0.7, 100),
    ("clean_4x576x1024", lambda: prob_maps(15, 4, 576, 1024, 0.7), 0.3, 0.7, 1000),
    ("odd_1x577x1023", lambda: prob_maps(16, 1, 577, 1023, 0.7), 0.3, 0.6, 100),
    ("odd_3x33x47", lambda: prob_maps(13, 3, 33, 47, 0.5), 0.3, 0.5, 1000),
    ("edges_2x200x300", lambda: _edge_maps(3, 2, 200, 300), 0.3, 0.7, 1000),
]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_boxes_from_maps_equal_oracle(case):
    from megreader_b200 import db_boxes
    _, make, thresh, box_thresh, maxc = case
    maps = make()
    got = db_boxes.boxes_from_maps(torch.from_numpy(maps).to(_dev()), None, thresh, box_thresh, maxc)
    n_boxes = _compare(got, _oracle(maps, maps, thresh, box_thresh, maxc), len(maps))
    # the noisy maps' first 100 contours (in cv2's order) are all specks: the reference finds no box there, nor does the device
    assert n_boxes == 0 if case[0] == "val_4x576x1024_c100" else n_boxes > 0


def test_unclip_leaves_the_image_and_clips():
    from megreader_b200 import db_boxes
    maps = _edge_maps(3, 2, 200, 300)
    boxes, _, count = db_boxes.boxes_from_maps(torch.from_numpy(maps).to(_dev()), None, 0.3, 0.7, 1000)
    b = np.concatenate([boxes[n, :count[n]].cpu().numpy() for n in range(2)])
    assert ((b[..., 0] == 0) | (b[..., 0] == 300)).any() and b.min() >= 0 and b[..., 0].max() <= 300 and b[..., 1].max() <= 200


def test_dest_thresh_binary_and_resize():
    """the bitmap from another map than the score (dest='thresh_binary'); resize=True to a destination size other than the map's"""
    from megreader_b200 import db_boxes
    binary = prob_maps(15, 3, 320, 480, 0.7)
    tb = np.clip(binary * np.float32(1.1) - np.float32(0.05), 0, 1).astype(np.float32)
    sizes = [(640, 960), (300, 500), (321, 479)]
    dev = _dev()
    got = db_boxes.boxes_from_maps(torch.from_numpy(binary).to(dev), torch.from_numpy(tb).to(dev), 0.3, 0.7, 1000,
                                   torch.tensor(sizes))
    assert _compare(got, _oracle(binary, tb, 0.3, 0.7, 1000, sizes), 3, scale=2.0) > 0
    rep = db_boxes.SegDetectorRepresenter(resize=True, dest='thresh_binary', max_candidates=1000)
    pred = {'binary': torch.from_numpy(binary).to(dev), 'thresh_binary': torch.from_numpy(tb).to(dev)}
    boxes_batch, out_pred = rep.represent({'image': torch.zeros(3, 3, 8, 8), 'shape': sizes}, pred)
    want = _oracle(binary, tb, 0.3, 0.7, 1000, sizes)
    assert out_pred is pred and len(boxes_batch) == 3
    for g, w in zip(boxes_batch, want):                 # the reference's structure: lists of [[x, y]] * 4 floats
        assert isinstance(g, list) and all(isinstance(v, float) for b in g for p in b for v in p)
        assert len(g) == len(w) and np.abs(np.array(g) - np.array(w)).max(initial=0) <= 2


def test_represent_structure_equals_oracle():
    from megreader_b200 import db_boxes
    from oracle.db_boxes_port import SegDetectorRepresenter as Oracle
    binary = prob_maps(15, 2, 288, 512, 0.7)
    x = torch.from_numpy(binary)
    batch = {'image': torch.zeros(2, 3, 288, 512), 'shape': [(288, 512), (288, 512)]}
    got, _ = db_boxes.SegDetectorRepresenter().represent(batch, {'binary': x.to(_dev())})
    want, _ = Oracle().represent(batch, {'binary': x})
    assert got == want


def test_boxes_graph_capture():
    from megreader_b200 import db_boxes
    dev = _dev()
    a = torch.from_numpy(prob_maps(15, 4, 576, 1024, 0.7)).to(dev)
    b = torch.flip(a, dims=(0, 3)).contiguous()
    eb = db_boxes.boxes_from_maps(b, None, 0.3, 0.7, 1000)
    static = a.clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        db_boxes.boxes_from_maps(static, None, 0.3, 0.7, 1000)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = db_boxes.boxes_from_maps(static, None, 0.3, 0.7, 1000)
    static.copy_(b)
    g.replay()
    torch.cuda.synchronize()
    assert all(torch.equal(u, v) for u, v in zip(out, eb)) and int(eb[2].sum()) > 0


def test_seg_detector_db_eval_and_boxes_in_one_graph():
    """seg_detector_db.yaml's model (deformable ResNet50 + SegDetector) in eval mode on the engine convolutions, then the boxes:
    one CUDA graph, replayed on a second batch, equal to the eager run"""
    import bench_trunks
    from megreader_b200 import db_boxes
    dev = _dev()
    torch.manual_seed(0)
    net, n = bench_trunks.build(6, dev, engine=True)
    assert n > 60
    net.eval()
    x1, _ = bench_trunks.synth_db(2, 2, (256, 256))
    x2, _ = bench_trunks.synth_db(3, 2, (256, 256))
    x1, x2 = x1.to(dev), x2.to(dev)

    def step(x):
        binary = net.decoder(net.backbone(x))
        binary = binary['binary'] if isinstance(binary, dict) else binary
        return db_boxes.boxes_from_maps(binary.float(), None, 0.3, 0.5, 100)
    with torch.no_grad():
        eager = step(x2)
        static = x1.clone()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            step(static)
        torch.cuda.current_stream().wait_stream(s)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            out = step(static)
        static.copy_(x2)
        g.replay()
        torch.cuda.synchronize()
    assert all(torch.equal(u, v) for u, v in zip(out, eager))
