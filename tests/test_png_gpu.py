"""GPU: mr_png_decode and mr_image_decode (csrc/png.cu) against cv2.imdecode(buf, cv2.IMREAD_COLOR), bit for bit: the PNG
corpus as one batch (broken files flagged with shape (0, 0), their neighbours exact), a mixed JPEG / PNG batch (every JPEG
also equal to mr_jpeg_decode's result for it alone), IIIT-like line batches and 1280 x 720 scenes, the capacities with
sentinel tails, graph capture and replay, and the chains into resize_normalize_packed and train_batch_packed."""
import numpy as np
import pytest
import torch

from tests import jpeg_cases as J
from tests import png_cases as C

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")


def _cv2(blob):
    return cv2.imdecode(np.frombuffer(blob, np.uint8), cv2.IMREAD_COLOR)


def _pixels(b):
    from megreader_b200 import jpeg, png
    return png.header_pixels(b) or jpeg._header_pixels(b)


def _check(blobs, res, flag=()):
    shapes, offs = res["shapes"].cpu().numpy(), res["image_offsets"].cpu().numpy()
    status, buf = res["status"].cpu().numpy(), res["buffer"].cpu().numpy()
    for i, b in enumerate(blobs):
        if i in flag:
            assert status[i] != 0 and tuple(shapes[i]) == (0, 0), i
            continue
        ref = _cv2(b)
        assert status[i] == 0, (i, status[i])
        h, w = shapes[i]
        got = buf[offs[i]:offs[i] + h * w * 3].reshape(h, w, 3)
        assert got.shape == ref.shape and np.array_equal(got, ref), i
    return status


def _decode(mod, blobs, cap=None, max_side=16384):
    from megreader_b200 import jpeg
    data, offs = jpeg.pack_bytes(blobs)
    cap = cap if cap is not None else sum(map(_pixels, blobs))
    return mod.decode_packed(data, offs, max_side, max_side, cap)


def lines(seed, n, pil=False):
    """IIIT-like word crops: RGB, 30-150 high, 100-600 wide, at cv2's default level or PIL's"""
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n):
        h, w = int(rng.integers(30, 151)), int(rng.integers(100, 601))
        img = J.image(rng, h, w)
        cv2.putText(img, "WORD", (5, h - 8), cv2.FONT_HERSHEY_SIMPLEX, h / 40, (20, 20, 20), 2)
        out.append(C.pil_encode(img[:, :, ::-1].copy(), "RGB") if (pil and i % 2) else C.cv2_encode(img))
    return out


def scenes(seed, n):
    from tests.test_jpeg_gpu import scene
    rng = np.random.default_rng(seed)
    return [C.cv2_encode(scene(rng, 720, 1280)) for _ in range(n)]


def test_corpus_one_batch():
    from megreader_b200 import png
    corpus = C.corpus()
    blobs = [b for _, b in corpus]
    flag = {i for i, (n, _) in enumerate(corpus) if n in C.EXPECTED_STATUS}
    st = _check(blobs, _decode(png, blobs), flag)
    for i, (n, _) in enumerate(corpus):
        if n in C.EXPECTED_STATUS:
            assert st[i] == C.EXPECTED_STATUS[n], (n, st[i])


def test_mixed_batch_equals_each_decoder():
    from megreader_b200 import image, jpeg
    jc, pc = J.corpus(), C.corpus()
    from tests.test_jpeg_cpu import EXPECTED_STATUS as JBAD
    items = []
    for k in range(max(len(jc), len(pc))):
        if k < len(jc):
            items.append(("j",) + jc[k])
        if k < len(pc):
            items.append(("p",) + pc[k])
    blobs = [b for _, _, b in items]
    flag = {i for i, (t, n, _) in enumerate(items) if n in (JBAD if t == "j" else C.EXPECTED_STATUS)}
    res = _decode(image, blobs)
    _check(blobs, res, flag)
    st, sh, offs, buf = (res[k].cpu().numpy() for k in ("status", "shapes", "image_offsets", "buffer"))
    for i, (t, n, b) in enumerate(items):
        if t != "j":
            continue
        alone = _decode(jpeg, [b])
        assert int(alone["status"][0]) == st[i] and alone["shapes"][0].tolist() == sh[i].tolist(), n
        if st[i] == 0:
            h, w = sh[i]
            assert np.array_equal(alone["buffer"][:h * w * 3].cpu().numpy(), buf[offs[i]:offs[i] + h * w * 3]), n


def test_lines_and_scenes():
    from megreader_b200 import png
    for n in (16, 512):
        ls = lines(n, n, pil=True)
        _check(ls, _decode(png, ls))
    sc = scenes(3, 4)
    _check(sc, _decode(png, sc))


SENTINEL = 0xA5


def _raw(entry, blobs, cap, tail=1 << 16):
    from megreader_b200 import _lib, jpeg
    L = _lib.lib()
    data, offs = jpeg.pack_bytes(blobs)
    N = len(blobs)
    need = getattr(L, "mr_%s_workspace_bytes" % entry)(N, data.numel(), cap)
    ws = torch.full((need + tail,), SENTINEL, dtype=torch.uint8, device="cuda")
    out = torch.full((3 * cap + tail,), SENTINEL, dtype=torch.uint8, device="cuda")
    res = dict(buffer=out, image_offsets=torch.empty(N, dtype=torch.int64, device="cuda"),
               shapes=torch.empty((N, 2), dtype=torch.int32, device="cuda"), status=torch.empty(N, dtype=torch.int32, device="cuda"))
    rc = getattr(L, "mr_%s_decode" % entry)(data.data_ptr(), data.numel(), offs.data_ptr(), N, 16384, 16384, cap, ws.data_ptr(), need,
                                            out.data_ptr(), res["image_offsets"].data_ptr(), res["shapes"].data_ptr(),
                                            res["status"].data_ptr(), torch.cuda.current_stream().cuda_stream)
    assert rc == 0
    torch.cuda.synchronize()
    return res, bool((ws[need:] == SENTINEL).all()) and bool((out[3 * cap:] == SENTINEL).all())


@pytest.mark.parametrize("entry", ["png", "image"])
def test_capacity_refusals(entry):
    ls = lines(40, 10)
    px = [_pixels(b) for b in ls]
    res, intact = _raw(entry, ls, sum(px[:6]))                       # the last four do not fit
    assert intact
    _check(ls, res, flag=set(range(6, 10)))
    assert all(int(s) == 8 for s in res["status"][6:].tolist())
    big = scenes(41, 1)[0]
    res, intact = _raw(entry, [big], 1000)
    assert intact and int(res["status"][0]) == 8 and res["shapes"][0].tolist() == [0, 0]
    rng = np.random.default_rng(42)
    exact = [C.cv2_encode(J.image(rng, 1, 100)), C.cv2_encode(J.image(rng, 33, 301))]
    res, intact = _raw(entry, exact, 100 + 33 * 301)                 # exact capacity
    assert intact
    _check(exact, res)


def test_graph_capture_and_replay():
    from megreader_b200 import image, jpeg
    a = lines(50, 32) + [x for _, x in J.corpus()[:8]]
    b = lines(51, 32) + [x for _, x in J.corpus(1)[:8]]
    size = max(sum(map(len, a)), sum(map(len, b)))
    cap = max(sum(map(_pixels, a)), sum(map(_pixels, b)))
    data = torch.zeros(size, dtype=torch.uint8, device="cuda")
    offs = torch.zeros(len(a) + 1, dtype=torch.int64, device="cuda")

    def load(blobs):
        d, o = jpeg.pack_bytes(blobs)
        data.zero_()
        data[:d.numel()].copy_(d)
        offs.copy_(o)

    load(a)
    res = image.decode_packed(data, offs, 16384, 16384, cap)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s), torch.cuda.graph(g, stream=s):
        image.decode_packed(data, offs, 16384, 16384, cap, out=res)
    torch.cuda.current_stream().wait_stream(s)
    load(b)
    g.replay()
    torch.cuda.synchronize()
    _check(b, res)
    first = res["buffer"].clone()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(first, res["buffer"])


def test_chains():
    from megreader_b200 import db_batch, image, input_pipeline
    ls = lines(60, 24)
    res = _decode(image, ls)
    imgs = [_cv2(b) for b in ls]
    for mode in ("resize", "pad"):
        got = input_pipeline.resize_normalize_packed(res["buffer"], res["image_offsets"], res["shapes"], (32, 128), mode)
        assert torch.equal(got, input_pipeline.resize_normalize(imgs, (32, 128), mode)), mode
    from tests.test_jpeg_gpu import _quads
    dev = torch.device("cuda")
    sc = scenes(61, 2) + [J.cv2_encode(np.ascontiguousarray(_cv2(scenes(62, 1)[0])), 90, "420")]
    P, T, O = _quads(3, 8, 720, 1280, dev)
    u = db_batch.draws(3, torch.Generator(device=dev).manual_seed(5))
    ref = db_batch.pack_images([torch.from_numpy(_cv2(b)).to(dev) for b in sc])
    want = db_batch.train_batch_packed(*ref, 1500, 2000, P, T, O, u)
    dec = _decode(image, sc)
    got = db_batch.train_batch_packed(dec["buffer"], dec["image_offsets"], dec["shapes"], 1500, 2000, P, T, O, u)
    for k in ("image", "polygons", "offsets", "status"):
        assert torch.equal(got[k], want[k]), k
