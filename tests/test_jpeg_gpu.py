"""GPU: mr_jpeg_decode (csrc/jpeg.cu) against cv2.imdecode(buf, cv2.IMREAD_COLOR), bit for bit: the seeded corpus as one
mixed batch (supported images exact, the others flagged with shape (0, 0) and exact neighbours), MLT-like scenes and text
lines, the synchronisation edge cases, the capacities, graph capture and replay, and the chains into db_batch,
resize_normalize_packed and crop_quads_packed."""
import numpy as np
import pytest
import torch

from tests import jpeg_cases as C

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")


def _cv2(blob):
    return cv2.imdecode(np.frombuffer(blob, np.uint8), cv2.IMREAD_COLOR)


def _check_batch(blobs, res, expect_flag=()):
    shapes = res["shapes"].cpu().numpy()
    offs = res["image_offsets"].cpu().numpy()
    status = res["status"].cpu().numpy()
    buf = res["buffer"].cpu().numpy()
    for i, b in enumerate(blobs):
        if i in expect_flag:
            assert status[i] != 0 and tuple(shapes[i]) == (0, 0), i
            continue
        ref = _cv2(b)
        assert status[i] == 0, (i, status[i])
        h, w = shapes[i]
        got = buf[offs[i]:offs[i] + h * w * 3].reshape(h, w, 3)
        assert got.shape == ref.shape and np.array_equal(got, ref), i
    return status


def _decode(blobs, cap=None, max_side=16384):
    from megreader_b200 import jpeg
    data, offs = jpeg.pack_bytes(blobs)
    cap = cap if cap is not None else sum(C_pixels(b) for b in blobs)
    return jpeg.decode_packed(data, offs, max_side, max_side, cap)


def C_pixels(b):
    from megreader_b200 import jpeg
    return jpeg._header_pixels(b)


def scene(rng, h, w):
    base = cv2.resize(rng.integers(0, 256, (h // 16, w // 16, 3), dtype=np.uint8), (w, h), interpolation=cv2.INTER_CUBIC)
    for _ in range(20):
        x, y = int(rng.integers(0, w - 200)), int(rng.integers(40, h - 20))
        cv2.putText(base, "TEXT%d" % rng.integers(1000), (x, y), cv2.FONT_HERSHEY_SIMPLEX, 1.5,
                    tuple(int(c) for c in rng.integers(0, 255, 3)), 3)
    return np.clip(base + rng.normal(0, 6, base.shape), 0, 255).astype(np.uint8)


def scenes(seed, n):
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n):
        h, w = int(rng.integers(720, 1501)), int(rng.integers(1280, 2001))
        b = C.cv2_encode(scene(rng, h, w), int(rng.integers(85, 96)), "420", rst=64 if i % 5 == 1 else 0)
        if i % 5 == 3:
            b = C.insert_after_soi(b, 0xE1, C.exif_bytes(int(rng.integers(2, 9))))
        out.append(b)
    return out


def lines(seed, n):
    rng = np.random.default_rng(seed)
    return [C.cv2_encode(C.image(rng, 32, int(rng.integers(64, 401)), "smooth"), int(rng.integers(70, 96)), "420") for _ in range(n)]


def test_corpus_one_batch():
    corpus = C.corpus()
    blobs = [b for _, b in corpus]
    from tests.test_jpeg_cpu import EXPECTED_STATUS
    flag = {i for i, (n, _) in enumerate(corpus) if n in EXPECTED_STATUS}
    _check_batch(blobs, _decode(blobs), flag)


def test_scenes_and_lines():
    _check_batch(scenes(1, 16), _decode(scenes(1, 16)))
    ls = lines(2, 512)
    _check_batch(ls, _decode(ls))


def test_sync_edge_cases():
    rng = np.random.default_rng(3)
    blobs = [C.cv2_encode(C.image(rng, 1, 1), 50, "420"),
             C.cv2_encode(C.image(rng, 200, 300), 90, "420", rst=1),
             C.cv2_encode(C.image(rng, 400, 600, "flat"), 90, "444"),
             C.cv2_encode(C.image(rng, 300, 400, "noise"), 100, "444"),
             C.cv2_encode(C.image(rng, 300, 400, "noise"), 100, "420", rst=7)]
    blobs += [C.random_case(rng) for _ in range(200)]
    _check_batch(blobs, _decode(blobs))


def test_capacity_and_refusals():
    from megreader_b200 import _lib, jpeg
    ls = lines(4, 20)
    px = [C_pixels(b) for b in ls]
    cap = sum(px[:12])
    _check_batch(ls, _decode(ls, cap=cap), expect_flag=set(range(12, 20)))
    res = _decode(ls, max_side=200)
    st = res["status"].cpu().numpy()
    for i, b in enumerate(ls):
        assert bool(st[i] & jpeg.STATUS["too_large"]) == (_cv2(b).shape[1] > 200)
    data, offs = jpeg.pack_bytes(ls)
    need = jpeg.workspace_bytes(20, data.numel(), cap)
    ws = torch.empty(need - 1, dtype=torch.uint8, device="cuda")
    out = torch.empty(3 * cap, dtype=torch.uint8, device="cuda")
    io = torch.empty(20, dtype=torch.int64, device="cuda")
    sh = torch.empty((20, 2), dtype=torch.int32, device="cuda")
    stt = torch.empty(20, dtype=torch.int32, device="cuda")
    rc = _lib.lib().mr_jpeg_decode(data.data_ptr(), data.numel(), offs.data_ptr(), 20, 16384, 16384, cap, ws.data_ptr(), need - 1,
                                   out.data_ptr(), io.data_ptr(), sh.data_ptr(), stt.data_ptr(), None)
    assert rc == 4
    assert _lib.lib().mr_jpeg_workspace_bytes(0, 10, 10) == 0


def test_graph_capture_and_replay():
    from megreader_b200 import jpeg
    a, b = lines(5, 64), lines(6, 64)
    size = max(sum(map(len, a)), sum(map(len, b)))
    cap = max(sum(map(C_pixels, a)), sum(map(C_pixels, b)))
    data = torch.zeros(size, dtype=torch.uint8, device="cuda")
    offs = torch.zeros(65, dtype=torch.int64, device="cuda")

    def load(blobs):
        d, o = jpeg.pack_bytes(blobs)
        data.zero_()
        data[:d.numel()].copy_(d)
        offs.copy_(o)

    load(a)
    res = jpeg.decode_packed(data, offs, 16384, 16384, cap)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            jpeg.decode_packed(data, offs, 16384, 16384, cap, out=res)
    torch.cuda.current_stream().wait_stream(s)
    load(b)
    g.replay()
    torch.cuda.synchronize()
    _check_batch(b, res)
    first = res["buffer"].clone()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(first, res["buffer"])


def test_chains():
    from megreader_b200 import db_batch, input_pipeline, text_crop
    ls = lines(7, 24)
    res = _decode(ls)
    imgs = [_cv2(b) for b in ls]
    for mode in ("resize", "pad"):
        got = input_pipeline.resize_normalize_packed(res["buffer"], res["image_offsets"], res["shapes"], (32, 128), mode)
        want = input_pipeline.resize_normalize(imgs, (32, 128), mode)
        assert torch.equal(got, want), mode
    sc = scenes(8, 3)
    res = _decode(sc)
    ref = db_batch.pack_images([torch.from_numpy(_cv2(b)).cuda() for b in sc])
    assert torch.equal(res["shapes"], ref[2])
    for k in range(3):
        o, h, w = int(res["image_offsets"][k]), *res["shapes"][k].tolist()
        ro = int(ref[1][k])
        assert torch.equal(res["buffer"][o:o + h * w * 3], ref[0][ro:ro + h * w * 3])
    quads = torch.tensor([[[[10, 10], [300, 12], [298, 60], [12, 58]]]] * 3, dtype=torch.int32, device="cuda")
    cnt = torch.ones(3, dtype=torch.int32, device="cuda")
    a = text_crop.crop_quads_packed(res["buffer"], res["image_offsets"], res["shapes"], quads, cnt)
    b = text_crop.crop_quads_packed(ref[0], ref[1], ref[2], quads, cnt)
    assert torch.equal(a["image"], b["image"])


SENTINEL = 0xA5


def _raw_decode(blobs, cap, max_side=16384, offsets=None, tail=1 << 16):
    """mr_jpeg_decode with workspace and output buffers that carry a sentinel tail: (result dict, tails untouched)"""
    from megreader_b200 import _lib, jpeg
    data, offs = jpeg.pack_bytes(blobs)
    if offsets is not None:
        offs = torch.tensor(offsets, dtype=torch.int64, device="cuda")
    N = offs.numel() - 1
    need = jpeg.workspace_bytes(N, data.numel(), cap)
    ws = torch.full((need + tail,), SENTINEL, dtype=torch.uint8, device="cuda")
    out = torch.full((3 * cap + tail,), SENTINEL, dtype=torch.uint8, device="cuda")
    res = dict(buffer=out, image_offsets=torch.empty(N, dtype=torch.int64, device="cuda"),
               shapes=torch.empty((N, 2), dtype=torch.int32, device="cuda"), status=torch.empty(N, dtype=torch.int32, device="cuda"))
    rc = _lib.lib().mr_jpeg_decode(data.data_ptr(), data.numel(), offs.data_ptr(), N, max_side, max_side, cap, ws.data_ptr(), need,
                                   out.data_ptr(), res["image_offsets"].data_ptr(), res["shapes"].data_ptr(), res["status"].data_ptr(),
                                   torch.cuda.current_stream().cuda_stream)
    assert rc == 0
    torch.cuda.synchronize()
    intact = bool((ws[need:] == SENTINEL).all()) and bool((out[3 * cap:] == SENTINEL).all())
    return res, intact


def test_capacity_stays_inside_the_workspace():
    rng = np.random.default_rng(21)
    big = scenes(22, 1)[0]
    res, intact = _raw_decode([big], 1000)                                 # a scene against a tiny pixel capacity
    assert intact and int(res["status"][0]) == 8 and res["shapes"][0].tolist() == [0, 0]
    for h, w in ((1, 100), (33, 300), (9, 17)):                            # 4:4:4, sides not multiples of 8, exact capacity
        b = C.cv2_encode(C.image(rng, h, w), 90, "444")
        res, intact = _raw_decode([b], h * w)
        assert intact
        _check_batch([b], res)
    lines_ = lines(23, 6)
    px = [C_pixels(b) for b in lines_]
    res, intact = _raw_decode(lines_ + [big], sum(px) + 500)               # the last image does not fit; earlier ones exact
    assert intact
    _check_batch(lines_ + [big], res, expect_flag={6})


def test_coefficient_capacity():
    """(6 P + 3072 N) / 64 blocks: a thin 4:4:4 image alone at exact pixel capacity needs more (flagged too_large); in a
    batch with room to spare it decodes exactly"""
    rng = np.random.default_rng(24)
    thin = C.cv2_encode(C.image(rng, 1, 200), 90, "444")
    res, intact = _raw_decode([thin], 200)
    assert intact and int(res["status"][0]) == 8 and res["shapes"][0].tolist() == [0, 0]
    other = C.cv2_encode(C.image(rng, 64, 64), 90, "420")
    res, intact = _raw_decode([other, thin], 200 + 64 * 64)
    assert intact
    _check_batch([other, thin], res)


def test_overlapping_offsets_are_flagged():
    rng = np.random.default_rng(25)
    blobs = [C.cv2_encode(C.image(rng, 20, 30 + 5 * i), 90, "420") for i in range(4)]
    n = [len(b) for b in blobs]
    ends = np.cumsum([0] + n).tolist()
    offs = [ends[0], ends[1], ends[0] + 20, ends[0] + 30, ends[4]]          # images 1 and 2 start inside image 0's bytes
    res, intact = _raw_decode(blobs, sum(C_pixels(b) for b in blobs), offsets=offs)
    st = res["status"].cpu().tolist()
    assert intact and st[0] == 0 and st[1] & 32 and st[2] & 32
    _check_batch(blobs[:1], {k: (v[:1] if k != "buffer" else v) for k, v in res.items()})


def _quads(n, k, h, w, dev):
    from megreader_b200 import db_targets
    g = torch.Generator().manual_seed(n)
    polys, tags = [], []
    for _ in range(n):
        x = torch.rand(k, generator=g) * (w - 200)
        y = torch.rand(k, generator=g) * (h - 60)
        q = torch.stack([torch.stack([x, y], -1), torch.stack([x + 180, y], -1), torch.stack([x + 180, y + 50], -1),
                         torch.stack([x, y + 50], -1)], 1)
        polys.append(q.float().to(dev))
        tags.append(torch.zeros(k, dtype=torch.uint8, device=dev))
    return db_targets.pack(polys, tags)


def test_scene_chain_one_graph():
    """bytes -> decode -> train_batch_packed -> make_targets_packed captured as one graph equals the same chain on
    pack_images of the cv2-decoded images with the same draws"""
    from megreader_b200 import db_batch, db_targets, jpeg
    dev = torch.device("cuda")
    sc = scenes(26, 4)
    P, T, O = _quads(4, 12, 720, 1280, dev)
    u = db_batch.draws(4, torch.Generator(device=dev).manual_seed(3))
    ref = db_batch.pack_images([torch.from_numpy(_cv2(b)).to(dev) for b in sc])
    want = db_batch.train_batch_packed(*ref, 1500, 2000, P, T, O, u)
    want_t = db_targets.make_targets_packed(want["polygons"], want["ignore_tags"], want["offsets"], (640, 640))
    data, offs = jpeg.pack_bytes(sc)
    cap = sum(C_pixels(b) for b in sc)
    dec = jpeg.decode_packed(data, offs, 1500, 2000, cap)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s), torch.cuda.graph(g, stream=s):
        jpeg.decode_packed(data, offs, 1500, 2000, cap, out=dec)
        got = db_batch.train_batch_packed(dec["buffer"], dec["image_offsets"], dec["shapes"], 1500, 2000, P, T, O, u)
        got_t = db_targets.make_targets_packed(got["polygons"], got["ignore_tags"], got["offsets"], (640, 640))
    torch.cuda.current_stream().wait_stream(s)
    g.replay()
    torch.cuda.synchronize()
    for k in ("image", "polygons", "offsets", "status"):
        assert torch.equal(got[k], want[k]), k
    for k in ("gt", "mask", "thresh_map", "thresh_mask"):
        assert torch.equal(got_t[k], want_t[k]), k
