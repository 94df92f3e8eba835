"""Device PNG decode (csrc/png.cu) timed with CUDA events: eager calls and graph replays for IIIT-like word crops (RGB,
30-150 x 100-600) in batches of 16, 512 and 4,096 at cv2's default level and at PIL's, four 1280 x 720 scenes, and a mixed
half-JPEG half-PNG line batch through image.decode_packed; cv2.imdecode on one host core beside each; one torch.profiler
pass for the split by kernel of a 512-line batch; the graph of 512 PNG lines -> decode -> resize_normalize_packed into
32 x 128.  Prints the card, its power limit and max SM clock.

    python -m benchmarks.png_decode
"""
import functools
import io
import os
import time

import numpy as np
import torch

from benchmarks.jpeg_decode import _encode, card, graph_of
from megreader_b200 import image, input_pipeline, jpeg, png

print = functools.partial(print, flush=True)  # noqa: A001


def _crop(rng):
    import cv2
    h, w = int(rng.integers(30, 151)), int(rng.integers(100, 601))
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    f = rng.uniform(5, 30, 3)
    img = np.stack([127 + 90 * np.sin(x / f[c] + c) * np.cos(y / (f[c] + 3) - c) for c in range(3)], -1)
    img = np.clip(img + rng.normal(0, 4, img.shape), 0, 255).astype(np.uint8)
    cv2.putText(img, "WORD%d" % rng.integers(100), (4, h - 6), cv2.FONT_HERSHEY_SIMPLEX, h / 45, (20, 20, 20), 2)
    return img


def lines(seed, n, pil=False):
    import cv2
    from PIL import Image
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        img = _crop(rng)
        if pil:
            bio = io.BytesIO()
            Image.fromarray(img[:, :, ::-1]).save(bio, "PNG")
            out.append(bio.getvalue())
        else:
            out.append(cv2.imencode(".png", img)[1].tobytes())
    return out


def scenes(seed, n):
    import cv2
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        base = cv2.resize(rng.integers(0, 256, (45, 80, 3), dtype=np.uint8), (1280, 720), interpolation=cv2.INTER_CUBIC)
        for _ in range(20):
            x, y = int(rng.integers(0, 1080)), int(rng.integers(40, 700))
            cv2.putText(base, "TEXT%d" % rng.integers(1000), (x, y), cv2.FONT_HERSHEY_SIMPLEX, 1.5,
                        tuple(int(c) for c in rng.integers(0, 255, 3)), 3)
        img = np.clip(base + rng.normal(0, 3, base.shape), 0, 255).astype(np.uint8)
        out.append(cv2.imencode(".png", img)[1].tobytes())
    return out


def timed(fn, min_s=0.5):
    """two windows of at least min_s, each call timed by CUDA events and synchronised (a call can take longer than its
    launches, so calls are never queued ahead): the mean ms per call in each window"""
    fn()
    torch.cuda.synchronize()
    res = []
    for _ in range(2):
        tot, n = 0.0, 0
        while tot < min_s * 1e3:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            e1.synchronize()
            tot += e0.elapsed_time(e1)
            n += 1
        res.append(tot / n)
    return res


def _pixels(b):
    return png.header_pixels(b) or jpeg._header_pixels(b)


def arm(name, blobs, mod=png):
    import cv2
    data, offs = jpeg.pack_bytes(blobs)
    cap = sum(map(_pixels, blobs))
    res = mod.decode_packed(data, offs, 16384, 16384, cap)
    torch.cuda.synchronize()
    assert int(res["status"].abs().sum()) == 0
    eager = timed(lambda: mod.decode_packed(data, offs, 16384, 16384, cap, out=res))
    g = graph_of(lambda: mod.decode_packed(data, offs, 16384, 16384, cap, out=res))
    graph = timed(g.replay)
    mb = sum(map(len, blobs)) / 1e6
    ms = min(graph)
    cv2.setNumThreads(1)
    t0 = time.perf_counter()
    for b in blobs:
        cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR)
    host = (time.perf_counter() - t0) * 1e3
    print("%-22s N=%5d  %6.2f MB  %7.2f MP  eager %s ms  graph %s ms  -> %.0f MP/s;  cv2 one host core %.2f ms (%.0f MP/s)"
          % (name, len(blobs), mb, cap / 1e6, " / ".join("%.3f" % x for x in eager), " / ".join("%.3f" % x for x in graph),
             cap / 1e6 / (ms / 1e3), host, cap / 1e6 / (host / 1e3)))
    return data, offs, cap, res


def profile_split(blobs):
    from torch.profiler import ProfilerActivity, profile
    data, offs = jpeg.pack_bytes(blobs)
    cap = sum(map(_pixels, blobs))
    res = png.decode_packed(data, offs, 16384, 16384, cap)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        png.decode_packed(data, offs, 16384, 16384, cap, out=res)
        torch.cuda.synchronize()
    print(prof.key_averages().table(sort_by="cuda_time_total", row_limit=12))


def main():
    print(card())
    print("host os.cpu_count() = %d" % os.cpu_count())
    profile_split(lines(4096, 512))
    for n in (16, 512):
        arm("%d lines cv2" % n, lines(n, n))
        arm("%d lines PIL" % n, lines(n + 1, n, pil=True))
    arm("4 scenes 1280x720", scenes(3, 4))
    rng = np.random.default_rng(5)
    mixed = [b if i % 2 else _encode(_crop(rng), 90) for i, b in enumerate(lines(6, 512))]
    arm("512 lines half JPEG", mixed, image)
    ls = lines(512, 512)
    data, offs = jpeg.pack_bytes(ls)
    host = data.cpu().pin_memory()
    cap = sum(map(_pixels, ls))
    dec = png.decode_packed(data, offs, 150, 600, cap)

    def chain():
        data.copy_(host, non_blocking=True)
        png.decode_packed(data, offs, 150, 600, cap, out=dec)
        input_pipeline.resize_normalize_packed(dec["buffer"], dec["image_offsets"], dec["shapes"], (32, 128))

    g = graph_of(chain)
    print("chain 512 PNG lines: copy bytes -> decode -> resize_normalize_packed into 32 x 128, one graph: %s ms"
          % " / ".join("%.3f" % x for x in timed(g.replay)))
    arm("4096 lines cv2", lines(4096, 4096))
    arm("4096 lines PIL", lines(4097, 4096, pil=True))


if __name__ == "__main__":
    main()
