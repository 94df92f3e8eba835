"""Device JPEG decode (csrc/jpeg.cu) timed with CUDA events: eager calls and graph replays for 16 and 4 MLT-like scenes and
512 / 4,096 text lines; cv2.imdecode on one host core and torchvision's nvJPEG decode beside it on the same bytes; one
torch.profiler pass for the split by kernel; the two graph chains bytes -> decode -> train_batch_packed -> make_targets_packed
(16 scenes into 640 x 640) and bytes -> decode -> resize_normalize_packed (512 lines into 32 x 128).  Prints the card, its
power limit and max SM clock.

    python -m benchmarks.jpeg_decode
"""
import functools
import os
import subprocess
import time

import numpy as np
import torch

from megreader_b200 import db_batch, db_targets, input_pipeline, jpeg

print = functools.partial(print, flush=True)  # noqa: A001


def _encode(img, quality, rst=0):
    import cv2
    p = [cv2.IMWRITE_JPEG_QUALITY, int(quality), cv2.IMWRITE_JPEG_SAMPLING_FACTOR, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420]
    if rst:
        p += [cv2.IMWRITE_JPEG_RST_INTERVAL, rst]
    return cv2.imencode(".jpg", img, p)[1].tobytes()


def scenes(seed, n):
    """MLT-like scenes: 1280 x 720 to 2000 x 1500, quality 85 to 95, 4:2:0, every fifth with a restart interval"""
    import cv2
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n):
        h, w = int(rng.integers(720, 1501)), int(rng.integers(1280, 2001))
        base = cv2.resize(rng.integers(0, 256, (h // 16, w // 16, 3), dtype=np.uint8), (w, h), interpolation=cv2.INTER_CUBIC)
        for _ in range(20):
            x, y = int(rng.integers(0, w - 200)), int(rng.integers(40, h - 20))
            cv2.putText(base, "TEXT%d" % rng.integers(1000), (x, y), cv2.FONT_HERSHEY_SIMPLEX, 1.5,
                        tuple(int(c) for c in rng.integers(0, 255, 3)), 3)
        img = np.clip(base + rng.normal(0, 6, base.shape), 0, 255).astype(np.uint8)
        out.append(_encode(img, int(rng.integers(85, 96)), 64 if i % 5 == 1 else 0))
    return out


def lines(seed, n):
    """text lines 32 x 64 to 32 x 400, quality 70 to 95, 4:2:0"""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        w = int(rng.integers(64, 401))
        y, x = np.mgrid[0:32, 0:w].astype(np.float64)
        f = rng.uniform(3, 20, 3)
        img = np.stack([127 + 90 * np.sin(x / f[c] + c) * np.cos(y / (f[c] + 3) - c) for c in range(3)], -1)
        img = np.clip(img + rng.normal(0, 10, img.shape), 0, 255).astype(np.uint8)
        out.append(_encode(img, int(rng.integers(70, 96))))
    return out


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, check=True).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return "nvidia-smi unavailable (%s)" % e


def timed(fn, min_s=0.5):
    fn()
    torch.cuda.synchronize()
    res = []
    for _ in range(2):
        n, t0 = 0, time.perf_counter()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        while time.perf_counter() - t0 < min_s:
            fn()
            n += 1
        e1.record()
        torch.cuda.synchronize()
        res.append(e0.elapsed_time(e1) / n)
    return res


def arm(name, blobs):
    import cv2
    data, offs = jpeg.pack_bytes(blobs)
    cap = sum(jpeg._header_pixels(b) for b in blobs)
    res = jpeg.decode_packed(data, offs, 16384, 16384, cap)
    torch.cuda.synchronize()
    assert int(res["status"].abs().sum()) == 0
    eager = timed(lambda: jpeg.decode_packed(data, offs, 16384, 16384, cap, out=res))
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s), torch.cuda.graph(g, stream=s):
        jpeg.decode_packed(data, offs, 16384, 16384, cap, out=res)
    torch.cuda.current_stream().wait_stream(s)
    graph = timed(g.replay)
    mb = sum(map(len, blobs)) / 1e6
    ms = min(graph)
    print("%-12s N=%5d  %6.1f MB  %7.1f MP  eager %s ms  graph %s ms  -> %.0f MP/s  %.0f MB/s"
          % (name, len(blobs), mb, cap / 1e6, " / ".join("%.3f" % x for x in eager), " / ".join("%.3f" % x for x in graph),
             cap / 1e6 / (ms / 1e3), mb / (ms / 1e3)))
    cv2.setNumThreads(1)
    t0 = time.perf_counter()
    for b in blobs:
        cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR)
    print("    cv2.imdecode one host core (os.cpu_count() = %d): %.2f ms" % (os.cpu_count(), (time.perf_counter() - t0) * 1e3))
    try:
        import torchvision
        from torchvision.io import decode_jpeg
        ts = [torch.frombuffer(bytearray(b), dtype=torch.uint8) for b in blobs]
        out = decode_jpeg(ts, device="cuda")
        torch.cuda.synchronize()
        t = timed(lambda: decode_jpeg(ts, device="cuda"))
        diff = max(int((o.permute(1, 2, 0).flip(-1).cpu().int() - torch.from_numpy(cv2.imdecode(np.frombuffer(b, np.uint8), 1)).int())
                       .abs().max()) if o.shape[1:] == cv2.imdecode(np.frombuffer(b, np.uint8), 1).shape[:2] else -1
                   for o, b in zip(out, blobs))
        print("    torchvision %s nvJPEG: %s ms, largest difference from cv2 %d" % (torchvision.__version__, " / ".join("%.3f" % x for x in t), diff))
    except Exception as e:  # noqa: BLE001
        print("    torchvision nvJPEG: not run (%s)" % str(e).splitlines()[0][:100])
    return data, offs, cap, res


def graph_of(fn):
    fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s), torch.cuda.graph(g, stream=s):
        fn()
    torch.cuda.current_stream().wait_stream(s)
    return g


def chains(sc, ls):
    """one graph each, replayed after the pinned bytes are copied into the captured device buffer"""
    dev = torch.device("cuda")
    data, offs = jpeg.pack_bytes(sc)
    host = data.cpu().pin_memory()
    cap = sum(jpeg._header_pixels(b) for b in sc)
    dec = jpeg.decode_packed(data, offs, 1500, 2000, cap)
    g = torch.Generator().manual_seed(0)
    polys, tags = [], []
    for _ in sc:
        x, y = torch.rand(20, generator=g) * 1000, torch.rand(20, generator=g) * 600
        polys.append(torch.stack([torch.stack([x, y], -1), torch.stack([x + 180, y], -1), torch.stack([x + 180, y + 50], -1),
                                  torch.stack([x, y + 50], -1)], 1).to(dev))
        tags.append(torch.zeros(20, dtype=torch.uint8, device=dev))
    P, T, O = db_targets.pack(polys, tags)
    u = db_batch.draws(len(sc), torch.Generator(device=dev).manual_seed(1))

    def scene_chain():
        data.copy_(host, non_blocking=True)
        jpeg.decode_packed(data, offs, 1500, 2000, cap, out=dec)
        o = db_batch.train_batch_packed(dec["buffer"], dec["image_offsets"], dec["shapes"], 1500, 2000, P, T, O, u)
        db_targets.make_targets_packed(o["polygons"], o["ignore_tags"], o["offsets"], (640, 640))

    gs = graph_of(scene_chain)
    print("chain 16 scenes: copy bytes -> decode -> train_batch_packed -> make_targets_packed, one graph: %s ms"
          % " / ".join("%.3f" % x for x in timed(gs.replay)))
    ldata, loffs = jpeg.pack_bytes(ls)
    lhost = ldata.cpu().pin_memory()
    lcap = sum(jpeg._header_pixels(b) for b in ls)
    ldec = jpeg.decode_packed(ldata, loffs, 32, 400, lcap)

    def line_chain():
        ldata.copy_(lhost, non_blocking=True)
        jpeg.decode_packed(ldata, loffs, 32, 400, lcap, out=ldec)
        input_pipeline.resize_normalize_packed(ldec["buffer"], ldec["image_offsets"], ldec["shapes"], (32, 128))

    gl = graph_of(line_chain)
    print("chain 512 lines: copy bytes -> decode -> resize_normalize_packed into 32 x 128, one graph: %s ms"
          % " / ".join("%.3f" % x for x in timed(gl.replay)))


def main():
    print(card())
    sc = scenes(11, 16)
    a = arm("16 scenes", sc)
    arm("4 scenes", scenes(12, 4))
    ls = lines(13, 512)
    arm("512 lines", ls)
    arm("4096 lines", lines(14, 4096))
    chains(sc, ls)
    data, offs, cap, res = a
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            jpeg.decode_packed(data, offs, 16384, 16384, cap, out=res)
        torch.cuda.synchronize()
    print(prof.key_averages().table(sort_by="cuda_time_total", row_limit=15))


if __name__ == "__main__":
    main()
