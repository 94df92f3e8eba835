"""Time text_crop.crop_quads_packed (eager and CUDA-graph replay) for 4 MLT-like images (1280 x 720 to 2000 x 1500) with 100,
500 and 1,000 quads each into 32 x 100 and 64 x 256, its output bytes per second against 3.35 TB/s, and the reference's host
ImageCropper loop (cv2 on one core, as oracle/text_crop_port restates it) on the same quads; then the detection-to-strings
chain replayed as one CUDA graph: DB eval at 4 x 576 x 1024 (engine convolutions, seeded weights), boxes_from_maps
(max_candidates 1000), the crops into 32 x 128, engine CRNN eval and ctc_greedy_decode.  Every timed window is at least
0.5 s of work.  Run it twice to see the spread.

    python -m benchmarks.text_crop"""
import json
import subprocess
import time

import numpy as np
import torch

from megreader_b200 import db_batch, text_crop
from tests import text_crop_cases as C

SIZES = [(720, 1280), (1080, 1920), (1500, 2000), (960, 1280)]


def gpu_info():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True).strip()
    except Exception as e:                                  # noqa: BLE001
        return "unknown (%s)" % e


WINDOW_S = 0.5


def timed(fn):
    """seconds per call of fn over a window of at least WINDOW_S, by CUDA events"""
    fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    reps = max(20, int(WINDOW_S / max(time.perf_counter() - t0, 1e-6)))
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / 1e3 / reps


def graph_of(fn):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = fn()
    return g, out


def chain_row(dev):
    import bench
    import bench_trunks
    from megreader_b200 import db_boxes, decode
    torch.manual_seed(0)
    det, _ = bench_trunks.build(6, dev, engine=True)
    det.eval()
    rec = bench.build_model(dev).eval()
    x, _ = bench_trunks.synth_db(2, 4, (576, 1024))
    x = x.to(dev)
    rng = np.random.default_rng(1)
    imgs = [C.image(rng, 576, 1024) for _ in range(4)]
    buf, offs, shapes = db_batch.pack_images([torch.from_numpy(i).to(dev) for i in imgs])

    def chain():
        binary = det.decoder(det.backbone(x))
        binary = binary["binary"] if isinstance(binary, dict) else binary
        boxes, _, count = db_boxes.boxes_from_maps(binary.float(), None, 0.3, 0.7, 1000)
        crops = text_crop.crop_quads_packed(buf, offs, shapes, boxes, count, (32, 128))
        return crops["total"], decode.ctc_greedy_decode(rec.decoder(rec.backbone(crops["image"]), train=False))

    with torch.no_grad():
        g, out = graph_of(chain)
        t = timed(g.replay)
    return dict(chain="DB eval 4x576x1024 + boxes + crops 32x128 + CRNN eval + decode", graph_ms=t * 1e3,
                boxes_found=int(out[0][0]), crnn_rows=4000)


def main():
    import cv2
    from oracle import text_crop_port as port
    cv2.setNumThreads(1)
    dev = torch.device("cuda")
    rng = np.random.default_rng(0)
    imgs = [C.image(rng, h, w) for h, w in SIZES]
    buf, offs, shapes = db_batch.pack_images([torch.from_numpy(i).to(dev) for i in imgs])
    res = dict(gpu=gpu_info(), rows=[])
    for per in (100, 500, 1000):
        qs = [np.stack([C.quad(rng, "rotated", h, w) for _ in range(per)]) for h, w in SIZES]
        q = torch.from_numpy(np.concatenate(qs)).to(dev)
        o = torch.tensor([0] + list(np.cumsum([per] * 4)), dtype=torch.int32, device=dev)
        for size in ((32, 100), (64, 256)):
            call = lambda: text_crop.crop_quads_packed(buf, offs, shapes, q, o, size)  # noqa: E731
            eager = timed(call)
            g, _ = graph_of(call)
            graph = timed(g.replay)
            out_bytes = 4 * per * 3 * size[0] * size[1] * 4
            t0 = time.perf_counter()
            n_host = 50
            for k in range(n_host):
                port.crop(imgs[k % 4], qs[k % 4][k], size, "resize")
            host = (time.perf_counter() - t0) / n_host * 4 * per
            row = dict(per_image=per, size=size, eager_ms=eager * 1e3, graph_ms=graph * 1e3,
                       out_TBps=out_bytes / graph / 1e12, share_of_3_35TBps=out_bytes / graph / 3.35e12, host_ms=host * 1e3)
            res["rows"].append(row)
            print(json.dumps(row))
    res["chain"] = chain_row(dev)
    print(json.dumps(res["chain"]))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
