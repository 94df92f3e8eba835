"""Time the DB validation measure (megreader_b200.db_measure) on two seeded workloads:

  yaml   4 x 576 x 1024, about 30 gt per image, detections from boxes_from_maps(max_candidates=1000) on maps rendered from the
         gt (make_targets_packed's text map plus noise), gt validated by make_targets_packed;
  dense  16 images with 100 gt and 1000 noisy int32 detections each.

For each: evaluate_packed eager and replayed from a CUDA graph (CUDA events after warm-up); for `yaml` also the whole
validation step of seg_detector_db.yaml in one graph (eval model on the engine convolutions, boxes_from_maps,
make_targets_packed, evaluate_packed into device totals); and the host evaluator of oracle/db_measure_port.py on the same
inputs.  That host figure is the oracle's exact-arithmetic restatement, an upper bound on the reference's shapely cost, not
the reference itself.  Prints the card and its power limit first.

    python benchmarks/db_measure.py [--iters 50]
"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from megreader_b200 import db_boxes, db_measure, db_targets  # noqa: E402
from oracle import db_measure_port as port  # noqa: E402
from tests.db_measure_cases import batch_case  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name()


def time_ms(fn, iters, warmup=5):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def graph_of(fn):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    return g


def host_oracle_s(images):
    t = time.perf_counter()
    for g, tg, d in images:
        port.evaluate_image([dict(points=g[i], ignore=bool(tg[i])) for i in range(len(g))], [dict(points=p) for p in d])
    return time.perf_counter() - t


def measure_inputs(dev, polys, tags, offsets, boxes, count, iters, label):
    totals = torch.zeros(3, dtype=torch.int64, device=dev)
    fn = lambda: db_measure.evaluate_packed(polys, tags, offsets, boxes, count, totals=totals)  # noqa: E731
    eager = time_ms(fn, iters)
    g = graph_of(fn)
    graph = time_ms(g.replay, iters)
    print("%-6s evaluate_packed: eager %.3f ms, graph %.3f ms  (max_dets %d, gt slots %d)"
          % (label, eager, graph, boxes.size(1), polys.size(0)))
    return eager, graph


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("db_measure benchmark: no CUDA device")
    dev = torch.device("cuda")
    print("card:", card())

    # yaml: 4 x 576 x 1024
    H, W = 576, 1024
    images = batch_case(101, 4, H, W, (25, 35), (0, 0))
    polys, tags, offsets = db_targets.pack([torch.from_numpy(g).to(dev) for g, _, _ in images],
                                           [torch.from_numpy(t).to(dev) for _, t, _ in images])
    t = db_targets.make_targets_packed(polys, tags, offsets, (H, W))
    gen = torch.Generator(device=dev).manual_seed(1)
    prob = (t["gt"] * 0.9 + 0.15 * torch.rand(t["gt"].shape, generator=gen, device=dev)).clamp(0, 1)
    boxes, _, count = db_boxes.boxes_from_maps(prob, None, 0.3, 0.7, 1000)
    measure_inputs(dev, t["polygons"], t["ignore_tags"], offsets, boxes, count, args.iters, "yaml")
    off, cn = offsets.cpu().numpy(), count.cpu().numpy()
    vp, vt, bx = t["polygons"].cpu().numpy(), t["ignore_tags"].cpu().numpy().astype(bool), boxes.cpu().numpy()
    host = [(vp[off[n]:off[n + 1]], vt[off[n]:off[n + 1]], bx[n, :cn[n]]) for n in range(4)]
    print("yaml   detections per image: %s" % cn.tolist())
    print("yaml   oracle host evaluator (exact-arithmetic restatement, not the reference): %.1f ms" % (1e3 * host_oracle_s(host)))

    import bench_trunks
    torch.manual_seed(0)
    net, _ = bench_trunks.build(6, dev, engine=True)
    net.eval()
    x, _ = bench_trunks.synth_db(2, 4, (H, W))
    x = x.to(dev)
    totals = torch.zeros(3, dtype=torch.int64, device=dev)

    def step():
        binary = net.decoder(net.backbone(x))
        binary = binary['binary'] if isinstance(binary, dict) else binary
        b, _, c = db_boxes.boxes_from_maps(binary.float(), None, 0.3, 0.7, 1000)
        tt = db_targets.make_targets_packed(polys, tags, offsets, (H, W))
        return db_measure.evaluate_packed(tt["polygons"], tt["ignore_tags"], offsets, b, c, totals=totals)
    with torch.no_grad():
        g = graph_of(step)
        full = time_ms(g.replay, max(5, args.iters // 5), warmup=2)
    print("yaml   validation step in one graph (model + boxes + targets + measure): %.2f ms" % full)

    # dense: 16 images, 100 gt, 1000 noisy detections
    images = batch_case(102, 16, 640, 640, (100, 100), (1000, 1000), np.float64, True, noise=0.5)
    polys, tags, offsets = db_targets.pack([torch.from_numpy(g).to(dev) for g, _, _ in images],
                                           [torch.from_numpy(t).to(dev) for _, t, _ in images])
    boxes = torch.from_numpy(np.stack([d for _, _, d in images])).to(dev)
    count = torch.full((16,), 1000, dtype=torch.int32, device=dev)
    measure_inputs(dev, polys, tags, offsets, boxes, count, args.iters, "dense")
    print("dense  oracle host evaluator (exact-arithmetic restatement, not the reference), first 2 images: %.1f s"
          % host_oracle_s(images[:2]))


if __name__ == "__main__":
    main()
