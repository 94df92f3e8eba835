"""Time the DB training targets (megreader_b200.db_targets, csrc/db_targets.cu) against the host processes they replace.

    python benchmarks/db_targets.py [--batch 16] [--size 640] [--quads 10 30] [--iters 50] [--host-images 4]

For each quad count: seeded rotated text boxes 10 to 80 px high at size x size (tests/db_targets_cases.py), a batch of
`batch` images; device time of make_targets_packed per batch from CUDA events after warm-up, eager and replayed from a CUDA
graph; and the host time of the oracle's MakeSegDetectionData + MakeBorderMap (oracle/db_targets_port.py: numpy, cv2 and the
Python Clipper restatement) per image on `host-images` of the same images, one core, scaled to the batch.  Prints the card's
name and power limit first; writes nothing."""
import argparse
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from megreader_b200 import db_targets  # noqa: E402
from oracle import db_targets_port as port  # noqa: E402
from tests.db_targets_cases import batch  # noqa: E402


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                       text=True).strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return torch.cuda.get_device_name(0) + ", power limit unknown"


def device_ms(fn, iters):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--size", type=int, default=640)
    ap.add_argument("--quads", type=int, nargs="+", default=[10, 30])
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--host-images", type=int, default=4)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("benchmarks/db_targets.py needs a CUDA device")
    print("device:", card())
    S = a.size
    for q in a.quads:
        images = batch(1000 + q, a.batch, S, S, q, q, np.float64, odd=0.0)
        polys, tags, offsets = db_targets.pack([torch.as_tensor(p, device="cuda") for p, _ in images],
                                               [torch.as_tensor(t, device="cuda") for _, t in images])
        run = lambda: db_targets.make_targets_packed(polys, tags, offsets, (S, S))  # noqa: E731
        for _ in range(3):
            run()
        torch.cuda.synchronize()
        eager = device_ms(run, a.iters)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            run()
        g.replay()
        torch.cuda.synchronize()
        graph = device_ms(g.replay, a.iters)
        t0 = time.perf_counter()
        for p, t in images[:a.host_images]:
            port.make_targets(p.copy(), t, (S, S))
        host = (time.perf_counter() - t0) / a.host_images * 1e3
        print("%d x %dx%d, %d quads per image: device %.3f ms eager, %.3f ms graph per batch; host oracle %.1f ms per image "
              "(%.0f ms per batch on one core)" % (a.batch, S, S, q, eager, graph, host, host * a.batch))


if __name__ == "__main__":
    main()
