"""CRNN layer 0 (Conv2d(3, 64, 3, 1, 1) -> ReLU -> MaxPool2d(2, 2), bf16) the unfused way against the fused stem kernels of
csrc/crnn_stem.cu, forward and backward, at the bench shape (512 x 3 x 32 x 256) and at a small batch (4 x 3 x 32 x 100).

    old forward  = nchw_to_nhwc + im2col + GEMM + bias/ReLU/pool          new forward  = mr_crnn_stem_fwd
    old backward = pool backward (dz, dbias) + weight-gradient GEMM       new backward = mr_crnn_stem_bwd
                   + the [64, 72] -> [64, 3, 3, 3] permute

Each arm is timed like bench._graph_time (20 calls captured in one CUDA graph, replayed after warm-up, CUDA events); old and
new alternate for --rounds rounds in one process and the median is reported.  Algorithmic bytes are what a fused stem has
to move (forward: x fp32 in, y bf16 and one routing byte per pooled value out; backward: x, dy and the routing bytes in),
and both arms are rated on those bytes against the data sheet's 3.35 TB/s.

    python benchmarks/crnn_stem.py --out DIR [--rounds 5]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from benchmarks.crnn_conv_layers import card  # noqa: E402
from megreader_b200 import crnn_engine  # noqa: E402
from megreader_b200 import nnops as ops  # noqa: E402

HBM_TBS = 3.35
SHAPES = [(512, 32, 256), (4, 32, 100)]


def arms(n, h, w, dev):
    torch.manual_seed(0)
    conv = torch.nn.Conv2d(3, 64, 3, 1, 1).to(dev)
    pool = torch.nn.MaxPool2d(2, 2)
    g = torch.Generator(device=dev).manual_seed(1)
    x = torch.randn((n, 3, h, w), generator=g, device=dev)
    dy = torch.randn((n, h // 2, w // 2, 64), generator=g, device=dev).to(torch.bfloat16)
    bf = torch.bfloat16
    a = ops.nchw_to_nhwc(x, 8, bf)
    col, ho, wo = ops.im2col(a, 3, 3, 1, 1, 72)
    Wm = ops.conv_weight_pack(conv.weight, 8, 72, bf, 0)
    z = ops.gemm(col, Wm, transB=True)
    y_old, idx_old = ops.bias_relu_pool_fwd(z, conv.bias.detach(), n, ho, wo, 64, (2, 2), (2, 2), (0, 0))
    _, idx_new = ops.crnn_stem_fwd(x, conv, pool, True)

    def old_fwd():
        a = ops.nchw_to_nhwc(x, 8, bf)
        col, _, _ = ops.im2col(a, 3, 3, 1, 1, 72)
        zz = ops.gemm(col, Wm, transB=True)
        return ops.bias_relu_pool_fwd(zz, conv.bias.detach(), n, ho, wo, 64, (2, 2), (2, 2), (0, 0))

    def old_bwd():
        dz, dbias = ops.bias_relu_pool_bwd(dy.view(-1, 64), y_old, idx_old, n, ho, wo, 64, (2, 2), (2, 2), (0, 0))
        dWm = ops.gemm(dz, col, transA=True, out_dtype=torch.float32)
        return crnn_engine._weight_grad(dWm, 3, 8, 3, 3), dbias

    pooled = n * (h // 2) * (w // 2) * 64
    xb = n * 3 * h * w * 4
    return [("fwd", xb + pooled * 3, old_fwd, lambda: ops.crnn_stem_fwd(x, conv, pool, True)),
            ("bwd", xb + pooled * 3, old_bwd, lambda: ops.crnn_stem_bwd(x, dy, idx_new, conv, pool))]


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--out", required=True, help="directory for the JSON record")
    ap.add_argument("--iters", type=int, default=20, help="calls per CUDA graph")
    ap.add_argument("--rounds", type=int, default=5, help="alternating old / new rounds (the median is reported)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("crnn_stem: needs a CUDA device")
    dev = torch.device("cuda:0")
    info = card()
    rows = []
    for n, h, w in SHAPES:
        cs = arms(n, h, w, dev)
        times = {}
        for _ in range(args.rounds):
            for kind, _, old, new in cs:
                times.setdefault((kind, "old"), []).append(bench._graph_time(old, args.iters))
                times.setdefault((kind, "new"), []).append(bench._graph_time(new, args.iters))
        for kind, nbytes, _, _ in cs:
            row = {"shape": [n, 3, h, w], "pass": kind, "algorithmic_mb": nbytes * 1e-6}
            for arm in ("old", "new"):
                ts = sorted(times[(kind, arm)])
                t = ts[len(ts) // 2]
                row[arm] = {"us": t * 1e6, "us_all": [v * 1e6 for v in times[(kind, arm)]], "gbs": nbytes / t * 1e-9,
                            "of_hbm_peak": nbytes / t * 1e-12 / HBM_TBS}
            rows.append(row)
            print("%4d x 3 x %d x %-4d %s  %7.1f MB   old %8.1f us (%5.1f%% of HBM)   new %8.1f us %7.0f GB/s (%5.1f%% of HBM)"
                  % (n, h, w, kind, row["algorithmic_mb"], row["old"]["us"], 100 * row["old"]["of_hbm_peak"],
                     row["new"]["us"], row["new"]["gbs"], 100 * row["new"]["of_hbm_peak"]), flush=True)
    rec = {"rows": rows, "iters_per_graph": args.iters, "rounds": args.rounds, "hbm_tbs": HBM_TBS, "card": info}
    os.makedirs(args.out, exist_ok=True)
    path = os.path.join(args.out, "crnn_stem.json")
    with open(path, "w") as f:
        json.dump(rec, f, indent=1)
    print("card: %s" % json.dumps(info))
    print("wrote", path)


if __name__ == "__main__":
    main()
