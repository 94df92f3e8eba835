"""wgmma GEMM (ours) vs cuBLAS on the CRNN conv GEMM shapes at batch 512 (fprop NT, dgrad NN, wgrad TN split-K)."""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from megreader_b200 import nnops  # noqa: E402

dev = torch.device("cuda:0")
LAYERS = [("conv0", 4194304, 64, 72), ("conv1", 1048576, 128, 576), ("conv2", 262144, 256, 1152),
          ("conv3", 262144, 256, 2304), ("conv4", 133120, 512, 2304), ("conv5", 133120, 512, 4608),
          ("conv6", 33280, 512, 2048)]


def t(fn, it=5):
    fn(); torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(it):
        fn()
    b.record(); torch.cuda.synchronize()
    return a.elapsed_time(b) / it * 1e3


for name, P, Cout, K in LAYERS:
    col = torch.randn(P, K, device=dev).bfloat16()
    W = torch.randn(Cout, K, device=dev).bfloat16()
    dz = torch.randn(P, Cout, device=dev).bfloat16()
    fl = 2.0 * P * Cout * K
    res = {"layer": name, "P": P, "Cout": Cout, "K": K}
    res["fprop_tc_us"] = t(lambda: nnops.gemm_tc(col, W))
    res["fprop_blas_us"] = t(lambda: nnops.gemm(col, W, transB=True))
    res["dgrad_tc_us"] = t(lambda: nnops.gemm_tc(dz, W, transA=False, transB=False))
    res["dgrad_blas_us"] = t(lambda: nnops.gemm(dz, W))
    out = torch.zeros(Cout, K, device=dev)
    for sp in (1, 4, 16, 64):
        res["wgrad_tc_s%d_us" % sp] = t(lambda: nnops.gemm_tc(dz, col, transA=True, transB=False, out=out, beta=1.0, splits=sp))
    res["wgrad_blas_us"] = t(lambda: nnops.gemm(dz, col, transA=True, out_dtype=torch.float32))
    res["TFLOPs"] = {k[:-3]: round(fl / v / 1e6, 1) for k, v in res.items() if k.endswith("_us")}
    print(json.dumps(res), flush=True)
    del col, W, dz
