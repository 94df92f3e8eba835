"""DCNv2 backward at the bench shapes: fused wgmma kernels vs the column-matrix + SGEMM route: python benchmarks/dcn_bwd.py"""
import os, sys, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from megreader_b200 import dcn
dev = torch.device("cuda:0")
B = 8
MODES = {"fused": (), "wgrad_fused": ("MR_DCN_UNFUSED_DGRAD",), "unfused": ("MR_DCN_UNFUSED_DGRAD", "MR_DCN_UNFUSED_WGRAD")}
for C, H in ((128, 64), (256, 32), (512, 16)):
    torch.manual_seed(0)
    x = torch.randn(B, C, H, H, device=dev)
    w = torch.randn(C, C, 3, 3, device=dev) / (3 * C ** 0.5)
    off = 2 * torch.randn(B, 18, H, H, device=dev)
    m = torch.sigmoid(torch.randn(B, 9, H, H, device=dev))
    go = torch.randn(B, C, H, H, device=dev)
    res, outs = {}, {}
    for mode, envs in MODES.items():
        for e in ("MR_DCN_UNFUSED_DGRAD", "MR_DCN_UNFUSED_WGRAD"):
            os.environ.pop(e, None)
        for e in envs:
            os.environ[e] = "1"
        gi, gw, goff, gm = torch.zeros_like(x), torch.zeros_like(w), torch.zeros_like(off), torch.zeros_like(m)
        def run():
            dcn.modulated_deform_conv_cuda_backward(x, w, None, None, off, m, None, gi, gw, None, goff, gm, go, 3, 3, 1, 1, 1, 1, 1, 1, 1, 1, False)
        for _ in range(3):
            run()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(10):
            run()
        b.record()
        torch.cuda.synchronize()
        res[mode] = a.elapsed_time(b) / 10 * 1e3
        gi.zero_(); gw.zero_(); run()
        outs[mode] = [t.clone() for t in (gi, gw, goff, gm)]
    err = [float((a - b).abs().max() / b.abs().max()) for a, b in zip(outs["fused"], outs["unfused"])]
    print("C%d@%d: bwd fused %.1f us | wgrad fused only %.1f us | unfused %.1f us | rel diff gi %.1e gw %.1e goff %.1e gm %.1e" % (
        C, H, res["fused"], res["wgrad_fused"], res["unfused"], *err), flush=True)
