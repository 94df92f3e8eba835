"""Deformable convolution in fp32 vs bf16 vs fp16 at the config-5 DCN layer shapes (batch 8, 3x3, deformable_group = 1,
fp32 master weights), forward and forward + backward, CUDA-event timed after warm-up:

    python benchmarks/dcn_half.py [--batch 8] [--iters 20]

  fp32   as the bf16 channels_last trunk calls the op today (refapi/backbones/resnet.py:_apply_conv2): input and offset field
         copied to fp32 NCHW, then the fp32 op (three bf16 MMAs per K block)
  bf16 / fp16   the input and offset field converted to the half dtype in NCHW, then the half-precision op (one MMA per K block)

Per shape and mode: time per call (us) and the tensor-pipe share: one GEMM of 2 * B * Cout * 9C * Ho * Wo flops per forward
(three per forward + backward: forward, weight and data gradients) against 989 TFLOP/s (H100 SXM dense bf16 / fp16).  The
device name and power limit are printed with the numbers.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from megreader_b200 import dcn  # noqa: E402

PEAK = 989e12
# (C, H of the input, stride): the first unit of the 128-channel stage has stride 2 and input-sized (128^2) offsets
SHAPES = [(128, 128, 2), (128, 64, 1), (256, 32, 1), (512, 16, 1)]


def device_info():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        q = "unknown"
    return {"device": name, "power_limit,max_sm_clock": q}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    print(json.dumps(device_info()), flush=True)
    B = args.batch
    for C, H, s in SHAPES:
        torch.manual_seed(0)
        Ho = (H - 1) // s + 1
        # the trunk's tensors: bf16 channels_last activations and offset field (offset conv at stride 1: input-sized)
        x_cl = torch.randn(B, C, H, H, device=dev).to(torch.bfloat16).to(memory_format=torch.channels_last)
        field_cl = torch.cat([2 * torch.randn(B, 18, H, H, device=dev), torch.randn(B, 9, H, H, device=dev)], 1)
        field_cl = field_cl.to(torch.bfloat16).to(memory_format=torch.channels_last)
        w = (torch.randn(C, C, 3, 3, device=dev) / (3 * C ** 0.5)).requires_grad_(True)
        go = torch.randn(B, C, Ho, Ho, device=dev)
        flops = 2.0 * B * C * 9 * C * Ho * Ho

        def run(mode, backward):
            dt = {"fp32": torch.float32, "bf16": torch.bfloat16, "fp16": torch.float16}[mode]
            x = x_cl.to(dt).contiguous().requires_grad_(backward)
            field = field_cl.to(dt).contiguous().requires_grad_(backward)
            out = dcn.modulated_deform_conv(x, field[:, :18], field[:, -9:].sigmoid(), w, None, s, 1, 1, 1, 1)
            if backward:
                w.grad = None
                out.backward(go.to(dt))
            return out

        res = {"B": B, "C": C, "H": H, "stride": s, "Ho": Ho}
        outs = {}
        for mode in ("fp32", "bf16", "fp16"):
            for backward in (False, True):
                for _ in range(3):
                    run(mode, backward)
                torch.cuda.synchronize()
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                for _ in range(args.iters):
                    run(mode, backward)
                b.record()
                torch.cuda.synchronize()
                us = a.elapsed_time(b) * 1e3 / args.iters
                key = "%s_%s" % (mode, "fwdbwd" if backward else "fwd")
                res[key + "_us"] = round(us, 1)
                res[key + "_tensor_pipe_pct"] = round(100 * (3 if backward else 1) * flops / (us * 1e-6) / PEAK, 1)
            with torch.no_grad():
                outs[mode] = run(mode, False).float()
        for mode in ("bf16", "fp16"):
            res[mode + "_rel_l2_vs_fp32"] = float((outs[mode] - outs["fp32"]).norm() / outs["fp32"].norm())
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
