"""The DB text detector of experiments/seg_detector/seg_detector_db.yaml (bench_trunks.py config 6) and its loss tail alone:

    python benchmarks/db_step.py [--steps 10] [--warmup 3] [--batch 16] [--tail-iters 20]

1. One JSON line from bench_trunks.run with config 6: deformable_resnet50 + SegDetector(adaptive, k=50) + L1BalanceCELoss on
   synthetic 3x640x640 scenes (tests/db_data.py), per-GPU batch 16 (the yaml's 16 per GPU; --batch 2 = 16 over 8 GPUs), SGD,
   the step captured in a CUDA graph.
2. The loss tail alone at the same batch and 640x640, forward + backward from the three maps, CUDA-event timed after warm-up:
     fused      megreader_b200.db_head.L1BalanceCELossFunction (csrc/db_head.cu, no host synchronisation)
     framework  the reference's composition (decoders.BalanceCrossEntropyLoss / MaskL1Loss / DiceLoss: torch.topk over the
                N*N*H*W broadcast values and two host synchronisations)
   Achieved bandwidth of the fused tail from algorithmic bytes: forward reads 7 fp32 maps in pass 1 and 3 maps (binary, gt, mask)
   in each of the 3 further select passes and the sum pass; backward reads 7 maps and writes 3.  Against 3.35 TB/s (H100 SXM HBM3).
The device name and power limit are printed with the numbers."""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
import bench_trunks  # noqa: E402
from benchmarks.dcn_half import device_info  # noqa: E402

HBM = 3.35e12


def tail_bytes(N, H, W):
    m = N * H * W * 4
    return {"forward": 7 * m + 4 * 3 * m, "backward": 7 * m + 3 * m}


def time_ms(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def loss_tail(N, H, W, iters):
    import megreader_b200
    from megreader_b200 import db_head
    from tests.db_data import db_batch
    megreader_b200.install_reference_api()
    import decoders
    dev = torch.device("cuda")
    g = torch.Generator(device=dev).manual_seed(0)
    batch = {k: torch.from_numpy(v).to(dev) for k, v in db_batch(1, N, H, W).items()}
    maps = [torch.rand((N, 1, H, W), generator=g, device=dev).clamp_(1e-4, 1 - 1e-4).requires_grad_(True) for _ in range(3)]
    bce, l1, dice = decoders.BalanceCrossEntropyLoss(), decoders.MaskL1Loss(), decoders.DiceLoss()

    def fused():
        loss = db_head.l1_balance_ce_loss(*maps, batch["gt"], batch["mask"], batch["thresh_map"], batch["thresh_mask"])[0]
        loss.backward()
        return loss

    def framework():
        loss = dice(maps[2], batch["gt"], batch["mask"]) + 10 * l1(maps[1], batch["thresh_map"], batch["thresh_mask"])[0] \
            + 5 * bce(maps[0], batch["gt"], batch["mask"])
        loss.backward()
        return loss

    lf, lr = float(fused().detach()), float(framework().detach())
    t_fused, t_frame = time_ms(fused, iters), time_ms(framework, iters)
    with torch.no_grad():
        t_fwd = time_ms(lambda: db_head.l1_balance_ce_loss(*maps, batch["gt"], batch["mask"], batch["thresh_map"],
                                                           batch["thresh_mask"]), iters)
    by = tail_bytes(N, H, W)
    return {"shape": [N, H, W], "fused_ms_fwd_bwd": t_fused, "fused_ms_fwd": t_fwd, "framework_ms_fwd_bwd": t_frame,
            "speedup": t_frame / t_fused, "loss_fused": lf, "loss_framework": lr,
            "fused_fwd_bwd_GBps": (by["forward"] + by["backward"]) / (t_fused * 1e-3) / 1e9,
            "fused_fwd_GBps": by["forward"] / (t_fwd * 1e-3) / 1e9,
            "fraction_of_3.35TBps": (by["forward"] + by["backward"]) / (t_fused * 1e-3) / HBM,
            "algorithmic_bytes": by}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=0, help="per-GPU batch (default 16)")
    ap.add_argument("--tail-iters", type=int, default=20)
    ap.add_argument("--skip-step", action="store_true")
    args = ap.parse_args()
    args.config, args.gpus, args.impl, args.strong, args.dump_outputs = 6, 1, "ours", False, None
    assert torch.cuda.is_available(), "benchmarks/db_step.py needs a GPU"
    if not args.skip_step:
        bench_trunks.run(args, bench.peaks(), bench.ClockSampler, bench.emit_json)
    out = {"loss_tail": loss_tail(args.batch or 16, 640, 640, args.tail_iters)}
    out.update(device_info())
    print(json.dumps(out))


if __name__ == "__main__":
    main()
