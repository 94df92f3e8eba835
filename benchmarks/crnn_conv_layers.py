"""Where the CRNN training step's time goes, convolution by convolution, at the bench shape (batch 512 of 3x32x256 lines,
bf16 NHWC activations).

(a) every implicit convolution of the step: L1-L6 forward, input gradient (dz convolved with the flipped, transposed
    weights, padding k-1-p) and weight gradient, on seeded inputs.  Each call runs through the one-tile-per-CTA entry
    (conv_fprop_tc / conv_wgrad_tc) and through the persistent entry (conv_fprop_pp / conv_wgrad_pp), the two
    alternating; each is timed like bench._graph_time (20 launches captured in a CUDA graph, replayed after warm-up).
    Forward and input-gradient outputs are compared bit for bit, weight gradients by their largest relative difference.
    Weight-gradient times include zeroing the fp32 output, which both entries need.
        python benchmarks/crnn_conv_layers.py --out DIR [--batch 512] [--rounds 3]
(b) torch.profiler over a few eager training steps of bench.build_model after warm-up, kernel time summed by name: the
    share of the step that the convolutions are.
        python benchmarks/crnn_conv_layers.py --profile --out DIR [--steps 3]

(c) the persistent kernels against each other, call by call, the arms alternating round after round: forward and input
    gradient on the 128-pixel ping-pong kernel (tile_m=128) and as mr_conv_fprop_pp selects (tile_m=0: the 256-pixel
    kernel from 36 K blocks on), L6's input gradient also as the engine's row split (two 1 x 2 convolutions), and the
    weight gradient with the planner's schedule on 128 x 256 tiles (its old arm is this script's (a) run from the parent
    build) and, at L1 and L2, as the engine runs it (crnn_engine._conv_wgrad: 128 x 192 tiles).  Beside
    TFLOP/s it prints the L2-to-SM rate implied by the kernel's operand bytes per FLOP, and for the weight gradient the
    share of the issued MMA work that multiplies real pixels and columns rather than zero fill.
        python benchmarks/crnn_conv_layers.py --changed --out DIR [--batch 512] [--rounds 3]

All write JSON into DIR together with the card's name, power limit and maximum SM clock.  L0 (Cin = 3) runs on the fused
stem kernels of csrc/crnn_stem.cu (benchmarks/crnn_stem.py) and is not an implicit convolution.
"""
import argparse
import json
import os
import re
import subprocess
import sys
from collections import defaultdict

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from megreader_b200 import nnops as ops  # noqa: E402

# (name, input H, W, C, Cout, k, padding) of the implicit convolutions of backbones/crnn.py at 32 x 256 lines
LAYERS = [("L1", 16, 128, 64, 128, 3, 1), ("L2", 8, 64, 128, 256, 3, 1), ("L3", 8, 64, 256, 256, 3, 1),
          ("L4", 4, 65, 256, 512, 3, 1), ("L5", 4, 65, 512, 512, 3, 1), ("L6", 2, 66, 512, 512, 2, 0)]


def card():
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30).stdout.strip().split(", ")
        info.update(power_limit_w=float(q[0]), max_sm_mhz=float(q[1]))
    except Exception as e:      # the figures are then missing from the record, not guessed
        info.update(power_limit_w=None, max_sm_mhz=None, query_error=str(e))
    return info


def calls(n, dev):
    """[(layer, kind, flop, old_fn, new_fn)] on seeded bf16 operands."""
    g = torch.Generator(device=dev).manual_seed(0)
    out = []
    for name, H, W, C, Cout, k, p in LAYERS:
        Ho, Wo = H + 2 * p - k + 1, W + 2 * p - k + 1
        flop = 2.0 * n * Ho * Wo * Cout * k * k * C
        x = torch.randn((n, H, W, C), generator=g, device=dev).to(torch.bfloat16)
        Wm = (torch.randn((Cout, k * k * C), generator=g, device=dev) / (k * k * C) ** 0.5).to(torch.bfloat16)
        dz = torch.randn((n, Ho, Wo, Cout), generator=g, device=dev).to(torch.bfloat16)
        Wd = (torch.randn((C, k * k * Cout), generator=g, device=dev) / (k * k * Cout) ** 0.5).to(torch.bfloat16)
        dW = torch.zeros((Cout, k * k * C), dtype=torch.float32, device=dev)
        out += [
            (name, "fprop", flop, lambda x=x, Wm=Wm, k=k, p=p: ops.conv_fprop_tc(x, Wm, k, k, p, p)[0],
             lambda x=x, Wm=Wm, k=k, p=p: ops.conv_fprop_pp(x, Wm, k, k, p, p)[0]),
            (name, "dgrad", flop, lambda dz=dz, Wd=Wd, k=k, p=p: ops.conv_fprop_tc(dz, Wd, k, k, k - 1 - p, k - 1 - p)[0],
             lambda dz=dz, Wd=Wd, k=k, p=p: ops.conv_fprop_pp(dz, Wd, k, k, k - 1 - p, k - 1 - p)[0]),
            (name, "wgrad", flop, lambda dz=dz, x=x, k=k, p=p, dW=dW: ops.conv_wgrad_tc(dz, x, k, k, p, p, out=dW.zero_()),
             lambda dz=dz, x=x, k=k, p=p, dW=dW: ops.conv_wgrad_pp(dz, x, k, k, p, p, out=dW.zero_())),
        ]
    return out


def run_layers(args):
    dev = torch.device("cuda:0")
    pk = bench.peaks()
    rows = []
    cs = calls(args.batch, dev)
    times = defaultdict(list)
    for _ in range(args.rounds):                      # old and new alternate, call by call, round after round
        for i, (_, _, _, old, new) in enumerate(cs):
            times[(i, "old")].append(bench._graph_time(old, args.iters))
            times[(i, "new")].append(bench._graph_time(new, args.iters))
    for i, (name, kind, flop, old, new) in enumerate(cs):
        row = {"layer": name, "kind": kind, "gflop": flop * 1e-9}
        for arm in ("old", "new"):
            t = sorted(times[(i, arm)])[len(times[(i, arm)]) // 2]
            row[arm] = {"us": t * 1e6, "us_all": [v * 1e6 for v in times[(i, arm)]], "tflops": flop / t * 1e-12,
                        "of_peak": flop / t * 1e-12 / pk["bf16_tflops"]}
        if kind != "wgrad":
            row["bit_identical"] = bool(torch.equal(old(), new()))
        else:                                         # fp32 atomics in a different order: relative difference
            a, b = old().clone(), new().clone()
            row["max_rel_diff"] = float((a - b).abs().max() / a.abs().max())
        rows.append(row)
        o, nw = row["old"], row["new"]
        print("%-3s %-6s %7.1f GFLOP  old %8.1f us %6.1f TFLOP/s %5.1f%%   new %s%s" % (
            name, kind, row["gflop"], o["us"], o["tflops"], 100 * o["of_peak"],
            "%8.1f us %6.1f TFLOP/s %5.1f%%" % (nw["us"], nw["tflops"], 100 * nw["of_peak"]),
            "  max rel diff %.1e" % row["max_rel_diff"] if kind == "wgrad" else
            ("  identical" if row["bit_identical"] else "  DIFFERENT")), flush=True)
    tot = {arm: sum(r[arm]["us"] for r in rows) for arm in ("old", "new")}
    print("all 18 calls: old %.1f us, new %.1f us" % (tot["old"], tot["new"]))
    return {"batch": args.batch, "iters_per_graph": args.iters, "rounds": args.rounds, "peaks": pk, "calls": rows,
            "total_us": tot}


# operand bytes loaded from L2 per FLOP: a 64-deep K block of a 128 x 128 tile (ping-pong), of two 128-pixel tiles sharing
# one 128-wide weight box (256-pixel kernel), of a 128 x 256 weight-gradient tile (RB rows: the same ratio)
B_PER_FLOP = {"pp128": 32768 / (2 * 128 * 128 * 64), "m256": 49152 / (2 * 256 * 128 * 64),
              "wgrad": (128 + 256) * 128 / (2 * 128 * 256 * 64), "wgrad_n192": (128 + 192) * 128 / (2 * 128 * 192 * 64)}


def changed_calls(n, dev):
    """[(layer, kind, flop, {arm: (fn, bytes per FLOP)})] on seeded bf16 operands."""
    from megreader_b200 import crnn_engine
    g = torch.Generator(device=dev).manual_seed(0)
    out = []
    for name, H, W, C, Cout, k, p in LAYERS:
        Ho, Wo = H + 2 * p - k + 1, W + 2 * p - k + 1
        flop = 2.0 * n * Ho * Wo * Cout * k * k * C
        x = torch.randn((n, H, W, C), generator=g, device=dev).to(torch.bfloat16)
        Wm = (torch.randn((Cout, k * k * C), generator=g, device=dev) / (k * k * C) ** 0.5).to(torch.bfloat16)
        dz = torch.randn((n, Ho, Wo, Cout), generator=g, device=dev).to(torch.bfloat16)
        Wd = (torch.randn((C, k * k * Cout), generator=g, device=dev) / (k * k * Cout) ** 0.5).to(torch.bfloat16)
        dW = torch.zeros((Cout, k * k * C), dtype=torch.float32, device=dev)
        for kind, a, w, pad, kb in (("fprop", x, Wm, p, k * k * C // 64), ("dgrad", dz, Wd, k - 1 - p, k * k * Cout // 64)):
            sel = "m256" if kb >= 36 else "pp128"
            arms = {"pp128": (lambda a=a, w=w, k=k, pad=pad: ops.conv_fprop_pp(a, w, k, k, pad, pad, tile_m=128)[0],
                              B_PER_FLOP["pp128"]),
                    "selected": (lambda a=a, w=w, k=k, pad=pad: ops.conv_fprop_pp(a, w, k, k, pad, pad)[0],
                                 B_PER_FLOP[sel])}
            if kind == "dgrad" and Ho == 1:
                arms["rows"] = (lambda a=a, w=w, k=k, p=p, H=H: crnn_engine._conv_dgrad(a, w, k, k, p, p, H),
                                B_PER_FLOP["pp128"])
            out.append((name, kind, flop, arms))
        arms = {"selected": (lambda dz=dz, x=x, k=k, p=p, dW=dW: ops.conv_wgrad_pp(dz, x, k, k, p, p, out=dW.zero_()),
                             B_PER_FLOP["wgrad"])}
        if k * k * C % 256 and k * k * C % 192 == 0:  # the engine runs these on 128 x 192 tiles
            arms["engine"] = (lambda dz=dz, x=x, k=k, p=p, dW=dW: crnn_engine._conv_wgrad(dz, x, k, k, p, p, out=dW.zero_()),
                              B_PER_FLOP["wgrad_n192"])
        out.append((name, "wgrad", flop, arms))
    return out


def wgrad_useful_mma(name, n, sms, n192=False):
    """Share of the weight gradient's issued MMA work that multiplies real operands: the useful products over the K blocks
    (RB pixels each, zero fill included) x 128 x 256 tiles of mr_conv_wgrad_pp's plan (n192: x 128 x 192 tiles of
    mr_conv_wgrad_n192's)."""
    _, H, W, C, Cout, k, p = next(lay for lay in LAYERS if lay[0] == name)
    Ho, Wo = H + 2 * p - k + 1, W + 2 * p - k + 1
    plan = (ops.conv_wgrad_n192_plan if n192 else ops.conv_wgrad_pp_plan)(n, H, W, C, Cout, k, k, p, p, sms)
    return n * Ho * Wo * Cout * k * k * C / (plan["kb_total"] * plan["RB"] * plan["tiles"] * 128 * (192 if n192 else 256))


def run_changed(args):
    dev = torch.device("cuda:0")
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    cs = changed_calls(args.batch, dev)
    times = defaultdict(list)
    for _ in range(args.rounds):
        for i, (_, _, _, arms) in enumerate(cs):
            for arm, (fn, _) in arms.items():
                times[(i, arm)].append(bench._graph_time(fn, args.iters))
    rows = []
    for i, (name, kind, flop, arms) in enumerate(cs):
        row = {"layer": name, "kind": kind, "gflop": flop * 1e-9}
        ref = None
        for arm, (fn, bpf) in arms.items():
            ts = times[(i, arm)]
            t = sorted(ts)[len(ts) // 2]
            row[arm] = {"us": t * 1e6, "us_all": [v * 1e6 for v in ts], "tflops": flop / t * 1e-12,
                        "l2_tb_s": flop / t * bpf * 1e-12}
            if kind != "wgrad":
                r = fn()
                ref = r.clone() if ref is None else ref
                row[arm]["same_bits_as_pp128"] = bool(torch.equal(r.view_as(ref), ref))
        if kind == "wgrad":
            row["useful_mma"] = wgrad_useful_mma(name, args.batch, sms)
            if "engine" in arms:
                row["engine"]["useful_mma"] = wgrad_useful_mma(name, args.batch, sms, n192=True)
        rows.append(row)
        print("%-3s %-6s %s" % (name, kind, "  ".join(
            "%s %7.1f us (%s) %6.1f TFLOP/s L2 %4.1f TB/s%s" % (
                arm, v["us"], "/".join("%.0f" % u for u in v["us_all"]), v["tflops"], v["l2_tb_s"],
                "" if v.get("same_bits_as_pp128", True) else " DIFFERENT")
            for arm, v in row.items() if isinstance(v, dict)) +
            ("  useful MMA %.1f %% of issued" % (100 * row["useful_mma"]) if kind == "wgrad" else "") +
            (" (engine %.1f %%)" % (100 * row["engine"]["useful_mma"]) if "engine" in row else "")), flush=True)
    return {"batch": args.batch, "iters_per_graph": args.iters, "rounds": args.rounds, "calls": rows}


def kernel_family(name):
    m = re.match(r"(?:void )?(?:\(anonymous namespace\)::)?([\w:]+?)(?:<|\(|$)", name)
    return m.group(1) if m else name


def run_profile(args):
    from torch.profiler import DeviceType, ProfilerActivity, profile
    from megreader_b200 import crnn_engine
    dev = torch.device("cuda:0")
    torch.backends.cudnn.benchmark = True
    net = bench.build_model(dev)
    crnn_engine.set_compute_dtype(torch.bfloat16)
    opt = torch.optim.Adam(net.parameters(), lr=1e-3, fused=True)
    x, y, l = [t.to(dev) for t in bench.synth_batch(0, args.batch)]

    def step():
        opt.zero_grad(set_to_none=True)
        loss, _ = net(x, y, l)
        loss.mean().backward()
        opt.step()

    for _ in range(3):
        step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            step()
        torch.cuda.synchronize()
    per = defaultdict(lambda: [0.0, 0])
    for e in prof.events():
        if e.device_type == DeviceType.CUDA:
            k = kernel_family(e.name)
            per[k][0] += e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
            per[k][1] += 1
    total = sum(v[0] for v in per.values())
    rows = sorted(({"kernel": k, "us_per_step": v[0] / args.steps, "launches_per_step": v[1] / args.steps,
                    "share": v[0] / total} for k, v in per.items()), key=lambda r: -r["us_per_step"])
    conv = sum(r["us_per_step"] for r in rows if re.match(r"conv_(fprop|wgrad)_", r["kernel"]))
    for r in rows[:25]:
        print("%9.1f us  %5.1f%%  %6.1f x  %s" % (r["us_per_step"], 100 * r["share"], r["launches_per_step"], r["kernel"]))
    print("kernel time per step %.1f us; implicit convolutions %.1f us (%.1f%%)" % (total / args.steps, conv,
                                                                                     100 * conv * args.steps / total))
    return {"batch": args.batch, "steps": args.steps, "kernel_us_per_step": total / args.steps,
            "conv_us_per_step": conv, "conv_share": conv * args.steps / total, "kernels": rows}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--out", required=True, help="directory for the JSON record")
    ap.add_argument("--batch", type=int, default=bench.BATCH_PER_GPU)
    ap.add_argument("--iters", type=int, default=20, help="launches per CUDA graph")
    ap.add_argument("--rounds", type=int, default=3, help="alternating old / new rounds (the median is reported)")
    ap.add_argument("--profile", action="store_true", help="(b): profile whole training steps instead")
    ap.add_argument("--changed", action="store_true", help="(c): the persistent kernels against each other")
    ap.add_argument("--steps", type=int, default=3, help="profiled steps for --profile")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("crnn_conv_layers: needs a CUDA device")
    info = card()
    rec = run_profile(args) if args.profile else run_changed(args) if args.changed else run_layers(args)
    rec["card"] = info
    os.makedirs(args.out, exist_ok=True)
    path = os.path.join(args.out, "crnn_conv_profile.json" if args.profile else
                        "crnn_conv_changed.json" if args.changed else "crnn_conv_layers.json")
    with open(path, "w") as f:
        json.dump(rec, f, indent=1)
    print("card: %s" % json.dumps(info))
    print("wrote", path)


if __name__ == "__main__":
    main()
