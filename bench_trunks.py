"""bench.py --config 3 | 4 | 5: the other configurations of BASELINE.json, same JSON contract as the headline line;
benchmarks/db_step.py runs config 6.

  config 3   resnet50dilated_ppm + CTCDecoder2D (res50-ppm-2d-ctc.yaml), 3x64x256 lines, feature map 8x32, 2D-CTC loss
  config 4   Resnet50FPN + AttentionDecoder (fpn50-attention-decoder.yaml), 3x64x256 lines (SURVEY.md D3)
  config 6   deformable_resnet50 + SegDetector(adaptive, k=50) + L1BalanceCELoss (seg_detector_db.yaml), 3x640x640 scenes, per-GPU
             batch 16, SGD (momentum 0.9, weight decay 1e-4) as in the yaml; the DB tail and loss on csrc/db_head.cu

One "step" = forward + backward + Adam (config 6: SGD) on one synthetic batch (per-GPU batch 32 = BASELINE's 256 over 8 GPUs;
config 5: 8, config 6: 16; --batch overrides).
bf16 compute on the repo's kernels: every convolution of trunk and head runs on the wgmma implicit-GEMM kernels
(megreader_b200.conv_engine), the 2D-CTC head epilogue + loss on csrc/ctc2d_head.cu + csrc/ctc2d.cu, the attention decoder's recurrent
loop on csrc/attn_decode.cu, the deformable units on csrc/dcn_tcgen05.cu, BatchNorm on the NHWC row kernels of csrc/nn_kernels.cu;
ReLU / residual adds / pooling / interpolation are library (ATen) kernels.  The step is captured in CUDA graphs (MR_BENCH_EAGER=1: eager launches).
"""
import os
import time

import numpy as np
import torch

CFG = {
    3: dict(name="ResNet50-dilated-PPM + 2D-CTC head (res50-ppm-2d-ctc.yaml)", hw=(64, 256), backbone="resnet50dilated_ppm",
            decoder="CTCDecoder2D", l_max=12),
    # BASELINE.json quotes 48x160, but the head's encoder (three height-halving pools + a 2-row closing conv,
    # decoders/attention_decoder.py:41-66) needs a 16-row feature map = 64 input rows at the FPN's stride 4 (SURVEY.md D3)
    4: dict(name="ResNet50-FPN + attention decoder (fpn50-attention-decoder.yaml)", hw=(64, 256), backbone="Resnet50FPN",
            decoder="AttentionDecoder", l_max=12),
    # no EAST yaml exists in the reference; SURVEY.md D4: FeaturePyramid(deformable_resnet50, FPNTopDown) -> EASTDecoder
    5: dict(name="deformable ResNet50 (DCNv2) + FPN + EAST head (SURVEY.md D4 composition)", hw=(512, 512), backbone="deformable_resnet50+FPN",
            decoder="EASTDecoder", l_max=0),
    6: dict(name="deformable ResNet50 (DCNv2) + DB head + L1BalanceCELoss (seg_detector_db.yaml)", hw=(640, 640),
            backbone="deformable_resnet50", decoder="SegDetector", l_max=0),
}


def synth_east(seed, n, hw):
    """SURVEY.md section 8d: uint8-like scenes, all-zero heat maps / dense boxes with unit weights (loss arithmetic only)."""
    rng = np.random.RandomState(seed)
    x = (rng.standard_normal((n, 3, hw[0], hw[1])) * 60 + 110).clip(0, 255).astype(np.float32)
    z = lambda c: torch.zeros(n, c, hw[0], hw[1])  # noqa: E731
    return torch.from_numpy(x), {"heatmap": z(1), "heatmap_weight": z(1) + 1, "densebox": z(8), "densebox_weight": z(8) + 1}


def synth(seed, n, hw, l_max, S=32, n_classes=38):
    rng = np.random.RandomState(seed)
    x = rng.standard_normal((n, 3, hw[0], hw[1])).astype(np.float32)
    lengths = rng.randint(1, l_max + 1, size=n).astype(np.int64)
    labels = np.zeros((n, S), np.int32)
    for b in range(n):
        labels[b, :lengths[b]] = rng.randint(2, n_classes, size=lengths[b])
    return torch.from_numpy(x), torch.from_numpy(labels), torch.from_numpy(lengths)


def _map(t, fn):
    if t is None:
        return None
    if isinstance(t, dict):
        return {k: fn(v) for k, v in t.items()}
    return fn(t)


def _nbytes(t):
    if t is None:
        return 0
    if isinstance(t, dict):
        return sum(v.numel() * v.element_size() for v in t.values())
    return t.numel() * t.element_size()


def synth_db(seed, n, hw):
    """seeded images + DB targets (tests/db_data.py: random axis-aligned / rotated text boxes, 5-15 % positive pixels)."""
    from tests.db_data import db_batch, db_images
    lab = {k: torch.from_numpy(v) for k, v in db_batch(seed, n, hw[0], hw[1]).items()}
    return torch.from_numpy(db_images(seed, n, hw[0], hw[1])), lab


def make_batch(cfg, seed, n):
    c = CFG[cfg]
    if cfg == 6:
        x, lab = synth_db(seed, n, c["hw"])
        return x, lab, None
    if cfg == 5:
        x, lab = synth_east(seed, n, c["hw"])
        return x, lab, None
    return synth(seed, n, c["hw"], c["l_max"])


def build(cfg, device, engine=True, wgrad_side_stream=None):
    import megreader_b200
    megreader_b200.install_reference_api()
    import backbones
    import decoders
    from tests.weights import fill_state_dict
    c = CFG[cfg]
    if cfg == 6:                         # seg_detector_db.yaml: SegDetectorModel(deformable_resnet50, SegDetector) + L1BalanceCELoss
        from decoders.seg_detector_loss import L1BalanceCELoss
        bb = backbones.deformable_resnet50(pretrained=False)
        dec = decoders.SegDetector(adaptive=True, in_channels=[256, 512, 1024, 2048], k=50)
        criterion = L1BalanceCELoss()
    elif cfg == 5:
        from backbones.feature_pyramid import FeaturePyramid
        from backbones.fpn_top_down import FPNTopDown
        bb = FeaturePyramid(backbones.deformable_resnet50(pretrained=False), FPNTopDown([2048, 1024, 512, 256], 256))
        dec = decoders.EASTDecoder(channels=256)
    else:
        bb = getattr(backbones, c["backbone"])(resnet_pretrained=False)
        dec = getattr(decoders, c["decoder"])(in_channels=256)

    class Net(torch.nn.Module):          # structure/model.py:16-24 BasicModel: decoder(backbone(x), **kw)
        def __init__(self):
            super().__init__()
            self.backbone = fill_state_dict(bb, "bb%d." % cfg)
            self.decoder = fill_state_dict(dec, "dec%d." % cfg)

        def forward(self, images, targets, lengths):
            if cfg == 6:                 # structure/model.py:140-155 SegDetectorModel: criterion(decoder(backbone(x)), batch)
                pred = self.decoder(self.backbone(images), training=True)
                loss, _ = criterion(pred, targets)
                return loss, pred
            if cfg == 5:                 # structure/model.py:63-87 DetectionModel: decoder(feature, label, meta, train)
                loss, pred, _ = self.decoder(self.backbone(images), targets, None, True)
                return loss, pred
            return self.decoder(self.backbone(images), targets=targets, lengths=lengths, train=True)
    net = Net().to(device).train()
    n_engine = 0
    if engine:
        from megreader_b200 import conv_engine
        n_engine = conv_engine.use_engine_convs(net, wgrad_side_stream=wgrad_side_stream)
    return net, n_engine


def conv_roofline(dev, peaks, cfg):
    """dominant contraction of the trunk on this repo's kernel: the dilated 3x3 512->512 convolution of layer4 (config 3:
    8x32 map) / the 3x3 512->512 of layer4 at stride-32 resolution (config 4), timed alone with CUDA events."""
    from megreader_b200 import nnops
    N = 256
    H, W, C, d = (8, 32, 512, 4) if cfg == 3 else ((16, 16, 512, 1) if cfg in (5, 6) else (6, 20, 512, 1))
    x = torch.randn(N, H, W, C, device=dev).bfloat16()
    wm = (torch.randn(C, 9 * C, device=dev) / 68).bfloat16()
    fn = lambda: nnops.conv2d_fprop_tc(x, wm, 3, 3, 1, 1, d, d, d, d)  # noqa: E731
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(10):
        fn()
    b.record()
    torch.cuda.synchronize()
    sec = a.elapsed_time(b) / 10 * 1e-3
    flops = 2.0 * N * H * W * C * 9 * C
    return {"kernel": "conv_fprop_tcgen05_kernel (3x3 512->512, dilation %d, %dx%d map, batch %d)" % (d, H, W, N),
            "bound": "tensor", "achieved": flops / sec / 1e12, "peak": peaks["bf16_tflops"], "unit": "TFLOP/s",
            "frac": flops / sec / 1e12 / peaks["bf16_tflops"], "traffic": None, "peak_source": peaks["source"],
            "alg_flops_per_launch": flops, "us_per_launch": sec * 1e6}


def cpu_arm(cfg, sample_n, steps, budget_s=25.0):
    """The same modules on the host cores (the reference's CPU path for these configurations is plain PyTorch modules; the
    native 2D-CTC op has no CPU implementation in the reference, so the config-3 arm times trunk + head convolutions
    forward + backward and says so)."""
    import megreader_b200
    megreader_b200.install_reference_api()
    import backbones
    from tests.weights import fill_state_dict
    c = CFG[cfg]
    cores = max(1, min(32, len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)))
    torch.set_num_threads(cores)
    if cfg in (5, 6):
        return {"value": None, "unit": "lines/s", "cores": cores, "kind": "port",
                "sample": "not timed: the reference has no CPU implementation of the DCN op (functions/deform_conv.py:40-41 raises)"}
    bb = fill_state_dict(getattr(backbones, c["backbone"])(resnet_pretrained=False), "bb%d." % cfg).train()
    x, _, _ = synth(0, sample_n, c["hw"], c["l_max"])
    opt = torch.optim.Adam(bb.parameters(), lr=1e-3)

    def step():
        opt.zero_grad()
        out = bb(x)
        out = out[-1] if isinstance(out, (tuple, list)) else out
        out.float().square().mean().backward()
        opt.step()
    step()
    t0 = time.perf_counter()
    done = 0
    for _ in range(steps):
        step()
        done += 1
        if time.perf_counter() - t0 > budget_s:
            break
    dt = time.perf_counter() - t0
    return {"value": sample_n * done / dt, "unit": "lines/s", "cores": cores, "kind": "port",
            "sample": "%d steps of a %d-line batch through the %s trunk (forward + backward + Adam, torch CPU fp32, %d threads); the "
                      "decoder / loss are not in this arm" % (done, sample_n, c["backbone"], cores),
            "ms_per_step": dt / done * 1e3}


def run(args, peaks, ClockSampler, emit_json):
    import torch.distributed as dist
    from megreader_b200 import _lib, dp
    cfg = args.config
    c = CFG[cfg]
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    torch.manual_seed(0)
    batch = args.batch or {5: 8, 6: 16}.get(cfg, 32)        # BASELINE.json: 256 (cfg 3/4) and 64 (cfg 5) over 8 GPUs; yaml: 16 (cfg 6)
    # one GPU: the convolutions' weight gradients run on a side stream (nothing reads a gradient before backward() returns here);
    # N > 1: they accumulate into the flat all-reduce buffer on the backward's stream.  MR_CONV_WGRAD_SIDE_STREAM=0 switches it off.
    side_wgrad = world == 1 and os.environ.get("MR_CONV_WGRAD_SIDE_STREAM", "1") != "0"
    net, n_engine = build(cfg, dev, wgrad_side_stream=side_wgrad)
    params = [p for p in net.parameters() if p.requires_grad]
    if cfg == 6:                                             # seg_detector_db.yaml: SGD lr 0.007, momentum 0.9, weight decay 1e-4
        opt = torch.optim.SGD(params, lr=0.007, momentum=0.9, weight_decay=1e-4)
        opt_name, opt_desc = "SGD", "SGD lr 0.007 momentum 0.9 weight decay 1e-4"
    else:
        opt = torch.optim.Adam(params, lr=1e-3, fused=True, capturable=True)
        opt_name, opt_desc = "Adam", "Adam lr 1e-3"
    # N > 1: gradients as views of one flat buffer, ONE in-place NCCL all-reduce (AVG) between the two graphs (megreader_b200/dp.py)
    fg = dp.FlatGrads(params) if world > 1 else None
    host = []
    for i in range(3):
        hb = make_batch(cfg, 100 * rank + i, batch)
        host.append(tuple(_map(t, lambda v: v.pin_memory()) for t in hb))
    dev_batches = [tuple(_map(t, lambda v: v.to(dev)) for t in hb) for hb in host]
    static = tuple(_map(t, lambda v: torch.empty_like(v)) for t in dev_batches[0])
    # config 4: the attention head's per-step random draws (teacher-forcing coin, step dropout) are made on the host before every
    # step in the reference's order and copied into static device tensors the captured forward reads (decoder.feedback_static)
    attn = net.decoder if cfg == 4 else None
    fb_static = None
    if attn is not None:
        fb_static = tuple(t.to(dev) for t in attn.draw_feedback(batch))
        attn.feedback_static = fb_static

    def refresh_feedback():
        if attn is not None:
            for dst, src in zip(fb_static, attn.draw_feedback(batch)):
                dst.copy_(src.pin_memory(), non_blocking=True)

    def fwd_bwd(x, y, l):
        if fg is not None:
            fg.zero()
        else:
            opt.zero_grad(set_to_none=True)
        loss, _ = net(x, y, l)
        loss = loss.mean()
        loss.backward()
        return loss

    def eager_step(x, y, l):
        refresh_feedback()
        loss = fwd_bwd(x, y, l)
        if fg is not None:
            fg.allreduce_()
        opt.step()
        return loss

    def barrier():
        if world > 1:
            dist.barrier(device_ids=[local])
        torch.cuda.synchronize()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for i in range(3):
            eager_step(*dev_batches[i % 3])
    torch.cuda.current_stream().wait_stream(side)
    barrier()
    _lib.reset_launch_count()
    eager_step(*dev_batches[0])
    torch.cuda.synchronize()
    launches_per_step = _lib.launch_count()
    # the step as CUDA graphs (graph A = zero + forward + backward [+ Adam when N = 1]; N > 1: NCCL all-reduce, then graph B = Adam):
    # ~4,000 launches per step are otherwise bound by the host.  MR_BENCH_EAGER=1 keeps the eager launch mode; a capture that fails
    # (every rank decides together) falls back to it and says so -- the kernels are the same either way.
    graph_a = graph_b = static_loss = None
    launch_mode = "eager (MR_BENCH_EAGER=1)"
    if not os.environ.get("MR_BENCH_EAGER"):
        ok = torch.ones(1, device=dev)
        try:
            graph_a = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph_a):
                static_loss = fwd_bwd(*static)
                if world == 1:
                    opt.step()
            if world > 1:
                graph_b = torch.cuda.CUDAGraph()
                with torch.cuda.graph(graph_b, pool=graph_a.pool()):
                    opt.step()
            launch_mode = "step captured in CUDA graph(s)" + ("; the NCCL all-reduce runs between two graphs" if world > 1 else "")
        except Exception as e:                         # launch mode only: the eager step runs the same kernels
            ok.zero_()
            launch_mode = "eager (CUDA-graph capture failed: %s)" % str(e).replace("\n", " ")[:160]
            torch.cuda.synchronize()
        if world > 1:
            dist.all_reduce(ok, op=dist.ReduceOp.MIN)
        if float(ok.item()) == 0.0:
            graph_a = graph_b = None
            if not launch_mode.startswith("eager"):
                launch_mode = "eager (CUDA-graph capture failed on another rank)"

    def step(x, y, l):
        if graph_a is None:
            return eager_step(x, y, l)
        refresh_feedback()
        for dst, src in zip(static, (x, y, l)):
            if dst is None:
                continue
            if isinstance(dst, dict):
                for k in dst:
                    dst[k].copy_(src[k], non_blocking=True)
            else:
                dst.copy_(src, non_blocking=True)
        graph_a.replay()
        if graph_b is not None:
            fg.allreduce_()
            graph_b.replay()
        return static_loss
    for i in range(max(3, args.warmup)):
        step(*dev_batches[i % 3])
    barrier()
    sampler = ClockSampler(local) if rank == 0 else None
    if sampler:
        sampler.start()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    barrier()
    e0.record()
    for i in range(args.steps):
        loss = step(*dev_batches[i % 3])
    e1.record()
    barrier()
    ms = e0.elapsed_time(e1)
    clocks = sampler.stop() if sampler else None
    final_loss = float(loss.item())
    # end to end: pinned host batches, copies inside the timed region, loss read back every step
    copy_stream = torch.cuda.Stream()
    h2d = sum(_nbytes(t) for t in host[0])

    def fetch(i):
        with torch.cuda.stream(copy_stream):
            b = tuple(_map(t, lambda v: v.to(dev, non_blocking=True)) for t in host[i % 3])
            ev = torch.cuda.Event()
            ev.record(copy_stream)
        return b, ev

    def e2e_loop(k):
        nxt = fetch(0)
        for i in range(k):
            (x, y, l), ev = nxt
            torch.cuda.current_stream().wait_event(ev)
            if i + 1 < k:
                nxt = fetch(i + 1)
            float(step(x, y, l).item())
    e2e_loop(3)
    barrier()
    f0, f1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    f0.record()
    e2e_loop(args.steps)
    f1.record()
    barrier()
    ms_e2e = f0.elapsed_time(f1)
    t = torch.tensor([ms, ms_e2e], device=dev, dtype=torch.float64)
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    ms, ms_e2e = float(t[0]), float(t[1])
    lines = batch * world * args.steps
    out = {
        "metric": "%s/sec %s train step (fwd+bwd+%s), %dx%d inputs, batch %d/GPU" % ("scenes" if cfg in (5, 6) else "text-lines", c["name"], opt_name, c["hw"][0], c["hw"][1], batch),
        "value": lines / (ms / 1e3), "unit": "scenes/s" if cfg in (5, 6) else "lines/s", "n_gpus": world, "steps": args.steps, "warmup": max(3, args.warmup),
        "ms_per_step": ms / args.steps, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "bf16",
        "data": "synthetic",
        "config": {"workload": "%s, 3x%dx%d fp32 input, bf16 compute, %s" % (c["name"], c["hw"][0], c["hw"][1], opt_desc),
                   "batch_per_gpu": batch, "global_batch": batch * world, "parallelism": "dp%d" % world,
                   "l2": "3 rotating input batches; weights + gradients + Adam state (> 400 MB) and activations exceed the 50 MB L2"},
        "e2e": {"value": lines / (ms_e2e / 1e3), "unit": "scenes/s" if cfg in (5, 6) else "lines/s", "h2d_bytes_per_step": h2d, "d2h_bytes_per_step": 4,
                "ms_per_step": ms_e2e / args.steps},
        "gpu_launches": launches_per_step * args.steps, "final_loss": final_loss, "clocks": clocks,
        "engine_convs": n_engine,
    }
    if rank == 0:
        out["roofline"] = conv_roofline(dev, peaks, cfg)
        out["cpu_baseline"] = cpu_arm(cfg, 2, 3)
        out["stages"] = {"convolutions (trunk + head, %d layers)" % n_engine: "megreader_b200 wgmma implicit-GEMM kernels (fprop, dgrad, wgrad)",
                         "BatchNorm": "megreader_b200 NHWC row kernels (conv_engine.EngineBatchNorm2d: column statistics through block partials, "
                                      "row-tiled normalisation, fused backward)",
                         "ReLU / residual add / pooling / interpolation": "library (ATen, channels_last bf16)",
                         "head": ("megreader_b200 fused 2D-CTC epilogue + DP kernels" if cfg == 3 else
                                  "attention decoder: the 32-step loop and its backward through time = megreader_b200 persistent cooperative kernels (csrc/attn_decode.cu), hoisted encoder projection; weight-gradient products over the saved rows: library GEMMs" if cfg == 4 else
                                  "DB head: convolutions and the 2x2 stride-2 transposed convolutions on the conv engine; sigmoid + step function and "
                                  "L1BalanceCELoss (hard-negative mining by an on-device radix select) on csrc/db_head.cu; "
                                  "DCNv2 units: fused wgmma kernels (csrc/dcn_tcgen05.cu)" if cfg == 6 else
                                  "EAST head: 3x3 / 1x1 convolutions and the 2x2 stride-2 transposed convolutions (as 1x1 convolutions + depth-to-space) on the conv engine, losses library; "
                                  "DCNv2 units: fused wgmma forward / weight-gradient / data-gradient kernels (csrc/dcn_tcgen05.cu)"),
                         "conv weight gradients": "side stream, joined at the end of the backward pass (conv_engine.WGRAD_SIDE_STREAM)"
                                                  if side_wgrad else "the backward's stream",
                         opt_name: "library (torch SGD, foreach)" if cfg == 6 else "library (torch fused, capturable)", "launch": launch_mode}
        emit_json(out)
    if world > 1:
        dist.destroy_process_group()
