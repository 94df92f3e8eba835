"""Lexicon-constrained CTC decoding (megreader_b200.lexicon.decode_packed) timed as CUDA-graph replays, next to the float64
restatement (tests/lexicon_port.py) on one CPU core.

    python -m benchmarks.lexicon_decode [--iters 20] [--host-samples 2]

Workloads, at crnn.yaml's input (32 x 128, W = 33) and community-base.yaml's (64 x 256, W = 65), C = 38: N = 3,000 with
per-image lists of 50 and of 1,000 words (IIIT5K-50 / 1k style, every word scored), N = 512 with one shared list of 50,000
words at delta = 3 and delta = None, and the 2D head at H = 8 with per-image lists of 50.  The probabilities are peaked
synthetic softmax outputs (a random word spelled with blanks between letters, over noise), so delta = 3 keeps the near
misses of the greedy result.  The host column is the restatement's time per sample on --host-samples samples with one torch
thread; it is the per-image word loop a user without the device path would run.  One JSON line per workload."""
import argparse
import json
import subprocess
import time

import numpy as np
import torch

from tests import lexicon_cases as lc
from tests import lexicon_port as port


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:
        q = torch.cuda.get_device_name()
    return q


def synth(rng, N, W, H, dev):
    """peaked probabilities (N, C, H, W) and, for H > 1, a mask; the words they spell"""
    truths = [lc.random_word(rng, 3, min(10, W // 2)) for _ in range(N)]
    z = np.empty((N, lc.C, 1, W), np.float32)
    for n, t in enumerate(truths):
        z[n, :, 0] = lc.peaked_logits(rng, t, W, 9.0)
    z = torch.from_numpy(z).to(dev)
    if H > 1:
        z = z + 0.3 * torch.randn((N, lc.C, H, W), device=dev, generator=torch.Generator(dev).manual_seed(1))
    prob = torch.softmax(z, 1)
    mask = torch.softmax(2 * torch.randn((N, 1, H, W), device=dev, generator=torch.Generator(dev).manual_seed(2)), 2) \
        if H > 1 else None
    return prob, mask, truths


def random_words(rng, n, lo, hi):
    lens = rng.integers(lo, hi + 1, n)
    chars = np.array(list(lc.LETTERS))[rng.integers(0, len(lc.LETTERS), int(lens.sum()))]
    return ["".join(w) for w in np.split(chars, np.cumsum(lens)[:-1])]


def per_image_lists(rng, truths, size):
    """the truth, 24 near misses of it (1 to 3 edits) and random words"""
    pool = iter(random_words(rng, len(truths) * (size - 25), 2, 10))
    out = []
    for t in truths:
        ws = [lc.edit(rng, t, int(rng.integers(1, 4))) for _ in range(24)] + [next(pool) for _ in range(size - 25)]
        ws.insert(int(rng.integers(0, size)), t)
        out.append(ws)
    return out


def time_graph(fn, iters):
    fn()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    for _ in range(3):
        g.replay()
    torch.cuda.synchronize()
    times = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        g.replay()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return float(np.median(times)), float(np.min(times)), float(np.max(times))


def run(name, W, H, N, layout, size, delta, args, dev, rng):
    from megreader_b200 import lexicon
    prob, mask, truths = synth(rng, N, W, H, dev)
    if layout == "per_image":
        words, ranges = lexicon.WordList.per_image(per_image_lists(rng, truths, size), lc.CS, dev)
    else:
        shared = sorted(set(random_words(rng, int(size * 1.2), 1, 10)) | set(truths[:size // 10]))[:size]
        words, ranges = lexicon.WordList(shared, lc.CS, dev), None
    out = lexicon.decode_packed(prob, words, ranges, delta, mask=mask)
    med, lo, hi = time_graph(lambda: lexicon.decode_packed(prob, words, ranges, delta, mask=mask, out=out), args.iters)
    cand = int(out["candidates"].sum())
    k = args.host_samples
    ids = [lc.ids(w) for w in words.words[:len(words) if ranges is None else int(ranges[k - 1, 1])]]
    torch.set_num_threads(1)
    t0 = time.perf_counter()
    want = port.decode(prob[:k].cpu(), ids, None if ranges is None else ranges[:k].cpu().numpy(), delta,
                       None if mask is None else mask[:k].cpu())
    host_ms = (time.perf_counter() - t0) * 1e3 / k
    agree = int((out["word"][:k].cpu().numpy() == want["word"]).sum())
    return dict(workload=name, N=N, W=W, H=H, words_per_sample=size, delta=delta, device_ms=round(med, 3),
                device_ms_min=round(lo, 3), device_ms_max=round(hi, 3), candidates=cand,
                pairs_per_s=round(cand / (med * 1e-3)), host_ms_per_sample=round(host_ms, 2), host_samples=k,
                host_agrees=f"{agree}/{k}", speedup_vs_host=round(host_ms * N / med, 1))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--host-samples", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("benchmarks.lexicon_decode: needs a CUDA device")
    dev = torch.device("cuda:0")
    print(json.dumps(dict(gpu=gpu_info())), flush=True)
    rng = np.random.default_rng(0)
    for W in (33, 65):
        for name, N, layout, size, delta in (("per_image_50", 3000, "per_image", 50, None),
                                             ("per_image_1000", 3000, "per_image", 1000, None),
                                             ("shared_50k_d3", 512, "shared", 50000, 3),
                                             ("shared_50k_all", 512, "shared", 50000, None)):
            print(json.dumps(run(name, W, 1, N, layout, size, delta, args, dev, rng)), flush=True)
    print(json.dumps(run("2d_h8_per_image_50", 33, 8, 3000, "per_image", 50, None, args, dev, rng)), flush=True)


if __name__ == "__main__":
    main()
