"""Time the text recognisers' validation measure on the device (megreader_b200.rec_measure) and the host path it replaces.

    python benchmarks/rec_measure.py

  * measure_labels alone, eager and replayed as a CUDA graph, at N = 16 / 512 / 4,096 and widths 33 / 65, with and without a
    lexicon of 3,209 random words (the size of the reference's train_lexicon.txt; 3,133 unique after the set);
  * a whole validation step in one graph (engine CRNN eval + ctc_greedy_decode + measure_labels with totals) at crnn.yaml's
    validation batch 16 x 3 x 32 x 128 and at the bench shape 512 x 3 x 32 x 256;
  * the host path on the same labels, on one core: the plain-Python restatement's representer loop (label_to_string, and the
    CTC collapse where the rows are argmax rows: the validation-step rows), its measurer and its gather_measure.  This is a
    host-side estimate, not the reference.  Its Levenshtein runs in Python / numpy, slower than editdistance's C.  Its loops
    run over host lists, faster than the reference's loops over CUDA tensor elements, which read the device once per element.
Device times are CUDA events after warm-up, median of 5 windows; the card's name and power limit are printed with them."""
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()[0]
    except Exception:
        q = torch.cuda.get_device_name()
    return q


def events_ms(fn, iters):
    ts = []
    for _ in range(5):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b) / iters)
    return float(np.median(ts))


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


def host_path(gt, pred, cs, words, collapse=False):
    """the restatement's represent (with the CTC collapse of argmax rows when `collapse`), measure and gather_measure on one
    core: seconds"""
    from oracle import rec_measure_port as port
    t = time.perf_counter()
    rows = [port.collapse(r, cs.blank, cs.unknown) for r in pred.tolist()] if collapse else pred.tolist()
    out = [{'label_string': port.fold(cs, g), 'pred_string': port.fold(cs, p)} for g, p in zip(gt.tolist(), rows)]
    m = port.SequenceRecognitionMeasurer(words)
    m.gather_measure([m.measure(None, out)])
    return time.perf_counter() - t


def main():
    import bench
    from megreader_b200 import decode, rec_measure
    from megreader_b200.charset import EnglishCharset
    from tests import rec_measure_cases as cases
    dev = torch.device("cuda:0")
    cs = EnglishCharset()
    table = rec_measure.fold_table(cs, dev)
    rng = np.random.default_rng(0)
    words = ["".join(rng.choice(list("ABCDEFGHIJKLMNOPQRSTUVWXYZ"), int(rng.integers(2, 12)))) for _ in range(3209)]
    lexicon = rec_measure.Lexicon(words, dev)
    rows = []
    print(json.dumps({"card": card(), "torch": torch.__version__}))
    for N in (16, 512, 4096):
        for W in (33, 65):
            gt_np, pred_np = cases.pair_corpus(rng, len(cs), N, 32 if W == 33 else 64, 25)
            pred_np = np.pad(pred_np, ((0, 0), (0, W - pred_np.shape[1])))
            gt, pred = torch.from_numpy(gt_np).to(dev, torch.int32), torch.from_numpy(pred_np).to(dev, torch.int32)
            for lex in (None, lexicon):
                totals = rec_measure.new_totals(dev)
                fn = (lambda: rec_measure.measure_labels(gt, pred, table, lex, totals))
                fn()                                # warm-up: module load, allocator growth
                torch.cuda.synchronize()
                eager = events_ms(fn, 20)
                g = graph_of(fn)
                graph = events_ms(g.replay, 50)
                row = dict(what="measure_labels", N=N, width=W, lexicon=len(lex) if lex else 0, eager_ms=round(eager, 4),
                           graph_ms=round(graph, 4))
                if lex is None and N <= 512:
                    row["host_path_ms"] = round(1e3 * min(host_path(gt_np, pred_np, cs, None) for _ in range(2)), 2)
                rows.append(row)
                print(json.dumps(row))
    net = bench.build_model(dev).eval()
    for N, Wimg in ((16, 128), (512, 256)):
        x = torch.randn(N, 3, 32, Wimg, device=dev)
        lab = torch.from_numpy(cases.label_rows(rng, 38, N, 32, 12).astype(np.int32)).to(dev)
        totals = rec_measure.new_totals(dev)

        def step():
            prob = net.decoder(net.backbone(x), train=False)
            return rec_measure.measure_labels(lab, decode.ctc_greedy_decode(prob), table, totals=totals)
        with torch.no_grad():
            g = graph_of(step)
            ms = events_ms(g.replay, 10)
            prob = net.decoder(net.backbone(x), train=False)
            argmax = prob.argmax(1)[:, 0, :].cpu().numpy()
        row = dict(what="validation step graph (CRNN eval + ctc_greedy_decode + measure_labels)", shape=[N, 3, 32, Wimg],
                   graph_ms=round(ms, 3), host_path_ms=round(1e3 * host_path(lab.cpu().numpy(), argmax, cs, None, True), 2))
        rows.append(row)
        print(json.dumps(row))


if __name__ == "__main__":
    main()
