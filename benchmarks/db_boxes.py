"""The DB detector's SegDetectorRepresenter up to the unclip (seg_detector_representer.py:60-96, 125-168) on the device against
the reference's host path, on seeded DB-like probability maps (tests/db_boxes_cases.prob_maps: the text
boxes of tests/db_data.db_batch, blurred, through a sigmoid, plus noise; a few thousand contours per image, small, broken and
holed ones included):

    python benchmarks/db_boxes.py [--iters 50] [--host-iters 5]

Shapes: the yaml's validation batch, 4 x 576x1024 with max_candidates 1000 (seg_detector_db.yaml), and 16 x 640x640.
  device  megreader_b200.db_boxes.find_contours, and find_contours + box_candidates (csrc/db_boxes.cu), CUDA events over
          --iters calls after warm-up, eager and replayed from a CUDA graph
  host    what the reference does for the same steps: the map to the host (.cpu().numpy()), the threshold,
          cv2.findContours(RETR_LIST, CHAIN_APPROX_NONE) per image, and per kept contour get_mini_boxes (cv2.minAreaRect +
          cv2.boxPoints + the corner order) and, where sside >= 3, box_score_fast (cv2.fillPoly + cv2.mean); host clock, after a
          device synchronise
  boxes   megreader_b200.db_boxes.boxes_from_maps (the whole representer: unclip, second box, rescale and compaction included),
          eager and graph, against the oracle's representer (oracle/db_boxes_port.py: the reference with its three environment
          fixes) on the host, D2H copy included
  eval    at the validation shape: seg_detector_db.yaml's model (deformable ResNet50 + SegDetector, engine convolutions, bf16) in
          eval mode plus boxes_from_maps, captured in one CUDA graph, per replay
The device contours are checked against cv2 before timing.  The device name and power limit are printed with the numbers."""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from benchmarks.dcn_half import device_info  # noqa: E402
from megreader_b200 import db_boxes  # noqa: E402
from tests.db_boxes_cases import box_score_fast, digest, get_mini_boxes, prob_maps  # noqa: E402

CASES = [(4, 576, 1024, 0.3, 1000, 11), (16, 640, 640, 0.3, 1000, 14)]


def events_ms(fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--host-iters", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("benchmarks/db_boxes.py needs a CUDA device")
    import cv2
    dev = torch.device("cuda:0")
    info = device_info()
    for N, H, W, thresh, maxc, seed in CASES:
        maps = torch.from_numpy(prob_maps(seed, N, H, W)).to(dev)
        out = db_boxes.find_contours(maps, thresh, maxc)
        got = db_boxes.contour_lists(*out[:3])

        def host():
            m = maps.cpu().numpy()
            return [cv2.findContours((m[n, 0] > thresh).astype(np.uint8) * 255, cv2.RETR_LIST, cv2.CHAIN_APPROX_NONE)[0][:maxc]
                    for n in range(N)]
        want = host()
        assert [digest(c) for c in got] == [digest(c) for c in want], "device contours differ from cv2"
        contours = lambda: db_boxes.find_contours(maps, thresh, maxc)  # noqa: E731
        both = lambda: db_boxes.box_candidates(maps, *contours()[:3])  # noqa: E731

        def host_boxes():
            from oracle.db_boxes_port import SegDetectorRepresenter
            rep = SegDetectorRepresenter(thresh, 0.7, maxc)
            m = maps.cpu()
            return [rep.boxes_from_bitmap(m[n], m[n] > thresh, W, H) for n in range(N)]

        def host_candidates():
            m = maps.cpu().numpy()
            out = []
            for n in range(N):
                for c in cv2.findContours((m[n, 0] > thresh).astype(np.uint8) * 255, cv2.RETR_LIST, cv2.CHAIN_APPROX_NONE)[0][:maxc]:
                    box, sside = get_mini_boxes(c)
                    out.append(box_score_fast(m[n, 0], box.reshape(-1, 2)) if sside >= 3 else None)
            return out
        timings = {}
        boxes = lambda: db_boxes.boxes_from_maps(maps, None, thresh, 0.7, maxc)  # noqa: E731
        for label, fn in (("contours", contours), ("candidates", both), ("boxes", boxes)):
            for _ in range(5):
                fn()
            torch.cuda.synchronize()
            timings["device_%s_eager_ms" % label] = round(events_ms(fn, args.iters), 4)
            g = torch.cuda.CUDAGraph()
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                fn()
            torch.cuda.current_stream().wait_stream(s)
            with torch.cuda.graph(g):
                fn()
            for _ in range(3):
                g.replay()
            torch.cuda.synchronize()
            timings["device_%s_graph_ms" % label] = round(events_ms(g.replay, args.iters), 4)
        for label, fn in (("contours", host), ("candidates", host_candidates), ("boxes", host_boxes)):
            fn()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(args.host_iters):
                fn()
            timings["host_%s_ms" % label] = round((time.perf_counter() - t0) * 1e3 / args.host_iters, 3)
        total = out[3].cpu().tolist()
        print(json.dumps({"step": "db_box_candidates", "shape": [N, 1, H, W], "thresh": thresh, "max_candidates": maxc,
                          "contours_per_image": total, **timings, **info}), flush=True)
    eval_step(info, args.iters)


def eval_step(info, iters):
    import bench_trunks
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    net, _ = bench_trunks.build(6, dev, engine=True)
    net.eval()
    x, _ = bench_trunks.synth_db(1, 4, (576, 1024))
    static = x.to(dev)

    def step():
        binary = net.decoder(net.backbone(static))
        binary = binary['binary'] if isinstance(binary, dict) else binary
        return db_boxes.boxes_from_maps(binary.float(), None, 0.3, 0.7, 1000)
    with torch.no_grad():
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(3):
                step()
        torch.cuda.current_stream().wait_stream(s)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            step()
        for _ in range(3):
            g.replay()
        torch.cuda.synchronize()
        ms = events_ms(g.replay, iters)
    print(json.dumps({"step": "db_eval_step_plus_boxes", "shape": [4, 3, 576, 1024], "graph_ms": round(ms, 3),
                      "model": "deformable ResNet50 + SegDetector(adaptive, k=50), engine convolutions (bf16), eval", **info}),
          flush=True)


if __name__ == "__main__":
    main()
