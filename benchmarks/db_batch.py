"""Device time of the DB detector's input batch (megreader_b200.db_batch), graph-replayed, and the oracle's host time per
image on one core for the same inputs.

    python -m benchmarks.db_batch [--iters 20]

Training: 16 MLT-like inputs (sides mixed from 1280 x 720 to 2000 x 1500, 10 to 30 quads each, scale draws spread over the
whole range) into 640 x 640, with and without make_targets_packed.  Validation: 4 inputs resized to 576 x 1024.  Prints one
JSON line with the card name and power limit."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from megreader_b200 import db_batch, db_targets  # noqa: E402
from tests import db_batch_cases as C  # noqa: E402

SIDES = [(720, 1280), (1080, 1920), (1200, 1600), (1500, 2000), (960, 1280), (768, 1024)]


def inputs(n, rng, validate=False):
    imgs, polys, tags = [], [], []
    for i in range(n):
        h, w = (576, 1024) if validate else SIDES[i % len(SIDES)]
        imgs.append(C.image(rng, h, w))
        k = int(rng.integers(10, 31))
        polys.append(C.quads(rng, h, w, k))
        tags.append((rng.random(k) < 0.15).astype(np.uint8))
    return imgs, polys, tags


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()[0]
        return [s.strip() for s in q.split(",")]
    except Exception:
        return [torch.cuda.get_device_name(0), "unknown"]


def graph_ms(fn, iters):
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
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(iters):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--host-images", type=int, default=4)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    rng = np.random.default_rng(0)
    imgs, polys, tags = inputs(16, rng)
    d_imgs = [torch.from_numpy(x).to(dev) for x in imgs]
    buf, ioff, shapes = db_batch.pack_images(d_imgs)
    P, T, O = db_targets.pack([torch.from_numpy(p).to(dev) for p in polys], [torch.from_numpy(t).to(dev) for t in tags])
    u = db_batch.draws(16, torch.Generator(device=dev).manual_seed(1))
    u[:, 2] = torch.linspace(0, 1, 16, device=dev)          # the scale draws span 0.5 .. 3.0
    max_h, max_w = 1500, 2000

    def train():
        return db_batch.train_batch_packed(buf, ioff, shapes, max_h, max_w, P, T, O, u)

    def train_targets():
        o = train()
        db_targets.make_targets_packed(o["polygons"], o["ignore_tags"], o["offsets"], (640, 640))

    vimgs, vpolys, vtags = inputs(4, rng, validate=True)
    vbuf, vioff, vshapes = db_batch.pack_images([torch.from_numpy(x).to(dev) for x in vimgs])
    VP, VT, VO = db_targets.pack([torch.from_numpy(p).to(dev) for p in vpolys], [torch.from_numpy(t).to(dev) for t in vtags])

    def validate():
        o = db_batch.validate_batch_packed(vbuf, vioff, vshapes, 576, 1024, VP, VT, VO)
        db_targets.make_targets_packed(o["polygons"], o["ignore_tags"], o["offsets"], (576, 1024))

    res = dict(train_batch16_ms=graph_ms(train, a.iters), train_batch16_with_targets_ms=graph_ms(train_targets, a.iters),
               validate_batch4_with_targets_ms=graph_ms(validate, a.iters))
    from oracle import db_batch_port as port
    uh = u.cpu().numpy()
    t0 = time.perf_counter()
    for i in range(a.host_images):
        port.train_sample(imgs[i], polys[i], tags[i], uh[i])
    res["oracle_host_ms_per_image"] = (time.perf_counter() - t0) * 1e3 / a.host_images
    name, power = card()
    res.update(gpu=name, power_limit=power, host_threads=1, torch_threads=torch.get_num_threads())
    print(json.dumps(res))


if __name__ == "__main__":
    import cv2
    cv2.setNumThreads(1)
    main()
