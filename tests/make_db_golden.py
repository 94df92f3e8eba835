"""Record tests/golden/seg_detector_ref.npz from the UNMODIFIED reference modules (oracle/ref_loader.py), so that the DB head
tests run where the reference tree is absent.

    python -m tests.make_db_golden          # needs the reference tree (MEGREADER_REFERENCE)

The case: the reference SegDetector(adaptive=True, k=50) with in_channels=[64,128,256,512] and inner_channels=256, weights from
tests.weights.fill_state_dict(salt "seg."), seeded features c2 16x16 .. c5 2x2 at N = 2, and a seeded DB batch at 64x64
(tests.db_data.db_batch).  Everything runs in float64 in the reference's own modules, train mode, criterion L1BalanceCELoss.
The features and the batch are regenerated from their seeds (features(), batch()).  Recorded: train maps, eval maps, loss and metrics, gradients w.r.t. the four features, a seeded sample of 16
entries of every parameter gradient (pg_idx:<name> / pg:<name>), and the state-dict names and shapes of the SegDetector and of
the full SegDetectorModel of experiments/seg_detector/seg_detector_db.yaml (JSON strings)."""
import json
import os
import subprocess
import sys
import types
import zlib

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
GOLD = os.path.join(ROOT, "tests", "golden", "seg_detector_ref.npz")
FEAT_SHAPES = [(2, 64, 16, 16), (2, 128, 8, 8), (2, 256, 4, 4), (2, 512, 2, 2)]
SALT = "seg."


def features():
    rng = np.random.RandomState(23)
    return [rng.standard_normal(s).astype(np.float64) for s in FEAT_SHAPES]


def batch():
    from tests.db_data import db_batch
    return {k: v.astype(np.float64) for k, v in db_batch(29, 2, 64, 64).items()}


def grad_sample(name, numel, n=16):
    rng = np.random.RandomState(zlib.crc32(name.encode()) & 0x7FFFFFFF)
    return np.sort(rng.choice(numel, min(n, numel), replace=False))


def main():
    from oracle import ref_loader
    from tests.weights import fill_state_dict
    assert ref_loader.install(), "reference tree not present"
    from decoders.seg_detector import SegDetector
    from decoders.seg_detector_loss import L1BalanceCELoss
    torch.set_num_threads(1)
    head = fill_state_dict(SegDetector(adaptive=True, k=50, in_channels=[64, 128, 256, 512]), SALT).double().train()
    feats = [torch.from_numpy(f).requires_grad_(True) for f in features()]
    b = {k: torch.from_numpy(v) for k, v in batch().items()}
    pred = head(feats, training=True)
    loss, metrics = L1BalanceCELoss()(pred, b)
    loss.backward()
    out = {}
    out.update({"train_" + k: v.detach().numpy() for k, v in pred.items()})
    out["loss"] = loss.detach().numpy()
    out.update({"m_" + k: v.detach().numpy() for k, v in metrics.items()})
    out.update({"gf%d" % i: f.grad.numpy() for i, f in enumerate(feats)})
    for name, p in head.named_parameters():
        idx = grad_sample(name, p.numel())
        out["pg_idx:" + name] = idx
        out["pg:" + name] = p.grad.reshape(-1).numpy()[idx]
    with torch.no_grad():
        ev = head.eval()(feats, training=False)
    out.update({"eval_" + k: v.numpy() for k, v in ev.items()})
    out["state_head"] = np.array(json.dumps([[k, list(v.shape)] for k, v in head.state_dict().items()]))
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "db_boundary_probe.py"), "reference"], capture_output=True,
                       text=True, check=True)
    probe = json.loads(r.stdout.strip().splitlines()[-1])
    out["state_model"] = np.array(json.dumps({"state": probe["state"], "n_params": probe["n_params"]}))
    np.savez_compressed(GOLD, **out)
    print("wrote %s: loss %.9f, %s" % (GOLD, float(loss), {k: float(v.detach()) for k, v in metrics.items()}))


if __name__ == "__main__":
    sys.modules.setdefault("assets.ops.dcn.deform_conv_cuda", types.ModuleType("assets.ops.dcn.deform_conv_cuda"))
    main()
