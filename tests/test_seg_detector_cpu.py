"""CPU: the DB detector head (decoders.SegDetector + L1BalanceCELoss) against tests/golden/seg_detector_ref.npz, recorded from the
reference's own modules in float64 (tests/make_db_golden.py), and the host-side checks of its C-ABI entries."""
import contextlib
import importlib
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import ref_loader
from tests import db_port
from tests.make_db_golden import GOLD, SALT, batch, features, grad_sample
from tests.weights import fill_state_dict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def gold():
    return dict(np.load(GOLD))


def _decoders():
    import megreader_b200.refapi.decoders as decoders      # by package path: `decoders` may be the reference's in this process
    return decoders


def _head():
    return fill_state_dict(_decoders().SegDetector(adaptive=True, k=50, in_channels=[64, 128, 256, 512]), SALT)


@contextlib.contextmanager
def _reference_decoders():
    """The reference's `decoders` package, imported while the refapi one (same name) is set aside; restored on exit."""
    assert ref_loader.install()
    names = lambda: [k for k in sys.modules if k == "decoders" or k.startswith("decoders.")]  # noqa: E731
    saved = {k: sys.modules.pop(k) for k in names()}
    sys.path.insert(0, ref_loader.REF)
    try:
        mod = importlib.import_module("decoders")
        assert mod.__file__.startswith(ref_loader.REF)
        yield mod
    finally:
        sys.path.remove(ref_loader.REF)
        for k in names():
            del sys.modules[k]
        sys.modules.update(saved)


def _rel(a, b):
    return float(np.abs(np.asarray(a) - np.asarray(b)).max() / max(np.abs(np.asarray(b)).max(), 1e-300))


def test_state_dict_matches_reference(gold):
    assert [[k, list(v.shape)] for k, v in _head().state_dict().items()] == json.loads(str(gold["state_head"]))


def test_exports():
    d = _decoders()
    for name in ("SegDetector", "DiceLoss", "MaskL1Loss", "BalanceCrossEntropyLoss"):
        assert hasattr(d, name)
    from megreader_b200.refapi.decoders.seg_detector_loss import SegDetectorLossBuilder, L1BalanceCELoss
    assert type(SegDetectorLossBuilder("L1BalanceCELoss").build()) is L1BalanceCELoss


def test_smooth_fails_at_construction_like_the_reference():
    with pytest.raises(TypeError):
        _decoders().SegDetector(adaptive=True, smooth=True)


def test_port_reproduces_golden(gold):
    head = _head().double().train()
    feats = [torch.from_numpy(f).requires_grad_(True) for f in features()]
    b = {k: torch.from_numpy(v) for k, v in batch().items()}
    pred = db_port.seg_detector_forward(head, feats)
    loss, metrics = db_port.l1_balance_ce(pred, b)
    loss.backward()
    assert _rel(loss.item(), gold["loss"]) < 1e-6
    for k, v in metrics.items():
        assert _rel(v.item(), gold["m_" + k]) < 1e-6, k
    for k, v in pred.items():
        assert _rel(v.detach().numpy(), gold["train_" + k]) < 1e-6, k
    for i, f in enumerate(feats):
        assert _rel(f.grad.numpy(), gold["gf%d" % i]) < 1e-6, i
    for name, p in head.named_parameters():
        idx = gold["pg_idx:" + name]
        assert np.array_equal(idx, grad_sample(name, p.numel()))
        ref = gold["pg:" + name]
        got = p.grad.reshape(-1).numpy()[idx]
        assert np.abs(got - ref).max() <= 1e-6 * max(np.abs(ref).max(), 1e-12), name
    with torch.no_grad():
        ev = db_port.seg_detector_forward(head.eval(), feats)
    for k, v in ev.items():
        assert _rel(v.numpy(), gold["eval_" + k]) < 1e-6, k


def _loss_cases():
    """(pred, batch) cases for pinning the port to the reference criterion: hard / soft gt, N = 1 and N = 3 (the broadcast)."""
    rng = np.random.RandomState(4)
    out = []
    for N, soft in ((1, False), (3, False), (2, True)):
        H, W = 12, 10
        gt = (rng.rand(N, 1, H, W) < 0.2).astype(np.float64)
        if soft:
            gt = np.where(rng.rand(N, 1, H, W) < 0.3, rng.rand(N, 1, H, W), gt)
        mask = (rng.rand(N, H, W) < 0.9).astype(np.float64)
        pred = {"binary": rng.uniform(0.01, 0.99, (N, 1, H, W)), "thresh": rng.uniform(0.2, 0.8, (N, 1, H, W)),
                "thresh_binary": rng.uniform(0.01, 0.99, (N, 1, H, W))}
        b = {"gt": gt, "mask": mask, "thresh_map": rng.uniform(0.3, 0.7, (N, H, W)),
             "thresh_mask": (rng.rand(N, H, W) < 0.4).astype(np.float64)}
        t = lambda d: {k: torch.from_numpy(v) for k, v in d.items()}  # noqa: E731
        out.append((t(pred), t(b)))
    return out


@pytest.mark.skipif(not ref_loader.available(), reason="reference tree not present")
def test_port_pinned_to_reference_criterion():
    for pred, b in _loss_cases():
        p_ref = {k: v.clone().requires_grad_(True) for k, v in pred.items()}
        p_port = {k: v.clone().requires_grad_(True) for k, v in pred.items()}
        with _reference_decoders():
            ref = importlib.import_module("decoders.seg_detector_loss")
            l_ref, m_ref = ref.L1BalanceCELoss()(p_ref, b)
        l_port, m_port = db_port.l1_balance_ce(p_port, b)
        l_ref.backward()
        l_port.backward()
        assert abs(l_ref.item() - l_port.item()) <= 1e-12 * abs(l_ref.item())
        for k in m_ref:
            assert abs(float(m_ref[k]) - float(m_port[k])) <= 1e-12 * abs(float(m_ref[k])) + 1e-15, k
        for k in pred:       # random float64 inputs: no ties at tau, so torch.topk's choice is the tie rule's
            assert torch.allclose(p_ref[k].grad, p_port[k].grad, rtol=1e-10, atol=1e-14), k


@pytest.mark.skipif(not ref_loader.available(), reason="reference tree not present")
def test_plain_compositions_match_reference():
    d = _decoders()
    with _reference_decoders() as ref:
        ref_mods = (ref.DiceLoss(), ref.MaskL1Loss(), ref.BalanceCrossEntropyLoss())
    for pred, b in _loss_cases():
        assert torch.equal(d.DiceLoss()(pred["thresh_binary"], b["gt"], b["mask"]),
                           ref_mods[0](pred["thresh_binary"], b["gt"], b["mask"]))
        assert torch.equal(d.MaskL1Loss()(pred["thresh"], b["thresh_map"], b["thresh_mask"])[0],
                           ref_mods[1](pred["thresh"], b["thresh_map"], b["thresh_mask"])[0])
        assert torch.equal(d.BalanceCrossEntropyLoss()(pred["binary"], b["gt"], b["mask"]),
                           ref_mods[2](pred["binary"], b["gt"], b["mask"]))


def _probe(mode):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "db_boundary_probe.py"), mode], capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


@pytest.mark.skipif(not ref_loader.available(), reason="reference tree not present")
def test_seg_detector_db_yaml_builds_on_refapi_with_identical_state_dict(gold):
    ours, ref = _probe("refapi"), _probe("reference")
    assert "refapi" in ours["decoders_file"] and ref["decoders_file"].startswith(ref_loader.REF)
    assert (ours["model"], ours["backbone"], ours["decoder"], ours["loss_class"]) == \
        ("SegDetectorModel", "deformable_resnet50", "SegDetector", "L1BalanceCELoss")
    assert ours["state"] == ref["state"]
    assert len(ours["state"]) == 398 and ours["n_params"] == ref["n_params"] == 28978313
    recorded = json.loads(str(gold["state_model"]))
    assert recorded["state"] == ours["state"] and recorded["n_params"] == ours["n_params"]


def test_surfaces_raise_on_cpu_tensors():
    from megreader_b200 import db_head
    z = torch.zeros(1, 1, 4, 4)
    with pytest.raises(NotImplementedError):
        db_head.step_function(z, z, 50.0)
    m = torch.zeros(1, 4, 4)
    with pytest.raises(NotImplementedError):
        db_head.l1_balance_ce_loss(z, z, z, z, m, m, m)
    with pytest.raises(NotImplementedError):
        _head()([torch.zeros(2, 64, 8, 8), torch.zeros(2, 128, 4, 4), torch.zeros(2, 256, 2, 2), torch.zeros(2, 512, 1, 1)])


def test_capi_argument_checks_without_gpu():
    """Host-side checks return before any CUDA call (aligned dummy pointers: nothing touches them)."""
    from megreader_b200 import _lib
    L = _lib.lib()
    MR_ERR_NULL_POINTER, MR_ERR_BAD_SHAPE = 1, 4
    p = [0x10000 * (i + 1) for i in range(12)]
    assert L.mr_db_step_fwd(p[0], p[1], 0, -1, 50.0, p[2], p[3], p[4], None) == MR_ERR_BAD_SHAPE
    assert L.mr_db_step_fwd(p[0], p[1], 3, 16, 50.0, p[2], p[3], p[4], None) == MR_ERR_BAD_SHAPE
    assert L.mr_db_step_fwd(p[0], p[1], 0, 0, 50.0, p[2], p[3], p[4], None) == 0            # empty: no-op
    assert L.mr_db_step_fwd(None, p[1], 0, 16, 50.0, p[2], p[3], p[4], None) == MR_ERR_NULL_POINTER
    assert L.mr_db_step_fwd(p[0], p[1], 1, 16, 50.0, p[2], None, p[4], None) == MR_ERR_NULL_POINTER
    assert L.mr_db_step_bwd(p[0], p[1], p[2], p[3], p[4], p[5], 0, 16, 50.0, None, p[6], None) == MR_ERR_NULL_POINTER
    assert L.mr_db_step_bwd(p[0], None, p[2], p[3], p[4], p[5], 0, 16, 50.0, p[6], p[7], None) == MR_ERR_NULL_POINTER
    assert L.mr_db_loss_workspace_bytes(2, 64, 64) > 0 and L.mr_db_loss_workspace_bytes(0, 64, 64) == 0
    maps = p[:7]
    fwd = lambda m, N, H, W, ws=p[7], out=p[8]: L.mr_db_loss_fwd_f32(*m, N, H, W, 1e-6, 1e-6, 10.0, 5.0, 3.0, ws, out, None)  # noqa: E731
    assert fwd(maps, 0, 8, 8) == MR_ERR_BAD_SHAPE
    assert fwd(maps, 2, 8, -1) == MR_ERR_BAD_SHAPE
    assert fwd(maps, 193, 8, 8) == _lib.MR_ERR_UNSUPPORTED
    assert fwd(maps[:3] + [None] + maps[4:], 2, 8, 8) == MR_ERR_NULL_POINTER
    assert fwd(maps, 2, 8, 8, ws=None) == MR_ERR_NULL_POINTER
    assert fwd(maps, 2, 8, 8, out=None) == MR_ERR_NULL_POINTER
    bwd = lambda m, N, ws=p[7], g=p[8], d=p[9]: L.mr_db_loss_bwd_f32(*m, N, 8, 8, 10.0, 5.0, ws, g, d, p[10], p[11], None)  # noqa: E731
    assert bwd(maps, 0) == MR_ERR_BAD_SHAPE
    assert bwd(maps, 2, g=None) == MR_ERR_NULL_POINTER
    assert bwd(maps, 2, d=None) == MR_ERR_NULL_POINTER
    assert bwd([None] + maps[1:], 2) == MR_ERR_NULL_POINTER
