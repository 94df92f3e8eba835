"""Every reachable CTC kernel instantiation of csrc/ctc2d.cu against a float64 reference, at the length, label and memory
edges where the dispatch and the sweeps branch.

Each case runs one entry point under torch.profiler, asserts that the instantiations tests/ctc_variants.py expects are the
ones that ran, and compares the result element by element:
  contract  ctc2d_forward + ctc2d_backward (fp32 fast / accurate, fp64) against the C oracle (oracle/ctc2d_oracle.c):
            nll, log_alpha with its exact -inf pattern, grad with its exact zero pattern;
  train     ctc_loss_2d with requires_grad (forward_train + backward_apply) against the same oracle;
  ctc1d     ctc1d.ctc_loss_from_logits against torch.nn.functional.ctc_loss on the CPU in float64 applied to
            log_softmax(logits), for zero_infinity on / off and every reduction: per-sample nll and the gradient with
            respect to the logits.  A sample that no alignment fits (L + repeats > Tb) has nll = inf with zero_infinity off;
            torch then returns NaN as its logits gradient for t < Tb (and 0 after), so only nll = inf is asserted for it.
            Torch gives an empty target the blank-only path: nll = -sum_{t<Tb} log p(t, blank).

Large-N cases (dp4 group sizes 4 / 6 / 8 come from N against the SM count) run the kernel on the whole batch and compare a
fixed subset of samples: samples are independent and the C oracle is serial.

Tolerances.  fp32: nll 1e-4 relative, log_alpha 1e-4 relative + 1e-4 absolute, grad 2e-4 relative + 2e-5 absolute; fp64:
nll 1e-10, log_alpha 1e-9, grad 1e-8 relative + 1e-10 absolute -- the suite's bounds, measured at T <= 64.  Beyond T = 64 the
gradient gets a term that grows with the sample's length Tb.  Every sweep step rounds log-domain values of magnitude at most
M = |nll| + max|log p| (2^-24 M) and, with fast math, adds the error of one ex2.approx / lg2.approx pair (< 2^-21 in log2
units); so R, Rb and nll each carry an absolute error below e = Tb (2^-24 M + 2^-21), and the posterior
exp(R + Rb + nll) a relative error below expm1(3 e).  The gradient element is exp(lp) go (1 - posterior), so its error is
bounded by |exp(lp) go - grad_ref| expm1(3 e) on top of the fixed bounds.  nll's relative error, 2^-24 Tb + 2^-21 Tb / |nll|,
stays below 1e-4 for every case here.  Zero and -inf patterns are exact.
"""
import numpy as np
import pytest
import torch

from oracle import capi
from tests import ctc_variants as cv

pytestmark = pytest.mark.gpu

SMS = cv.device_limits()[0]


# ---------------------------------------------------------------- inputs
def _target(rng, L, kind, C, blank):
    """A target of L labels.  kind: rand (no blank), rep (every label doubled: L // 2 repeats), blank (the blank at every third
    position), high (labels >= 32)."""
    pool = [c for c in range(C) if c != blank]
    if kind == "high":
        pool = [c for c in pool if c >= 32] or pool
    lab = list(rng.choice(pool, size=L))
    if kind == "rep":
        lab = [lab[j // 2] for j in range(L)]
    if kind == "blank":
        for j in range(0, L, 3):
            lab[j] = blank
    return lab


def _repeats(lab):
    return sum(1 for a, b in zip(lab, lab[1:]) if a == b)


def make_inputs(case, dtype=np.float32):
    """Seeded (lp [T,H,N,C] = log_softmax_H(mask) + log_softmax_C(classify), targets [N,S], il, tl).  case["samples"] is a
    list of (Tb, L, kind) repeated over the batch; Tb = None: T, "=": exactly L + repeats (the feasibility boundary), "<":
    one step below it."""
    T, H, N, C, S, blank = (case[k] for k in ("T", "H", "N", "C", "S", "blank"))
    rng = np.random.RandomState(case["seed"])
    tg = rng.randint(0, C, size=(N, S)).astype(np.int64)   # padding past L holds arbitrary classes: never read
    il = np.empty(N, np.int64)
    tl = np.empty(N, np.int64)
    spec = case["samples"]
    for b in range(N):
        Tb, L, kind = spec[b % len(spec)]
        lab = _target(rng, L, kind, C, blank)
        tg[b, :L] = lab
        tl[b] = L
        il[b] = T if Tb is None else (L + _repeats(lab) + (0 if Tb == "=" else -1) if isinstance(Tb, str) else Tb)
        assert 1 <= il[b] <= T, (case["id"], b, il[b])
    m = rng.standard_normal((T, H, N))
    c = rng.standard_normal((T, H, N, C))
    m = m - np.log(np.exp(m).sum(1, keepdims=True))
    c = c - np.log(np.exp(c).sum(3, keepdims=True))
    return np.ascontiguousarray((m[..., None] + c).astype(dtype)), tg, il, tl


# ---------------------------------------------------------------- the case list
MIX3 = [(None, 5, "rand"), (17, 8, "blank"), ("=", 20, "rep"), (None, 32, "rand"), (1, 0, "rand"), (9, 0, "rand"),
        (2, 1, "rand"), ("<", 12, "rep")]          # dp4: ns = 1, 2, 3 in one round; L = 0 / 1; Tb = 1, 2, odd, boundary


def _case(id, entry, T, H, N, C, S, samples, blank=0, fast=True, real="float", env=None, offset=False, scalar_go=False,
          strided=False, subset=None, seed=0):
    return dict(id=id, entry=entry, T=T, H=H, N=N, C=C, S=S, samples=samples, blank=blank, fast=fast, real=real,
                env=env or {}, offset=offset, scalar_go=scalar_go, strided=strided, subset=subset, seed=seed)


def _sub(N):
    return np.r_[0:12, N - 9:N]


CASES = [
    # ---- dp4 (fast fp32, S <= 32, C <= 64)
    _case("dp4-fac-h8-blanklabel", "train", 32, 8, 7, 38, 32, MIX3, seed=1),
    _case("dp4-fac-blank40-high", "train", 20, 3, 5, 64, 16,
          [(None, 9, "blank"), (None, 7, "high"), (13, 0, "rand"), ("=", 8, "rep"), (1, 1, "high")], blank=40, seed=2),
    _case("dp4-grad-h8-blankC-1", "contract", 32, 8, 9, 38, 32, MIX3 + [(None, 11, "high")], blank=37, seed=3),
    _case("dp4-grad-h1-offset-scalar-go", "contract", 15, 1, 6, 12, 7,
          [(None, 7, "rand"), (2, 1, "rand"), ("=", 6, "rep"), (4, 0, "rand"), (15, 5, "blank")], blank=11,
          offset=True, scalar_go=True, seed=4),
    _case("dp4-fac-G4", "train", 32, 8, 4 * SMS + 1, 38, 32, MIX3, subset=_sub(4 * SMS + 1), seed=5),
    _case("dp4-fac-G6", "train", 32, 8, 6 * SMS + 1, 38, 32, MIX3, subset=_sub(6 * SMS + 1), seed=6),
    _case("dp4-grad-G8", "contract", 32, 8, 8 * SMS, 38, 32, MIX3, subset=_sub(8 * SMS), seed=7),
    _case("dp4-fac-oddG-T48", "train", 48, 8, 8 * SMS + 3, 38, 32, MIX3, subset=_sub(8 * SMS + 3), seed=8),
    _case("dp4-fac-offset", "train", 12, 2, 5, 6, 4, [(None, 4, "rep"), (3, 2, "rand"), (12, 0, "rand")],
          offset=True, strided=True, seed=9),
    _case("dp4-fac-C1", "train", 10, 4, 3, 2, 3, [(None, 3, "rand"), (5, 2, "rand"), (3, 0, "rand")], blank=1, seed=10),
    # ---- dpg (C > 64)
    _case("dpg-fac-C65-blanklabel", "train", 32, 4, 9, 65, 32, MIX3, seed=11),
    _case("dpg-grad-C500-h8", "contract", 16, 8, 6, 500, 12,
          [(None, 7, "blank"), (5, 0, "rand"), ("=", 8, "rep"), ("<", 6, "rep"), (1, 1, "rand"), (16, 12, "rand")],
          blank=499, seed=12),
    _case("dpg-grad-C4001-unstaged", "contract", 6, 4, 3, 4001, 3, [(None, 3, "rand"), (2, 1, "rand"), (6, 0, "rand")],
          blank=2000, seed=13),
    # ---- dp4 refuses at large T: dp_warp, one state per lane
    _case("T420-fac-h8", "train", 420, 8, 3, 38, 8, [(None, 8, "rep"), (211, 5, "rand"), (1, 1, "rand")], seed=14),
    _case("T420-grad-h2", "contract", 420, 2, 3, 38, 8, [(None, 8, "rep"), (300, 0, "rand"), (2, 1, "rand")], seed=15),
    # ---- block kernels: accurate math, MR_CTC2D_BLOCK_DP=1, fp64
    _case("block-acc-grad-h8", "contract", 32, 8, 9, 38, 32, MIX3 + [(None, 11, "blank")], blank=37, fast=False, seed=16),
    _case("block-acc-grad-h2", "contract", 12, 2, 5, 9, 6, [(None, 6, "rep"), (1, 1, "rand"), (7, 0, "rand"), ("<", 4, "rep")],
          blank=8, fast=False, seed=28),
    _case("block-acc-grad-h5-unstaged", "contract", 6, 5, 3, 4001, 3, [(None, 3, "rand"), (6, 0, "rand"), (1, 1, "rand")],
          fast=False, seed=17),
    _case("block-acc-fac-h8", "train", 32, 8, 10, 38, 32, MIX3, blank=37, fast=False, seed=18),
    _case("block-acc-fac-h3-offset", "train", 32, 3, 5, 70, 32, MIX3[:3] + [(14, 0, "rand"), (2, 1, "blank")],
          fast=False, offset=True, seed=19),
    _case("block-acc-fac-h2", "train", 9, 2, 4, 7, 4, [(None, 4, "rep"), (1, 1, "rand"), (5, 0, "rand")],
          fast=False, seed=20),
    _case("block-env-grad-h8", "contract", 32, 8, 7, 38, 32, MIX3, fast=True, env={"MR_CTC2D_BLOCK_DP": "1"}, seed=21),
    _case("block-env-grad-h1", "contract", 16, 1, 5, 40, 12, [(None, 5, "rand"), ("=", 6, "rep"), (3, 0, "rand"), (16, 12, "blank")],
          blank=39, env={"MR_CTC2D_BLOCK_DP": "1"}, seed=22),
    _case("block-env-fac-h8", "train", 32, 8, 7, 38, 32, MIX3, blank=37, env={"MR_CTC2D_BLOCK_DP": "1"}, seed=23),
    _case("block-env-fac-h2", "train", 18, 2, 6, 9, 6, [(None, 6, "rep"), ("<", 6, "rep"), (1, 0, "rand")],
          env={"MR_CTC2D_BLOCK_DP": "1"}, strided=True, seed=24),
    _case("f64-grad-h8", "contract", 32, 8, 7, 38, 32, MIX3, blank=37, real="double", seed=25),
    _case("f64-grad-h3", "contract", 12, 3, 6, 10, 6, [(None, 6, "rep"), (1, 1, "rand"), (7, 0, "rand"), ("<", 4, "rep")],
          real="double", scalar_go=True, seed=26),
    _case("f64-grad-unstaged", "contract", 6, 8, 3, 1000, 3, [(None, 3, "blank"), (2, 1, "rand"), (6, 0, "rand")],
          blank=500, real="double", seed=27),
]

# dp_warp: every NSMAX for GRAD (contract) and FAC (train), H = 8 and H != 8.  NS = 1, 2, 3 need MR_CTC2D_DP_V3=1 (S <= 32 goes
# to dp4 otherwise); S = 48 / 64 / 160 / 256 reach NS = 4 / 8 / 16 / 32 on their own.  Within one launch, samples of every
# smaller sweep width run next to the widest; targets longer than Tb are infeasible (nll = inf, zero gradient).
_WARP = [
    (1, 15, 20, [(None, 15, "rand"), (3, 0, "rand"), (1, 1, "rand"), ("=", 6, "rep"), ("<", 6, "rep")]),
    (2, 24, 30, [(None, 24, "rand"), (None, 7, "blank"), (4, 0, "rand"), (2, 1, "rand")]),
    (3, 32, 40, [(None, 32, "rand"), (None, 20, "rep"), (None, 5, "high"), (5, 0, "rand")]),
    (4, 48, 56, [(None, 48, "rand"), (None, 40, "rand"), (None, 20, "rand"), (None, 5, "blank"), (1, 0, "rand")]),
    (8, 64, 80, [(None, 64, "rand"), (None, 60, "rand"), (None, 40, "rep"), (None, 20, "rand"), (None, 5, "rand"),
                 (3, 0, "rand")]),
    (16, 160, 24, [(None, 150, "rand"), (None, 100, "rand"), (None, 3, "rand"), (24, 12, "blank")]),
    (32, 256, 12, [(None, 256, "rand"), (None, 200, "rand"), (None, 3, "rand"), (7, 0, "rand")]),
]
for _ns, _S, _T, _smp in _WARP:
    _env = {"MR_CTC2D_DP_V3": "1"} if _ns <= 3 else None
    CASES.append(_case("warp%d-grad-h8" % _ns, "contract", _T, 8, 5, 38, _S, _smp, blank=37, env=_env, seed=100 + _ns))
    CASES.append(_case("warp%d-grad-h1" % _ns, "contract", _T, 1, 6, 40, _S, _smp, env=_env, scalar_go=_ns == 8,
                       seed=200 + _ns))
    CASES.append(_case("warp%d-fac-h8" % _ns, "train", _T, 8, 6, 38, _S, _smp, env=_env, seed=300 + _ns))
    CASES.append(_case("warp%d-fac-h3" % _ns, "train", _T, 3, 6, 12, _S, _smp, blank=11, env=_env, strided=_ns == 2,
                       seed=400 + _ns))

# the 1D loss (H = 1, no label equal to the blank): dp_warp for fast math, whatever S gives; the block kernel otherwise
_SEQ = [(None, 0, "rand"), (1, 0, "rand"), (2, 0, "rand"), (1, 1, "rand"), ("=", 6, "rep"), ("<", 6, "rep"),
        (9, 3, "rand"), (None, 16, "high")]
CASES += [
    _case("1d-crnn-bench", "ctc1d", 65, 1, 512, 38, 32,
          [(None, 16, "rand"), (None, 0, "rand")] + [(t, L, k) for t, L, k in _SEQ if L <= 16] + [(33, 16, "rep")],
          subset=np.r_[0:40], seed=500),
    _case("1d-acc", "ctc1d", 40, 1, 10, 38, 20, _SEQ, fast=False, strided=True, seed=501),
    _case("1d-block-env", "ctc1d", 40, 1, 10, 38, 20, _SEQ, env={"MR_CTC2D_BLOCK_DP": "1"}, seed=502),
]
for _ns, _S, _T, _smp in _WARP:
    CASES.append(_case("1d-warp%d" % _ns, "ctc1d", max(_T, 17), 1, 8, 38, _S,
                       [s for s in _smp if s[2] != "blank"] + _SEQ[:3], blank=0 if _ns % 2 else 37, seed=600 + _ns))

IDS = [c["id"] for c in CASES]
assert len(set(IDS)) == len(IDS)


def expected(case):
    return cv.expected_kernels(case["entry"], case["T"], case["H"], case["N"], case["C"], case["S"], fast=case["fast"],
                               real=case["real"], aligned=not case["offset"], env=case["env"])


VARIANTS = set()
for _c in CASES:
    VARIANTS |= expected(_c)


# ---------------------------------------------------------------- helpers
def _on(dev, a, offset=False, strided=False):
    t = torch.from_numpy(np.ascontiguousarray(a))
    if offset:   # a contiguous view 4 bytes past a 16-byte boundary: every vector path must step aside
        buf = torch.zeros(t.numel() + 1, dtype=t.dtype, device=dev)
        v = buf[1:].view(t.shape)
        v.copy_(t)
        return v
    if strided:  # targets with a column stride of 2
        wide = torch.zeros(t.shape[0], 2 * t.shape[1], dtype=t.dtype, device=dev)
        wide[:, ::2] = t.to(dev)
        return wide[:, ::2]
    return t.to(dev)


def _grad_bound(g_ref, lp, go, nll_ref, il, T, rt, at, axis_n):
    """Element-wise bound of the module docstring; the Tb-dependent term only where T > 64."""
    bnd = rt * np.abs(g_ref) + at
    if T > 64:
        shape = [1] * g_ref.ndim
        shape[axis_n] = -1
        M = np.abs(np.where(np.isfinite(nll_ref), nll_ref, 0)) + np.abs(lp).max()
        e = il * (2.0 ** -24 * M + 2.0 ** -21)
        bnd = bnd + np.abs(np.exp(lp.astype(np.float64)) * go.reshape(shape) - g_ref) * np.expm1(3 * e).reshape(shape)
    return bnd


def _assert_within(got, ref, bnd, what):
    err = np.abs(got.astype(np.float64) - ref)
    bad = ~(err <= bnd)
    assert not bad.any(), "%s: %d of %d elements outside the bound; first at %s: got %r, want %r" % (
        what, int(bad.sum()), bad.size, np.argwhere(bad)[0], got[tuple(np.argwhere(bad)[0])], ref[tuple(np.argwhere(bad)[0])])


@pytest.fixture
def env(monkeypatch):
    for k in ("MR_CTC2D_BLOCK_DP", "MR_CTC2D_DP_V3"):
        monkeypatch.delenv(k, raising=False)

    def set_case(case):
        from megreader_b200 import ctc2d
        monkeypatch.setattr(ctc2d, "FAST_MATH", case["fast"])
        monkeypatch.setattr(ctc2d, "CONTRACT_PATH", False)
        for k, v in case["env"].items():
            monkeypatch.setenv(k, v)
    return set_case


# ---------------------------------------------------------------- 2D
CASES_2D = [c for c in CASES if c["entry"] != "ctc1d"]


@pytest.mark.parametrize("case", CASES_2D, ids=[c["id"] for c in CASES_2D])
def test_ctc2d_variant_vs_oracle(cuda, case, env):
    from megreader_b200 import ctc2d
    env(case)
    dtype = np.float64 if case["real"] == "double" else np.float32
    T, H, N, C, S, blank = (case[k] for k in ("T", "H", "N", "C", "S", "blank"))
    lp, tg, il, tl = make_inputs(case, dtype)
    go = (1.0 + np.arange(N) % 5 / 4.0).astype(dtype)
    if case["scalar_go"]:
        go[:] = 0.75
    d_lp = _on(cuda, lp, offset=case["offset"])
    d_tg = _on(cuda, tg, strided=case["strided"])
    d_il, d_tl = _on(cuda, il), _on(cuda, tl)
    d_go = torch.tensor(0.75, dtype=d_lp.dtype, device=cuda) if case["scalar_go"] else _on(cuda, go)
    assert (d_lp.data_ptr() % 16 != 0) == case["offset"]
    want = expected(case)

    if case["entry"] == "contract":
        def run():
            nll, la = ctc2d.ctc2d_forward(d_lp, d_tg, d_il, d_tl, blank, 0.0)
            return nll, la, ctc2d.ctc2d_backward(d_go, d_lp, d_tg, d_il, d_tl, nll, la, blank)
        nll, la, gr = cv.run_expecting(want, run)
    else:
        if case["offset"]:   # keep the misaligned storage: the gradient is taken with respect to the view itself
            x = d_lp._base.requires_grad_(True)[1:].view(d_lp.shape)
        else:
            x = d_lp.detach().requires_grad_(True)

        def run():
            loss = ctc2d.ctc_loss_2d(x, d_tg, d_il, d_tl, blank)
            g, = torch.autograd.grad((loss * d_go).sum(), x)
            return loss, None, g
        nll, la, gr = cv.run_expecting(want, run)
        assert (x.data_ptr() % 16 != 0) == case["offset"]

    sel = case["subset"] if case["subset"] is not None else np.arange(N)
    lps = np.ascontiguousarray(lp[:, :, sel]).astype(np.float64)
    nll_ref, la_ref = capi.ctc2d_forward(lps, tg[sel], il[sel], tl[sel], blank)
    gr_ref = capi.ctc2d_backward(go[sel].astype(np.float64), lps, tg[sel], il[sel], tl[sel], nll_ref, la_ref, blank)
    f64 = dtype == np.float64
    nll = nll.detach().cpu().numpy()[sel]
    assert np.array_equal(np.isinf(nll), np.isinf(nll_ref)), (nll, nll_ref)
    np.testing.assert_allclose(nll, nll_ref, rtol=1e-10 if f64 else 1e-4)
    if la is not None:
        la = la.cpu().numpy()[sel]
        fin = np.isfinite(la_ref)
        assert np.array_equal(np.isfinite(la), fin), "log_alpha -inf pattern differs"
        assert np.all(la[~fin] == la_ref[~fin])
        np.testing.assert_allclose(la[fin], la_ref[fin], rtol=1e-9 if f64 else 1e-4, atol=1e-9 if f64 else 1e-4)
    g = gr.cpu().numpy()[:, :, sel]
    assert np.array_equal(g == 0, gr_ref == 0), "zero pattern of the gradient differs (K3 :506-513)"
    bnd = _grad_bound(gr_ref, lps, go[sel], nll_ref, il[sel], T, 1e-8 if f64 else 2e-4, 1e-10 if f64 else 2e-5, 2)
    _assert_within(g, gr_ref, bnd, "grad")


# ---------------------------------------------------------------- 1D
CASES_1D = [c for c in CASES if c["entry"] == "ctc1d"]


@pytest.mark.parametrize("reduction", ["none", "mean", "sum"])
@pytest.mark.parametrize("zero_inf", [True, False], ids=["zinf", "inf"])
@pytest.mark.parametrize("case", CASES_1D, ids=[c["id"] for c in CASES_1D])
def test_ctc1d_variant_vs_torch(cuda, case, zero_inf, reduction, env):
    from megreader_b200 import ctc1d
    env(case)
    T, N, C, S, blank = (case[k] for k in ("T", "N", "C", "S", "blank"))
    lp, tg, il, tl = make_inputs(case)
    logits = (lp[:, 0] * 1.5).astype(np.float32)           # [T, N, C]; any logits: the op applies log_softmax itself
    w = (1.0 + np.arange(N) % 3).astype(np.float64)        # reduction none: a per-sample output gradient
    feas = np.array([int(tl[b]) + _repeats(list(tg[b, :tl[b]])) <= il[b] for b in range(N)])
    x = _on(cuda, logits).requires_grad_(True)

    def run():
        loss, _ = ctc1d.ctc_loss_from_logits(x, _on(cuda, tg, strided=case["strided"]), _on(cuda, il), _on(cuda, tl), blank,
                                             zero_inf, reduction)
        nll, _ = ctc1d.LogSoftmaxCTCFunction.apply(x.detach(), _on(cuda, tg), _on(cuda, il), _on(cuda, tl), blank, zero_inf)
        out = loss * torch.from_numpy(w).float().to(cuda) if reduction == "none" else loss
        g, = torch.autograd.grad(out.sum(), x)
        return loss.detach(), nll, g
    loss, nll, g = cv.run_expecting(expected(case), run)

    xr = torch.from_numpy(logits).double().requires_grad_(True)
    lr = torch.nn.functional.log_softmax(xr, dim=2)
    args = (lr, torch.from_numpy(tg), torch.from_numpy(il), torch.from_numpy(tl))
    nll_ref = torch.nn.functional.ctc_loss(*args, blank=blank, reduction="none", zero_infinity=zero_inf).detach().numpy()
    loss_ref = torch.nn.functional.ctc_loss(*args, blank=blank, reduction=reduction, zero_infinity=zero_inf)
    out_ref = loss_ref * torch.from_numpy(w) if reduction == "none" else loss_ref
    g_ref, = torch.autograd.grad(out_ref.sum(), xr)
    g_ref = g_ref.numpy()

    sel = case["subset"] if case["subset"] is not None else np.arange(N)
    nll = nll.cpu().numpy()
    assert np.array_equal(np.isinf(nll[sel]), ~feas[sel] & (not zero_inf))
    assert np.array_equal(nll[sel] == 0, nll_ref[sel] == 0)
    np.testing.assert_allclose(nll[sel], nll_ref[sel], rtol=1e-4)
    if zero_inf or feas.all():
        np.testing.assert_allclose(loss.cpu().numpy(), loss_ref.detach().numpy(), rtol=1e-4)
    else:
        assert np.isinf(loss.cpu().numpy()).any()
    keep = sel[feas[sel] | zero_inf]                      # torch's gradient of an infeasible sample without zero_infinity: NaN
    g, g_ref = g.cpu().numpy()[:, keep], g_ref[:, keep]
    # exact zeros: t >= Tb, and every column of a sample that zero_infinity drops (its factors are zero, so p f - p sum p f
    # is exactly 0; a factor of 1 would cancel only up to the rounding of sum p)
    assert np.array_equal(g == 0, g_ref == 0), "zero pattern of the logits gradient differs"
    # d loss / d logits = scale (p fac - p sum_c p fac): the logits gradient carries the fp32 log_softmax on top of the CTC
    # factors, one more 2^-24 |p| per class sum -- inside the 2e-4 relative bound
    scale = {"none": w[keep], "mean": 1.0 / (N * np.maximum(tl[keep], 1)), "sum": np.ones(len(keep))}[reduction]
    bnd = 2e-4 * np.abs(g_ref) + 2e-5 * scale[None, :, None]
    if T > 64:   # the Tb-dependent term of the module docstring, through p (fac - sum_c p fac): at most twice the posterior's
        p = np.exp(lr.detach().numpy()[:, keep])
        M = np.abs(np.where(np.isfinite(nll_ref[keep]), nll_ref[keep], 0)) + np.abs(lr.detach().numpy()).max()
        bnd = bnd + 2 * scale[None, :, None] * p * np.expm1(3 * il[keep] * (2.0 ** -24 * M + 2.0 ** -21))[None, :, None]
    _assert_within(g, g_ref, bnd, "grad_logits")
