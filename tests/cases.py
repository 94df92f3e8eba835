"""Seeded synthetic inputs shared by the oracle tests, the GPU parity tests, smoke() and bench.py."""
import numpy as np


def ctc2d_case(seed, T, H, N, C, S, Lmax=None, peak=0.0, ragged_T=False, dtype=np.float32, blank=0):
    """SURVEY.md §8d synthetic 2D-CTC inputs: lp = log_softmax_H(mask)[...,None] + log_softmax_C(classify).
    Targets avoid the blank; feasibility (2L+1 <= T_b... loosely L <= T_b) is kept so nll is finite."""
    rng = np.random.RandomState(seed)
    Lmax = min(S, Lmax or S)
    il = np.full((N,), T, np.int64)
    if ragged_T:
        il = rng.randint(max(1, T // 2), T + 1, size=N).astype(np.int64)
    tl = np.empty((N,), np.int64)
    targets = np.zeros((N, S), np.int64)
    labels = [c for c in range(C) if c != blank]
    for b in range(N):
        lim = max(1, min(Lmax, int(il[b]) // 2))
        tl[b] = rng.randint(1, lim + 1)
        targets[b, :tl[b]] = rng.choice(labels, size=tl[b])
    m = rng.standard_normal((T, H, N)).astype(np.float64)
    c = rng.standard_normal((T, H, N, C)).astype(np.float64)
    if peak:
        for b in range(N):
            L = int(tl[b])
            for t in range(int(il[b])):
                k = min(L - 1, t * L // int(il[b]))
                c[t, :, b, targets[b, k]] += peak
    m = m - np.log(np.exp(m).sum(1, keepdims=True))
    c = c - np.log(np.exp(c).sum(3, keepdims=True))
    lp = (m[..., None] + c).astype(dtype)
    return np.ascontiguousarray(lp), targets, il, tl


def load_head_golden():
    """tests/golden/ctc2d_head_ref_<case>.npz (oracle/make_golden.py) merged into one {"<case>.<name>": array} dict."""
    import glob
    import os
    out = {}
    for f in sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "ctc2d_head_ref_*.npz"))):
        with np.load(f) as g:
            out.update({k: g[k] for k in g.files})
    assert out, "no ctc2d_head_ref_*.npz under tests/golden"
    return out


GOLDEN_SAMPLE = 512


def sample_indices(ref):
    """Which elements of a reference array the reference-kernel goldens keep: None (all of them) up to GOLDEN_SAMPLE elements,
    otherwise a fixed seeded choice of GOLDEN_SAMPLE flat indices, three quarters of them drawn from the non-zero finite entries
    (gradients over large alphabets are mostly structural zeros) and the rest from everywhere."""
    ref = np.asarray(ref).reshape(-1)
    if ref.size <= GOLDEN_SAMPLE:
        return None
    rng = np.random.RandomState(ref.size % (1 << 31))
    nz = np.flatnonzero((ref != 0) & np.isfinite(ref))
    take = min(nz.size, GOLDEN_SAMPLE * 3 // 4)
    picked = rng.choice(nz, take, replace=False) if take else np.zeros(0, np.int64)
    rest = np.setdiff1d(np.arange(ref.size), picked, assume_unique=False)
    picked = np.concatenate([picked, rng.choice(rest, GOLDEN_SAMPLE - take, replace=False)])
    return np.sort(picked).astype(np.int64)
