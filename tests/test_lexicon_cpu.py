"""CPU: the PRODUCT's arithmetic of lexicon-constrained CTC decoding (megreader_b200/csrc/lexicon_core.cuh -- the code the CUDA
kernels of csrc/lexicon.cu run) compiled for the host by tests/host_harness/lexicon_core_host.cpp, in float and in double,
against the float64 restatement (tests/lexicon_port.py) on the seeded cases of tests/lexicon_cases.py; the banded Levenshtein
distance and the (score, index) ordering on their own; WordList's refusals and per-image packing; and the C-ABI's argument
checks, which return before any CUDA call."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

from oracle.rec_measure_port import levenshtein
from tests import lexicon_cases as lc
from tests import lexicon_port as port

HERE = os.path.dirname(os.path.abspath(__file__))
CASES = lc.all_cases()


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    gxx = shutil.which("g++")
    if not gxx:
        pytest.skip("g++ not available")
    so = str(tmp_path_factory.mktemp("harness") / "liblexicon_core_host.so")
    subprocess.check_call([gxx, "-O2", "-std=c++17", "-shared", "-fPIC", "-ffp-contract=off",
                           "-I", os.path.join(HERE, "..", "megreader_b200", "csrc"),
                           os.path.join(HERE, "host_harness", "lexicon_core_host.cpp"), "-o", so])
    lib = ctypes.CDLL(so)
    lib.host_word_score_f32.restype = ctypes.c_float
    lib.host_word_score_f64.restype = ctypes.c_double
    lib.host_score_key.restype = ctypes.c_uint64
    lib.host_score_key.argtypes = [ctypes.c_float, ctypes.c_int]
    lib.host_lpe_f32.argtypes = lib.host_lpe_f64.argtypes = [ctypes.c_void_p] * 2 + [ctypes.c_int] * 4 + [ctypes.c_float,
                                                                                                          ctypes.c_void_p]
    for f in (lib.host_decode_f32, lib.host_decode_f64):
        f.argtypes = [ctypes.c_void_p] * 2 + [ctypes.c_int] * 5 + [ctypes.c_float, ctypes.c_void_p, ctypes.c_void_p,
                                                                    ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_int] \
            + [ctypes.c_void_p] * 5
    return lib


def _p(a):
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


def table(words):
    ids = [lc.ids(w) for w in words]
    off = np.zeros(len(ids) + 1, np.int32)
    np.cumsum([len(r) for r in ids], out=off[1:])
    cls = np.array([c for r in ids for c in r], np.int32)
    return ids, cls, off


def host_decode(lib, c, real, max_words=None):
    prob = np.ascontiguousarray(c["prob"], np.float32)
    mask = None if c["mask"] is None else np.ascontiguousarray(c["mask"], np.float32)
    N, C, H, W = prob.shape
    _, cls, off = table(c["words"])
    ranges = None if c["ranges"] is None else np.ascontiguousarray(c["ranges"], np.int64)
    labels = np.ascontiguousarray(port.greedy(prob, mask).numpy(), np.int32)
    word, cand, status = (np.zeros(N, np.int32) for _ in range(3))
    score = np.zeros(N, np.float64 if real == "f64" else np.float32)
    M = len(c["words"]) if max_words is None else max_words
    delta = -1 if c["delta"] is None else c["delta"]
    getattr(lib, "host_decode_" + real)(_p(prob), _p(mask), N, C, H, W, 0, port.TINY, _p(cls), _p(off), len(c["words"]),
                                        _p(ranges), M, delta, _p(labels), _p(word), _p(score), _p(cand), _p(status))
    return dict(labels=labels, word=word, score=score, candidates=cand, status=status)


def host_lpe(lib, c, real):
    prob = np.ascontiguousarray(c["prob"], np.float32)
    mask = None if c["mask"] is None else np.ascontiguousarray(c["mask"], np.float32)
    N, C, H, W = prob.shape
    lpe = np.zeros((N, W, C), np.float64 if real == "f64" else np.float32)
    getattr(lib, "host_lpe_" + real)(_p(prob), _p(mask), N, C, H, W, port.TINY, _p(lpe))
    return lpe


def assert_scores(got, want, rtol):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    assert np.array_equal(np.isneginf(got), np.isneginf(want)), (got, want)
    f = np.isfinite(want)
    np.testing.assert_allclose(got[f], want[f], rtol=rtol, atol=0)


@pytest.mark.parametrize("name", sorted(CASES))
@pytest.mark.parametrize("real,rtol", [("f64", 1e-9), ("f32", 1e-5)])
def test_decode_equals_oracle(harness, name, real, rtol):
    c = CASES[name]
    want = port.decode(c["prob"], [lc.ids(w) for w in c["words"]], c["ranges"], c["delta"], c["mask"])
    got = host_decode(harness, c, real)
    for k in ("word", "candidates", "status", "labels"):
        np.testing.assert_array_equal(got[k], want[k], err_msg=k)
    assert_scores(got["score"], want["score"], rtol)


@pytest.mark.parametrize("name", sorted(CASES))
@pytest.mark.parametrize("real,rtol", [("f64", 1e-9), ("f32", 1e-5)])
def test_every_candidate_score(harness, name, real, rtol):
    """the score of every scored (sample, word) pair, -inf for the words that cannot be aligned"""
    c = CASES[name]
    ids, _, _ = table(c["words"])
    want = port.decode(c["prob"], ids, c["ranges"], c["delta"], c["mask"])["scores"]
    lpe = host_lpe(harness, c, real)
    fn = getattr(harness, "host_word_score_" + real)
    ptr = ctypes.POINTER(ctypes.c_double if real == "f64" else ctypes.c_float)
    W, C = lpe.shape[1:]
    pairs = 0
    for n, scores in enumerate(want):
        row = np.ascontiguousarray(lpe[n])
        got = [fn(row.ctypes.data_as(ptr), W, C, _p(np.array(ids[k], np.int32)), len(ids[k]), 0) for k in scores]
        assert_scores(got, list(scores.values()), rtol)
        pairs += len(scores)
    assert pairs > 0


def test_cases_cover_the_edges():
    got = {name: port.decode(c["prob"], [lc.ids(w) for w in c["words"]], c["ranges"], c["delta"], c["mask"])
           for name, c in CASES.items()}
    d0 = got["1d_peaked_d0"]
    assert (d0["word"][[2, 3]] == -1).all() and d0["candidates"][2] == 0     # empty range: greedy
    allinf = got["1d_peaked_dNone"]
    assert allinf["candidates"][3] == 2 and allinf["word"][3] == -1            # all infeasible: greedy
    assert all(np.isneginf(s) for s in allinf["scores"][3].values())
    words = CASES["1d_peaked_dNone"]["words"]
    assert any(words[k] in ("LL", "BOOK") for k in allinf["word"] if k >= 0)
    for name in ("1d_peaked_dNone", "2d_peaked_dNone", "1d_flat", "2d_flat"):
        c = CASES[name]
        for n, k in enumerate(got[name]["word"]):
            if k < 0:
                continue
            b = c["ranges"][n][0]
            first = [j for j in range(b, c["ranges"][n][1]) if c["words"][j] == c["words"][k]][0]
            assert k == first, (name, n)                                      # duplicates: the lowest index
    lw = got["long_words"]["scores"][0]
    assert np.isfinite(lw[0]) and np.isneginf(lw[1]) and np.isfinite(lw[2])     # 64 classes; 64 + 32 repeats > 65 frames
    assert sum(len(s) for s in got["1d_peaked_d3"]["scores"]) < sum(len(s) for s in got["1d_peaked_dNone"]["scores"])


def test_banded_levenshtein(harness):
    rng = np.random.default_rng(5)
    for _ in range(3000):
        w = rng.integers(2, 8, rng.integers(1, 65)).astype(np.int32)
        g = rng.integers(2, 8, rng.integers(0, 70)).astype(np.int32)
        if rng.random() < 0.5:
            g = np.array(lc.ids(lc.edit(rng, "".join(lc.LETTERS[c] for c in w), int(rng.integers(0, 5)))), np.int32)
        d = levenshtein(list(w), list(g))
        for delta in (0, 1, 2, 3, 5, 200):
            got = harness.host_levenshtein(_p(w), len(w), _p(g), len(g), delta)
            assert got == min(d, delta + 1), (list(w), list(g), delta)


def test_oracle_levenshtein_many():
    rng = np.random.default_rng(6)
    words = [list(rng.integers(2, 6, rng.integers(1, 20))) for _ in range(300)]
    for _ in range(20):
        g = list(rng.integers(2, 6, rng.integers(0, 25)))
        assert port.levenshtein_many(words, g).tolist() == [levenshtein(w, g) for w in words]


def test_score_key_orders_score_then_lowest_index(harness):
    vals = [-np.inf, -1e30, -5.5, -5.5, -1e-30, -0.0, 0.0, 1e-30, 3.0, np.nan]
    key = harness.host_score_key
    assert key(float("-inf"), 3) == 0 and key(float("nan"), 3) == 0
    assert key(-0.0, 7) == key(0.0, 7)
    finite = [v for v in vals if np.isfinite(v)]
    for a in finite:
        for b in finite:
            for i, j in ((0, 1), (1, 0), (5, 5)):
                want = (np.float32(a), -i) > (np.float32(b), -j)
                assert (key(a, i) > key(b, j)) == want, (a, i, b, j)


def test_overflow_and_bad_range(harness):
    c = dict(CASES["1d_peaked_dNone"])
    want_greedy = port.greedy(c["prob"]).numpy()
    got = host_decode(harness, c, "f64", max_words=10)
    lens = c["ranges"][:, 1] - c["ranges"][:, 0]
    assert (got["status"] == np.where(lens > 10, 1, 0)).all() and (lens > 10).any()
    over = lens > 10
    assert (got["word"][over] == -1).all() and np.array_equal(got["labels"][over], want_greedy[over])
    c["ranges"] = c["ranges"].copy()
    c["ranges"][0] = (5, 4)
    assert host_decode(harness, c, "f64")["status"][0] == 2


def test_wordlist_refuses_bad_words():
    from megreader_b200.lexicon import WordList
    with pytest.raises(ValueError, match="'AB-C'"):
        WordList(["AB", "AB-C"], lc.CS, device="cpu")
    with pytest.raises(ValueError, match="empty"):
        WordList(["AB", ""], lc.CS, device="cpu")
    with pytest.raises(ValueError, match="'%s'" % ("Z" * 65)):
        WordList(["Z" * 65], lc.CS, device="cpu")
    w = WordList(["book", "Z" * 64, "BOOK"], lc.CS, device="cpu")
    assert w.offsets.tolist() == [0, 4, 68, 72] and w.cls[:4].tolist() == lc.ids("BOOK") and w.max_list == 3


def test_wordlist_per_image_ranges(tmp_path):
    from megreader_b200.lexicon import WordList
    path = tmp_path / "lex.txt"
    path.write_text("ZETA alpha\nALPHA zeta ZETA\n")
    words, ranges = WordList.per_image([["A", "B"], [], ["C", "A", "A"], str(path)], lc.CS, device="cpu")
    assert ranges.dtype.is_floating_point is False and ranges.tolist() == [[0, 2], [2, 2], [2, 5], [5, 9]]
    assert words.words[5:] == ["ALPHA", "ZETA", "alpha", "zeta"] and words.max_list == 4 and len(words) == 9
    shared = WordList(str(path), lc.CS, device="cpu")
    assert shared.words == ["ALPHA", "ZETA", "alpha", "zeta"] and shared.max_list == 4


def test_capi_argument_checks():
    from megreader_b200 import _lib, build
    build.build()
    L = _lib.lib()
    r = lambda n: -(-n // 256) * 256  # noqa: E731
    for N, M in ((1, 0), (3, 50), (512, 50000), (65535, 7)):
        assert L.mr_lexicon_workspace_bytes(N, M) == 2 * r(4 * N) + r(8 * N) + r(4 * N * M)
    assert L.mr_lexicon_workspace_bytes(65536, 1) == 0 and L.mr_lexicon_workspace_bytes(-1, 1) == 0
    assert L.mr_lexicon_workspace_bytes(1, -1) == 0 and L.mr_lexicon_workspace_bytes(65535, 2 ** 20) == 0
    P = 0x10000                                                # never dereferenced: every check comes first
    ws = L.mr_lexicon_workspace_bytes(4, 10)

    def call(N=4, C=38, H=1, W=33, blank=0, tiny=1e-38, cls=P, off=P, n_words=20, M=10, delta=-1, workspace=P, nbytes=ws,
             labels=P, out=P):
        return L.mr_lexicon_ctc_decode(P, None, N, C, H, W, 1, 1, 1, 1, 0, 0, 0, blank, 1, tiny, cls, off, n_words, None, M,
                                       delta, workspace, nbytes, labels, out, out, out, out, None)
    BAD, NULL = 4, 1
    assert call(delta=-2) == BAD and call(N=-1) == BAD and call(N=65536) == BAD and call(W=0) == BAD
    assert call(C=0) == BAD and call(M=-1) == BAD and call(n_words=-1) == BAD and call(tiny=0.0) == BAD
    assert call(blank=38) == 2 and call(blank=-1) == 2
    assert call(cls=None) == NULL and call(off=None) == NULL and call(workspace=None) == NULL
    assert call(labels=None) == NULL and call(out=None) == NULL
    assert call(nbytes=ws - 1) == BAD and call(M=100) == BAD
    assert call(W=2000) == _lib.MR_ERR_UNSUPPORTED                      # 2000 x 38 log-probabilities: no room
    assert call(N=0) == 0
