"""CPU: the PRODUCT's arithmetic of the text recognisers' validation measure (megreader_b200/csrc/rec_measure_core.cuh -- the code
the CUDA kernels of csrc/rec_measure.cu run) compiled for the host by tests/host_harness/rec_measure_core_host.cpp, checked against
  * the plain-Python oracle (oracle/rec_measure_port.py) on 20,000 seeded label pairs of lengths 0 to 200 over four charsets
    (English, EnglishPrintable, a Chinese-size one, a custom one with expanding and supplementary-plane characters);
  * np.sum for every length from 1 to 1,100 (numpy's pairwise order), and the meter updates of gather_measure;
and the oracle against the golden recorded from the reference's own measurer and representers, plus the reference's lexicon
quirks (skipped where the reference tree is absent) and the fold table's refusal."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

from oracle import rec_measure_port as port
from tests import rec_measure_cases as cases

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    gxx = shutil.which("g++")
    if not gxx:
        pytest.skip("g++ not available")
    so = str(tmp_path_factory.mktemp("harness") / "librec_measure_core_host.so")
    subprocess.check_call([gxx, "-O2", "-std=c++17", "-shared", "-fPIC", "-ffp-contract=off",
                           "-I", os.path.join(HERE, "..", "megreader_b200", "csrc"),
                           os.path.join(HERE, "host_harness", "rec_measure_core_host.cpp"), "-o", so])
    lib = ctypes.CDLL(so)
    lib.host_pairwise_sum.restype = ctypes.c_double
    lib.host_pairwise_two_pass.restype = ctypes.c_double
    lib.host_hash.restype = ctypes.c_uint64
    return lib


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def table(charset):
    from megreader_b200.rec_measure import fold_table
    t = fold_table(charset, "cpu")
    return np.ascontiguousarray(t.len.numpy()), np.ascontiguousarray(t.cp.numpy())


def host_pairs(lib, gt, pred, tab):
    gt, pred = np.ascontiguousarray(gt, np.int64), np.ascontiguousarray(pred, np.int64)
    n = len(gt)
    gl, pl, st, d = (np.zeros(n, np.int32) for _ in range(4))
    score = np.zeros(n)
    lib.host_pairs(_p(gt), gt.shape[1], _p(pred), pred.shape[1], n, _p(tab[0]), _p(tab[1]), len(tab[0]), _p(gl), _p(pl), _p(st),
                   _p(d), _p(score))
    return gl, pl, st, d, score


@pytest.mark.parametrize("name", ["english", "printable", "chinese", "custom"])
def test_core_equals_oracle(harness, name):
    cs = cases.charsets()[name]
    tab = table(cs)
    rng = np.random.default_rng(["english", "printable", "chinese", "custom"].index(name) + 20)
    gt, pred = cases.pair_corpus(rng, len(cs), 5000)
    gl, pl, st, d, score = host_pairs(harness, gt, pred, tab)
    assert not st.any()
    equal = 0
    for i in range(len(gt)):
        g, p = port.fold(cs, gt[i]), port.fold(cs, pred[i])
        assert (gl[i], pl[i]) == (len(g), len(p)), i
        want = port.levenshtein(g, p)
        assert d[i] == want, (i, g, p)
        assert score[i] == port.edit_score(g, p), i
        equal += g == p
    assert equal > 100 and gl.max() > 150 and (gl == 0).sum() > 5
    if name == "custom":
        assert (gl > np.count_nonzero(gt > 1, axis=1)).any()      # 'ß' and 'ﬁ' expanded


def test_bad_labels(harness):
    cs = cases.charsets()["english"]
    tab = table(cs)
    gt = np.array([[2, 3, 38, 0], [2, 3, 0, 0], [-1, 2, 0, 0]])
    pred = np.array([[2, 3, 0, 0], [2, -5, 0, 0], [2, 0, 0, 0]])
    _, _, st, _, _ = host_pairs(harness, gt, pred, tab)
    assert st.tolist() == [1, 1, 1]


def test_fold_table():
    from megreader_b200.rec_measure import fold_table
    cs = cases.charsets()["custom"]
    lens, cps = table(cs)
    for i in range(len(cs)):
        want = "" if i < 2 else cs[i].upper()
        assert "".join(chr(c) for c in cps[i, :lens[i]]) == want
    assert lens.max() == 2 and (cps[:, :] >= 0x10000).any()
    from megreader_b200.charset import EnglishCharset
    lens, _ = table(EnglishCharset())
    assert lens.tolist() == [0, 0] + [1] * 36

    class Long(cases.ListCharset):
        pass
    with pytest.raises(ValueError, match="more than 4"):
        fold_table(Long(["ab", "hello"]), "cpu")


def test_pairwise_sum_equals_numpy(harness):
    rng = np.random.default_rng(3)
    for n in range(1, 1101):
        a = np.ascontiguousarray(rng.random(n) * 10.0 ** rng.integers(-6, 7, n))
        want = np.array(list(a)).sum()
        assert harness.host_pairwise_sum(_p(a), n) == want, n
        assert harness.host_pairwise_two_pass(_p(a), n) == want, n
        assert port.pairwise_sum(a) == want, n
    for n in (4096, 4099, 65536 + 13, 300001):       # deeper trees, as the batch kernel sums them (leaves, then the tree)
        a = np.ascontiguousarray(rng.random(n) * 10.0 ** rng.integers(-6, 7, n))
        assert harness.host_pairwise_two_pass(_p(a), n) == a.sum() == harness.host_pairwise_sum(_p(a), n), n
    assert harness.host_pairwise_sum(_p(np.zeros(1)), 0) == harness.host_pairwise_two_pass(_p(np.zeros(1)), 0) == 0.0


def test_hash_depends_on_every_symbol(harness):
    seen = set()
    for w in ["", "A", "B", "AB", "BA", "AA", "A\0", "\U00010400"]:
        cp = np.frombuffer(w.encode("utf-32-le"), np.int32).copy() if w else np.zeros(1, np.int32)
        seen.add(harness.host_hash(_p(cp), len(w)))
    assert len(seen) == 8


def meters_of(totals):
    from megreader_b200 import rec_measure
    return rec_measure.gather(totals)


def same_meters(got, want):
    assert sorted(got) == sorted(want)
    for k in want:
        g = [got[k].val, got[k].sum, got[k].count, got[k].avg]
        w = [want[k].val, want[k].sum, want[k].count, want[k].avg]
        assert np.array_equal(np.array(g, np.float64), np.array(w, np.float64), equal_nan=True), (k, g, w)
        assert g[2] == w[2] and type(g[2]) is int


@pytest.mark.parametrize("lexicon", [False, True])
def test_meter_updates_equal_oracle(harness, lexicon):
    rng = np.random.default_rng(11 + lexicon)
    sizes = [16, 3, 1, 200, 9, 700]
    acc = (rng.random(sum(sizes)) < 0.3).astype(np.uint8)
    ed = np.where(acc, 1.0, rng.random(sum(sizes)))
    ed[rng.random(len(ed)) < 0.1] = 0.0
    inl = (rng.random(sum(sizes)) < 0.4).astype(np.uint8)
    inl[16:19] = 1                                    # a batch with no out-of-lexicon sample
    inl[19] = 0
    inl[:16] = 0                                      # and one without in-lexicon samples before any other
    totals = np.zeros(25)
    harness.host_totals(_p(np.array(sizes, np.int32)), len(sizes), _p(acc), _p(ed), _p(inl), int(lexicon), _p(totals))
    raw, o = [], 0
    for n in sizes:
        m = dict(accuracy=[bool(v) for v in acc[o:o + n]], edit_distance=[float(v) for v in ed[o:o + n]])
        if lexicon:
            m["in_lexicon"] = [bool(v) for v in inl[o:o + n]]
        raw.append(m)
        o += n
    want = port.SequenceRecognitionMeasurer(["X"] if lexicon else None).gather_measure(raw)
    same_meters(meters_of(totals), want)
    from megreader_b200.rec_measure import SequenceRecognitionMeasurer
    m = SequenceRecognitionMeasurer()
    m._words = {"X"} if lexicon else None
    same_meters(m.gather_measure(raw), want)


# ---- the oracle against the golden of the reference's measurer and representers ----

def golden():
    return np.load(os.path.join(HERE, "golden", "rec_measure_ref.npz"))


def golden_cases():
    from oracle.make_rec_measure_golden import CASES
    return CASES


@pytest.mark.parametrize("lexicon", [False, True])
def test_oracle_equals_golden(lexicon):
    z = golden()
    words = set(z["lexicon"].tolist())
    for name, rep, seed, N, W, batches in golden_cases():
        m = port.SequenceRecognitionMeasurer(words if lexicon else None)
        raw = []
        for b in range(batches):
            out = [{'label_string': g, 'pred_string': p} for g, p in zip(z["%s/%d/label_string" % (name, b)].tolist(),
                                                                         z["%s/%d/pred_string" % (name, b)].tolist())]
            r = m.measure(None, out)
            assert r["accuracy"] == z["%s/%d/accuracy" % (name, b)].tolist()
            assert r["edit_distance"] == z["%s/%d/edit_distance" % (name, b)].tolist()
            if lexicon:
                assert r["in_lexicon"] == z["%s/%d/in_lexicon" % (name, b)].tolist()
            raw.append(r)
        g = m.gather_measure(raw)
        tag = "lexicon" if lexicon else "plain"
        names = z["%s/%s/meters" % (name, tag)].tolist()
        got = np.array([[float(g[k].val), float(g[k].sum), float(g[k].count), float(g[k].avg)] for k in names])
        assert np.array_equal(got, z["%s/%s/values" % (name, tag)], equal_nan=True), name


def test_golden_strings_follow_the_port():
    """the golden's strings are the representers' collapse of the seeded inputs, label_to_string'd (labels as recorded)"""
    from oracle.make_rec_measure_golden import case_batch
    z = golden()
    cs = cases.charsets()["english"]
    for name, rep, seed, N, W, batches in golden_cases():
        for b in range(batches):
            labels, pred = case_batch(rep, seed * 100 + b, N, W)
            assert np.array_equal(z["%s/%d/labels" % (name, b)], labels)
            if rep == "CTCRepresenter":
                rows = [port.collapse(r) for r in pred[:, :, 0, :].argmax(1)]
            elif rep == "SequenceRecognitionRepresenter":
                rows = [port.blank_after_first_blank(r) for r in pred]
            else:
                continue                                   # the 2D path is checked on the GPU against the golden
            want = ["".join(cs[i] for i in r if i > 1) for r in rows]
            assert z["%s/%d/pred_string" % (name, b)].tolist() == want


@pytest.fixture(scope="module")
def reference():
    from oracle import make_rec_measure_golden as gen
    ref = gen.reference()
    if ref is None:
        pytest.skip("reference tree not present")
    return ref


def test_golden_is_current(reference, tmp_path):
    from oracle import make_rec_measure_golden as gen
    reps, mm = reference
    path = str(tmp_path / "lexicon.txt")
    words = gen.lexicon_file(path)
    z = golden()
    assert z["lexicon"].tolist() == words
    for name, rep, seed, N, W, batches in gen.CASES:
        for k, v in gen.run_case(reps, mm, path, rep, seed, N, W, batches).items():
            assert np.array_equal(z[name + "/" + k], v, equal_nan=v.dtype.kind == "f"), (name, k)


def test_reference_lexicon_quirks(reference, tmp_path):
    """an empty lexicon file is falsy (no in / out split); lowercase words never match; words with characters outside the
    charset are kept and match only an equal upper-cased string"""
    from megreader_b200.rec_measure import SequenceRecognitionMeasurer
    _, mm = reference
    out = [{'label_string': 'hello', 'pred_string': 'HELLO'}, {'label_string': 'ÉTÉ', 'pred_string': ''},
           {'label_string': 'abc', 'pred_string': 'abd'}]
    empty = tmp_path / "empty.txt"
    empty.write_text("\n  \n")
    r = mm.SequenceRecognitionMeasurer(nori_lexicon_path=str(empty))
    assert sorted(r.measure(None, out)) == ["accuracy", "edit_distance"]
    assert sorted(r.gather_measure([r.measure(None, out)], None)) == ["accuracy", "edit_distance"]
    assert SequenceRecognitionMeasurer(str(empty)).nori_lexicon is None
    words = tmp_path / "words.txt"
    words.write_text("hello ABC\nÉTÉ abc\n")
    r = mm.SequenceRecognitionMeasurer(nori_lexicon_path=str(words))
    assert r.measure(None, out)["in_lexicon"] == [False, True, True]
    assert port.SequenceRecognitionMeasurer({"hello", "ABC", "ÉTÉ", "abc"}).measure(None, out) == r.measure(None, out)


def test_measurer_takes_config_keywords():
    from megreader_b200 import rec_measure
    m = rec_measure.SequenceRecognitionMeasurer(**{'class': 'structure.measurers.SequenceRecognitionMeasurer'}, cmd={})
    assert m.nori_lexicon is None and m.validate_measure.__func__ is m.evaluate_measure.__func__


def test_measurer_empty_batch():
    """an empty output list gives the reference's structures with empty lists, as the reference's loops do"""
    from megreader_b200 import rec_measure
    assert rec_measure.SequenceRecognitionMeasurer().measure(None, []) == dict(accuracy=[], edit_distance=[])
    m = rec_measure.SequenceRecognitionMeasurer()
    m._words = {"X"}
    assert m.measure(None, []) == dict(accuracy=[], edit_distance=[], in_lexicon=[])
    assert port.SequenceRecognitionMeasurer({"X"}).measure(None, []) == m.measure(None, [])
