"""GPU: lexicon-constrained CTC decoding (megreader_b200.lexicon, csrc/lexicon.cu) against the float64 restatement
(tests/lexicon_port.py) on the seeded cases of tests/lexicon_cases.py, against the project's own CTC ops (ctc1d for H = 1,
ctc2d_forward for H = 8) on the chosen words, end to end after a seeded CRNN at crnn.yaml's input size with per-image and
shared word lists, under CUDA-graph replay with new probabilities and ranges, and with a range longer than
max_words_per_sample."""
import numpy as np
import pytest
import torch

from tests import lexicon_cases as lc
from tests import lexicon_port as port

pytestmark = pytest.mark.gpu
CASES = lc.all_cases()


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def run(c, dev, **kw):
    from megreader_b200 import lexicon
    words = lexicon.WordList(c["words"], lc.CS, dev)
    ranges = None if c["ranges"] is None else torch.from_numpy(np.asarray(c["ranges"], np.int64)).to(dev)
    mask = None if c["mask"] is None else torch.from_numpy(c["mask"]).to(dev)
    out = lexicon.decode_packed(torch.from_numpy(c["prob"]).to(dev), words, ranges, c["delta"], mask=mask, **kw)
    return {k: v.cpu().numpy() for k, v in out.items()}


def assert_scores(got, want, rtol=1e-5):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    assert np.array_equal(np.isneginf(got), np.isneginf(want)), (got, want)
    f = np.isfinite(want)
    np.testing.assert_allclose(got[f], want[f], rtol=rtol, atol=0)


@pytest.mark.parametrize("name", sorted(CASES))
def test_device_equals_oracle(name):
    dev = _dev()
    c = CASES[name]
    want = port.decode(c["prob"], [lc.ids(w) for w in c["words"]], c["ranges"], c["delta"], c["mask"])
    got = run(c, dev)
    for k in ("word", "candidates", "status", "labels"):
        np.testing.assert_array_equal(got[k], want[k], err_msg=k)
    assert_scores(got["score"], want["score"])


@pytest.mark.parametrize("name", ["1d_flat", "1d_peaked_dNone", "2d_flat", "2d_peaked_dNone", "1d_w65", "long_words"])
def test_chosen_scores_equal_the_ctc_ops(name):
    """every sample's rows repeated once per candidate word and fed to the existing CTC ops: their nll of every candidate
    equals -score of the float64 restatement, and the nll of the chosen word equals -score of the device"""
    from megreader_b200 import ctc1d, ctc2d
    dev = _dev()
    c = CASES[name]
    ids = [lc.ids(w) for w in c["words"]]
    want = port.decode(c["prob"], ids, c["ranges"], c["delta"], c["mask"])
    got = run(c, dev)
    lp = port.log_probs(c["prob"], c["mask"]).float()                      # (W, H, N, C)
    T, H, N, C = lp.shape
    checked = 0
    for n in range(N):
        ks = [k for k, s in want["scores"][n].items() if np.isfinite(s)]
        if not ks:
            continue
        S = max(len(ids[k]) for k in ks)
        tg = torch.zeros((len(ks), S), dtype=torch.int64)
        for i, k in enumerate(ks):
            tg[i, :len(ids[k])] = torch.tensor(ids[k])
        tl = torch.tensor([len(ids[k]) for k in ks], dtype=torch.int64)
        il = torch.full((len(ks),), T, dtype=torch.int64)
        x = lp[:, :, n:n + 1].expand(T, H, len(ks), C).contiguous().to(dev)
        if H == 1:
            nll, _ = ctc1d.ctc_loss_from_logits(x[:, 0].contiguous(), tg.to(dev), il.to(dev), tl.to(dev), zero_infinity=False,
                                                reduction="none")
        else:
            nll, _ = ctc2d.ctc2d_forward(x, tg.to(dev), il.to(dev), tl.to(dev), 0)
        nll = nll.double().cpu().numpy()
        np.testing.assert_allclose(nll, [-want["scores"][n][k] for k in ks], rtol=1e-5)
        if got["word"][n] >= 0:
            np.testing.assert_allclose(nll[ks.index(int(got["word"][n]))], -got["score"][n], rtol=1e-5)
            checked += 1
    assert checked > 0


def _crnn_probs(dev, N, seed):
    import bench
    torch.manual_seed(0)
    net = bench.build_model(dev).eval()
    rng = np.random.default_rng(seed)
    x = torch.from_numpy(rng.standard_normal((N, 3, 32, 128)).astype(np.float32)).to(dev)
    with torch.no_grad():
        return net.decoder(net.backbone(x), train=False)                    # (N, C, 1, 33)


def _compare_choices(got_word, got_score, want, words):
    """the device's words equal the restatement's except where its two best scores are within 1e-4 relative"""
    near = 0
    for n, scores in enumerate(want["scores"]):
        if got_word[n] == want["word"][n]:
            continue
        top = sorted((s for s in scores.values() if np.isfinite(s)), reverse=True)[:2]
        assert len(top) == 2 and abs(top[0] - top[1]) <= 1e-4 * abs(top[0]), (n, got_word[n], want["word"][n], top)
        assert np.isclose(got_score[n], top[0], rtol=1e-5)
        near += 1
    assert near <= 0.01 * len(want["scores"]), near
    return near


def test_crnn_end_to_end_per_image_and_shared():
    """crnn.yaml (32 x 128, W = 33), seeded weights, N = 512: LexiconCTCRepresenter with per-image lists of 50 holding the
    ground truth, and with one shared list of 50,000 words at delta = 3; measure_labels accepts the labels"""
    from megreader_b200 import lexicon, rec_measure
    dev = _dev()
    N = 512
    prob = _crnn_probs(dev, N, 3)
    rng = np.random.default_rng(4)
    truths = [lc.random_word(rng, 3, 10) for _ in range(N)]
    lists = []
    for t in truths:
        ws = [lc.edit(rng, t, int(rng.integers(1, 4))) for _ in range(30)] + [lc.random_word(rng, 2, 10) for _ in range(19)]
        ws.insert(int(rng.integers(0, 50)), t)
        lists.append(ws)
    words, ranges = lexicon.WordList.per_image(lists, lc.CS, dev)
    gt = torch.zeros((N, 32), dtype=torch.int32)
    for n, t in enumerate(truths):
        gt[n, :len(t)] = torch.tensor(lc.ids(t))
    batch = {'label': gt.to(dev), 'lexicon_ranges': ranges}
    rep = lexicon.LexiconCTCRepresenter(words)
    g, labels = rep.represent_labels(batch, prob)
    out = lexicon.decode_packed(prob, words, ranges)
    assert torch.equal(labels, out["labels"])
    ids = [lc.ids(w) for w in words.words]
    want = port.decode(prob.cpu(), ids, ranges.cpu().numpy())
    _compare_choices(out["word"].cpu().numpy(), out["score"].cpu().numpy(), want, ids)
    np.testing.assert_array_equal(out["candidates"].cpu().numpy(), 50)
    res = rec_measure.measure_labels(g, labels, rec_measure.fold_table(lc.CS, dev))
    assert int(res["status"].sum()) == 0
    strings = rep.represent(batch, prob)
    chosen = out["word"].cpu().numpy()
    assert all(s["pred_string"] == words.words[k] for s, k in zip(strings, chosen) if k >= 0)
    assert all(s["label_string"] == t for s, t in zip(strings, truths))

    # one shared list of 50,000 words, delta = 3: the oracle on the first 128 samples
    shared = sorted({lc.random_word(rng, 1, 10) for _ in range(60000)})[:50000]
    words = lexicon.WordList(shared, lc.CS, dev)
    rep = lexicon.LexiconCTCRepresenter(words, max_edit_distance=3)
    _, labels = rep.represent_labels({'label': gt.to(dev)}, prob)
    out = lexicon.decode_packed(prob, words, max_edit_distance=3)
    assert torch.equal(labels, out["labels"])
    ids = [lc.ids(w) for w in shared]
    k = 128
    want = port.decode(prob[:k].cpu(), ids, None, 3)
    _compare_choices(out["word"][:k].cpu().numpy(), out["score"][:k].cpu().numpy(), want, ids)
    np.testing.assert_array_equal(out["candidates"][:k].cpu().numpy(), want["candidates"])
    assert (out["word"] >= 0).sum() > N // 4
    assert int(rec_measure.measure_labels(g, labels, rec_measure.fold_table(lc.CS, dev))["status"].sum()) == 0


def test_graph_replay_with_new_probs_and_ranges():
    from megreader_b200 import lexicon
    dev = _dev()
    cs = [lc.case(s, N=6, W=16, H=8, delta=2) for s in (40, 41, 42)]
    words = lexicon.WordList([w for c in cs for w in c["words"]], lc.CS, dev)
    offsets = np.cumsum([0] + [len(c["words"]) for c in cs])
    inputs = [(torch.from_numpy(c["prob"]).to(dev), torch.from_numpy(c["mask"]).to(dev),
               torch.from_numpy(np.asarray(c["ranges"], np.int64) + offsets[i]).to(dev)) for i, c in enumerate(cs)]
    M = max(int((r[:, 1] - r[:, 0]).max()) for _, _, r in inputs)
    eager = [lexicon.decode_packed(p, words, r, 2, mask=m, max_words_per_sample=M) for p, m, r in inputs]
    static = [t.clone() for t in inputs[0]]
    out = lexicon.decode_packed(static[0], words, static[2], 2, mask=static[1], max_words_per_sample=M)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        lexicon.decode_packed(static[0], words, static[2], 2, mask=static[1], out=out, max_words_per_sample=M)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        lexicon.decode_packed(static[0], words, static[2], 2, mask=static[1], out=out, max_words_per_sample=M)
    for i in (2, 0, 1):
        for t, x in zip(static, inputs[i]):
            t.copy_(x)
        g.replay()
        torch.cuda.synchronize()
        for k in out:
            assert torch.equal(out[k], eager[i][k]), (i, k)
    assert len({int(e["word"].sum()) for e in eager}) == 3


def test_overflow_keeps_greedy_and_leaves_the_others():
    from megreader_b200 import decode
    dev = _dev()
    c = CASES["1d_peaked_dNone"]
    lens = c["ranges"][:, 1] - c["ranges"][:, 0]
    full = run(c, dev)
    M = 10
    got = run(c, dev, max_words_per_sample=M)
    over = lens > M
    assert over.any() and (~over).any()
    greedy = decode.ctc_greedy_decode(torch.from_numpy(c["prob"]).to(dev)).cpu().numpy()
    np.testing.assert_array_equal(got["status"], np.where(over, 1, 0))
    np.testing.assert_array_equal(got["labels"][over], greedy[over])
    assert (got["word"][over] == -1).all() and np.isneginf(got["score"][over]).all() and (got["candidates"][over] == 0).all()
    for k in ("labels", "word", "score", "candidates"):
        np.testing.assert_array_equal(got[k][~over], full[k][~over], err_msg=k)
