"""GPU: the text recognisers' validation measure (megreader_b200.rec_measure, csrc/rec_measure.cu) and the device representers
(megreader_b200.decode) against the plain-Python oracle (oracle/rec_measure_port.py) and the golden of the reference's own
measurer and representers (tests/golden/rec_measure_ref.npz): integers equal, float64 bit for bit, meters field for field."""
import os

import numpy as np
import pytest
import torch

from oracle import rec_measure_port as port
from tests import rec_measure_cases as cases

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def golden():
    return np.load(os.path.join(HERE, "golden", "rec_measure_ref.npz"))


def english():
    from megreader_b200.charset import EnglishCharset
    return EnglishCharset()


def meter_rows(g, names):
    return np.array([[float(g[k].val), float(g[k].sum), float(g[k].count), float(g[k].avg)] for k in names])


@pytest.mark.parametrize("name,dtype", [("english", torch.int32), ("printable", torch.int64), ("chinese", torch.int32),
                                        ("custom", torch.int64)])
def test_device_equals_oracle(name, dtype):
    from megreader_b200 import rec_measure
    dev = _dev()
    cs = cases.charsets()[name]
    gt, pred = cases.pair_corpus(np.random.default_rng(100 + len(name)), len(cs), 2500)
    pred = pred[:, :150]                                  # different widths
    table = rec_measure.fold_table(cs, dev)
    out = rec_measure.measure_labels(torch.from_numpy(gt).to(dev, dtype), torch.from_numpy(pred).to(dev, dtype), table)
    h = {k: v.cpu().numpy() for k, v in out.items() if k != "workspace"}
    assert not h["status"].any() and not h["in_lexicon"].any()
    for i in range(len(gt)):
        g, p = port.fold(cs, gt[i]), port.fold(cs, pred[i])
        assert (h["gt_length"][i], h["pred_length"][i]) == (len(g), len(p)), i
        assert h["distance"][i] == port.levenshtein(g, p), (i, g, p)
        assert h["edit_distance"][i] == port.edit_score(g, p) and h["accuracy"][i] == (g == p), i
    assert h["accuracy"].sum() > 50


def run_golden_case(z, name, batches, lexicon, dev, labels_of=None):
    """measure_strings (or measure_labels through labels_of(b)) over the case's batches into one totals"""
    from megreader_b200 import rec_measure
    totals = rec_measure.new_totals(dev)
    for b in range(batches):
        if labels_of is None:
            out = rec_measure.measure_strings(z["%s/%d/label_string" % (name, b)].tolist(), z["%s/%d/pred_string" % (name, b)].tolist(),
                                              lexicon, totals, dev)
        else:
            out = rec_measure.measure_labels(*labels_of(b), rec_measure.fold_table(english(), dev), lexicon, totals)
        assert out["accuracy"].cpu().numpy().tolist() == z["%s/%d/accuracy" % (name, b)].tolist()
        assert np.array_equal(out["edit_distance"].cpu().numpy(), z["%s/%d/edit_distance" % (name, b)])
        if lexicon:
            assert out["in_lexicon"].cpu().numpy().tolist() == z["%s/%d/in_lexicon" % (name, b)].tolist()
    return totals


@pytest.mark.parametrize("with_lexicon", [False, True])
def test_golden_strings_and_meters(with_lexicon):
    from megreader_b200 import rec_measure
    from oracle.make_rec_measure_golden import CASES
    dev = _dev()
    z = golden()
    lexicon = rec_measure.Lexicon(z["lexicon"].tolist(), dev) if with_lexicon else None
    tag = "lexicon" if with_lexicon else "plain"
    for name, rep, seed, N, W, batches in CASES:
        totals = run_golden_case(z, name, batches, lexicon, dev)
        names = z["%s/%s/meters" % (name, tag)].tolist()
        g = rec_measure.gather(totals)
        assert sorted(g) == names
        assert np.array_equal(meter_rows(g, names), z["%s/%s/values" % (name, tag)], equal_nan=True), name


def representer_inputs(rep, seed, N, W, dev):
    from oracle.make_rec_measure_golden import case_batch
    labels, pred = case_batch(rep, seed, N, W)
    batch = {'label': torch.from_numpy(labels)}
    if isinstance(pred, tuple):
        return batch, tuple(torch.from_numpy(p).to(dev) for p in pred)
    return batch, torch.from_numpy(pred).to(dev)


@pytest.mark.parametrize("with_lexicon", [False, True])
def test_representers_golden(with_lexicon):
    """represent's strings equal the reference loops' (golden); represent_labels -> measure_labels gives the same per-sample
    results and meters as the string form"""
    from megreader_b200 import decode, rec_measure
    from oracle.make_rec_measure_golden import CASES
    dev = _dev()
    z = golden()
    lexicon = rec_measure.Lexicon(z["lexicon"].tolist(), dev) if with_lexicon else None
    tag = "lexicon" if with_lexicon else "plain"
    for name, rep, seed, N, W, batches in CASES:
        r = getattr(decode, rep)(english())
        inputs = [representer_inputs(rep, seed * 100 + b, N, W, dev) for b in range(batches)]
        for b, (batch, pred) in enumerate(inputs):
            res = r.represent(batch, pred.clone() if torch.is_tensor(pred) else pred)
            assert [d['label_string'] for d in res] == z["%s/%d/label_string" % (name, b)].tolist(), (name, b)
            assert [d['pred_string'] for d in res] == z["%s/%d/pred_string" % (name, b)].tolist(), (name, b)
            if rep == "CTCRepresenter2D":
                assert torch.equal(res[0]['mask'], pred[1][0][0].cpu()) and torch.equal(res[0]['classify'], pred[0][0].cpu())
        totals = run_golden_case(z, name, batches, lexicon, dev, lambda b: r.represent_labels(*inputs[b]))
        names = z["%s/%s/meters" % (name, tag)].tolist()
        assert np.array_equal(meter_rows(rec_measure.gather(totals), names), z["%s/%s/values" % (name, tag)], equal_nan=True)


def test_no_host_sync_and_graph_replay():
    from megreader_b200 import rec_measure
    dev = _dev()
    cs = cases.charsets()["printable"]
    table = rec_measure.fold_table(cs, dev)
    rng = np.random.default_rng(5)
    batches = [tuple(torch.from_numpy(a).to(dev) for a in cases.pair_corpus(rng, len(cs), 64, 40, 40)) for _ in range(4)]
    words = [port.fold(cs, r) for r in batches[0][0].cpu().numpy()[:20]] + ["lower", ""]
    lexicon = rec_measure.Lexicon(words, dev)
    eager = rec_measure.new_totals(dev)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        eager_out = [rec_measure.measure_labels(g, p, table, lexicon, eager) for g, p in batches]
    finally:
        torch.cuda.set_sync_debug_mode(0)
    static = [t.clone() for t in batches[0]]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        rec_measure.measure_labels(*static, table, lexicon)
    torch.cuda.current_stream().wait_stream(s)
    totals = rec_measure.new_totals(dev)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = rec_measure.measure_labels(*static, table, lexicon, totals)
    totals.zero_()
    for k, (gt, pred) in enumerate(batches):
        static[0].copy_(gt)
        static[1].copy_(pred)
        g.replay()
        for key in ("accuracy", "distance", "edit_distance", "in_lexicon", "status"):
            assert torch.equal(out[key], eager_out[k][key]), (k, key)
    torch.cuda.synchronize()
    assert torch.equal(totals, eager) and eager[4 * 2 + 3] == 4 and eager_out[0]["in_lexicon"].sum() >= 15
    assert sorted(rec_measure.gather(totals)) == sorted(rec_measure.gather(eager))


def test_bad_labels_and_refusals():
    from megreader_b200 import rec_measure
    dev = _dev()
    table = rec_measure.fold_table(english(), dev)
    gt = torch.tensor([[2, 3, 0], [2, 38, 0], [-1, 2, 0], [2, 2, 2]], dtype=torch.int64, device=dev)
    pred = torch.tensor([[2, 3, 0], [2, 3, 0], [2, 0, 0], [2, -7, 0]], dtype=torch.int64, device=dev)
    totals = rec_measure.new_totals(dev)
    out = rec_measure.measure_labels(gt, pred, table, totals=totals)
    assert out["status"].tolist() == [0, rec_measure.BAD_LABEL, rec_measure.BAD_LABEL, rec_measure.BAD_LABEL]
    assert totals[:24].abs().sum() == 0 and totals[24] == 1
    with pytest.raises(RuntimeError, match="refused|not counted"):
        rec_measure.gather(totals)
    m = rec_measure.SequenceRecognitionMeasurer(charset=english())
    with pytest.raises(RuntimeError, match="outside the charset"):
        m.measure(None, (gt, pred))
    assert m.measure(None, (gt[:1], pred[:1])) == dict(accuracy=[True], edit_distance=[1.0])
    with pytest.raises(NotImplementedError):
        rec_measure.measure_labels(gt.cpu(), pred.cpu(), table)
    with pytest.raises(NotImplementedError):
        rec_measure.measure_labels(gt, pred.cpu(), table)
    with pytest.raises(NotImplementedError):
        from megreader_b200 import decode
        decode.CTCRepresenter(english()).represent_labels({'label': gt.cpu()}, torch.zeros(1, 38, 1, 4))
    with pytest.raises(RuntimeError, match="totals"):
        rec_measure.measure_labels(gt, pred, table, totals=torch.zeros(25, device=dev))


def test_measurer_structures(tmp_path):
    from megreader_b200 import rec_measure
    dev = _dev()
    out = [{'label_string': 'straße', 'pred_string': 'STRASSE'}, {'label_string': 'ab', 'pred_string': 'abc'},
           {'label_string': '', 'pred_string': 'x'}, {'label_string': 'x\U00010428', 'pred_string': 'X\U00010400'}]
    words = tmp_path / "w.txt"
    words.write_text("STRASSE ab\nX\U00010400\n")
    for path in (None, str(words)):
        m = rec_measure.SequenceRecognitionMeasurer(path, device=dev)
        p = port.SequenceRecognitionMeasurer({"STRASSE", "ab", "X\U00010400"} if path else None)
        got = [m.measure(None, out), m.measure(None, out[1:])]
        want = [p.measure(None, out), p.measure(None, out[1:])]
        assert got == want
        gm, gp = m.gather_measure(got), p.gather_measure(want)
        assert sorted(gm) == sorted(gp)
        for k in gp:
            assert np.array_equal(np.array([gm[k].val, gm[k].sum, gm[k].count, gm[k].avg], np.float64),
                                  np.array([gp[k].val, gp[k].sum, gp[k].count, gp[k].avg], np.float64), equal_nan=True), k


def test_crnn_validation_step_in_one_graph():
    """crnn.yaml's validation batch (16 x 3 x 32 x 128): engine CRNN eval, ctc_greedy_decode and measure_labels(totals) in one
    CUDA graph, replayed over seeded batches; gather(totals) equals the measurer on the host strings of the same labels"""
    import bench
    from megreader_b200 import decode, rec_measure
    dev = _dev()
    torch.manual_seed(0)
    net = bench.build_model(dev).eval()
    table = rec_measure.fold_table(english(), dev)
    rng = np.random.default_rng(9)
    xs = [torch.from_numpy(rng.standard_normal((16, 3, 32, 128)).astype(np.float32)).to(dev) for _ in range(3)]
    labels = [torch.from_numpy(cases.label_rows(rng, 38, 16, 32, 10).astype(np.int32)).to(dev) for _ in range(3)]
    rep = decode.CTCRepresenter(english())

    def step(x, lab, totals):
        prob = net.decoder(net.backbone(x), train=False)
        return rec_measure.measure_labels(lab, decode.ctc_greedy_decode(prob), table, totals=totals)

    with torch.no_grad():
        static = [xs[0].clone(), labels[0].clone()]
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            step(*static, None)
        torch.cuda.current_stream().wait_stream(s)
        totals = rec_measure.new_totals(dev)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            step(*static, totals)
        totals.zero_()
        raw = []
        for x, lab in zip(xs, labels):
            static[0].copy_(x)
            static[1].copy_(lab)
            g.replay()
            raw.append(port.SequenceRecognitionMeasurer().measure(None, rep.represent({'label': lab}, net.decoder(net.backbone(x),
                                                                                                                  train=False))))
        torch.cuda.synchronize()
    got, want = rec_measure.gather(totals), port.SequenceRecognitionMeasurer().gather_measure(raw)
    for k in want:
        assert [got[k].val, got[k].sum, got[k].count, got[k].avg] == [want[k].val, want[k].sum, want[k].count, want[k].avg], k
    assert got["accuracy"].count == 48


def _graph_chain(step, inputs, represent):
    """capture step(*static, totals) once, replay it over `inputs` copied into the static tensors; returns gather(totals) and
    the port measurer's gather_measure over represent(*inputs[k]) (the host strings of the same labels)"""
    from megreader_b200 import rec_measure
    dev = inputs[0][0].device
    static = [t.clone() for t in inputs[0]]
    with torch.no_grad():
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            step(*static, None)
        torch.cuda.current_stream().wait_stream(s)
        totals = rec_measure.new_totals(dev)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            step(*static, totals)
        totals.zero_()
        raw = []
        for x in inputs:
            for a, b in zip(static, x):
                a.copy_(b)
            g.replay()
            raw.append(port.SequenceRecognitionMeasurer().measure(None, represent(*x)))
        torch.cuda.synchronize()
    return rec_measure.gather(totals), port.SequenceRecognitionMeasurer().gather_measure(raw)


def _same_gather(got, want, n):
    assert sorted(got) == sorted(want)
    for k in want:
        assert [got[k].val, got[k].sum, got[k].count, got[k].avg] == [want[k].val, want[k].sum, want[k].count, want[k].avg], k
    assert got["accuracy"].count == n


def test_ctc2d_validation_step_in_one_graph():
    """res50-ppm-2d-ctc.yaml's chain at a small size: CTCDecoder2D eval, ctc2d_greedy_decode (via represent_labels) and
    measure_labels(totals) in one CUDA graph, replayed over seeded batches; gather(totals) equals the measurer on the host strings
    of represent()"""
    import megreader_b200
    from megreader_b200 import decode, rec_measure
    megreader_b200.install_reference_api()
    import decoders
    dev = _dev()
    torch.manual_seed(3)
    head = decoders.CTCDecoder2D(16, inner_channels=8).to(dev).eval()
    table = rec_measure.fold_table(english(), dev)
    rep = decode.CTCRepresenter2D(english())
    rng = np.random.default_rng(13)
    inputs = [(torch.from_numpy(rng.standard_normal((4, 16, 8, 32)).astype(np.float32)).to(dev),
               torch.from_numpy(cases.label_rows(rng, 38, 4, 32, 10).astype(np.int32)).to(dev)) for _ in range(3)]

    def step(x, lab, totals):
        return rec_measure.measure_labels(*rep.represent_labels({'label': lab}, head(x)), table, totals=totals)

    def represent(x, lab):
        with torch.no_grad():
            return rep.represent({'label': lab}, head(x))
    got, want = _graph_chain(step, inputs, represent)
    _same_gather(got, want, 12)


def test_attention_validation_step_in_one_graph():
    """fpn50-attention-decoder.yaml's chain at a small size: AttentionDecoder eval (the persistent greedy-decoding kernel),
    blank_after_first_blank_ (via represent_labels) and measure_labels(totals) in one CUDA graph, replayed over seeded batches;
    gather(totals) equals the measurer on the host strings of represent()"""
    import megreader_b200.refapi.decoders as md
    from megreader_b200 import decode, rec_measure
    dev = _dev()
    torch.manual_seed(4)
    head = md.AttentionDecoder(32, inner_channels=64, max_size=16, height=1).to(dev).eval()
    table = rec_measure.fold_table(english(), dev)
    rep = decode.SequenceRecognitionRepresenter(english())
    rng = np.random.default_rng(14)
    inputs = [(torch.from_numpy(rng.standard_normal((4, 32, 16, 32)).astype(np.float32)).to(dev),
               torch.from_numpy(cases.label_rows(rng, 38, 4, 32, 10).astype(np.int32)).to(dev)) for _ in range(3)]

    def step(x, lab, totals):
        return rec_measure.measure_labels(*rep.represent_labels({'label': lab}, head(x)), table, totals=totals)

    def represent(x, lab):
        with torch.no_grad():
            return rep.represent({'label': lab}, head(x))
    got, want = _graph_chain(step, inputs, represent)
    _same_gather(got, want, 12)
