"""Generate tests/golden/rec_measure_ref.npz with the REFERENCE's own representers (CTCRepresenter, CTCRepresenter2D,
SequenceRecognitionRepresenter) and SequenceRecognitionMeasurer (structure/, loaded unmodified through oracle/ref_loader).

    python -m oracle.make_rec_measure_golden

One environment fix, as make_db_measure_golden.py binds Polygon: editdistance is not a dependency of this project, so the
measurer module's `ed.eval` is bound to the Wagner-Fischer DP of oracle/rec_measure_port.py.  Per case the file holds, per
batch, the labels (the scores / predictions are regenerated from the seeds of tests/rec_measure_cases.py), the strings and the
measurer's per-sample results with and without a lexicon; and gather_measure's meters over the case's batches as
[meters, 4] (val, sum, count, avg) in the order of the `.../meters` names."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import rec_measure_port as port  # noqa: E402
from tests import rec_measure_cases as cases  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "rec_measure_ref.npz")
# name, representer, seed, N, W, batches
CASES = [
    ("ctc", "CTCRepresenter", 1, 16, 33, 3),
    ("ctc_wide", "CTCRepresenter", 2, 9, 65, 2),
    ("ctc2d", "CTCRepresenter2D", 3, 7, 32, 3),
    ("attn", "SequenceRecognitionRepresenter", 4, 11, 32, 3),
]
H2D = 4


def reference():
    """(module of representers, measurer module) or None where the reference tree is absent"""
    from oracle import ref_loader
    if not ref_loader.install():
        return None
    m = ref_loader.load("structure.measurers.sequence_recognition_measurer")
    m.ed.eval = port.levenshtein
    reps = {name: getattr(ref_loader.load(mod), name) for name, mod in (
        ("CTCRepresenter", "structure.representers.ctc_representer"),
        ("CTCRepresenter2D", "structure.representers.ctc_representer2d"),
        ("SequenceRecognitionRepresenter", "structure.representers.sequence_recognition_representer"))}
    return reps, m


def case_batch(rep, seed, N, W):
    """the representer's inputs for one batch: labels and pred as numpy arrays (pred a tuple for the 2D representer)"""
    C = 38
    if rep == "CTCRepresenter":
        return cases.ctc_batch(seed, N, C, W)
    if rep == "CTCRepresenter2D":
        labels, cls, mask = cases.ctc2d_batch(seed, N, C, H2D, W)
        return labels, (cls, mask)
    return cases.attn_batch(seed, N, C, W)


def run_case(reps, mm, lexicon_path, rep, seed, N, W, batches):
    import torch
    r = reps[rep]()
    out = {}
    raw, raw_lex = [], []
    plain = mm.SequenceRecognitionMeasurer()
    lexm = mm.SequenceRecognitionMeasurer(nori_lexicon_path=lexicon_path)
    for b in range(batches):
        labels, pred = case_batch(rep, seed * 100 + b, N, W)
        tp = tuple(torch.from_numpy(p) for p in pred) if isinstance(pred, tuple) else torch.from_numpy(pred.copy())
        res = r.represent({'label': torch.from_numpy(labels), 'image': torch.zeros(N, 1)}, tp)
        out["%d/labels" % b] = labels
        out["%d/label_string" % b] = np.array([d['label_string'] for d in res], dtype=str)
        out["%d/pred_string" % b] = np.array([d['pred_string'] for d in res], dtype=str)
        m = plain.measure(None, res)
        ml = lexm.measure(None, res)
        raw.append(m)
        raw_lex.append(ml)
        out["%d/accuracy" % b] = np.array(m['accuracy'], bool)
        out["%d/edit_distance" % b] = np.array(m['edit_distance'], np.float64)
        out["%d/in_lexicon" % b] = np.array(ml['in_lexicon'], bool)
    for tag, meas, r_ in (("plain", plain, raw), ("lexicon", lexm, raw_lex)):
        g = meas.gather_measure(r_, None)
        names = sorted(g)
        out[tag + "/meters"] = np.array(names, dtype=str)
        out[tag + "/values"] = np.array([[float(g[k].val), float(g[k].sum), float(g[k].count), float(g[k].avg)] for k in names])
    return out


def lexicon_file(path):
    rng = np.random.default_rng(7)
    strings = []
    for name, rep, seed, N, W, batches in CASES:
        for b in range(batches):
            labels, _ = case_batch(rep, seed * 100 + b, N, W)
            strings += [port.fold(cases.ListCharset("0123456789ABCDEFGHIJKLMNOPQRSTUVWXYZ"), row) for row in labels]
    words = cases.lexicon_words(rng, strings)
    with open(path, "w") as f:
        f.write("\n".join(words) + "\n")
    return words


def main():
    import tempfile
    ref = reference()
    if ref is None:
        raise SystemExit("reference tree not present")
    reps, mm = ref
    arrays = {}
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "lexicon.txt")
        words = lexicon_file(path)
        arrays["lexicon"] = np.array(words, dtype=str)
        for name, rep, seed, N, W, batches in CASES:
            for k, v in run_case(reps, mm, path, rep, seed, N, W, batches).items():
                arrays[name + "/" + k] = v
    np.savez_compressed(OUT, **arrays)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
