"""Plain-Python restatement of the text recognisers' validation measure: SequenceRecognitionMeasurer
(structure/measurers/sequence_recognition_measurer.py) with editdistance.eval restated as the Wagner-Fischer DP, numpy's
pairwise_sum and concern.AverageMeter, plus the string side of the three representers (label_to_string on collapsed labels).

Used by tests/test_rec_measure_*.py as the reference the device (megreader_b200.rec_measure) is compared with, and by
oracle/make_rec_measure_golden.py to stand in for editdistance, which is not a dependency of this project."""
import numpy as np


def levenshtein(a, b):
    """editdistance.eval(a, b): unit-cost insert / delete / substitute over the symbols of two sequences (the Wagner-Fischer
    DP, one row at a time: the insertions along a row are the running minimum of row[k] - k, plus j)"""
    a = [ord(c) if isinstance(c, str) else int(c) for c in a]
    b = np.array([ord(c) if isinstance(c, str) else int(c) for c in b], np.int64)
    idx = np.arange(len(b) + 1)
    prev = idx.copy()
    for i, x in enumerate(a, 1):
        cur = np.empty_like(prev)
        cur[0] = i
        cur[1:] = np.minimum(prev[1:] + 1, prev[:-1] + (b != x))
        prev = np.minimum.accumulate(cur - idx) + idx
    return int(prev[-1])


def edit_score(label, pred):
    """one entry of SequenceRecognitionMeasurer.edit_distance for upper-cased strings"""
    length = len(label)
    if length == 0:
        return 0.0
    return float(1 - min(length, levenshtein(label, pred)) * 1.0 / length)


def pairwise_sum(a):
    """numpy's pairwise_sum (the order of np.array(list_of_floats).sum()) in float64"""
    a = [float(v) for v in a]

    def rec(lo, n):
        if n < 8:
            res = 0.0
            for i in range(n):
                res += a[lo + i]
            return res
        if n <= 128:
            r = a[lo:lo + 8]
            i = 8
            while i < n - n % 8:
                for k in range(8):
                    r[k] += a[lo + i + k]
                i += 8
            res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]))
            while i < n:
                res += a[lo + i]
                i += 1
            return res
        h = n // 2
        h -= h % 8
        return rec(lo, h) + rec(lo + h, n - h)
    return rec(0, len(a))


class AverageMeter:
    """concern.AverageMeter"""

    def __init__(self):
        self.val = 0
        self.avg = 0
        self.sum = 0
        self.count = 0

    def update(self, val, n=1):
        self.val = val
        self.sum += val * n
        self.count += n
        with np.errstate(invalid="ignore", divide="ignore"):
            self.avg = np.float64(self.sum) / self.count
        return self


def fold(charset, label):
    """charset.label_to_string(label).upper(), the string the measurer compares; IndexError for an id >= len(charset)"""
    empty = (charset.blank, charset.unknown)
    return "".join(charset[int(i)] for i in label if int(i) not in empty).upper()


def collapse(pred, blank=0, unknown=1):
    """the CTC representers' greedy collapse of one argmax row (ctc_representer.py:22-34): repeats merged, unknown skipped
    without resetting the previous symbol, blanks dropped; blank-padded to the row's width"""
    out = [blank] * len(pred)
    valid, previous = 0, blank
    for c in pred:
        c = int(c)
        if c == previous or c == unknown:
            continue
        if c != blank:
            out[valid] = c
            valid += 1
        previous = c
    return out


def blank_after_first_blank(pred, blank=0):
    """SequenceRecognitionRepresenter.represent's mask: everything from the first blank on becomes blank"""
    out, seen = [], False
    for c in pred:
        seen = seen or int(c) == blank
        out.append(blank if seen else int(c))
    return out


class SequenceRecognitionMeasurer:
    """the reference measurer with editdistance.eval restated"""

    def __init__(self, lexicon=None):
        self.nori_lexicon = set(lexicon) if lexicon is not None else None

    def measure(self, batch, output):
        labels = [o['label_string'].upper() for o in output]
        preds = [o['pred_string'].upper() for o in output]
        res = dict(accuracy=[g == p for g, p in zip(labels, preds)], edit_distance=[edit_score(g, p) for g, p in zip(labels, preds)])
        if self.nori_lexicon:
            res['in_lexicon'] = [g in self.nori_lexicon for g in labels]
        return res

    def gather_measure(self, raw_metrics):
        def meter(batches, part=None):
            m = AverageMeter()
            for b in batches:
                values, in_lex = (b, None) if part is None else b
                if part is None:
                    m.update(pairwise_sum(values) / len(values), len(values))
                else:
                    sub = [v for v, f in zip(values, in_lex) if f == part]
                    m.update(pairwise_sum(sub) / max(len(sub), 1), len(sub))
            return m

        def as_float(values):
            return [float(v) for v in values]
        acc = [as_float(m['accuracy']) for m in raw_metrics]
        ed = [m['edit_distance'] for m in raw_metrics]
        if not self.nori_lexicon:
            return dict(accuracy=meter(acc), edit_distance=meter(ed))
        lex = [m['in_lexicon'] for m in raw_metrics]
        return dict(total_edit_distance=meter(ed), in_lexicon_edit_distance=meter(list(zip(ed, lex)), True),
                    out_lexicon_edit_distance=meter(list(zip(ed, lex)), False), total_accuracy=meter(acc),
                    in_lexicon_accuracy=meter(list(zip(acc, lex)), True), out_lexicon_accuracy=meter(list(zip(acc, lex)), False))
