"""Validation measure of the text recognisers on the device: SequenceRecognitionMeasurer
(structure/measurers/sequence_recognition_measurer.py) for a whole batch (csrc/rec_measure.cu).

    fold_table(charset, device)                               -> class id -> code points of charset[id].upper()
    Lexicon(words_or_path, device)                            -> the nori lexicon as a device hash table
    measure_labels(gt, pred, table, lexicon, totals)          -> dict of device tensors; never synchronises with the host, so
                                                                it can be captured in a CUDA graph, with `totals` updated
    measure_strings(gt_strings, pred_strings, lexicon, ...)   -> the same from host strings
    gather(totals)                                            -> gather_measure's meters, with one host read
    SequenceRecognitionMeasurer().measure / validate_measure / evaluate_measure / gather_measure -> the reference's structures

Per sample: accuracy (the upper-cased strings are equal), the exact Levenshtein distance over code points, the score
1 - min(L, d) / L (0.0 for an empty gt) and whether the upper-cased gt is a word of the lexicon.  `totals` holds the
AverageMeters of gather_measure, updated per batch from numpy's pairwise sums, so gather(totals) equals the reference's
gather_measure bit for bit.  Class ids outside [0, C) are refused (DESIGN §7).  CUDA only; no CPU fallback."""
import os

import numpy as np
import torch

from . import _lib
from .db_measure import AverageMeter

# status bits (include/megreader_b200.h)
BAD_LABEL, BAD_LENGTH = 1, 2
FOLD_MAX = 4
TOTALS = 25
METERS = ("accuracy", "edit_distance", "in_lexicon_accuracy", "out_lexicon_accuracy", "in_lexicon_edit_distance",
          "out_lexicon_edit_distance")


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _require_cuda(t, what):
    if not (torch.is_tensor(t) and t.is_cuda):
        raise NotImplementedError("megreader_b200: rec_measure runs on CUDA only (no CPU fallback); %s is not a CUDA tensor" % what)


class FoldTable:
    """len int32 [C] and cp int32 [C, 4] on one device: the code points of charset[id].upper(), none for blank and unknown
    (the ids charset.label_to_string drops)."""

    def __init__(self, lengths, cps):
        self.len, self.cp = lengths, cps

    def __len__(self):
        return self.len.numel()


def fold_table(charset, device=None):
    """the FoldTable of any charset with len(), [] and .blank / .unknown (the project's EnglishCharset or a reference Charset).
    Raises ValueError for a class whose upper case is longer than 4 code points."""
    C = len(charset)
    lengths = np.zeros(C, np.int32)
    cps = np.zeros((C, FOLD_MAX), np.int32)
    empty = (int(charset.blank), int(charset.unknown))
    for i in range(C):
        if i in empty:
            continue
        s = charset[i].upper()
        if len(s) > FOLD_MAX:
            raise ValueError("rec_measure.fold_table: class %d (%r) upper-cases to %d code points, more than %d"
                             % (i, charset[i], len(s), FOLD_MAX))
        lengths[i] = len(s)
        cps[i, :len(s)] = [ord(c) for c in s]
    dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
    return FoldTable(torch.from_numpy(lengths).to(dev), torch.from_numpy(cps).to(dev))


def _encode(strings, width=None):
    """host strings -> int32 code points [N, width] (zero padded) and lengths [N]"""
    lens = np.array([len(s) for s in strings], np.int32)
    w = int(lens.max()) if len(strings) and width is None else (width or 0)
    cp = np.zeros((len(strings), w), np.int32)
    for n, s in enumerate(strings):
        if s:
            cp[n, :len(s)] = np.frombuffer(s.encode("utf-32-le"), np.uint32).view(np.int32)
    return cp, lens


class Lexicon:
    """The measurer's lexicon: set(open(path).read().split()) or the set of the given words, as code points plus an
    open-addressing hash table on `device`.  Membership is case-sensitive on the word side, as in the reference: the upper-cased
    gt is looked up, so lowercase words never match.  An empty lexicon is falsy, and the measure then treats it as none."""

    def __init__(self, words_or_path, device=None):
        if isinstance(words_or_path, (str, os.PathLike)):
            with open(words_or_path) as f:
                words = set(f.read().split())
        else:
            words = set(words_or_path)
        self.words = frozenset(words)
        ordered = sorted(self.words)
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        lens = np.array([len(w) for w in ordered], np.int64)
        offsets = np.zeros(len(ordered) + 1, np.int64)
        np.cumsum(lens, out=offsets[1:])
        if offsets[-1] >= 2 ** 31:
            raise ValueError("rec_measure.Lexicon: %d code points, at most 2^31 - 1" % offsets[-1])
        joined = "".join(ordered)
        cp = np.frombuffer(joined.encode("utf-32-le"), np.uint32).view(np.int32) if joined else np.zeros(0, np.int32)
        self.cp = torch.from_numpy(cp.copy()).to(self.device)
        self.offsets = torch.from_numpy(offsets.astype(np.int32)).to(self.device)
        L = _lib.lib()
        nbytes = int(L.mr_rec_lexicon_build_bytes(len(ordered)))
        if nbytes <= 0:
            raise ValueError("rec_measure.Lexicon: %d words is too many" % len(ordered))
        self.table = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(L.mr_rec_lexicon_build(self.cp.data_ptr(), self.offsets.data_ptr(), len(ordered), self.table.data_ptr(),
                                              nbytes, _stream()), "rec_measure lexicon")

    def __len__(self):
        return len(self.words)

    def __bool__(self):
        return len(self.words) > 0

    def __contains__(self, word):
        return word in self.words


def _measure(gt, gt_len, pred, pred_len, table, lexicon, totals):
    folded = table is not None
    for name, t in (("gt", gt), ("pred", pred)) + ((("fold table", table.len),) if folded else ()):
        _require_cuda(t, name)
    if gt.dim() != 2 or pred.dim() != 2 or gt.size(0) != pred.size(0):
        raise RuntimeError("rec_measure: gt and pred must be [N, width] with the same N, got %s and %s"
                           % (tuple(gt.shape), tuple(pred.shape)))
    ok = (torch.int32, torch.int64) if folded else (torch.int32,)
    if gt.dtype not in ok or pred.dtype not in ok:
        raise RuntimeError("rec_measure: gt and pred must be %s, got %s and %s" % (" or ".join(map(str, ok)), gt.dtype, pred.dtype))
    dev = gt.device
    tensors = [("pred", pred)] + ([("fold table", table.len), ("fold table", table.cp)] if folded else
                                  [("gt lengths", gt_len), ("pred lengths", pred_len)])
    if lexicon:
        tensors.append(("lexicon", lexicon.table))
    for name, t in tensors:
        if t.device != dev:
            raise RuntimeError("rec_measure: %s is on %s, gt on %s" % (name, t.device, dev))
    if totals is not None and (not torch.is_tensor(totals) or totals.dtype != torch.float64 or totals.shape != (TOTALS,)
                               or not totals.is_contiguous() or totals.device != dev):
        raise RuntimeError("rec_measure: totals must be a contiguous float64 [%d] tensor on %s" % (TOTALS, dev))
    gt, pred = gt.contiguous(), pred.contiguous()
    N, Lg, Wp = gt.size(0), gt.size(1), pred.size(1)
    if N == 0:
        raise ValueError("rec_measure: an empty batch has no per-batch mean (the reference's gather_measure would add nan to "
                         "its meters); SequenceRecognitionMeasurer.measure returns empty lists for it")
    L = _lib.lib()
    nbytes = int(L.mr_rec_measure_workspace_bytes(N, Lg, Wp, int(folded)))
    if nbytes <= 0:
        raise RuntimeError("rec_measure: unsupported sizes N=%d, gt width %d, pred width %d" % (N, Lg, Wp))
    i32 = dict(dtype=torch.int32, device=dev)
    out = dict(accuracy=torch.empty(N, dtype=torch.bool, device=dev), distance=torch.empty(N, **i32),
               edit_distance=torch.empty(N, dtype=torch.float64, device=dev), in_lexicon=torch.empty(N, dtype=torch.bool, device=dev),
               gt_length=torch.empty(N, **i32), pred_length=torch.empty(N, **i32), status=torch.empty(N, **i32))
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    nw = len(lexicon) if lexicon else 0
    with torch.cuda.device(dev):
        _lib.check(L.mr_rec_measure(gt.data_ptr(), int(gt.dtype == torch.int64), gt_len.data_ptr() if gt_len is not None else None, Lg,
                                    pred.data_ptr(), int(pred.dtype == torch.int64),
                                    pred_len.data_ptr() if pred_len is not None else None, Wp, N,
                                    table.len.data_ptr() if folded else None, table.cp.data_ptr() if folded else None,
                                    len(table) if folded else 0, lexicon.cp.data_ptr() if nw else None,
                                    lexicon.offsets.data_ptr() if nw else None, nw, lexicon.table.data_ptr() if nw else None,
                                    ws.data_ptr(), nbytes, out["accuracy"].data_ptr(), out["distance"].data_ptr(),
                                    out["edit_distance"].data_ptr(), out["in_lexicon"].data_ptr(), out["gt_length"].data_ptr(),
                                    out["pred_length"].data_ptr(), out["status"].data_ptr(),
                                    totals.data_ptr() if totals is not None else None, _stream()), "rec_measure")
    out["workspace"] = ws
    return out


def measure_labels(gt, pred, table, lexicon=None, totals=None):
    """SequenceRecognitionMeasurer.measure for the label rows gt [N, Lg] and pred [N, Wp] (int32 or int64 class ids on one CUDA
    device, e.g. batch['label'] and ctc_greedy_decode's output) through the FoldTable `table`; no host synchronisation.

    Returns accuracy bool [N], distance int32 [N] (Levenshtein over the folded code points), edit_distance float64 [N],
    in_lexicon bool [N] (False without a lexicon), gt_length / pred_length int32 [N] (folded lengths) and status int32 [N]
    (BAD_LABEL: an id outside [0, C)).  totals, optional, float64 [25] on the same device (zeros to start): the AverageMeters
    of gather_measure, updated once per call; a batch with a bad sample updates no meter and is counted as refused, and
    gather() then raises.  The shorter width may hold at most 512 classes; N must be at least 1 (ValueError)."""
    _require_cuda(gt, "gt")
    return _measure(gt, None, pred, None, table, lexicon, totals)


def measure_strings(gt_strings, pred_strings, lexicon=None, totals=None, device=None):
    """measure_labels for host strings (the representers' label_string / pred_string): upper-cased and encoded as code
    points on the host, then the same kernels without a fold table."""
    if len(gt_strings) != len(pred_strings):
        raise ValueError("rec_measure: %d gt strings for %d predictions" % (len(gt_strings), len(pred_strings)))
    dev = torch.device(device) if device is not None else (lexicon.device if lexicon else torch.device("cuda", torch.cuda.current_device()))
    g, gl = _encode([s.upper() for s in gt_strings])
    p, pl = _encode([s.upper() for s in pred_strings])
    t = [torch.from_numpy(a).to(dev) for a in (g, gl, p, pl)]
    return _measure(t[0], t[1], t[2], t[3], None, lexicon, totals)


def new_totals(device=None):
    """zeroed totals for measure_labels / measure_strings"""
    return torch.zeros(TOTALS, dtype=torch.float64, device=device if device is not None else "cuda")


def _meter(row):
    val, s, count, updates = (float(v) for v in row)
    m = AverageMeter()
    if updates == 0:
        return m
    m.val, m.sum, m.count = np.float64(val), np.float64(s), int(count)
    with np.errstate(invalid="ignore", divide="ignore"):
        m.avg = m.sum / m.count                      # nan for a subset meter that has seen no sample yet, as numpy gives it
    return m


def gather(totals):
    """gather_measure's result from the totals of measure_labels / measure_strings (one host read): {'accuracy',
    'edit_distance'} without a lexicon; {'total_edit_distance', 'in_lexicon_edit_distance', 'out_lexicon_edit_distance',
    'total_accuracy', 'in_lexicon_accuracy', 'out_lexicon_accuracy'} with one."""
    t = totals.tolist() if torch.is_tensor(totals) else list(totals)
    if len(t) != TOTALS:
        raise ValueError("rec_measure.gather: totals must hold %d values" % TOTALS)
    if t[-1]:
        raise RuntimeError("rec_measure.gather: %d batches had class ids outside the charset or bad lengths and were not counted"
                           % int(t[-1]))
    m = [_meter(t[4 * k:4 * k + 4]) for k in range(6)]
    if t[4 * 2 + 3] == 0:
        return dict(accuracy=m[0], edit_distance=m[1])
    return dict(total_edit_distance=m[1], in_lexicon_edit_distance=m[4], out_lexicon_edit_distance=m[5], total_accuracy=m[0],
                in_lexicon_accuracy=m[2], out_lexicon_accuracy=m[3])


class SequenceRecognitionMeasurer:
    """The reference's SequenceRecognitionMeasurer on the device.  measure(batch, output) takes the representers' list of
    {'label_string', 'pred_string'} dicts, or the (gt, pred) label tensors of decode's represent_labels (folded through
    `charset`, the project's default charset unless given).  An empty lexicon file is falsy, as in the reference: the results
    then have no in / out-of-lexicon split.

    The constructor also takes, and ignores, the keywords the reference's config builder passes to every class it builds
    (concern/config.py: `cls(**args, cmd=cmd)` with `class` still in args)."""

    def __init__(self, nori_lexicon_path=None, charset=None, device=None, **config_kwargs):
        self.nori_lexicon_path = nori_lexicon_path
        self.device = device
        self.charset = charset
        self._words = None
        if nori_lexicon_path:
            with open(nori_lexicon_path) as f:
                self._words = set(f.read().split())
        self._lexicons = {}
        self._tables = {}

    @property
    def nori_lexicon(self):
        return self._words or None

    def _lexicon(self, dev):
        if not self._words:
            return None
        if dev not in self._lexicons:
            self._lexicons[dev] = Lexicon(self._words, dev)
        return self._lexicons[dev]

    def _table(self, dev):
        if dev not in self._tables:
            from .charset import default_charset
            self._tables[dev] = fold_table(self.charset if self.charset is not None else default_charset(), dev)
        return self._tables[dev]

    def measure(self, batch, output):
        labels = isinstance(output, (tuple, list)) and len(output) == 2 and torch.is_tensor(output[0])
        if (output[0].size(0) if labels else len(output)) == 0:
            # the reference's structures for an empty batch, without a launch (the kernels need N >= 1)
            return dict(accuracy=[], edit_distance=[], **({"in_lexicon": []} if self._words else {}))
        if labels:
            gt, pred = output
            _require_cuda(gt, "gt")
            dev = gt.device
            out = measure_labels(gt, pred, self._table(dev), self._lexicon(dev))
        else:
            dev = torch.device(self.device) if self.device is not None else torch.device("cuda", torch.cuda.current_device())
            out = measure_strings([o['label_string'] for o in output], [o['pred_string'] for o in output], self._lexicon(dev),
                                  device=dev)
        status = out["status"].cpu()
        if status.any():
            raise RuntimeError("rec_measure.SequenceRecognitionMeasurer: class ids outside the charset (status %s)" % status.tolist())
        res = dict(accuracy=out["accuracy"].tolist(), edit_distance=out["edit_distance"].tolist())
        if self._words:
            res["in_lexicon"] = out["in_lexicon"].tolist()
        return res

    def validate_measure(self, batch, output):
        return self.measure(batch, output), []

    evaluate_measure = validate_measure

    def gather_measure(self, raw_metrics, logger=None):
        """the reference's folding of the per-batch host lists measure() returned: numpy sums per batch into AverageMeters (the
        graph path keeps the same meters on the device: measure_labels(totals=...) and gather)"""
        if not self._words:
            return dict(accuracy=self._fold([m['accuracy'] for m in raw_metrics]),
                        edit_distance=self._fold([m['edit_distance'] for m in raw_metrics]))
        ed = self._fold_split([(m['edit_distance'], m['in_lexicon']) for m in raw_metrics])
        acc = self._fold_split([(m['accuracy'], m['in_lexicon']) for m in raw_metrics])
        return dict(total_edit_distance=ed[0], in_lexicon_edit_distance=ed[1], out_lexicon_edit_distance=ed[2],
                    total_accuracy=acc[0], in_lexicon_accuracy=acc[1], out_lexicon_accuracy=acc[2])

    @staticmethod
    def _fold(batches):
        meter = AverageMeter()
        for values in batches:
            meter.update(np.array(values).sum() / len(values), len(values))
        return meter

    @staticmethod
    def _fold_split(batches):
        meters = AverageMeter(), AverageMeter(), AverageMeter()
        with np.errstate(invalid="ignore", divide="ignore"):
            for values, in_lexicon in batches:
                values, in_lexicon = np.array(values), np.array(in_lexicon)
                meters[0].update(values.sum() / len(values), len(values))
                for meter, part in ((meters[1], values[in_lexicon == True]), (meters[2], values[in_lexicon == False])):  # noqa: E712
                    meter.update(part.sum() / max(len(part), 1), len(part))
        return meters
