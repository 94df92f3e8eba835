"""Lexicon-constrained transcription of the CTC heads on the device (csrc/lexicon.cu; DESIGN §7): Shi, Bai & Yao 2015,
§2.3.2 -- the word l of a lexicon D with the largest p(l | y), searched over the words within edit distance delta of the
greedy result, or over all of D.

    WordList(words_or_path, charset)              -> one word list as class ids on the device
    WordList.per_image(lists, charset)            -> (WordList, ranges int64 [N, 2]): every image's list, packed
    decode_packed(prob, words, ranges, ...)       -> dict of device tensors: labels (N, W), word, score, candidates, status;
                                                     no host synchronisation, so it can be captured in a CUDA graph
    LexiconCTCRepresenter / LexiconCTCRepresenter2D -> decode.CTCRepresenter / CTCRepresenter2D with the lexicon

The score of a word is its CTC log-likelihood (the 2D-CTC one for CTCDecoder2D) over the whole width; on equal scores the
lowest word index wins; a sample with no candidate of finite score keeps its greedy labels with word -1 and score -inf.
The attention head has no CTC likelihood and is not covered.  CUDA only; no CPU fallback."""
import os

import numpy as np
import torch

from . import _lib
from . import decode as _decode

MAX_WORD = 64                                   # MR_LEXICON_MAX_WORD
OVERFLOW, BAD_RANGE, BAD_WORD = 1, 2, 4         # status bits (include/megreader_b200.h)
TINY = float(torch.finfo(torch.float32).tiny)


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _read_words(words_or_path):
    if isinstance(words_or_path, (str, os.PathLike)):
        with open(words_or_path) as f:
            return sorted(set(f.read().split()))           # what rec_measure.Lexicon reads, in a fixed order
    return list(words_or_path)


class WordList:
    """Words as class ids through charset.index() (the mapping of MakeRecognitionLabel; EnglishCharset upper-cases), in the
    given order, duplicates kept: cls int32 [total] and offsets int32 [n + 1] on `device`.  A path is read as
    rec_measure.Lexicon reads it, and sorted.  Raises ValueError, naming the word, for an empty word, a word with a character
    the charset maps to `unknown`, or a word of more than 64 classes."""

    def __init__(self, words_or_path, charset=None, device=None):
        if charset is None:
            from .charset import default_charset
            charset = default_charset()
        self.charset = charset
        self.words = _read_words(words_or_path)
        ids = []
        lut = {}
        for w in self.words:
            if not isinstance(w, str) or not w:
                raise ValueError("lexicon.WordList: empty word %r" % (w,))
            if len(w) > MAX_WORD:
                raise ValueError("lexicon.WordList: word %r has %d classes, at most %d" % (w, len(w), MAX_WORD))
            for c in w:
                if c not in lut:
                    lut[c] = int(charset.index(c))
            row = [lut[c] for c in w]
            if int(charset.unknown) in row or int(charset.blank) in row:
                raise ValueError("lexicon.WordList: word %r has a character outside the charset" % w)
            ids.append(row)
        offsets = np.zeros(len(ids) + 1, np.int64)
        np.cumsum([len(r) for r in ids], out=offsets[1:])
        if offsets[-1] >= 2 ** 31 or len(ids) >= 2 ** 31:
            raise ValueError("lexicon.WordList: %d classes in %d words, at most 2^31 - 1" % (offsets[-1], len(ids)))
        flat = np.fromiter((c for r in ids for c in r), np.int32, int(offsets[-1]))
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        self.cls = torch.from_numpy(flat).to(self.device)
        self.offsets = torch.from_numpy(offsets.astype(np.int32)).to(self.device)
        self.max_list = len(ids)                    # the longest range a sample reads: the default max_words_per_sample

    def __len__(self):
        return len(self.words)

    @classmethod
    def per_image(cls, lists, charset=None, device=None):
        """lists: one word list (or path) per image -> (WordList of them all, ranges int64 [N, 2] on the same device)"""
        lists = [_read_words(x) for x in lists]
        words = cls([w for ws in lists for w in ws], charset, device)
        lens = np.array([len(ws) for ws in lists], np.int64)
        ends = np.cumsum(lens)
        ranges = np.stack([ends - lens, ends], axis=1) if len(lists) else np.zeros((0, 2), np.int64)
        words.max_list = int(lens.max()) if len(lists) else 0
        return words, torch.from_numpy(np.ascontiguousarray(ranges)).to(words.device)


def _outputs(N, W, device):
    return dict(labels=torch.empty((N, W), dtype=torch.int32, device=device),
                word=torch.empty(N, dtype=torch.int32, device=device),
                score=torch.empty(N, dtype=torch.float32, device=device),
                candidates=torch.empty(N, dtype=torch.int32, device=device),
                status=torch.empty(N, dtype=torch.int32, device=device))


def decode_packed(prob, words, ranges=None, max_edit_distance=None, mask=None, out=None, max_words_per_sample=None):
    """prob (N, C, 1, W) of CRNNDecoder / CTCDecoder, or classify (N, C, H, W) with mask (N, 1, H, W) of CTCDecoder2D, read
    through their strides in float32; words: a WordList; ranges int64 [N, 2] on the device (None: the whole list for every
    sample); max_edit_distance: delta >= 0, or None for every word of the range.  max_words_per_sample (default:
    words.max_list) sizes the candidate workspace; a longer range sets status bit OVERFLOW and keeps the greedy labels.
    `out` (a dict returned before, same shapes) is filled in place, so a captured graph can replay into the same tensors.
    -> dict labels int32 (N, W), word int32 [N], score float32 [N], candidates int32 [N], status int32 [N]"""
    if not prob.is_cuda or (mask is not None and not mask.is_cuda):
        raise NotImplementedError("megreader_b200.lexicon: CUDA tensors only (no CPU fallback)")
    if prob.dim() != 4:
        raise RuntimeError("lexicon.decode_packed: prob must be (N, C, H, W), got %s" % (tuple(prob.shape),))
    prob = prob.float()
    N, C, H, W = prob.shape
    if mask is None:
        if H != 1:
            raise RuntimeError("lexicon.decode_packed: H = %d needs the 2D head's mask" % H)
        m_ptr, ms = None, (0, 0, 0)
    else:
        mask = mask.float()
        if tuple(mask.shape) != (N, 1, H, W):
            raise RuntimeError("lexicon.decode_packed: mask must be (N, 1, H, W), got %s" % (tuple(mask.shape),))
        m_ptr, ms = mask.data_ptr(), (mask.stride(0), mask.stride(2), mask.stride(3))
    if ranges is not None:
        if ranges.dtype != torch.int64 or not ranges.is_cuda or tuple(ranges.shape) != (N, 2):
            raise RuntimeError("lexicon.decode_packed: ranges must be a CUDA int64 (N, 2) tensor")
        ranges = ranges.contiguous()
    delta = -1 if max_edit_distance is None else int(max_edit_distance)
    if max_edit_distance is not None and delta < 0:
        raise ValueError("lexicon.decode_packed: max_edit_distance must be >= 0 or None, got %r" % (max_edit_distance,))
    M = words.max_list if max_words_per_sample is None else int(max_words_per_sample)
    L = _lib.lib()
    nbytes = int(L.mr_lexicon_workspace_bytes(N, M))
    if nbytes <= 0:
        raise RuntimeError("lexicon.decode_packed: N = %d, max_words_per_sample = %d is too large" % (N, M))
    if out is None:
        out = _outputs(N, W, prob.device)
    workspace = torch.empty(nbytes, dtype=torch.uint8, device=prob.device)
    cs = words.charset
    with torch.cuda.device(prob.device):
        _lib.check(L.mr_lexicon_ctc_decode(
            prob.data_ptr(), m_ptr, N, C, H, W, prob.stride(0), prob.stride(1), prob.stride(2), prob.stride(3), *ms,
            int(cs.blank), int(cs.unknown), TINY, words.cls.data_ptr(), words.offsets.data_ptr(), len(words),
            ranges.data_ptr() if ranges is not None else None, M, delta, workspace.data_ptr(), nbytes,
            out["labels"].data_ptr(), out["word"].data_ptr(), out["score"].data_ptr(), out["candidates"].data_ptr(),
            out["status"].data_ptr(), _stream()), "lexicon_ctc_decode")
    return out


class LexiconCTCRepresenter(_decode.CTCRepresenter):
    """CTCRepresenter with lexicon-constrained decoding: `words` is a WordList (shared, or per image with the ranges in
    batch['lexicon_ranges']); represent / represent_labels as decode.CTCRepresenter's."""

    def __init__(self, words, charset=None, max_edit_distance=None, max_words_per_sample=None, cmd={}, **kwargs):
        super().__init__(charset if charset is not None else words.charset, cmd, **kwargs)
        self.words, self.max_edit_distance, self.max_words_per_sample = words, max_edit_distance, max_words_per_sample

    def _lexicon(self, batch, pred, mask=None):
        return decode_packed(pred, self.words, batch.get('lexicon_ranges'), self.max_edit_distance, mask=mask,
                             max_words_per_sample=self.max_words_per_sample)["labels"]

    def _labels(self, batch, pred):
        if not pred.is_cuda:
            raise NotImplementedError("megreader_b200.lexicon: CUDA tensors only")
        return batch['label'].to(pred.device), self._lexicon(batch, pred)


class LexiconCTCRepresenter2D(_decode.CTCRepresenter2D):
    """CTCRepresenter2D with lexicon-constrained decoding over the 2D-CTC likelihood; pred = (classify, mask)."""

    def __init__(self, words, charset=None, max_edit_distance=None, max_words_per_sample=None, max_size=32, cmd={}, **kwargs):
        super().__init__(charset if charset is not None else words.charset, max_size, cmd, **kwargs)
        self.words, self.max_edit_distance, self.max_words_per_sample = words, max_edit_distance, max_words_per_sample

    _lexicon = LexiconCTCRepresenter._lexicon

    def _labels(self, batch, pred):
        classify, mask = pred
        if not (classify.is_cuda and mask.is_cuda):
            raise NotImplementedError("megreader_b200.lexicon: CUDA tensors only")
        return batch['label'].to(classify.device), self._lexicon(batch, classify, mask)
