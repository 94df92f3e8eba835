"""Greedy decoders on the GPU: the integer core of the reference's representers (SURVEY.md §8f row N1) —
`CTCRepresenter.represent` (structure/representers/ctc_representer.py:22-34), `CTCRepresenter2D.represent`
(ctc_representer2d.py:27-51) and `SequenceRecognitionRepresenter.represent` (sequence_recognition_representer.py:23-28).
The functions return int32 label tensors.  The representer classes below build on them:

    represent(batch, pred)        -> the reference's list of {'label_string', 'pred_string'} dicts (CTCRepresenter2D adds the
                                     per-sample 'mask' / 'classify' CPU tensors its visualiser reads); the strings come from one
                                     device-to-host copy and a numpy lookup of the charset's strings
    represent_labels(batch, pred) -> the device (gt, pred) label tensors, for rec_measure.measure_labels (no host
                                     synchronisation, so a whole validation step can be captured in a CUDA graph)"""
import numpy as np
import torch

from . import _lib


def _st():
    return torch.cuda.current_stream().cuda_stream


def ctc_greedy_decode(prob, blank=0, unknown=1):
    """prob (N, C, 1, W) class scores (CRNNDecoder eval output) -> int32 (N, W) collapsed labels, blank-padded."""
    if not prob.is_cuda:
        raise NotImplementedError("megreader_b200.decode: CUDA tensors only")
    prob = prob.float()
    N, C, H, W = prob.shape
    out = torch.empty((N, W), dtype=torch.int32, device=prob.device)
    _lib.check(_lib.lib().mr_ctc_greedy_decode(prob.data_ptr(), None, N, C, 1, W, prob.stride(0), prob.stride(1),
                                               prob.stride(2), prob.stride(3), 0, 0, 0, blank, unknown, out.data_ptr(),
                                               _st()), "ctc_greedy_decode")
    return out


def ctc2d_greedy_decode(classify, mask, blank=0, unknown=1):
    """classify (N, C, H, W), mask (N, 1, H, W) (CTCDecoder2D eval output) -> int32 (N, W)."""
    if not classify.is_cuda:
        raise NotImplementedError("megreader_b200.decode: CUDA tensors only")
    classify, mask = classify.float(), mask.float()
    N, C, H, W = classify.shape
    out = torch.empty((N, W), dtype=torch.int32, device=classify.device)
    _lib.check(_lib.lib().mr_ctc_greedy_decode(classify.data_ptr(), mask.data_ptr(), N, C, H, W, classify.stride(0),
                                               classify.stride(1), classify.stride(2), classify.stride(3),
                                               mask.stride(0), mask.stride(2), mask.stride(3), blank, unknown,
                                               out.data_ptr(), _st()), "ctc2d_greedy_decode")
    return out


def blank_after_first_blank_(pred, blank=0):
    """In place on an int32 (N, W) tensor: everything from the first blank on becomes blank."""
    assert pred.dtype == torch.int32 and pred.is_contiguous() and pred.is_cuda
    _lib.check(_lib.lib().mr_blank_after_first_blank(pred.data_ptr(), pred.size(0), pred.size(1), blank, _st()),
               "blank_after_first_blank")
    return pred


class SequenceRecognitionRepresenter:
    """structure/representers/sequence_recognition_representer.py on the device: pred (N, W) class ids (AttentionDecoder's eval
    output); everything from the first blank on is blank (in place on an int32 contiguous pred, like the reference)."""

    def __init__(self, charset=None, cmd={}, **kwargs):
        if charset is None:
            from .charset import default_charset
            charset = default_charset()
        self.charset = charset
        strings = [charset[i] for i in range(len(charset))]
        strings[charset.blank] = strings[charset.unknown] = ""
        self._strings = np.array(strings, dtype=object)

    def label_to_string(self, label):
        return "".join(self._strings[np.asarray(label, dtype=np.int64)])

    def _decode(self, pred):
        pred = pred.to(torch.int32).contiguous()
        return blank_after_first_blank_(pred, self.charset.blank)

    def _labels(self, batch, pred):
        if not pred.is_cuda:
            raise NotImplementedError("megreader_b200.decode: CUDA tensors only")
        return batch['label'].to(pred.device), self._decode(pred)

    def represent_labels(self, batch, pred):
        return self._labels(batch, pred)

    def _strings_of(self, gt, pred):
        """one device-to-host copy of both label matrices, then one lookup per row"""
        gt, pred = gt.to(torch.int64), pred.to(torch.int64)
        both = torch.cat([gt.reshape(-1), pred.reshape(-1)]).cpu().numpy()
        g, p = both[:gt.numel()].reshape(gt.shape), both[gt.numel():].reshape(pred.shape)
        return [self.label_to_string(r) for r in g], [self.label_to_string(r) for r in p]

    def represent(self, batch, pred):
        gt, out = self._labels(batch, pred)
        labels, preds = self._strings_of(gt, out)
        return [{'label_string': g, 'pred_string': p} for g, p in zip(labels, preds)]


class CTCRepresenter(SequenceRecognitionRepresenter):
    """structure/representers/ctc_representer.py on the device: pred (N, C, 1, W) class scores (CRNNDecoder's eval output)."""

    def _decode(self, pred):
        return ctc_greedy_decode(pred, self.charset.blank, self.charset.unknown)


class CTCRepresenter2D(SequenceRecognitionRepresenter):
    """structure/representers/ctc_representer2d.py on the device: pred = (classify (N, C, H, W), mask (N, 1, H, W))
    (CTCDecoder2D's eval output)."""

    def __init__(self, charset=None, max_size=32, cmd={}, **kwargs):
        super().__init__(charset, cmd, **kwargs)
        self.max_size = max_size

    def _labels(self, batch, pred):
        classify, mask = pred
        if not (classify.is_cuda and mask.is_cuda):
            raise NotImplementedError("megreader_b200.decode: CUDA tensors only")
        return batch['label'].to(classify.device), ctc2d_greedy_decode(classify, mask, self.charset.blank, self.charset.unknown)

    def represent(self, batch, pred):
        result = super().represent(batch, pred)
        classify, mask = (t.to('cpu') for t in pred)
        for i, r in enumerate(result):
            r['mask'] = mask[i][0]
            r['classify'] = classify[i]
        return result
