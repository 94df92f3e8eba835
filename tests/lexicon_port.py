"""Float64 restatement of lexicon-constrained CTC decoding (megreader_b200.lexicon, DESIGN §7), the reference the host harness
and the device are compared with.  The reference project has no lexicon decoder, so this restates the definition from the
quantities it does define:
  * the greedy labels: oracle.crnn_port.greedy_ctc_decode (for the 2D head, on the columns of the arg-max-height path, as
    ctc_representer2d.py picks them);
  * the Levenshtein distance: oracle.rec_measure_port.levenshtein's recurrence over class ids, for many words at once;
  * the score of a word: -F.ctc_loss in float64 on the CPU for H = 1, -oracle.capi.ctc2d_forward (the float64 restatement of
    the reference's 2D-CTC kernel) for H > 1, both over lp = log(max(mask * classify, tiny)) formed in float32;
  * the choice: the candidate with the largest finite score, the lowest index among equal float32 scores; without one the
    greedy labels, word -1 and score -inf."""
import numpy as np
import torch

from oracle import capi
from oracle.crnn_port import greedy_ctc_decode

TINY = float(torch.finfo(torch.float32).tiny)
OVERFLOW, BAD_RANGE = 1, 2


def log_probs(prob, mask=None, tiny=TINY):
    """(N, C, H, W) float32 [+ mask (N, 1, H, W)] -> lp (W, H, N, C) float64: the product in float32, its log in float64"""
    prob = torch.as_tensor(prob, dtype=torch.float32)
    m = torch.ones_like(prob[:, :1]) if mask is None else torch.as_tensor(mask, dtype=torch.float32)
    lp = torch.log(torch.clamp_min(m * prob, tiny).double())
    return lp.permute(3, 2, 0, 1).contiguous()


def greedy(prob, mask=None):
    prob = torch.as_tensor(prob, dtype=torch.float32)
    if mask is None:
        return greedy_ctc_decode(prob)
    heat = prob * torch.as_tensor(mask, dtype=torch.float32)
    C = prob.shape[1]
    path = heat.max(1, keepdim=True)[0].argmax(2, keepdim=True).repeat(1, C, 1, 1)
    return greedy_ctc_decode(heat.gather(2, path))


def levenshtein_many(words, g):
    """levenshtein(w, g) for every w of `words` (lists of class ids) at once: rec_measure_port's row recurrence, with the
    words down the rows (padded with -1, which never equals a class) and g along the columns"""
    if not words:
        return np.zeros(0, np.int64)
    lens = np.array([len(w) for w in words])
    pad = np.full((len(words), lens.max()), -1, np.int64)
    for i, w in enumerate(words):
        pad[i, :len(w)] = w
    idx = np.arange(pad.shape[1] + 1)
    prev = np.broadcast_to(idx, (len(words), len(idx))).copy()
    for j, x in enumerate(g, 1):
        cur = np.empty_like(prev)
        cur[:, 0] = j
        cur[:, 1:] = np.minimum(prev[:, 1:] + 1, prev[:, :-1] + (pad != x))
        prev = np.minimum.accumulate(cur - idx, axis=1) + idx
    return prev[np.arange(len(words)), lens]


def word_scores(lp, n, words):
    """float64 log-likelihoods of `words` (lists of class ids) for sample n of lp (W, H, N, C)"""
    if not words:
        return np.zeros(0)
    T, H, _, C = lp.shape
    k = len(words)
    S = max(len(w) for w in words)
    tg = np.zeros((k, S), np.int64)
    for i, w in enumerate(words):
        tg[i, :len(w)] = w
    tl = np.array([len(w) for w in words], np.int64)
    x = lp[:, :, n:n + 1, :].expand(T, H, k, C).contiguous()
    if H == 1:
        nll = torch.nn.functional.ctc_loss(x[:, 0], torch.from_numpy(tg), torch.full((k,), T, dtype=torch.int64),
                                           torch.from_numpy(tl), blank=0, reduction="none", zero_infinity=False).numpy()
    else:
        nll, _ = capi.ctc2d_forward(x.numpy(), tg, np.full(k, T, np.int64), tl)
    return -np.asarray(nll, np.float64)


def decode(prob, words, ranges=None, delta=None, mask=None, max_words=None):
    """words: list of class-id lists; ranges (N, 2) or None -> dict labels (N, W) int32, word, score (float64), candidates,
    status, and `scores`: per sample {word index: score} of its candidates"""
    prob = torch.as_tensor(prob, dtype=torch.float32)
    N, _, _, W = prob.shape
    lp = log_probs(prob, mask)
    labels = greedy(prob, mask).numpy().astype(np.int32)
    M = len(words) if max_words is None else max_words
    out = dict(word=np.full(N, -1, np.int32), score=np.full(N, -np.inf), candidates=np.zeros(N, np.int32),
               status=np.zeros(N, np.int32), scores=[])
    for n in range(N):
        b, e = (0, len(words)) if ranges is None else (int(ranges[n][0]), int(ranges[n][1]))
        scores = {}
        if b < 0 or e < b or e > len(words):
            out["status"][n] = BAD_RANGE
        elif e - b > M:
            out["status"][n] = OVERFLOW
        else:
            g = [int(c) for c in labels[n] if c != 0]
            ks = np.arange(b, e)
            if delta is not None:
                ks = ks[levenshtein_many(words[b:e], g) <= delta]
            cand = [int(k) for k in ks]
            scores = dict(zip(cand, word_scores(lp, n, [words[k] for k in cand])))
            out["candidates"][n] = len(cand)
            finite = [k for k in cand if np.isfinite(scores[k])]
            if finite:
                k = max(finite, key=lambda k: (np.float32(scores[k]), -k))
                out["word"][n], out["score"][n] = k, scores[k]
                labels[n] = 0
                labels[n, :len(words[k])] = words[k]
        out["scores"].append(scores)
    out["labels"] = labels
    return out
