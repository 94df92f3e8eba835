"""Seeded inputs of the text recognisers' validation measure tests (tests/test_rec_measure_*.py,
oracle/make_rec_measure_golden.py): charsets, label-row corpora and representer batches."""
import string

import numpy as np


class ListCharset:
    """a reference-style charset: blank '\\t' (0), unknown '\\n' (1), then the given characters sorted"""
    blank, unknown = 0, 1

    def __init__(self, chars):
        self._charset = ['\t', '\n'] + sorted(set(chars) - {'\t', '\n'})

    def __len__(self):
        return len(self._charset)

    def __getitem__(self, i):
        return self._charset[i]


def charsets():
    """English (38 classes), EnglishPrintable (lowercase classes fold to uppercase), a Chinese-size charset (5,384 characters
    + blank and unknown) and a custom one with characters whose upper case expands or lies outside the BMP"""
    cjk = [chr(0x4E00 + i) for i in range(5384 - 26)] + list(string.ascii_uppercase)
    return {
        "english": ListCharset(string.digits + string.ascii_uppercase),
        "printable": ListCharset(string.digits + string.ascii_letters + string.punctuation),
        "chinese": ListCharset(cjk),
        "custom": ListCharset("abSßﬁ\U00010428\U00010400ŉẖx"),   # ß -> SS, ﬁ -> FI, 𐐨 -> 𐐀, ŉ -> ʼN, ẖ -> H̱
    }


def label_rows(rng, C, n, width, max_len):
    """n rows of class ids [n, width] int64: up to max_len symbols with blanks and unknowns sprinkled in, blank padded"""
    rows = np.zeros((n, width), np.int64)
    for i in range(n):
        L = int(rng.integers(0, max_len + 1))
        r = rng.integers(2, C, L)
        junk = rng.random(L) < 0.1
        r[junk] = rng.integers(0, 2, int(junk.sum()))
        rows[i, :L] = r
    return rows


def pair_corpus(rng, C, n, width=200, max_len=200):
    """gt and pred rows: pred an edited copy of gt (equal on about a tenth of the rows), or an unrelated row"""
    gt = label_rows(rng, C, n, width, max_len)
    pred = label_rows(rng, C, n, width, max_len)
    for i in range(n):
        if rng.random() < 0.6:
            row = [int(v) for v in gt[i] if v != 0]
            for _ in range(int(rng.integers(0, 4)) if rng.random() > 0.15 else 0):
                k = int(rng.integers(0, len(row) + 1))
                op = rng.integers(0, 3)
                if op == 0:
                    row.insert(k, int(rng.integers(0, C)))
                elif row and k < len(row):
                    if op == 1:
                        del row[k]
                    else:
                        row[k] = int(rng.integers(0, C))
            row = row[:width]
            pred[i] = 0
            pred[i, :len(row)] = row
    return gt, pred


def ctc_batch(seed, N, C, W, Lg=32, max_len=12):
    """labels [N, Lg] int32 and CTC class scores [N, C, 1, W] float32 whose argmax often spells the label"""
    rng = np.random.default_rng(seed)
    labels = label_rows(rng, C, N, Lg, max_len).astype(np.int32)
    logits = rng.standard_normal((N, C, 1, W)).astype(np.float32)
    for i in range(N):
        lab = [int(v) for v in labels[i] if v > 1]
        if rng.random() < 0.5:
            for k, c in enumerate(lab):
                for t in range(2 * k + 1, min(2 * k + 3, W)):
                    logits[i, c, 0, t] += 6.0
            logits[i, 0, 0, :] += 4.0
    return labels, logits


def ctc2d_batch(seed, N, C, H, W, Lg=32, max_len=12):
    """labels [N, Lg] int32, classify [N, C, H, W] and mask [N, 1, H, W] (softmaxed, as CTCDecoder2D's eval gives them)"""
    labels, logits = ctc_batch(seed, N, C, W, Lg, max_len)
    rng = np.random.default_rng(seed + 1)
    cls = np.repeat(logits, H, axis=2) + 0.5 * rng.standard_normal((N, C, H, W)).astype(np.float32)
    cls = np.exp(cls - cls.max(1, keepdims=True))
    cls /= cls.sum(1, keepdims=True)
    mask = rng.standard_normal((N, 1, H, W)).astype(np.float32)
    mask = np.exp(mask) / np.exp(mask).sum(2, keepdims=True)
    return labels, cls.astype(np.float32), mask.astype(np.float32)


def attn_batch(seed, N, C, W, Lg=32, max_len=12):
    """labels [N, Lg] int32 and attention predictions [N, W] int32 (a symbol sequence ending in blanks)"""
    rng = np.random.default_rng(seed)
    labels = label_rows(rng, C, N, Lg, max_len).astype(np.int32)
    pred = rng.integers(0, C, (N, W)).astype(np.int32)
    for i in range(N):
        lab = [int(v) for v in labels[i] if v > 1]
        if rng.random() < 0.5:
            pred[i, :len(lab)] = lab
            pred[i, len(lab):] = 0 if rng.random() < 0.7 else pred[i, len(lab):]
    return labels, pred


def lexicon_words(rng, strings, extra=20):
    """words for a lexicon: half of the given (upper-cased) gt strings, their lowercase forms and some random words"""
    words = [s.upper() for s in strings if s and rng.random() < 0.5]
    words += [w.lower() for w in words[:10]]
    words += ["".join(rng.choice(list(string.ascii_uppercase), int(rng.integers(1, 8)))) for _ in range(extra)]
    return words
