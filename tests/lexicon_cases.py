"""Seeded cases of lexicon-constrained CTC decoding shared by tests/test_lexicon_cpu.py and tests/test_lexicon_gpu.py: 1D and
2D (H = 8) heads, peaked and flat distributions, words that need a blank between repeated letters, infeasible words, words of
length 1 and of the maximum length, duplicates, empty and all-infeasible ranges, at delta = 0, 1, 3 and None."""
import numpy as np

from megreader_b200.charset import EnglishCharset

CS = EnglishCharset()
C = len(CS)
LETTERS = "ABCDEFGHIJKLMNOPQRSTUVWXYZ0123456789"


def ids(word):
    return [CS.index(c) for c in word]


def random_word(rng, lo=1, hi=8):
    return "".join(rng.choice(list(LETTERS), rng.integers(lo, hi + 1)))


def edit(rng, word, k):
    """word with k random single-character edits"""
    w = list(word)
    for _ in range(k):
        op = rng.integers(3) if len(w) > 1 else 0
        i = int(rng.integers(len(w) + (op == 0)))
        if op == 0:
            w.insert(i, rng.choice(list(LETTERS)))
        elif op == 1:
            w.pop(min(i, len(w) - 1))
        else:
            w[min(i, len(w) - 1)] = rng.choice(list(LETTERS))
    return "".join(w)


def peaked_logits(rng, word, W, peak):
    """(C, W) logits whose arg-max path spells `word` (a blank between letters), on top of noise"""
    z = rng.normal(size=(C, W))
    z[0] += 6.0
    L = len(word)
    start = int(rng.integers(0, max(1, W - 2 * L + 1)))
    for i, c in enumerate(ids(word)):
        f = start + 2 * i
        if f < W:
            z[c, f] += peak
    return z


def softmax(z, axis):
    z = z - z.max(axis=axis, keepdims=True)
    e = np.exp(z)
    return e / e.sum(axis=axis, keepdims=True)


def make_prob(rng, truths, W, H, kind):
    """classify (N, C, H, W) float32 and mask (N, 1, H, W) (None for H = 1)"""
    N = len(truths)
    z = np.empty((N, C, H, W))
    for n, word in enumerate(truths):
        base = peaked_logits(rng, word, W, 9.0) if kind == "peaked" else 0.0      # one alignment for every height
        for h in range(H):
            z[n, :, h] = base + rng.normal(size=(C, W)) * (0.3 if kind == "peaked" else 0.5)
    prob = softmax(z, 1).astype(np.float32)
    if H == 1:
        return prob, None
    mask = softmax(rng.normal(size=(N, 1, H, W)) * 2.0, 2).astype(np.float32)
    return prob, mask


def word_list(rng, truth, W, n_random=12):
    """a list around `truth`: itself, near misses at 1 to 4 edits, repeats, a duplicate, random words, an infeasible word"""
    words = [truth] + [edit(rng, truth, k) for k in (1, 1, 2, 3, 4)] + ["LL", "BOOK", "A", truth]
    words += [random_word(rng) for _ in range(n_random)]
    words.append("X" * ((W + 1) // 2 + 1))                           # repeats: needs 2L - 1 > W frames
    return words


def case(seed, N=6, W=33, H=1, kind="peaked", delta=None, layout="per_image"):
    """-> dict(prob, mask, words (strings), ranges (N, 2) int64 or None, delta)"""
    rng = np.random.default_rng(seed)
    truths = [random_word(rng, 1, 8) for _ in range(N)]
    truths[0] = "BOOK"
    truths[1 % N] = "LL"
    prob, mask = make_prob(rng, truths, W, H, kind)
    if layout == "shared":
        words = sorted({w for t in truths for w in word_list(rng, t, W, 4)}) + ["BOOK"]
        return dict(prob=prob, mask=mask, words=words, ranges=None, delta=delta)
    lists = [word_list(rng, t, W) for t in truths]
    if N >= 4:
        lists[2] = []                                                # empty range
        lists[3] = ["Q" * min(W, 64), "ZZ" * min(W // 2 + 1, 32)]     # nothing feasible
    words = [w for ws in lists for w in ws]
    lens = np.array([len(ws) for ws in lists], np.int64)
    ends = np.cumsum(lens)
    return dict(prob=prob, mask=mask, words=words, ranges=np.stack([ends - lens, ends], 1), delta=delta)


def long_word_case(seed):
    """words of the maximum length (64 classes) at W = 65: one feasible, one with a repeat more than the frames allow"""
    rng = np.random.default_rng(seed)
    feasible = "".join(LETTERS[i % 36] for i in range(64))
    prob, mask = make_prob(rng, [feasible, "A"], 65, 1, "peaked")
    words = [feasible, "A" * 33 + feasible[:31], "A", feasible[:63] + "Z", random_word(rng)]
    return dict(prob=prob, mask=mask, words=words, ranges=None, delta=None)


def all_cases():
    out = {}
    for d in (0, 1, 3, None):
        out["1d_peaked_d%s" % d] = case(10 + (9 if d is None else d), delta=d)
        out["2d_peaked_d%s" % d] = case(20 + (9 if d is None else d), W=16, H=8, delta=d)
    out["1d_flat"] = case(31, kind="flat")
    out["2d_flat"] = case(32, W=16, H=8, kind="flat")
    out["1d_shared_d1"] = case(33, layout="shared", delta=1)
    out["1d_w65"] = case(34, W=65, delta=3)
    out["long_words"] = long_word_case(35)
    return out
