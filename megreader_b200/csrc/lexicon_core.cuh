// Arithmetic of lexicon-constrained CTC decoding (DESIGN §7, Shi, Bai & Yao 2015 §2.3.2) shared by the CUDA kernels
// (lexicon.cu) and by a host-side harness (tests/host_harness/lexicon_core_host.cpp) that runs the SAME routines on the CPU,
// in float as the kernels do and in double.
//
//   * frame_log_prob / log_sum_exp: lp[t, h, c] = log(max(mask * classify, tiny)) and its log-sum over the heights.  The 2D-CTC
//     recurrence adds lp[t, h, cur] to a term that does not depend on h, so the likelihood summed over the heights is ordinary
//     CTC over lpe[t, c] = logsumexp_h lp[t, h, c];
//   * log_add3 / ctc_state: one state of the log-space CTC forward; ctc_word_score runs the whole forward of one word;
//   * banded_levenshtein: the Levenshtein distance of a word and the greedy labels, inside a band of half-width delta, with an
//     early exit as soon as every cell of a column exceeds delta;
//   * score_key: a (score, word index) pair as one 64-bit integer whose maximum is the largest score, then the lowest index.
#pragma once
#include <math.h>
#include <stdint.h>
#include <string.h>

#if !defined(__CUDACC__) && !defined(__host__)
#define __host__
#define __device__
#endif

namespace mr_lexicon {

constexpr int kMaxWord = 64;                    // classes per word
constexpr int kMaxStates = 2 * kMaxWord + 1;
// status bits per sample
constexpr int kOverflow = 1;                    // the range holds more words than max_words_per_sample
constexpr int kBadRange = 2;                    // begin < 0, end < begin or end > n_words
constexpr int kBadWord = 4;                     // a word of the range is empty, too long, or holds blank or a class >= C

template <class R> __host__ __device__ inline R r_exp(R x);
template <class R> __host__ __device__ inline R r_log1p(R x);
template <> __host__ __device__ inline float r_exp<float>(float x) { return expf(x); }
template <> __host__ __device__ inline double r_exp<double>(double x) { return exp(x); }
template <> __host__ __device__ inline float r_log1p<float>(float x) { return log1pf(x); }
template <class R> __host__ __device__ inline R r_log(R x);
template <> __host__ __device__ inline float r_log<float>(float x) { return logf(x); }
template <> __host__ __device__ inline double r_log<double>(double x) { return log(x); }
template <> __host__ __device__ inline double r_log1p<double>(double x) { return log1p(x); }

template <class R> __host__ __device__ inline R neg_inf() { return -(R)INFINITY; }

// the per-frame log-probability of the 2D-CTC head (ctc2d_head.head_log_probs): the product in float, the log in R
template <class R>
__host__ __device__ inline R frame_log_prob(float mask, float classify, float tiny) {
    const float p = mask * classify;
    return r_log<R>((R)(p > tiny ? p : tiny));
}

// log(sum_i exp(v(i))) over i < n: the maximum plus log1p of the other terms, so that a sum dominated by one term keeps the
// precision of that term
template <class R, class V>
__host__ __device__ inline R log_sum_exp(int n, const V &v) {
    R m = neg_inf<R>();
    int at = 0;
    for (int i = 0; i < n; ++i) {
        const R x = v(i);
        if (x > m) { m = x; at = i; }
    }
    if (m == neg_inf<R>()) return m;
    R s = 0;
    for (int i = 0; i < n; ++i)
        if (i != at) s += r_exp<R>(v(i) - m);
    return m + r_log1p<R>(s);
}

template <class R>
__host__ __device__ inline R log_add3(R a, R b, R c) {
    R m = a, x = b, y = c;
    if (b > m && b >= c) { m = b; x = a; y = c; }
    else if (c > m) { m = c; x = a; y = b; }
    if (m == neg_inf<R>()) return m;
    return m + r_log1p<R>(r_exp<R>(x - m) + r_exp<R>(y - m));
}

// state s of the extended label sequence (blank, w0, blank, w1, ..., blank): its class and whether it may be entered from
// state s - 2 (a letter that differs from the previous letter)
__host__ __device__ inline int state_class(const int *w, int s, int blank) { return (s & 1) ? w[s >> 1] : blank; }
__host__ __device__ inline bool state_skips(const int *w, int s) { return (s & 1) && s >= 3 && w[s >> 1] != w[(s >> 1) - 1]; }

// alpha_t[s] from alpha_{t-1}[s], [s - 1] and [s - 2] (pass -inf for the ones that do not exist or may not be entered)
template <class R>
__host__ __device__ inline R ctc_state(R stay, R from1, R from2, R lp) {
    const R a = log_add3<R>(stay, from1, from2);
    return a == neg_inf<R>() ? a : a + lp;
}

// frames a word needs: one per letter and one blank between equal neighbours
__host__ __device__ inline int ctc_min_frames(const int *w, int L) {
    int n = L;
    for (int i = 1; i < L; ++i) n += w[i] == w[i - 1];
    return n;
}

// log p(w | lpe) for lpe [T, ld] (the first C entries of a row are the classes), 1 <= L <= kMaxWord; -inf when the word
// cannot be aligned in T frames.  One thread; the scoring kernel runs the same states with one lane per state.
template <class R>
__host__ __device__ inline R ctc_word_score(const R *lpe, int T, int ld, const int *w, int L, int blank) {
    if (ctc_min_frames(w, L) > T) return neg_inf<R>();
    const int S = 2 * L + 1;
    R a[kMaxStates], b[kMaxStates];
    for (int s = 0; s < S; ++s) a[s] = s < 2 ? lpe[state_class(w, s, blank)] : neg_inf<R>();
    for (int t = 1; t < T; ++t) {
        const R *row = lpe + (int64_t)t * ld;
        for (int s = 0; s < S; ++s)
            b[s] = ctc_state<R>(a[s], s > 0 ? a[s - 1] : neg_inf<R>(), state_skips(w, s) ? a[s - 2] : neg_inf<R>(),
                                row[state_class(w, s, blank)]);
        for (int s = 0; s < S; ++s) a[s] = b[s];
    }
    return log_add3<R>(a[S - 1], a[S - 2], neg_inf<R>());
}

// Levenshtein distance of w [m] (m <= kMaxWord) and g [n] when it is at most delta >= 0, else delta + 1.  Column j of the DP
// holds the distances of every prefix of w to g[0, j); only the cells with |i - j| <= delta are kept (a path through any other
// cell costs more than delta), and the scan stops at the first column whose band is all above delta.
__host__ __device__ inline int banded_levenshtein(const int *w, int m, const int *g, int n, int delta) {
    const int big = delta + 1;
    if (m - n > delta || n - m > delta) return big;
    int D[kMaxWord + 1];
    for (int i = 0; i <= m; ++i) D[i] = i <= delta ? i : big;
    for (int j = 1; j <= n; ++j) {
        const int lo = j - delta > 0 ? j - delta : 0, hi = j + delta < m ? j + delta : m;
        int i = lo, diag, left, best;
        if (lo == 0) {
            diag = D[0];
            D[0] = left = best = j;
            i = 1;
        } else {
            diag = D[lo - 1];
            left = best = big;
        }
        for (; i <= hi; ++i) {
            const int up = D[i];
            int v = (up < left ? up : left) + 1;
            const int sub = diag + (w[i - 1] != g[j - 1]);
            v = sub < v ? sub : v;
            v = v < big ? v : big;
            diag = up;
            D[i] = left = v;
            best = v < best ? v : best;
        }
        if (best > delta) return big;
    }
    return D[m] < big ? D[m] : big;
}

// status of a sample's word range [begin, end) of a table of n_words words, at most max_words words per sample
__host__ __device__ inline int range_status(int64_t begin, int64_t end, int64_t n_words, int64_t max_words) {
    if (begin < 0 || end < begin || end > n_words) return kBadRange;
    return end - begin > max_words ? kOverflow : 0;
}

// 0 for a score that cannot win (-inf or NaN); else the order of the score in the high half, the complement of the index in
// the low half, so that the maximum key is the largest score and, among equal scores, the lowest index
__host__ __device__ inline uint64_t score_key(float score, int index) {
    if (!(score > -INFINITY)) return 0;
    if (score == 0.f) score = 0.f;                              // -0 and +0 are one score
    uint32_t bits;
    memcpy(&bits, &score, 4);
    bits = (bits & 0x80000000u) ? ~bits : bits | 0x80000000u;
    return ((uint64_t)bits << 32) | (uint32_t)~(uint32_t)index;
}

__host__ __device__ inline int key_index(uint64_t key) { return (int)~(uint32_t)key; }

__host__ __device__ inline float key_score(uint64_t key) {
    uint32_t bits = (uint32_t)(key >> 32);
    bits = (bits & 0x80000000u) ? bits & 0x7fffffffu : ~bits;
    float s;
    memcpy(&s, &bits, 4);
    return s;
}

}  // namespace mr_lexicon
