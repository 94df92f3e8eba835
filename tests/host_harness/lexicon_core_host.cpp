// Host-side harness: runs the PRODUCT's arithmetic of lexicon-constrained CTC decoding (megreader_b200/csrc/lexicon_core.cuh,
// the code the CUDA kernels in lexicon.cu execute) on the CPU, in float as the kernels do and in double, so that tests can
// compare it with the float64 restatement without a GPU.  Built on demand by tests/test_lexicon_cpu.py with g++.
#include <vector>

#include "lexicon_core.cuh"

using namespace mr_lexicon;

namespace {

// lpe [W, C] of sample n of prob [N, C, H, W] (contiguous) and mask [N, 1, H, W] (null: all ones)
template <class R>
void sample_lpe(const float *prob, const float *mask, int n, int C, int H, int W, float tiny, R *lpe) {
    const float *p = prob + (long long)n * C * H * W;
    const float *m = mask ? mask + (long long)n * H * W : nullptr;
    for (int t = 0; t < W; ++t)
        for (int c = 0; c < C; ++c)
            lpe[t * C + c] = log_sum_exp<R>(H, [&](int h) {
                return frame_log_prob<R>(m ? m[h * W + t] : 1.f, p[((long long)c * H + h) * W + t], tiny);
            });
}

// the whole decode of lexicon.cu for N samples, one thread: greedy [N, W] (what mr_ctc_greedy_decode wrote) is overwritten
// with the chosen words
template <class R>
void decode(const float *prob, const float *mask, int N, int C, int H, int W, int blank, float tiny, const int *cls,
            const int *off, int n_words, const long long *ranges, int max_words, int delta, int *labels, int *word, R *score,
            int *candidates, int *status) {
    std::vector<R> lpe((size_t)W * C);
    for (int n = 0; n < N; ++n) {
        const long long b = ranges ? ranges[2 * n] : 0, e = ranges ? ranges[2 * n + 1] : n_words;
        int *g = labels + (long long)n * W;
        int len = 0;
        while (len < W && g[len] != blank) ++len;
        status[n] = range_status(b, e, n_words, max_words);
        candidates[n] = 0;
        uint64_t best = 0;
        R best_score = neg_inf<R>();
        if (!status[n]) {
            sample_lpe<R>(prob, mask, n, C, H, W, tiny, lpe.data());
            for (long long k = b; k < e; ++k) {
                const int *w = cls + off[k], m = off[k + 1] - off[k];
                bool ok = m >= 1 && m <= kMaxWord;
                for (int i = 0; ok && i < m; ++i) ok = w[i] >= 0 && w[i] < C && w[i] != blank;
                if (!ok) { status[n] |= kBadWord; continue; }
                if (delta >= 0 && banded_levenshtein(w, m, g, len, delta) > delta) continue;
                ++candidates[n];
                const R s = ctc_word_score<R>(lpe.data(), W, C, w, m, blank);
                const uint64_t key = score_key((float)s, (int)k);
                if (key > best) { best = key; best_score = s; }
            }
        }
        word[n] = best ? key_index(best) : -1;
        score[n] = best_score;
        if (best) {
            const int k = key_index(best), m = off[k + 1] - off[k];
            for (int t = 0; t < W; ++t) g[t] = t < m ? cls[off[k] + t] : blank;
        }
    }
}

}  // namespace

extern "C" {

void host_lpe_f32(const float *prob, const float *mask, int N, int C, int H, int W, float tiny, float *lpe) {
    for (int n = 0; n < N; ++n) sample_lpe<float>(prob, mask, n, C, H, W, tiny, lpe + (long long)n * W * C);
}
void host_lpe_f64(const float *prob, const float *mask, int N, int C, int H, int W, float tiny, double *lpe) {
    for (int n = 0; n < N; ++n) sample_lpe<double>(prob, mask, n, C, H, W, tiny, lpe + (long long)n * W * C);
}

float host_word_score_f32(const float *lpe, int T, int C, const int *w, int L, int blank) {
    return ctc_word_score<float>(lpe, T, C, w, L, blank);
}
double host_word_score_f64(const double *lpe, int T, int C, const int *w, int L, int blank) {
    return ctc_word_score<double>(lpe, T, C, w, L, blank);
}

int host_levenshtein(const int *w, int m, const int *g, int n, int delta) { return banded_levenshtein(w, m, g, n, delta); }

unsigned long long host_score_key(float score, int index) { return score_key(score, index); }

void host_decode_f32(const float *prob, const float *mask, int N, int C, int H, int W, int blank, float tiny, const int *cls,
                     const int *off, int n_words, const long long *ranges, int max_words, int delta, int *labels, int *word,
                     float *score, int *candidates, int *status) {
    decode<float>(prob, mask, N, C, H, W, blank, tiny, cls, off, n_words, ranges, max_words, delta, labels, word, score, candidates,
                  status);
}
void host_decode_f64(const float *prob, const float *mask, int N, int C, int H, int W, int blank, float tiny, const int *cls,
                     const int *off, int n_words, const long long *ranges, int max_words, int delta, int *labels, int *word,
                     double *score, int *candidates, int *status) {
    decode<double>(prob, mask, N, C, H, W, blank, tiny, cls, off, n_words, ranges, max_words, delta, labels, word, score,
                   candidates, status);
}

}  // extern "C"
