// Lexicon-constrained CTC decoding on the device (DESIGN §7): for each sample, the word of its range of a word table with the
// highest CTC likelihood among the words within edit distance delta of the greedy result.
//   0. mr_ctc_greedy_decode writes the greedy labels into `labels`;
//   1. lexicon_filter_kernel, one thread per (sample, word of its range): the banded Levenshtein distance of the word to the
//      greedy labels (staged per block), and the survivors compacted into the sample's candidate list (warp-aggregated
//      atomics: the list's order varies, the arg-max below does not depend on it);
//   2. lexicon_score_kernel, a few blocks per sample: the sample's per-frame log-probabilities, summed over the heights, are
//      staged once in shared memory; then one warp per candidate runs the log-space CTC forward with one lane per state, and
//      the (score, index) key goes into the sample's maximum with one 64-bit atomicMax;
//   3. lexicon_select_kernel, one thread per label: the winner's classes (blank-padded) over the greedy labels, and the
//      word index, score, candidate count and status.
// Nothing is allocated and nothing is read back to the host, so the call can be captured in a CUDA graph.
#include "common.cuh"
#include "lexicon_core.cuh"

using namespace mr;
using namespace mr_lexicon;

namespace {

constexpr int kFilterThreads = 256;
constexpr int kScoreWarps = 8;
constexpr int kWordsPerWarp = 8;                // the score grid gives each warp about this many candidates of a full range
constexpr int kMaxScoreBlocks = 32;             // blocks per sample
constexpr int kSelectThreads = 256;
constexpr int64_t kMaxSmem = 232448;

int64_t r256(int64_t b) { return round_up(b, 256); }

struct Layout {
    int64_t o_count, o_flags, o_best, o_cand, total;
};

Layout layout(int64_t N, int64_t max_words) {
    Layout l;
    int64_t o = 0;
    l.o_count = o; o += r256(N * 4);
    l.o_flags = o; o += r256(N * 4);
    l.o_best = o;  o += r256(N * 8);
    l.o_cand = o;  o += r256(N * max_words * 4);
    l.total = o;
    return l;
}

struct Words {
    const int *cls, *off;
    const long long *ranges;        // [N, 2], or null: every sample reads the whole table
    int n_words, max_words;
};

__device__ __forceinline__ void sample_range(const Words &wd, int n, int64_t *b, int64_t *e) {
    *b = wd.ranges ? wd.ranges[2 * (int64_t)n] : 0;
    *e = wd.ranges ? wd.ranges[2 * (int64_t)n + 1] : wd.n_words;
}

// blockIdx.y = sample; thread i of the row of blocks = word i of its range
__global__ void __launch_bounds__(kFilterThreads) lexicon_filter_kernel(Words wd, const int *__restrict__ labels, int W, int C,
                                                                        int blank, int delta, int *__restrict__ count,
                                                                        int *__restrict__ flags, int *__restrict__ cand) {
    extern __shared__ int g[];
    const int n = blockIdx.y;
    int64_t b, e;
    sample_range(wd, n, &b, &e);
    if (range_status(b, e, wd.n_words, wd.max_words)) return;
    const int64_t i = (int64_t)blockIdx.x * kFilterThreads + threadIdx.x;
    if ((int64_t)blockIdx.x * kFilterThreads >= e - b) return;
    int nonblank = 0;
    for (int t = threadIdx.x; t < W; t += kFilterThreads) {
        g[t] = labels[(int64_t)n * W + t];
        nonblank += g[t] != blank;
    }
    __shared__ int s_len;
    if (threadIdx.x == 0) s_len = 0;
    __syncthreads();
    if (nonblank) atomicAdd(&s_len, nonblank);
    __syncthreads();
    const int len = s_len;                  // the greedy labels are a blank-free prefix of the row
    bool take = false;
    if (i < e - b) {
        const int word = (int)(b + i);
        const int o = wd.off[word], m = wd.off[word + 1] - o;
        const int *w = wd.cls + o;
        bool ok = m >= 1 && m <= kMaxWord;
        for (int k = 0; ok && k < m; ++k) ok = w[k] >= 0 && w[k] < C && w[k] != blank;
        if (!ok) atomicOr(flags + n, kBadWord);
        else take = delta < 0 || banded_levenshtein(w, m, g, len, delta) <= delta;
    }
    const unsigned ballot = __ballot_sync(0xffffffffu, take);
    if (!ballot) return;
    const int lane = threadIdx.x & 31, leader = __ffs(ballot) - 1;
    int base = 0;
    if (lane == leader) base = atomicAdd(count + n, __popc(ballot));
    base = __shfl_sync(0xffffffffu, base, leader);
    if (take) cand[(int64_t)n * wd.max_words + base + __popc(ballot & ((1u << lane) - 1))] = (int)(b + i);
}

struct Probs {
    const float *prob, *mask;       // mask null for the 1D heads
    int C, H, W;
    int64_t sN, sC, sH, sW, mN, mH, mW;
    float tiny;
};

// blockIdx.y = sample; the blocks of a sample share its candidates out warp by warp
__global__ void __launch_bounds__(32 * kScoreWarps) lexicon_score_kernel(Probs p, Words wd, int blank,
                                                                         const int *__restrict__ count,
                                                                         const int *__restrict__ cand,
                                                                         unsigned long long *__restrict__ best) {
    extern __shared__ float lpe[];                                     // [W, C], then per warp two alpha rows and the word
    const int n = blockIdx.y;
    const int cnt = count[n];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int first = blockIdx.x * kScoreWarps;
    if (first >= cnt) return;
    const int W = p.W, C = p.C, H = p.H;
    const float *cls = p.prob + (int64_t)n * p.sN;
    const float *msk = p.mask ? p.mask + (int64_t)n * p.mN : nullptr;
    for (int k = threadIdx.x; k < W * C; k += blockDim.x) {
        const int t = k / C, c = k % C;
        lpe[k] = log_sum_exp<float>(H, [&](int h) {
            return frame_log_prob<float>(msk ? msk[h * p.mH + t * p.mW] : 1.f, cls[c * p.sC + h * p.sH + t * p.sW], p.tiny);
        });
    }
    float *a = lpe + W * C + warp * (2 * kMaxStates + kMaxWord);
    float *b = a + kMaxStates;
    int *w = (int *)(b + kMaxStates);
    __syncthreads();
    const float ninf = -INFINITY;
    for (int k = first + warp; k < cnt; k += gridDim.x * kScoreWarps) {
        const int word = cand[(int64_t)n * wd.max_words + k];
        const int o = wd.off[word], L = wd.off[word + 1] - o;
        for (int j = lane; j < L; j += 32) w[j] = wd.cls[o + j];
        __syncwarp();
        float score = ninf;
        if (ctc_min_frames(w, L) <= W) {
            const int S = 2 * L + 1;
            for (int s = lane; s < S; s += 32) a[s] = s < 2 ? lpe[state_class(w, s, blank)] : ninf;
            __syncwarp();
            float *x = a, *y = b;
            for (int t = 1; t < W; ++t) {
                const float *row = lpe + t * C;
                for (int s = lane; s < S; s += 32)
                    y[s] = ctc_state<float>(x[s], s > 0 ? x[s - 1] : ninf, state_skips(w, s) ? x[s - 2] : ninf,
                                            row[state_class(w, s, blank)]);
                __syncwarp();
                float *z = x; x = y; y = z;
            }
            score = log_add3<float>(x[S - 1], x[S - 2], ninf);
        }
        const unsigned long long key = score_key(score, word);
        if (lane == 0 && key) atomicMax(best + n, key);
        __syncwarp();                                                  // w, a and b are rewritten for the next word
    }
}

__global__ void lexicon_select_kernel(Words wd, int N, int W, int blank, const int *__restrict__ count,
                                      const int *__restrict__ flags, const unsigned long long *__restrict__ best,
                                      int *__restrict__ labels, int *__restrict__ word, float *__restrict__ score,
                                      int *__restrict__ candidates, int *__restrict__ status) {
    const int64_t k = (int64_t)blockIdx.x * kSelectThreads + threadIdx.x;
    if (k >= (int64_t)N * W) return;
    const int n = (int)(k / W), t = (int)(k % W);
    const unsigned long long key = best[n];
    if (t == 0) {
        int64_t b, e;
        sample_range(wd, n, &b, &e);
        word[n] = key ? key_index(key) : -1;
        score[n] = key ? key_score(key) : -INFINITY;
        candidates[n] = count[n];
        status[n] = range_status(b, e, wd.n_words, wd.max_words) | flags[n];
    }
    if (!key) return;                                                  // the greedy labels stay
    const int idx = key_index(key), o = wd.off[idx], L = wd.off[idx + 1] - o;
    labels[k] = t < L ? wd.cls[o + t] : blank;
}

int64_t score_smem(int C, int W) { return ((int64_t)W * C + kScoreWarps * (2 * kMaxStates + kMaxWord)) * 4; }

}  // namespace

extern "C" {

int64_t mr_lexicon_workspace_bytes(int64_t N, int64_t max_words_per_sample) {
    if (N < 0 || N > 65535 || max_words_per_sample < 0 || max_words_per_sample > INT32_MAX ||
        N * max_words_per_sample > ((int64_t)1 << 33))
        return 0;
    return layout(N, max_words_per_sample).total;
}

int mr_lexicon_ctc_decode(const float *prob, const float *mask, int N, int C, int H, int W, int64_t sN, int64_t sC, int64_t sH,
                          int64_t sW, int64_t mN, int64_t mH, int64_t mW, int blank, int unknown, float tiny, const int *word_cls,
                          const int *word_offsets, int n_words, const long long *ranges, int max_words_per_sample,
                          int max_edit_distance, void *workspace, int64_t workspace_bytes, int *labels, int *word, float *score,
                          int *candidates, int *status, void *stream) {
    if (N < 0 || N > 65535 || C < 1 || H < 1 || W < 1 || n_words < 0 || max_words_per_sample < 0 || max_edit_distance < -1 ||
        !(tiny > 0.f))
        return MR_ERR_BAD_SHAPE;
    if (blank < 0 || blank >= C) return MR_ERR_BLANK_RANGE;
    if (N == 0) return MR_OK;
    if (!prob || !word_offsets || (n_words > 0 && !word_cls) || !workspace || !labels || !word || !score || !candidates || !status)
        return MR_ERR_NULL_POINTER;
    const int64_t need = mr_lexicon_workspace_bytes(N, max_words_per_sample);
    if (need <= 0 || workspace_bytes < need) return MR_ERR_BAD_SHAPE;
    const int64_t smem = score_smem(C, W);
    if (smem > kMaxSmem || (int64_t)W * 4 > 48 * 1024) return MR_ERR_UNSUPPORTED;
    cudaStream_t st = (cudaStream_t)stream;
    const Layout l = layout(N, max_words_per_sample);
    char *ws = (char *)workspace;
    int *count = (int *)(ws + l.o_count), *flags = (int *)(ws + l.o_flags), *cand = (int *)(ws + l.o_cand);
    unsigned long long *best = (unsigned long long *)(ws + l.o_best);
    MR_CUDA_TRY(cudaMemsetAsync(ws, 0, l.o_cand, st), "lexicon workspace memset");
    int rc = mr_ctc_greedy_decode(prob, mask, N, C, H, W, sN, sC, sH, sW, mN, mH, mW, blank, unknown, labels, stream);
    if (rc) return rc;
    const Words wd{word_cls, word_offsets, ranges, n_words, max_words_per_sample};
    if (max_words_per_sample > 0) {
        const dim3 fgrid((unsigned)ceil_div(max_words_per_sample, kFilterThreads), (unsigned)N);
        lexicon_filter_kernel<<<fgrid, kFilterThreads, (size_t)W * 4, st>>>(wd, labels, W, C, blank, max_edit_distance, count,
                                                                           flags, cand);
        if ((rc = check_launch("lexicon_filter_kernel"))) return rc;
        if ((rc = ensure_dyn_smem((const void *)lexicon_score_kernel, (size_t)smem, "lexicon_score_kernel smem"))) return rc;
        const int64_t blocks = ceil_div(max_words_per_sample, kScoreWarps * kWordsPerWarp);
        const dim3 sgrid((unsigned)(blocks < kMaxScoreBlocks ? blocks : kMaxScoreBlocks), (unsigned)N);
        const Probs p{prob, mask, C, H, W, sN, sC, sH, sW, mN, mH, mW, tiny};
        lexicon_score_kernel<<<sgrid, 32 * kScoreWarps, (size_t)smem, st>>>(p, wd, blank, count, cand, best);
        if ((rc = check_launch("lexicon_score_kernel"))) return rc;
    }
    lexicon_select_kernel<<<(unsigned)ceil_div((int64_t)N * W, kSelectThreads), kSelectThreads, 0, st>>>(
        wd, N, W, blank, count, flags, best, labels, word, score, candidates, status);
    return check_launch("lexicon_select_kernel");
}

}  // extern "C"
