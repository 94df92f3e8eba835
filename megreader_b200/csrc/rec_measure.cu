// The text recognisers' validation measure on the device: SequenceRecognitionMeasurer.measure and gather_measure
// (structure/measurers/sequence_recognition_measurer.py) for a batch, from the label tensors of the greedy decoders or from
// already-folded code points.
//   1. rec_measure_sample_kernel: one warp per sample.  Folds the gt and prediction rows through the fold table (class id ->
//      code points of charset[id].upper(), nothing for blank and unknown) into the workspace, computes the exact Levenshtein
//      distance with Hyyrö's bit-parallel recurrence (the shorter string is the pattern, lane b holds block b's state, the Eq
//      mask of a text symbol is two ballots over the pattern), accuracy (distance 0), the edit-distance score and the lexicon
//      membership of the folded gt;
//   2. rec_measure_batch_kernel, only with totals: one block.  The whole batch's and, with a lexicon, the in /
//      out-of-lexicon subsets' sums in numpy's pairwise order (the subsets compacted in sample order first; the trees' leaves
//      summed on separate threads, then added in the tree's order), the per-batch means of gather_measure, and the
//      AverageMeter updates into the caller's float64 totals.  A batch with any bad sample adds nothing to the meters and
//      counts as refused instead.
// rec_measure_lexicon_build_kernel fills the lexicon's open-addressing table (atomicCAS on word indices, keyed by lex_hash).
// Nothing is read back to the host, so the calls can be captured in a CUDA graph.
#include "common.cuh"
#include "rec_measure_core.cuh"

using namespace mr;
using namespace mr_recmeas;

namespace {

constexpr int kWarpsPerBlock = 4;
constexpr int kBatchThreads = 256;

int64_t r256(int64_t b) { return round_up(b, 256); }

struct Layout {
    int64_t o_gt, o_pred, o_in, o_out, o_leaf, total;
};

Layout layout(int64_t N, int64_t Lg, int64_t Wp, bool folded) {
    Layout l;
    int64_t o = 0;
    l.o_gt = o;   o += folded ? r256(N * Lg * kFoldMax * 4) : 0;
    l.o_pred = o; o += folded ? r256(N * Wp * kFoldMax * 4) : 0;
    l.o_in = o;   o += r256(N * 8);
    l.o_out = o;  o += r256(N * 8);
    l.o_leaf = o; o += r256(3 * ((N + 7) / 8) * 8);
    l.total = o > 256 ? o : 256;
    return l;
}

int64_t lexicon_capacity(int64_t n_words) {
    int64_t cap = 16;
    while (cap < 2 * n_words) cap <<= 1;
    return cap;
}

// fold row[0..L) into out (warp-wide); returns the folded length, *bad set when an id lies outside [0, C)
template <class T>
__device__ int fold_row(const T *__restrict__ row, int L, int C, const int *__restrict__ fold_len, const int *__restrict__ fold_cp,
                        int *out, bool *bad) {
    const int lane = threadIdx.x & 31;
    int pos = 0;
    bool b = false;
    for (int base = 0; base < L; base += 32) {
        const int i = base + lane;
        int cp[kFoldMax];
        int n = i < L ? fold_class((int64_t)row[i], C, fold_len, fold_cp, cp) : 0;
        b |= n < 0;
        n = n < 0 ? 0 : n;
        int incl = n;
        for (int s = 1; s < 32; s <<= 1) {
            const int v = __shfl_up_sync(0xffffffffu, incl, s);
            if (lane >= s) incl += v;
        }
        for (int k = 0; k < n; ++k) out[pos + incl - n + k] = cp[k];
        pos += __shfl_sync(0xffffffffu, incl, 31);
    }
    *bad = __any_sync(0xffffffffu, b);
    __syncwarp();
    return pos;
}

// Levenshtein distance of p[0..m) and t[0..n), m <= kMaxPattern (warp-wide, every lane returns it)
__device__ int warp_levenshtein(const int *p, int m, const int *t, int n) {
    if (m == 0) return n;
    if (n == 0) return m;
    const int lane = threadIdx.x & 31;
    const int nb = (m + 63) >> 6, last = (m - 1) & 63;
    uint64_t Pv = ~0ull, Mv = 0ull;             // block `lane`
    int score = m;
    for (int j = 0; j < n; ++j) {
        const int c = t[j];
        int h = 1;
        for (int b = 0; b < nb; ++b) {
            const int r0 = 64 * b + lane, r1 = r0 + 32;
            const unsigned lo = __ballot_sync(0xffffffffu, r0 < m && p[r0] == c);
            const unsigned hi = __ballot_sync(0xffffffffu, r1 < m && p[r1] == c);
            int hout = 0;
            if (lane == b) hout = myers_step(Pv, Mv, (uint64_t)lo | ((uint64_t)hi << 32), h, b == nb - 1 ? last : 63);
            h = __shfl_sync(0xffffffffu, hout, b);
        }
        score += h;
    }
    return score;
}

__device__ bool lexicon_has(const int *q, int n, const int *__restrict__ lex_cp, const int *__restrict__ lex_offsets,
                            const unsigned long long *__restrict__ hashes, const int *__restrict__ slots, int64_t cap) {
    const uint64_t h = lex_hash(q, n);
    for (int64_t s = (int64_t)(h & (uint64_t)(cap - 1));; s = (s + 1) & (cap - 1)) {
        const int w = slots[s];
        if (w < 0) return false;
        if (hashes[w] != h) continue;
        const int o = lex_offsets[w];
        if (lex_offsets[w + 1] - o != n) continue;
        bool eq = true;
        for (int k = 0; k < n && eq; ++k) eq = lex_cp[o + k] == q[k];
        if (eq) return true;
    }
}

template <class TG, class TP>
__global__ void __launch_bounds__(32 * kWarpsPerBlock)
rec_measure_sample_kernel(const TG *__restrict__ gt, const int *__restrict__ gt_len, int Lg, const TP *__restrict__ pred,
                          const int *__restrict__ pred_len, int Wp, int N, const int *__restrict__ fold_len,
                          const int *__restrict__ fold_cp, int C, const int *__restrict__ lex_cp, const int *__restrict__ lex_offsets,
                          int n_words, const unsigned long long *__restrict__ hashes, const int *__restrict__ slots, int64_t cap,
                          int *ws_gt, int *ws_pred, unsigned char *accuracy, int *distance, double *edit_distance,
                          unsigned char *in_lexicon, int *gt_folded, int *pred_folded, int *status) {
    const int n = blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
    if (n >= N) return;
    const int lane = threadIdx.x & 31;
    const int *g, *p;
    int lg, lp, st = 0;
    if (fold_len) {
        bool bg, bp;
        int *og = ws_gt + (int64_t)n * Lg * kFoldMax, *op = ws_pred + (int64_t)n * Wp * kFoldMax;
        lg = fold_row(gt + (int64_t)n * Lg, Lg, C, fold_len, fold_cp, og, &bg);
        lp = fold_row(pred + (int64_t)n * Wp, Wp, C, fold_len, fold_cp, op, &bp);
        st = (bg || bp) ? kBadLabel : 0;
        g = og;
        p = op;
    } else {
        lg = gt_len[n];
        lp = pred_len[n];
        if (lg < 0 || lg > Lg || lp < 0 || lp > Wp) st = kBadLength;
        lg = lg < 0 ? 0 : lg > Lg ? Lg : lg;
        lp = lp < 0 ? 0 : lp > Wp ? Wp : lp;
        g = (const int *)gt + (int64_t)n * Lg;
        p = (const int *)pred + (int64_t)n * Wp;
    }
    const int d = lg <= lp ? warp_levenshtein(g, lg, p, lp) : warp_levenshtein(p, lp, g, lg);
    if (lane == 0) {
        accuracy[n] = d == 0;
        distance[n] = d;
        edit_distance[n] = edit_score(lg, d);
        in_lexicon[n] = n_words > 0 && lexicon_has(g, lg, lex_cp, lex_offsets, hashes, slots, cap);
        gt_folded[n] = lg;
        pred_folded[n] = lp;
        status[n] = st;
    }
}

// exclusive prefix count of flag over the block (blockDim.x == kBatchThreads); *total the block's count
__device__ int block_scan(bool flag, int *warp_sums, int *total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned ballot = __ballot_sync(0xffffffffu, flag);
    if (lane == 0) warp_sums[warp] = __popc(ballot);
    __syncthreads();
    int before = 0, all = 0;
    for (int w = 0; w < kBatchThreads / 32; ++w) {
        before += w < warp ? warp_sums[w] : 0;
        all += warp_sums[w];
    }
    __syncthreads();
    *total = all;
    return before + __popc(ballot & ((1u << lane) - 1u));
}

__global__ void __launch_bounds__(kBatchThreads)
rec_measure_batch_kernel(int N, const unsigned char *__restrict__ accuracy, const double *__restrict__ edit_distance,
                         const unsigned char *__restrict__ in_lexicon, const int *__restrict__ status, int lexicon, double *in_vals,
                         double *out_vals, double *leaf_sums, double *totals) {
    __shared__ int warp_sums[kBatchThreads / 32];
    __shared__ double sums[3];
    const int tid = threadIdx.x;
    int n_in = 0, bad = 0, acc = 0, acc_in = 0;
    for (int base = 0; base < N; base += kBatchThreads) {
        const int i = base + tid;
        const bool v = i < N;
        const bool in = v && lexicon && in_lexicon[i];
        bad += __syncthreads_or(v && status[i] != 0);
        acc += __syncthreads_count(v && accuracy[i]);
        acc_in += __syncthreads_count(in && accuracy[i]);
        if (lexicon) {
            int chunk;
            const int k = block_scan(in, warp_sums, &chunk);
            if (in) in_vals[n_in + k] = edit_distance[i];
            else if (v) out_vals[base - n_in + tid - k] = edit_distance[i];
            n_in += chunk;
        }
    }
    __syncthreads();
    // numpy's pairwise sums of the batch and of the two subsets: every leaf of the three trees summed by its own thread, then
    // one thread per tree adds the leaves in the tree's order
    const int64_t n_sum[3] = {N, lexicon ? n_in : 0, lexicon ? N - n_in : 0};
    const double *src[3] = {edit_distance, in_vals, out_vals};
    const int64_t chunks = ((int64_t)N + 7) / 8;
    for (int64_t j = tid; j < 3 * chunks; j += kBatchThreads) {
        const int t = (int)(j / chunks);
        const int64_t p = 8 * (j % chunks);
        if (p < n_sum[t]) pairwise_leaf_pass(src[t], n_sum[t], p, leaf_sums + t * chunks);
    }
    __syncthreads();
    if ((tid & 31) == 0 && tid < 96) sums[tid >> 5] = pairwise_combine(n_sum[tid >> 5], leaf_sums + (tid >> 5) * chunks);
    __syncthreads();
    if (tid == 0) {
        if (bad) {
            totals[kTotals - 1] = mr_recmeas::dadd(totals[kTotals - 1], 1.0);
        } else {
            batch_update(totals, N, acc, sums[0], lexicon != 0, n_in, acc_in, lexicon ? sums[1] : 0.0, N - n_in, acc - acc_in,
                         lexicon ? sums[2] : 0.0);
        }
    }
}

__global__ void rec_measure_lexicon_build_kernel(const int *__restrict__ cp, const int *__restrict__ offsets, int n_words,
                                                 unsigned long long *hashes, int *slots, int64_t cap) {
    const int w = blockIdx.x * blockDim.x + threadIdx.x;
    if (w >= n_words) return;
    const uint64_t h = lex_hash(cp + offsets[w], offsets[w + 1] - offsets[w]);
    hashes[w] = h;
    for (int64_t s = (int64_t)(h & (uint64_t)(cap - 1));; s = (s + 1) & (cap - 1))
        if (atomicCAS(slots + s, -1, w) == -1) return;
}

template <class TG, class TP>
void launch_samples(const void *gt, const int *gt_len, int Lg, const void *pred, const int *pred_len, int Wp, int N, const int *fold_len,
                    const int *fold_cp, int C, const int *lex_cp, const int *lex_offsets, int n_words,
                    const unsigned long long *hashes, const int *slots, int64_t cap, int *ws_gt, int *ws_pred,
                    unsigned char *accuracy, int *distance, double *edit_distance, unsigned char *in_lexicon, int *gt_folded,
                    int *pred_folded, int *status, cudaStream_t st) {
    rec_measure_sample_kernel<TG, TP><<<(unsigned)ceil_div(N, kWarpsPerBlock), 32 * kWarpsPerBlock, 0, st>>>(
        (const TG *)gt, gt_len, Lg, (const TP *)pred, pred_len, Wp, N, fold_len, fold_cp, C, lex_cp, lex_offsets, n_words, hashes,
        slots, cap, ws_gt, ws_pred, accuracy, distance, edit_distance, in_lexicon, gt_folded, pred_folded, status);
}

}  // namespace

extern "C" {

int64_t mr_rec_lexicon_build_bytes(int64_t n_words) {
    if (n_words < 0 || n_words > ((int64_t)1 << 28)) return 0;
    return r256(n_words * 8) + lexicon_capacity(n_words) * 4;
}

int mr_rec_lexicon_build(const int *cp, const int *offsets, int n_words, void *table, int64_t table_bytes, void *stream) {
    if (n_words < 0 || n_words > (1 << 28)) return MR_ERR_BAD_SHAPE;
    if (!table || (n_words > 0 && (!cp || !offsets))) return MR_ERR_NULL_POINTER;
    if (table_bytes < mr_rec_lexicon_build_bytes(n_words)) return MR_ERR_BAD_SHAPE;
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t cap = lexicon_capacity(n_words);
    unsigned long long *hashes = (unsigned long long *)table;
    int *slots = (int *)((char *)table + r256((int64_t)n_words * 8));
    if (cudaMemsetAsync(slots, 0xff, cap * 4, st) != cudaSuccess) return check_launch("rec_measure lexicon memset");
    if (n_words == 0) return MR_OK;
    rec_measure_lexicon_build_kernel<<<(unsigned)ceil_div(n_words, 128), 128, 0, st>>>(cp, offsets, n_words, hashes, slots, cap);
    return check_launch("rec_measure lexicon build");
}

int64_t mr_rec_measure_workspace_bytes(int64_t N, int64_t gt_width, int64_t pred_width, int folded) {
    if (N <= 0 || N > ((int64_t)1 << 24) || gt_width < 0 || pred_width < 0 || gt_width > (1 << 20) || pred_width > (1 << 20) ||
        N * (gt_width + pred_width) > ((int64_t)1 << 30))
        return 0;
    return layout(N, gt_width, pred_width, folded != 0).total;
}

int mr_rec_measure(const void *gt, int gt_dtype, const int *gt_len, int gt_width, const void *pred, int pred_dtype, const int *pred_len,
                   int pred_width, int N, const int *fold_len, const int *fold_cp, int C, const int *lex_cp, const int *lex_offsets,
                   int n_words, const void *lex_table, void *workspace, int64_t workspace_bytes, unsigned char *accuracy,
                   int *distance, double *edit_distance, unsigned char *in_lexicon, int *gt_folded_len, int *pred_folded_len,
                   int *status, double *totals, void *stream) {
    const bool folded = fold_len != nullptr;
    const int64_t need = mr_rec_measure_workspace_bytes(N, gt_width, pred_width, folded);
    if (need <= 0 || (gt_dtype != 0 && gt_dtype != 1) || (pred_dtype != 0 && pred_dtype != 1) || n_words < 0) return MR_ERR_BAD_SHAPE;
    if (!folded && (gt_dtype != 0 || pred_dtype != 0)) return MR_ERR_BAD_SHAPE;        // code points are int32
    if (folded && (C < 1 || !fold_cp)) return MR_ERR_BAD_SHAPE;
    // the shorter folded string is the pattern, one 64-bit block per lane
    if ((int64_t)(gt_width < pred_width ? gt_width : pred_width) * (folded ? kFoldMax : 1) > kMaxPattern) return MR_ERR_UNSUPPORTED;
    if (!workspace || !accuracy || !distance || !edit_distance || !in_lexicon || !gt_folded_len || !pred_folded_len || !status)
        return MR_ERR_NULL_POINTER;
    if ((gt_width > 0 && !gt) || (pred_width > 0 && !pred) || (!folded && (!gt_len || !pred_len))) return MR_ERR_NULL_POINTER;
    if (n_words > 0 && (!lex_cp || !lex_offsets || !lex_table)) return MR_ERR_NULL_POINTER;
    if (workspace_bytes < need) return MR_ERR_BAD_SHAPE;
    cudaStream_t st = (cudaStream_t)stream;
    const Layout l = layout(N, gt_width, pred_width, folded);
    char *ws = (char *)workspace;
    int *ws_gt = (int *)(ws + l.o_gt), *ws_pred = (int *)(ws + l.o_pred);
    const unsigned long long *hashes = (const unsigned long long *)lex_table;
    const int *slots = n_words > 0 ? (const int *)((const char *)lex_table + r256((int64_t)n_words * 8)) : nullptr;
    const int64_t cap = lexicon_capacity(n_words);
#define MR_REC_LAUNCH(TG, TP)                                                                                                   \
    launch_samples<TG, TP>(gt, gt_len, gt_width, pred, pred_len, pred_width, N, fold_len, fold_cp, C, lex_cp, lex_offsets, n_words, \
                           hashes, slots, cap, ws_gt, ws_pred, accuracy, distance, edit_distance, in_lexicon, gt_folded_len,     \
                           pred_folded_len, status, st)
    if (gt_dtype == 0 && pred_dtype == 0) MR_REC_LAUNCH(int, int);
    else if (gt_dtype == 0) MR_REC_LAUNCH(int, long long);
    else if (pred_dtype == 0) MR_REC_LAUNCH(long long, int);
    else MR_REC_LAUNCH(long long, long long);
#undef MR_REC_LAUNCH
    int rc;
    if ((rc = check_launch("rec_measure samples"))) return rc;
    if (!totals) return MR_OK;                  // the batch stage only updates the meters
    rec_measure_batch_kernel<<<1, kBatchThreads, 0, st>>>(N, accuracy, edit_distance, in_lexicon, status, n_words > 0,
                                                          (double *)(ws + l.o_in), (double *)(ws + l.o_out),
                                                          (double *)(ws + l.o_leaf), totals);
    return check_launch("rec_measure batch");
}

}  // extern "C"
