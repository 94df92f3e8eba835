// Arithmetic of the text recognisers' validation measure (SequenceRecognitionMeasurer,
// structure/measurers/sequence_recognition_measurer.py) shared by the CUDA kernels (rec_measure.cu) and by a host-side harness
// (tests/host_harness/rec_measure_core_host.cpp) that runs the SAME routines on the CPU.  float64, every operation rounded on
// its own (no fused multiply-add), so host and device give the same bits.
//
//   * fold_class: a class id to the code points of charset[id].upper() (up to 4; none for blank and unknown), the rule of
//     label_to_string followed by the measurer's str.upper();
//   * myers_step / levenshtein: exact Levenshtein distance with unit costs (what editdistance.eval returns), Hyyrö's
//     bit-parallel form of Myers' recurrence over 64-bit blocks of the pattern;
//   * edit_score: the measurer's 1 - min(L, d) * 1.0 / L;
//   * lex_hash: the 64-bit hash of a code-point sequence that keys the lexicon table;
//   * pairwise_sum / pairwise_leaf_pass + pairwise_combine: numpy's pairwise_sum, the order in which
//     np.array(list_of_floats).sum() adds, in one thread or with the leaves on separate threads;
//   * meter_update: concern.AverageMeter.update(val, n).
#pragma once
#include <stdint.h>

#if !defined(__CUDACC__) && !defined(__host__)
#define __host__
#define __device__
#endif

namespace mr_recmeas {

constexpr int kFoldMax = 4;             // code points per class after str.upper()
constexpr int kMaxPattern = 2048;       // the shorter folded string of a pair: 32 blocks of 64, one per lane of a warp
constexpr int kPairwiseBlock = 128;     // numpy's PW_BLOCKSIZE
constexpr int kTreeDepth = 40;          // pairwise_sum splits halve n: enough for any int64 length
// status bits per sample
constexpr int kBadLabel = 1;            // a class id outside [0, C)
constexpr int kBadLength = 2;           // a code-point length outside [0, width]
// totals: 6 meters of 4 doubles (val, sum, count, updates), then the number of refused batches
enum { kMeterAccuracy = 0, kMeterEditDistance = 1, kMeterInAccuracy = 2, kMeterOutAccuracy = 3, kMeterInEditDistance = 4,
       kMeterOutEditDistance = 5, kMeters = 6 };
constexpr int kTotals = 4 * kMeters + 1;

#ifdef __CUDA_ARCH__
__device__ __forceinline__ double dadd(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double dmul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double ddiv(double a, double b) { return __ddiv_rn(a, b); }
#else
inline double dadd(double a, double b) { return a + b; }
inline double dmul(double a, double b) { return a * b; }
inline double ddiv(double a, double b) { return a / b; }
#endif

// code points of class `id` into cp[0..len); returns len, or -1 for an id outside [0, C).  fold_len [C] holds 0..kFoldMax,
// fold_cp [C, kFoldMax] the code points.
__host__ __device__ inline int fold_class(int64_t id, int C, const int *fold_len, const int *fold_cp, int *cp) {
    if (id < 0 || id >= C) return -1;
    const int n = fold_len[id];
    for (int k = 0; k < n; ++k) cp[k] = fold_cp[id * kFoldMax + k];
    return n;
}

// One column step of one 64-row block.  Pv / Mv: the block's vertical +1 / -1 deltas, Eq: the rows whose pattern symbol equals
// the text symbol, hin: the horizontal delta entering the block's top row (-1, 0, +1).  Returns the horizontal delta leaving
// row `bit` of the block (63 for a full block, the pattern's last row in the last one; rows above it never feed rows below).
__host__ __device__ inline int myers_step(uint64_t &Pv, uint64_t &Mv, uint64_t Eq, int hin, int bit) {
    const uint64_t hneg = hin < 0 ? 1ull : 0ull, hpos = hin > 0 ? 1ull : 0ull;
    const uint64_t Xv = Eq | Mv;
    Eq |= hneg;
    const uint64_t Xh = (((Eq & Pv) + Pv) ^ Pv) | Eq;
    uint64_t Ph = Mv | ~(Xh | Pv);
    uint64_t Mh = Pv & Xh;
    const int hout = (int)((Ph >> bit) & 1ull) - (int)((Mh >> bit) & 1ull);
    Ph = (Ph << 1) | hpos;
    Mh = (Mh << 1) | hneg;
    Pv = Mh | ~(Xv | Ph);
    Mv = Ph & Xv;
    return hout;
}

// Eq mask of symbol c over pattern block b (one thread; the kernel builds it with two warp ballots instead)
__host__ __device__ inline uint64_t eq_mask(const int *p, int m, int b, int c) {
    uint64_t eq = 0;
    for (int k = 0; k < 64 && 64 * b + k < m; ++k)
        if (p[64 * b + k] == c) eq |= 1ull << k;
    return eq;
}

// Levenshtein distance of p[0..m) and t[0..n), m <= kMaxPattern, one thread
__host__ __device__ inline int levenshtein(const int *p, int m, const int *t, int n) {
    if (m == 0) return n;
    if (n == 0) return m;
    uint64_t Pv[kMaxPattern / 64], Mv[kMaxPattern / 64];
    const int nb = (m + 63) >> 6, last = (m - 1) & 63;
    for (int b = 0; b < nb; ++b) { Pv[b] = ~0ull; Mv[b] = 0ull; }
    int score = m;
    for (int j = 0; j < n; ++j) {
        int h = 1;                                    // row 0 of column j is j: +1 per column
        for (int b = 0; b < nb; ++b) h = myers_step(Pv[b], Mv[b], eq_mask(p, m, b, t[j]), h, b == nb - 1 ? last : 63);
        score += h;
    }
    return score;
}

// the measurer's score of one sample: 0.0 for an empty gt, else float(1 - min(L, d) * 1.0 / L)
__host__ __device__ inline double edit_score(int L, int d) {
    if (L == 0) return 0.0;
    return dadd(1.0, -ddiv((double)(d < L ? d : L), (double)L));
}

// 64-bit hash of a code-point sequence (FNV-1a over 32-bit symbols, then the splitmix64 finaliser so that the low bits that
// index the table depend on every symbol)
__host__ __device__ inline uint64_t lex_hash(const int *cp, int n) {
    uint64_t h = 0xcbf29ce484222325ull ^ (uint64_t)(uint32_t)n;
    for (int i = 0; i < n; ++i) {
        h ^= (uint64_t)(uint32_t)cp[i];
        h *= 0x100000001b3ull;
    }
    h ^= h >> 30;
    h *= 0xbf58476d1ce4e5b9ull;
    h ^= h >> 27;
    h *= 0x94d049bb133111ebull;
    return h ^ (h >> 31);
}

// numpy's pairwise_sum below the split: a running sum from 0.0 below 8 elements; else eight strided accumulators combined as
// ((r0 + r1) + (r2 + r3)) + ((r4 + r5) + (r6 + r7)), then the tail one by one.  n <= kPairwiseBlock.
__host__ __device__ inline double pairwise_leaf(const double *a, int64_t n) {
    if (n < 8) {
        double res = 0.0;
        for (int64_t i = 0; i < n; ++i) res = dadd(res, a[i]);
        return res;
    }
    double r[8];
    for (int k = 0; k < 8; ++k) r[k] = a[k];
    int64_t i = 8;
    for (; i < n - (n % 8); i += 8)
        for (int k = 0; k < 8; ++k) r[k] = dadd(r[k], a[i + k]);
    double res = dadd(dadd(dadd(r[0], r[1]), dadd(r[2], r[3])), dadd(dadd(r[4], r[5]), dadd(r[6], r[7])));
    for (; i < n; ++i) res = dadd(res, a[i]);
    return res;
}

// The leaf of numpy's pairwise_sum tree over n elements that holds element p: above kPairwiseBlock a node splits at n / 2
// rounded down to a multiple of 8, so every leaf starts at a multiple of 8 and is at most kPairwiseBlock long.
__host__ __device__ inline void pairwise_leaf_at(int64_t n, int64_t p, int64_t *off, int64_t *len) {
    int64_t o = 0, l = n;
    while (l > kPairwiseBlock) {
        int64_t h = l / 2;
        h -= h % 8;
        if (p < o + h) {
            l = h;
        } else {
            o += h;
            l -= h;
        }
    }
    *off = o;
    *len = l;
}

// numpy's pairwise_sum over n elements, given leaf(off, len) -> the sum of one leaf: the leaves' sums added in the tree's
// order, sum(left half) + sum(right half) at every node.  The recursion runs on an explicit stack.
template <class Leaf>
__host__ __device__ inline double pairwise_tree(int64_t n, const Leaf &leaf) {
    int64_t off[kTreeDepth], len[kTreeDepth];
    double left[kTreeDepth];
    int stage[kTreeDepth];
    int sp = 0;
    off[0] = 0; len[0] = n; stage[0] = 0;
    double ret = 0.0;
    for (;;) {
        if (stage[sp] == 0 && len[sp] <= kPairwiseBlock) {
            ret = leaf(off[sp], len[sp]);
        } else if (stage[sp] < 2) {
            int64_t h = len[sp] / 2;
            h -= h % 8;
            if (stage[sp] == 1) left[sp] = ret;
            off[sp + 1] = stage[sp] == 0 ? off[sp] : off[sp] + h;
            len[sp + 1] = stage[sp] == 0 ? h : len[sp] - h;
            stage[sp + 1] = 0;
            ++stage[sp];
            ++sp;
            continue;
        } else {
            ret = dadd(left[sp], ret);
        }
        if (sp == 0) return ret;
        --sp;
    }
}

struct LeafSum {            // a leaf summed in place
    const double *a;
    __host__ __device__ double operator()(int64_t off, int64_t len) const { return pairwise_leaf(a + off, len); }
};

struct LeafTable {          // a leaf's sum computed beforehand, stored at its start / 8
    const double *sums;
    __host__ __device__ double operator()(int64_t off, int64_t len) const { return len ? sums[off / 8] : 0.0; }
};

// numpy's pairwise_sum(a, n), one thread
__host__ __device__ inline double pairwise_sum(const double *a, int64_t n) { return pairwise_tree(n, LeafSum{a}); }

// the same in two passes, as the batch kernel runs it: every leaf's sum into leaf_sums[start / 8] (ceil(n / 8) entries; each
// 8-aligned position p finds its leaf and sums it if the leaf starts there, so the leaves can go to different threads), then
// the leaves combined in the tree's order
__host__ __device__ inline void pairwise_leaf_pass(const double *a, int64_t n, int64_t p, double *leaf_sums) {
    int64_t off, len;
    pairwise_leaf_at(n, p, &off, &len);
    if (off == p) leaf_sums[p / 8] = pairwise_leaf(a + off, len);
}

__host__ __device__ inline double pairwise_combine(int64_t n, const double *leaf_sums) { return pairwise_tree(n, LeafTable{leaf_sums}); }

// concern.AverageMeter.update(val, n) on m = (val, sum, count, updates): val = mean; sum += mean * n; count += n
__host__ __device__ inline void meter_update(double *m, double mean, int64_t n) {
    m[0] = mean;
    m[1] = dadd(m[1], dmul(mean, (double)n));
    m[2] = dadd(m[2], (double)n);
    m[3] = dadd(m[3], 1.0);
}

// the per-batch means of gather_measure: accuracy and edit-distance sums over the whole batch (N samples) and, with a lexicon,
// over the n_in in-lexicon and n_out out-of-lexicon samples; added into totals (kTotals doubles)
__host__ __device__ inline void batch_update(double *totals, int64_t N, int64_t acc, double ed, bool lexicon, int64_t n_in,
                                             int64_t acc_in, double ed_in, int64_t n_out, int64_t acc_out, double ed_out) {
    meter_update(totals + 4 * kMeterAccuracy, ddiv((double)acc, (double)N), N);
    meter_update(totals + 4 * kMeterEditDistance, ddiv(ed, (double)N), N);
    if (!lexicon) return;
    const double d_in = (double)(n_in > 1 ? n_in : 1), d_out = (double)(n_out > 1 ? n_out : 1);
    meter_update(totals + 4 * kMeterInAccuracy, ddiv((double)acc_in, d_in), n_in);
    meter_update(totals + 4 * kMeterOutAccuracy, ddiv((double)acc_out, d_out), n_out);
    meter_update(totals + 4 * kMeterInEditDistance, ddiv(ed_in, d_in), n_in);
    meter_update(totals + 4 * kMeterOutEditDistance, ddiv(ed_out, d_out), n_out);
}

}  // namespace mr_recmeas
