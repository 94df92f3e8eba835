// Host-side harness: runs the PRODUCT's arithmetic of the text recognisers' validation measure
// (megreader_b200/csrc/rec_measure_core.cuh, the code the CUDA kernels in rec_measure.cu execute) on the CPU, so that tests can
// compare it with the plain-Python oracle without a GPU.  Built on demand by tests/test_rec_measure_cpu.py with g++.
#include "rec_measure_core.cuh"

using namespace mr_recmeas;

extern "C" {

// for n pairs of class-id rows (gt [n, Lg], pred [n, Wp] int64) through the fold table: folded lengths, status, Levenshtein
// distance and edit-distance score, as the sample kernel computes them (the shorter folded string is the pattern)
void host_pairs(const long long *gt, int Lg, const long long *pred, int Wp, int n, const int *fold_len, const int *fold_cp, int C,
                int *gt_len, int *pred_len, int *status, int *distance, double *score) {
    static int g[4 * 4096], p[4 * 4096];
    for (int i = 0; i < n; ++i) {
        int lg = 0, lp = 0, st = 0, cp[kFoldMax];
        for (int k = 0; k < Lg; ++k) {
            const int m = fold_class(gt[(long long)i * Lg + k], C, fold_len, fold_cp, cp);
            if (m < 0) st = kBadLabel;
            for (int j = 0; j < m; ++j) g[lg++] = cp[j];
        }
        for (int k = 0; k < Wp; ++k) {
            const int m = fold_class(pred[(long long)i * Wp + k], C, fold_len, fold_cp, cp);
            if (m < 0) st = kBadLabel;
            for (int j = 0; j < m; ++j) p[lp++] = cp[j];
        }
        const int d = lg <= lp ? levenshtein(g, lg, p, lp) : levenshtein(p, lp, g, lg);
        gt_len[i] = lg;
        pred_len[i] = lp;
        status[i] = st;
        distance[i] = d;
        score[i] = edit_score(lg, d);
    }
}

double host_pairwise_sum(const double *a, long long n) { return pairwise_sum(a, n); }

// the batch kernel's form: the leaf pass at every 8-aligned position (in reverse, as threads may run in any order), then the
// ordered combine
double host_pairwise_two_pass(const double *a, long long n) {
    static double leaf_sums[1 << 17];
    for (long long p = ((n + 7) / 8 - 1) * 8; p >= 0; p -= 8) pairwise_leaf_pass(a, n, p, leaf_sums);
    return pairwise_combine(n, leaf_sums);
}

unsigned long long host_hash(const int *cp, int n) { return lex_hash(cp, n); }

// batch_update over `batches` batches: sizes[b] samples each, acc / ed / in_lexicon concatenated in sample order
void host_totals(const int *sizes, int batches, const unsigned char *acc, const double *ed, const unsigned char *in_lexicon, int lexicon,
                 double *totals) {
    static double in_vals[1 << 16], out_vals[1 << 16];
    long long o = 0;
    for (int b = 0; b < batches; ++b) {
        const int N = sizes[b];
        long long a = 0, a_in = 0, n_in = 0, n_out = 0;
        for (int i = 0; i < N; ++i) {
            a += acc[o + i];
            if (lexicon && in_lexicon[o + i]) { a_in += acc[o + i]; in_vals[n_in++] = ed[o + i]; }
            else if (lexicon) out_vals[n_out++] = ed[o + i];
        }
        batch_update(totals, N, a, host_pairwise_two_pass(ed + o, N), lexicon != 0, n_in, a_in, host_pairwise_two_pass(in_vals, n_in),
                     n_out, a - a_in, host_pairwise_two_pass(out_vals, n_out));
        o += N;
    }
}

}  // extern "C"
