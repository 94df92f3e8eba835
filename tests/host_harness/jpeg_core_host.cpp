// Host-side harness: runs the PRODUCT's JPEG routines (megreader_b200/csrc/jpeg_core.cuh, the code the CUDA kernels in jpeg.cu
// execute) on the CPU, so that tests can compare them with cv2.imdecode without a GPU.  Built on demand with g++
// -ffp-contract=off.
#include <stdlib.h>
#include <string.h>

#include <vector>

#include "jpeg_core.cuh"

using namespace mr_jpeg;

namespace {

struct Scan {
    std::vector<uint8_t> s;              // unstuffed stream
    std::vector<int64_t> seg;            // segment start bytes, then the stream's end
    int status = 0;
};

// the scan bytes split as the device's split kernel does, byte by byte with classify()
Scan split(const uint8_t *p, int64_t n, const Info &I) {
    Scan S;
    const uint8_t *b = p + I.scan;
    const int64_t m = n - I.scan;
    S.seg.push_back(0);
    int rst = 0;
    for (int64_t i = 0; i < m; ++i) {
        const int k = classify(b, m, i);
        if (k == kEnd) break;
        if (k == kData) S.s.push_back(b[i]);
        if (k == kRst) {
            if (b[i + 1] - 0xD0 != (rst & 7)) S.status |= kCorrupt;
            ++rst;
            S.seg.push_back((int64_t)S.s.size());
        }
    }
    S.seg.push_back((int64_t)S.s.size());
    const int64_t mcus = (int64_t)I.mcus_x * I.mcus_y;
    const int64_t want = I.ri ? (mcus + I.ri - 1) / I.ri : 1;
    if ((int64_t)S.seg.size() - 1 != want) S.status |= kCorrupt;
    return S;
}

int64_t seg_blocks(const Info &I, int64_t k) {
    const int64_t mcus = (int64_t)I.mcus_x * I.mcus_y;
    if (!I.ri) return mcus * I.bpm;
    const int64_t lo = k * I.ri, hi = lo + I.ri < mcus ? lo + I.ri : mcus;
    return (hi - lo) * I.bpm;
}

// coefficients of every block with one sequential decode per segment (run = the whole segment)
int decode_coefs(const Info &I, const Scan &S, std::vector<int16_t> &coef) {
    int status = S.status;
    const int64_t nblk = (int64_t)I.mcus_x * I.mcus_y * I.bpm;
    coef.assign(nblk * 64, 0);
    const int64_t nseg = (int64_t)S.seg.size() - 1;
    int64_t base = 0;
    for (int64_t k = 0; k < nseg; ++k) {
        const int64_t nb = seg_blocks(I, k);
        if (base + nb > nblk) break;
        St st{(int32_t)(8 * S.seg[k]), 0, 0};
        const int dc0[3] = {0, 0, 0};
        RunOut o = decode_run<true>(I, S.s.data(), (int64_t)S.s.size(), 8 * S.seg[k + 1], st, 8 * S.seg[k + 1], coef.data() + base * 64, 0,
                                    nb, dc0);
        if (o.err || !o.done) status |= kCorrupt;
        base += nb;
    }
    return status;
}

// The synchronising decode of jpeg.cu as host loops over runs of `run_bits`: phase 1 (every run from the assumed state),
// kRelax passes (every run from its predecessor's latest exit), phase 2 (every run from its predecessor's exit), the walker (runs whose entry was not that exit are decoded from
// the true one), the segmented prefix sums, and the write pass.  Counts how many runs the walker decoded.
int decode_coefs_sync(const Info &I, const Scan &S, int run_bits, std::vector<int16_t> &coef, int *fixed) {
    constexpr int kRelax = 2;            // as jpeg.cu
    int status = S.status;
    const int64_t nblk = (int64_t)I.mcus_x * I.mcus_y * I.bpm;
    coef.assign(nblk * 64, 0);
    const int64_t nseg = (int64_t)S.seg.size() - 1;
    const uint8_t *s = S.s.data();
    const int64_t end = (int64_t)S.s.size();
    int64_t base = 0;
    *fixed = 0;
    for (int64_t k = 0; k < nseg; ++k) {
        const int64_t nb = seg_blocks(I, k);
        if (base + nb > nblk) break;
        const int64_t b0 = 8 * S.seg[k], b1 = 8 * S.seg[k + 1];
        const int64_t nr = b1 > b0 ? (b1 - b0 + run_bits - 1) / run_bits : 1;
        auto r_end = [&](int64_t r) { return b0 + (r + 1) * run_bits < b1 ? b0 + (r + 1) * run_bits : b1; };
        std::vector<St> X(nr), Y(nr), E(nr);
        std::vector<RunOut> C(nr);
        for (int64_t r = 0; r < nr; ++r) {
            X[r] = St{(int32_t)(b0 + r * run_bits), 0, 0};
            decode_run<false>(I, s, end, b1, X[r], r_end(r));
        }
        for (int i = 0; i < kRelax; ++i) {
            std::vector<St> Z(nr);
            for (int64_t r = 0; r < nr; ++r) {
                Z[r] = r ? X[r - 1] : St{(int32_t)b0, 0, 0};
                decode_run<false>(I, s, end, b1, Z[r], r_end(r));
            }
            X.swap(Z);
        }
        for (int64_t r = 0; r < nr; ++r) {
            E[r] = r ? X[r - 1] : St{(int32_t)b0, 0, 0};
            Y[r] = E[r];
            C[r] = decode_run<false>(I, s, end, b1, Y[r], r_end(r));
        }
        for (int64_t r = 1; r < nr; ++r) {
            if (same(Y[r - 1], X[r - 1])) continue;       // the true entry is the exit phase 2 started from
            E[r] = Y[r - 1];
            Y[r] = E[r];
            C[r] = decode_run<false>(I, s, end, b1, Y[r], r_end(r));
            ++*fixed;
        }
        int64_t first = 0;
        int dc[3] = {0, 0, 0};
        bool done = false;
        for (int64_t r = 0; r < nr; ++r) {
            St st = E[r];
            RunOut o = decode_run<true>(I, s, end, b1, st, r_end(r), coef.data() + base * 64, first, nb, dc);
            if (o.err && first < nb) status |= kCorrupt;
            done |= o.done != 0;
            first += C[r].blocks;
            for (int c = 0; c < 3; ++c) dc[c] += C[r].dc[c];
        }
        if (!done) status |= kCorrupt;
        base += nb;
    }
    return status;
}

int pixels(const Info &I, std::vector<int16_t> &coef, uint8_t *out) {
    const int64_t nblk = (int64_t)coef.size() / 64;
    std::vector<uint8_t> blocks(nblk * 128);
    for (int64_t b = 0; b < nblk; ++b) idct_islow(coef.data() + 64 * b, I.qt[I.mcu_comp[b % I.bpm]], blocks.data() + 128 * b);
    for (int y = 0; y < I.out_h; ++y)
        for (int x = 0; x < I.out_w; ++x) output_pixel(I, blocks.data(), y, x, out + 3 * ((int64_t)y * I.out_w + x));
    return 0;
}

}  // namespace

extern "C" {

// header of one image: info[0..7] = status, out_h, out_w, colour space, orientation, ncomp, restart interval, blocks per MCU
int host_header(const uint8_t *p, int64_t n, int *info) {
    static Info I;
    parse(p, n, I);
    const int v[8] = {I.status, I.out_h, I.out_w, I.cs, I.orient, I.ncomp, I.ri, I.bpm};
    memcpy(info, v, sizeof(v));
    return I.status;
}

// cv2.imdecode(IMREAD_COLOR) of one image into out (capacity `cap` bytes): status; shape in hw[2].  run_bits > 0 decodes the
// coefficients with the synchronising decode at that run size (fixed[0] = runs the walker decoded), else sequentially.
int host_decode(const uint8_t *p, int64_t n, int run_bits, int64_t cap, uint8_t *out, int *hw, int *fixed) {
    static Info I;
    hw[0] = hw[1] = 0;
    fixed[0] = 0;
    if (parse(p, n, I)) return I.status;
    if ((int64_t)I.out_h * I.out_w * 3 > cap) return kTooLarge;
    Scan S = split(p, n, I);
    std::vector<int16_t> coef;
    const int st = run_bits > 0 ? decode_coefs_sync(I, S, run_bits, coef, fixed) : decode_coefs(I, S, coef);
    if (st) return st;
    pixels(I, coef, out);
    hw[0] = I.out_h;
    hw[1] = I.out_w;
    return 0;
}

// the coefficients of both decodes (sequential into a, synchronising at run_bits into b; int16 [cap]); returns the block
// count, or -1 when the header or the scan split fails
int64_t host_coefs(const uint8_t *p, int64_t n, int run_bits, int64_t cap, int16_t *a, int16_t *b, int *fixed) {
    static Info I;
    if (parse(p, n, I)) return -1;
    Scan S = split(p, n, I);
    std::vector<int16_t> ca, cb;
    const int s1 = decode_coefs(I, S, ca), s2 = decode_coefs_sync(I, S, run_bits, cb, fixed);
    if (s1 != s2 || (int64_t)ca.size() > cap) return -1;
    memcpy(a, ca.data(), ca.size() * 2);
    memcpy(b, cb.data(), cb.size() * 2);
    return (int64_t)ca.size() / 64;
}

}  // extern "C"

#ifdef JPEG_HARNESS_MAIN
// Sanitizer build: decodes every file named on the command line at a 32-bit run size; exit status 0 unless a check fires.
#include <stdio.h>

int main(int argc, char **argv) {
    for (int a = 1; a < argc; ++a) {
        FILE *f = fopen(argv[a], "rb");
        if (!f) return 2;
        std::vector<uint8_t> b;
        int c;
        while ((c = fgetc(f)) != EOF) b.push_back((uint8_t)c);
        fclose(f);
        int info[8], hw[2], fixed[1];
        host_header(b.data(), (int64_t)b.size(), info);
        std::vector<uint8_t> out(3 * (size_t)(info[1] > 0 ? info[1] : 1) * (size_t)(info[2] > 0 ? info[2] : 1));
        host_decode(b.data(), (int64_t)b.size(), 32, (int64_t)out.size(), out.data(), hw, fixed);
    }
    return 0;
}
#endif
