// Host-side harness: runs the PRODUCT's PNG routines (megreader_b200/csrc/png_core.cuh, the code the CUDA kernels in png.cu
// execute) on the CPU, so that tests can compare them with cv2.imdecode without a GPU.  Built on demand with g++.
#include <stdlib.h>
#include <string.h>

#include <vector>

#include "png_core.cuh"

using namespace mr_png;

namespace {

uint32_t g_tab[256];

void init_tab() {
    for (uint32_t i = 0; i < 256; ++i) g_tab[i] = crc_table_entry(i);
}

// the first IDAT run's payloads, CRCs checked (each chunk's CRC formed from two parts and crc_combine, as the kernel
// combines its threads' parts); false on a CRC error
bool gather(const uint8_t *p, const Info &I, std::vector<uint8_t> &z) {
    int64_t i = I.idat;
    while (be32(p + i + 4) == kIDAT) {
        const int64_t len = be32(p + i);
        const uint8_t *t = p + i + 4;
        const int64_t cut = (len * 5) / 7;
        const uint32_t a = crc_update(g_tab, 0, t, 4 + cut), b = crc_update(g_tab, 0, t + 4 + cut, len - cut);
        if (crc_combine(a, b, len - cut) != be32(t + 4 + len)) return false;
        z.insert(z.end(), t + 4, t + 4 + len);
        i += 12 + len;
    }
    return true;
}

struct CopySink {                        // the serial inflate: matches copied at once
    uint8_t *out;
    void operator()(int64_t dst, int dist, int len) {
        for (int k = 0; k < len; ++k) out[dst + k] = out[dst + k - dist];
    }
};

struct RecordSink {                      // the kernels' form: matches recorded
    std::vector<int64_t> dst;
    std::vector<int> dist, len;
    void operator()(int64_t d, int s, int l) { dst.push_back(d); dist.push_back(s); len.push_back(l); }
};

// the kernels' resolution of the recorded matches: src[b] = b - dist inside a match, then src[b] = src[src[b]] in rounds
// until nothing changes, then every match byte from its literal source
int resolve(const RecordSink &R, uint8_t *out, int64_t n) {
    std::vector<int64_t> src(n);
    for (int64_t b = 0; b < n; ++b) src[b] = b;
    for (size_t m = 0; m < R.dst.size(); ++m)
        for (int k = 0; k < R.len[m]; ++k) src[R.dst[m] + k] = R.dst[m] + k - R.dist[m];
    int rounds = 0;
    for (bool changed = true; changed; ++rounds) {
        changed = false;
        std::vector<int64_t> next(src);
        for (int64_t b = 0; b < n; ++b)
            if (src[src[b]] != src[b]) { next[b] = src[src[b]]; changed = true; }
        src.swap(next);
    }
    for (int64_t b = 0; b < n; ++b) out[b] = out[src[b]];
    return rounds;
}

}  // namespace

extern "C" {

// header of one image: info[0..7] = status, out_h, out_w, colour type, bit depth, interlace, orientation, palette entries
int host_header(const uint8_t *p, int64_t n, int *info) {
    static Info I;
    init_tab();
    parse(p, n, g_tab, I);
    const int v[8] = {I.status, I.out_h, I.out_w, I.ctype, I.depth, I.interlace, I.orient, I.npal};
    memcpy(info, v, sizeof(v));
    return I.status;
}

// cv2.imdecode(IMREAD_COLOR) of one image into out (capacity `cap` bytes): status; shape in hw[2].  jump != 0 resolves the
// matches as the kernels do (recorded, then pointer jumping; rounds[0] = rounds taken), else the inflate copies them.
int host_decode(const uint8_t *p, int64_t n, int jump, int64_t cap, uint8_t *out, int *hw, int *rounds) {
    static Info I;
    static Tables T;
    init_tab();
    hw[0] = hw[1] = 0;
    rounds[0] = 0;
    if (parse(p, n, g_tab, I)) return I.status;
    if ((int64_t)I.out_h * I.out_w * 3 > cap) return kTooLarge;
    std::vector<uint8_t> z;
    if (!gather(p, I, z)) return kBadHeader;
    const int64_t raw = I.poff[7];
    std::vector<uint8_t> d(raw + 1);
    InflateResult r;
    if (jump) {
        RecordSink S;
        r = inflate(z.data(), (int64_t)z.size(), d.data(), I, I.split, T, S);
        if (r.status) return r.status;
        rounds[0] = resolve(S, d.data(), r.written);
    } else {
        CopySink S{d.data()};
        r = inflate(z.data(), (int64_t)z.size(), d.data(), I, I.split, T, S);
        if (r.status) return r.status;
    }
    if (r.check && adler32(d.data(), raw) != r.adler) return kCorrupt;
    for (int q = 0; q < I.npass; ++q) {
        if (!I.pw[q]) continue;
        for (int y = 0; y < I.ph[q]; ++y) {
            uint8_t *row = d.data() + I.poff[q] + (int64_t)y * (I.rb[q] + 1) + 1;
            if (!unfilter_row(row, y ? row - I.rb[q] - 1 : nullptr, I.rb[q], I.fbpp)) return kCorrupt;
        }
    }
    for (int y = 0; y < I.out_h; ++y)
        for (int x = 0; x < I.out_w; ++x) output_pixel(I, d.data(), y, x, out + 3 * ((int64_t)y * I.out_w + x));
    hw[0] = I.out_h;
    hw[1] = I.out_w;
    return 0;
}

}  // extern "C"

#ifdef PNG_HARNESS_MAIN
// Sanitizer build: decodes every file named on the command line both ways; exit status 0 unless a check fires.
#include <stdio.h>

int main(int argc, char **argv) {
    for (int a = 1; a < argc; ++a) {
        FILE *f = fopen(argv[a], "rb");
        if (!f) return 2;
        std::vector<uint8_t> b;
        int c;
        while ((c = fgetc(f)) != EOF) b.push_back((uint8_t)c);
        fclose(f);
        int info[8], hw[2], rounds[1];
        host_header(b.data(), (int64_t)b.size(), info);
        std::vector<uint8_t> out(3 * (size_t)(info[1] > 0 ? info[1] : 1) * (size_t)(info[2] > 0 ? info[2] : 1));
        for (int j = 0; j < 2; ++j) host_decode(b.data(), (int64_t)b.size(), j, (int64_t)out.size(), out.data(), hw, rounds);
    }
    return 0;
}
#endif
