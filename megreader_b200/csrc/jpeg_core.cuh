// Baseline JPEG decoding as cv2.imdecode(buf, cv2.IMREAD_COLOR) does it with libjpeg-turbo's defaults (JDCT_ISLOW, fancy
// upsampling, table-driven YCbCr -> BGR) and OpenCV's EXIF orientation, shared by the CUDA kernels (jpeg.cu) and by a host
// harness (tests/host_harness/jpeg_core_host.cpp).  Integer arithmetic only.
//
//   parse()          the markers up to SOS: quantisation and Huffman tables (libjpeg's maxcode / valoffset plus a 9-bit
//                    first-level table), frame and MCU geometry, restart interval, colour space, orientation, status
//   classify()       one byte of the entropy-coded data: data byte, stuffed zero, RSTn, or the marker that ends the scan
//   decode_run()     the Huffman decode of the symbols that start inside one run of bits of a restart segment, from a given
//                    state (bit position, block in MCU, zig-zag index); optionally writing coefficients
//   idct_islow()     jpeg_idct_islow of one block as libjpeg-turbo's x86 SIMD computes it (16-bit wraps and saturations)
//   output_pixel()   upsampling (h2v1 / h2v2 / h1v2 fancy where libjpeg-turbo applies it, box replication elsewhere),
//                    colour conversion and orientation of one output pixel
#pragma once
#include <stdint.h>

#ifndef __CUDACC__
#define __host__
#define __device__
#endif

namespace mr_jpeg {

// per-image status bits
enum Status { kBadHeader = 1, kUnsupportedProcess = 2, kUnsupportedComponents = 4, kTooLarge = 8, kCorrupt = 16, kBadOffsets = 32 };
enum ColorSpace { kGray = 0, kYCbCr = 1, kRGB = 2 };

constexpr int kMaxSide = 16384;
constexpr int kMaxBlocksInMCU = 10;
constexpr int kLookBits = 9;

struct Huff {
    int32_t maxcode[18];                 // libjpeg's derived table: largest code of each length, -1 if none (maxcode[17] sentinel)
    int32_t valoffset[18];               // symbol index = code + valoffset[length]
    uint16_t look[1 << kLookBits];       // first level: (length << 8) | symbol for codes of up to 9 bits, 0 otherwise
    uint8_t val[256];
};

struct Comp {
    int id, h, v, tq, td, ta;
    int lh, lv;                          // blocks of this component in one MCU of the scan (1 x 1 for a one-component scan)
    int first;                           // its first block in the MCU
    int dw, dh;                          // downsampled width and height
};

struct Info {
    int status;
    int h, w;                            // the frame
    int out_h, out_w;                    // after the orientation
    int ncomp, cs, orient, adobe, jfix;
    int hmax, vmax;
    int mcus_x, mcus_y, bpm;             // MCU grid of the scan and blocks per MCU
    int ri;                              // restart interval in MCUs (0: none)
    int64_t scan;                        // byte offset of the first entropy-coded byte (relative to the image's bytes)
    int nseg;                            // restart segments found in the scan
    int runs;                            // runs of the image's segments
    int64_t run_base;                    // its first run in the batch
    int64_t coef;                        // its first coefficient block in the workspace
    int64_t out;                         // its first output pixel
    Comp c[3];                           // in frame order
    int so[3];                           // the scan's order of the frame components
    int8_t mcu_comp[kMaxBlocksInMCU];
    int16_t qt[3][64];                   // per component, natural order (libjpeg's ISLOW_MULT_TYPE is short with SIMD)
    Huff dc[3], ac[3];                   // per component
};

__host__ __device__ constexpr int zigzag(int k) {
    constexpr int z[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                           41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                           30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};
    return z[k];
}

// ---------------------------------------------------------------- header

struct Reader {
    const uint8_t *p;
    int64_t n, i;
    __host__ __device__ int u8() { return i < n ? p[i++] : (i++, -1); }
    __host__ __device__ int u16() { const int a = u8(), b = u8(); return (a < 0 || b < 0) ? -1 : (a << 8) | b; }
};

// libjpeg's jpeg_make_d_derived_tbl; false for a table it refuses
__host__ __device__ inline bool make_huff(const uint8_t bits[17], const uint8_t *vals, int nvals, bool dc, Huff &t) {
    int size[257], code[257];
    int p = 0;
    for (int l = 1; l <= 16; ++l) {
        if (p + bits[l] > 256) return false;
        for (int i = 0; i < bits[l]; ++i) size[p++] = l;
    }
    size[p] = 0;
    if (p != nvals) return false;
    int c = 0, si = size[0];
    p = 0;
    while (size[p]) {
        while (size[p] == si) code[p++] = c++;
        if (c >= (1 << si)) return false;
        c <<= 1;
        ++si;
    }
    p = 0;
    for (int l = 1; l <= 16; ++l) {
        if (bits[l]) {
            t.valoffset[l] = p - code[p];
            p += bits[l];
            t.maxcode[l] = code[p - 1];
        } else {
            t.maxcode[l] = -1;
        }
    }
    t.valoffset[17] = 0;
    t.maxcode[17] = 0xFFFFF;
    for (int i = 0; i < (1 << kLookBits); ++i) t.look[i] = 0;
    for (int i = 0; i < 256; ++i) t.val[i] = i < nvals ? vals[i] : 0;
    p = 0;
    for (int l = 1; l <= kLookBits; ++l)
        for (int i = 0; i < bits[l]; ++i, ++p) {
            const int base = code[p] << (kLookBits - l);
            for (int j = 0; j < (1 << (kLookBits - l)); ++j) t.look[base + j] = (uint16_t)((l << 8) | vals[p]);
        }
    if (dc)
        for (int i = 0; i < nvals; ++i)
            if (vals[i] > 15) return false;
    return true;
}

// OpenCV's EXIF orientation from TIFF data t[0, tn) (a JPEG APP1 payload after "Exif\0\0", or a PNG eXIf chunk): IFD0 tag
// 0x0112, either byte order; 1 when absent
__host__ __device__ inline int tiff_orientation(const uint8_t *t, int64_t tn) {
    if (tn < 8) return 1;
    bool le;
    if (t[0] == 'I' && t[1] == 'I') le = true;
    else if (t[0] == 'M' && t[1] == 'M') le = false;
    else return 1;
    auto g16 = [&](int64_t o) -> int { return le ? t[o] | (t[o + 1] << 8) : (t[o] << 8) | t[o + 1]; };
    auto g32 = [&](int64_t o) -> int64_t {
        return le ? (int64_t)((uint32_t)t[o] | ((uint32_t)t[o + 1] << 8) | ((uint32_t)t[o + 2] << 16) | ((uint32_t)t[o + 3] << 24))
                  : (int64_t)(((uint32_t)t[o] << 24) | ((uint32_t)t[o + 1] << 16) | ((uint32_t)t[o + 2] << 8) | (uint32_t)t[o + 3]);
    };
    if (g16(2) != 42) return 1;
    const int64_t ifd = g32(4);
    if (ifd < 8 || ifd + 2 > tn) return 1;
    const int cnt = g16(ifd);
    for (int e = 0; e < cnt; ++e) {
        const int64_t o = ifd + 2 + 12 * (int64_t)e;
        if (o + 12 > tn) return 1;
        if (g16(o) == 0x0112) {
            const int v = g16(o + 8);
            return v >= 1 && v <= 8 ? v : 1;
        }
    }
    return 1;
}

// the first APP1 "Exif\0\0" segment's orientation
__host__ __device__ inline int exif_orientation(const uint8_t *d, int64_t n) {
    if (n < 14 || d[0] != 'E' || d[1] != 'x' || d[2] != 'i' || d[3] != 'f' || d[4] != 0 || d[5] != 0) return 1;
    return tiff_orientation(d + 6, n - 6);
}

__host__ __device__ inline int ceil_div_i(int a, int b) { return (a + b - 1) / b; }

// Walks the markers of one image to its first SOS and fills I; returns I.status.  The tables are located in a first walk
// and built after it, from their last definition before SOS.
__host__ __device__ inline int parse(const uint8_t *p, int64_t n, Info &I) {
    I.status = 0;
    I.orient = 1;
    I.adobe = -1;
    I.jfix = 0;
    I.ri = 0;
    I.nseg = 0;
    I.runs = 0;
    I.h = I.w = I.out_h = I.out_w = 0;
    I.ncomp = 0;
    I.scan = n;
    bool have_q[4] = {false, false, false, false}, have_h[2][4] = {{false, false, false, false}, {false, false, false, false}};
    bool frame = false, exif_seen = false;
    int fid[3] = {0, 0, 0}, fh[3], fv[3], ftq[3];
    Reader r{p, n, 0};
    if (r.u8() != 0xFF || r.u8() != 0xD8) return I.status = kBadHeader;
    int64_t dqt_at[4] = {-1, -1, -1, -1}, dht_at[2][4] = {{-1, -1, -1, -1}, {-1, -1, -1, -1}};
    for (;;) {
        int c = r.u8();
        while (c >= 0 && c != 0xFF) c = r.u8();          // garbage before a marker (libjpeg warns and skips it)
        while (c == 0xFF) c = r.u8();                     // fill bytes
        if (c < 0) return I.status = kBadHeader;
        if (c == 0xD8 || c == 0xD9 || (c >= 0xD0 && c <= 0xD7) || c == 0x01) {
            if (c == 0xD9) return I.status = kBadHeader;  // EOI before any scan
            continue;
        }
        const int len = r.u16();
        if (len < 2 || r.i + len - 2 > n) return I.status = kBadHeader;
        const int64_t seg = r.i, end = r.i + len - 2;
        if (c == 0xC0 || c == 0xC1) {
            if (frame) return I.status = kBadHeader;
            frame = true;
            const int prec = r.u8();
            I.h = r.u16();
            I.w = r.u16();
            const int nf = r.u8();
            if (prec != 8) return I.status = kUnsupportedProcess;
            if (I.h == 0) return I.status = kUnsupportedProcess;   // height in a DNL marker
            if (I.w == 0 || nf < 1 || end - seg != 6 + 3 * (int64_t)nf) return I.status = kBadHeader;
            if (nf != 1 && nf != 3) return I.status = kUnsupportedComponents;
            I.ncomp = nf;
            for (int i = 0; i < nf; ++i) {
                fid[i] = r.u8();
                const int hv = r.u8();
                fh[i] = hv >> 4;
                fv[i] = hv & 15;
                ftq[i] = r.u8();
                if (fh[i] < 1 || fh[i] > 4 || fv[i] < 1 || fv[i] > 4 || ftq[i] > 3) return I.status = kBadHeader;
            }
        } else if ((c >= 0xC2 && c <= 0xCF && c != 0xC4 && c != 0xC8 && c != 0xCC) || c == 0xDC) {
            return I.status = kUnsupportedProcess;        // progressive, lossless, hierarchical, arithmetic; DNL
        } else if (c == 0xC4) {
            while (r.i < end) {
                const int64_t at = r.i;
                const int tc = r.u8();
                if (tc < 0 || (tc >> 4) > 1 || (tc & 15) > 3) return I.status = kBadHeader;
                int cnt = 0;
                for (int l = 1; l <= 16; ++l) cnt += r.u8();
                if (cnt > 256 || r.i + cnt > end) return I.status = kBadHeader;
                r.i += cnt;
                dht_at[tc >> 4][tc & 15] = at;
                have_h[tc >> 4][tc & 15] = true;
            }
        } else if (c == 0xDB) {
            while (r.i < end) {
                const int64_t at = r.i;
                const int pq = r.u8();
                if (pq < 0 || (pq >> 4) > 1 || (pq & 15) > 3) return I.status = kBadHeader;
                r.i += (pq >> 4) ? 128 : 64;
                if (r.i > end) return I.status = kBadHeader;
                dqt_at[pq & 15] = at;
                have_q[pq & 15] = true;
            }
        } else if (c == 0xDD) {
            if (len != 4) return I.status = kBadHeader;
            I.ri = r.u16();
        } else if (c == 0xE0) {
            if (len - 2 >= 14 && p[seg] == 'J' && p[seg + 1] == 'F' && p[seg + 2] == 'I' && p[seg + 3] == 'F' && p[seg + 4] == 0)
                I.jfix = 1;
        } else if (c == 0xE1) {
            if (!exif_seen) I.orient = exif_orientation(p + seg, end - seg);
            exif_seen = true;
        } else if (c == 0xEE) {
            if (len - 2 >= 12 && p[seg] == 'A' && p[seg + 1] == 'd' && p[seg + 2] == 'o' && p[seg + 3] == 'b' && p[seg + 4] == 'e')
                I.adobe = p[seg + 11];
        } else if (c == 0xDA) {
            if (!frame) return I.status = kBadHeader;
            const int ns = r.u8();
            if (ns < 1 || ns > 4 || end - seg != 4 + 2 * (int64_t)ns) return I.status = kBadHeader;
            if (ns != I.ncomp) return I.status = kUnsupportedProcess;   // the frame is coded in more than one scan
            int order[3];
            for (int i = 0; i < ns; ++i) {
                const int cs = r.u8(), t = r.u8();
                int k = -1;
                for (int j = 0; j < I.ncomp; ++j)
                    if (fid[j] == cs) k = j;
                if (k < 0) return I.status = kBadHeader;
                for (int j = 0; j < i; ++j)
                    if (order[j] == k) return I.status = kBadHeader;
                order[i] = k;
                I.so[i] = k;
                Comp &C = I.c[k];
                C.id = cs; C.h = fh[k]; C.v = fv[k]; C.tq = ftq[k]; C.td = t >> 4; C.ta = t & 15;
                if (C.td > 3 || C.ta > 3 || !have_h[0][C.td] || !have_h[1][C.ta] || !have_q[C.tq]) return I.status = kBadHeader;
            }
            const int ss = r.u8(), se = r.u8(), a = r.u8();
            if (ss != 0 || se != 63 || a != 0) return I.status = kBadHeader;
            I.scan = end;
            break;
        }
        r.i = end;
    }
    // geometry: blocks of an MCU in scan order, components in frame order
    I.hmax = I.vmax = 1;
    for (int i = 0; i < I.ncomp; ++i) {
        I.hmax = I.c[i].h > I.hmax ? I.c[i].h : I.hmax;
        I.vmax = I.c[i].v > I.vmax ? I.c[i].v : I.vmax;
    }
    for (int i = 0; i < I.ncomp; ++i)
        if (I.hmax % I.c[i].h || I.vmax % I.c[i].v) return I.status = kUnsupportedComponents;   // fractional sampling
    if (I.ncomp == 1) {
        I.so[0] = 0;
        Comp &C = I.c[0];
        C.dw = ceil_div_i(I.w * C.h, I.hmax);
        C.dh = ceil_div_i(I.h * C.v, I.vmax);
        C.lh = C.lv = 1;
        C.first = 0;
        I.mcus_x = ceil_div_i(C.dw, 8);
        I.mcus_y = ceil_div_i(C.dh, 8);
        I.bpm = 1;
        I.mcu_comp[0] = 0;
    } else {
        I.mcus_x = ceil_div_i(I.w, 8 * I.hmax);
        I.mcus_y = ceil_div_i(I.h, 8 * I.vmax);
        I.bpm = 0;
        for (int j = 0; j < I.ncomp; ++j) {
            const int i = I.so[j];
            Comp &C = I.c[i];
            C.dw = ceil_div_i(I.w * C.h, I.hmax);
            C.dh = ceil_div_i(I.h * C.v, I.vmax);
            C.lh = C.h;
            C.lv = C.v;
            C.first = I.bpm;
            if (I.bpm + C.h * C.v > kMaxBlocksInMCU) return I.status = kBadHeader;
            for (int b = 0; b < C.h * C.v; ++b) I.mcu_comp[I.bpm++] = (int8_t)i;
        }
    }
    // colour space: libjpeg's default_decompress_parms, on the frame's component ids
    if (I.ncomp == 1) I.cs = kGray;
    else if (I.jfix) I.cs = kYCbCr;
    else if (I.adobe >= 0) I.cs = I.adobe == 0 ? kRGB : kYCbCr;
    else I.cs = (fid[0] == 'R' && fid[1] == 'G' && fid[2] == 'B') ? kRGB : kYCbCr;
    // tables of the scan's components
    for (int i = 0; i < I.ncomp; ++i) {
        Comp &C = I.c[i];
        Reader q{p, n, dqt_at[C.tq]};
        const int pq = q.u8() >> 4;
        for (int k = 0; k < 64; ++k) I.qt[i][zigzag(k)] = (int16_t)(pq ? q.u16() : q.u8());
        for (int cls = 0; cls < 2; ++cls) {
            Reader h{p, n, dht_at[cls][cls ? C.ta : C.td] + 1};
            uint8_t bits[17];
            bits[0] = 0;
            int cnt = 0;
            for (int l = 1; l <= 16; ++l) cnt += bits[l] = (uint8_t)h.u8();
            if (!make_huff(bits, p + h.i, cnt, cls == 0, cls ? I.ac[i] : I.dc[i])) return I.status = kBadHeader;
        }
    }
    const bool transpose = I.orient >= 5;
    I.out_h = transpose ? I.w : I.h;
    I.out_w = transpose ? I.h : I.w;
    return I.status;
}

// ---------------------------------------------------------------- entropy-coded data

enum ByteKind { kData = 0, kDrop = 1, kRst = 2, kEnd = 3 };

// Byte i of the scan bytes b[0, n): kData (one byte of the stream; for 0xFF 0x00 the 0xFF is the data byte), kDrop (a stuffed
// zero, fill 0xFF, or the code of an RSTn), kRst (0xFF of an RSTn: a new restart segment starts at the next data byte) or
// kEnd (0xFF of any other marker: the scan ends here).  The end of the bytes also ends the scan.
__host__ __device__ inline int classify(const uint8_t *b, int64_t n, int64_t i) {
    const int x = b[i];
    if (x == 0xFF) {
        const int y = i + 1 < n ? b[i + 1] : -1;
        if (y == 0xFF) return kDrop;                      // a run of 0xFF: only its last one counts
        if (y == 0x00) return kData;
        if (y >= 0xD0 && y <= 0xD7) return kRst;
        return y < 0 ? kDrop : kEnd;
    }
    if (i == 0) return kData;
    const int w = b[i - 1];
    if (w != 0xFF) return kData;
    return kDrop;                                         // a stuffed zero or the code byte of a marker
}

struct St {
    int32_t pos;                         // bit position in the image's unstuffed stream
    int16_t blk;                         // block within the MCU
    int16_t zz;                          // next zig-zag index (0: the DC symbol)
};
__host__ __device__ inline bool same(const St &a, const St &b) { return a.pos == b.pos && a.blk == b.blk && a.zz == b.zz; }

// 32 bits from bit position pos of the stream s[0, end) (zero past end)
__host__ __device__ inline uint32_t peek32(const uint8_t *s, int64_t end, int64_t pos) {
    const int64_t b = pos >> 3;
    uint64_t v = 0;
    for (int k = 0; k < 5; ++k) v = (v << 8) | (b + k < end ? s[b + k] : 0);
    return (uint32_t)(v >> (8 - (pos & 7)));
}

// one Huffman symbol at the top of w: returns (length << 8) | symbol, or 0 for an invalid code
__host__ __device__ inline int huff_decode(const Huff &t, uint32_t w) {
    const int f = t.look[w >> (32 - kLookBits)];
    if (f) return f;
    for (int l = kLookBits + 1; l <= 16; ++l) {
        const int32_t code = (int32_t)(w >> (32 - l));
        if (code <= t.maxcode[l]) return (l << 8) | t.val[(code + t.valoffset[l]) & 255];
    }
    return 0;
}

__host__ __device__ inline int extend(uint32_t v, int s) { return (int)v < (1 << (s - 1)) ? (int)v - (1 << s) + 1 : (int)v; }

struct RunOut {
    int blocks;                          // DC symbols decoded (blocks started)
    int dc[3];                           // sum of their DC differences per component
    int err;                             // an invalid code, a coefficient past 63, or bits past the segment's end
    int done;                            // WRITE: the segment's last block was completed
};

// Decodes the symbols that start before bit `stop` from state s (in place), within a segment ending at bit seg_end.  Without
// WRITE it only counts.  With WRITE, coef points at the segment's first block, `first` is the segment-relative index of the
// first block started in this run (blocks started in earlier runs), dc_base the DC predictions at that point, and decoding
// ends when block seg_blocks would start; coefficients go to coef in natural order (blocks zeroed beforehand).
template <bool WRITE>
__host__ __device__ inline RunOut decode_run(const Info &I, const uint8_t *s, int64_t end_byte, int64_t seg_end, St &st, int64_t stop,
                                             int16_t *coef = nullptr, int64_t first = 0, int64_t seg_blocks = 0, const int *dc_base = nullptr) {
    RunOut o{0, {0, 0, 0}, 0, 0};
    int64_t cur = first - (st.zz ? 1 : 0);               // the block being decoded (WRITE)
    int dcs[3] = {0, 0, 0};
    if (WRITE) {
        if (cur >= seg_blocks) return o;
        for (int c = 0; c < 3; ++c) dcs[c] = dc_base[c];
    }
    while (st.pos < stop) {
        if (WRITE && st.zz == 0 && first + o.blocks >= seg_blocks) break;
        const int comp = I.mcu_comp[st.blk];
        const uint32_t w = peek32(s, end_byte, st.pos);
        int nbits;
        if (st.zz == 0) {
            const int f = huff_decode(I.dc[comp], w);
            if (!f) { o.err = 1; st.pos += 16; st.zz = 1; continue; }
            const int l = f >> 8, sz = f & 15;
            nbits = l + sz;
            const int diff = sz ? extend((w << l) >> (32 - sz), sz) : 0;
            o.blocks++;
            o.dc[comp] += diff;
            if (WRITE) {
                cur = first + o.blocks - 1;
                dcs[comp] += diff;
                coef[cur * 64] = (int16_t)dcs[comp];
            }
            st.zz = 1;
        } else {
            const int f = huff_decode(I.ac[comp], w);
            if (!f) { o.err = 1; st.pos += 16; st.zz = 0; st.blk = (int16_t)((st.blk + 1) % I.bpm); continue; }
            const int l = f >> 8, rs = f & 255, r = rs >> 4, sz = rs & 15;
            nbits = l + sz;
            int k = st.zz;
            if (sz) {
                k += r;
                if (k > 63) { o.err = 1; k = 63; }
                else if (WRITE) coef[cur * 64 + zigzag(k)] = (int16_t)extend((w << l) >> (32 - sz), sz);
                k += 1;
            } else {
                k = r == 15 ? k + 16 : 64;
            }
            st.zz = (int16_t)k;
        }
        st.pos += nbits;
        if (st.pos > seg_end) o.err = 1;
        if (st.zz >= 64) {
            st.zz = 0;
            st.blk = (int16_t)(st.blk + 1 == I.bpm ? 0 : st.blk + 1);
            if (WRITE && cur + 1 == seg_blocks) o.done = 1;
        }
    }
    return o;
}

// ---------------------------------------------------------------- IDCT

// libjpeg-turbo's jsimd_idct_islow (the x86 SIMD form of jpeg_idct_islow that cv2 runs): in int16 [64] natural order,
// quantisation q [64] (ISLOW_MULT_TYPE short); out 8 x 8 samples (row stride 8).  Its arithmetic differs from the C form
// only where values leave 16 bits:
//   * dequantisation keeps the low 16 bits of coef * q (pmullw);
//   * in0 +- in4 and the odd part's z3 = in7 + in3, z4 = in5 + in1 are 16-bit sums (paddw, wrapping); every product
//     and the other sums are 32-bit (pmaddwd with the constant pairs below, equal to the C form's terms);
//   * pass 1 stores its descaled results saturated to int16 (packssdw), and when rows 1..7 of the whole block are zero
//     it stores in0 << PASS1_BITS in 16 bits (psllw, wrapping) instead;
//   * pass 2 saturates its descaled results to int8 (packssdw, packsswb) and adds CENTERJSAMPLE, where the C form masks
//     with RANGE_MASK.
__host__ __device__ inline void idct_islow(const int16_t *in, const int16_t *q, uint8_t *out) {
    constexpr int CB = 13, P1 = 2;
    constexpr int32_t F0298 = 2446, F0390 = 3196, F0541 = 4433, F0765 = 6270, F0899 = 7373, F1175 = 9633, F1501 = 12299, F1847 = 15137,
                      F1961 = 16069, F2053 = 16819, F2562 = 20995, F3072 = 25172;
    auto w16 = [](int32_t x) -> int32_t { return (int32_t)(int16_t)(uint16_t)(uint32_t)x; };
    auto s16 = [](int32_t x) -> int32_t { return x < -32768 ? -32768 : x > 32767 ? 32767 : x; };
    // one 1-D pass over v[8] (int16 values) -> the 8 outputs before descaling
    auto pass = [&](const int32_t *v, int32_t *o) {
        const int32_t z2 = v[2], z3 = v[6];
        const int32_t tmp3 = z2 * (F0541 + F0765) + z3 * F0541;
        const int32_t tmp2 = z2 * F0541 + z3 * (F0541 - F1847);
        const int32_t tmp0 = w16(v[0] + v[4]) * (1 << CB);
        const int32_t tmp1 = w16(v[0] - v[4]) * (1 << CB);
        const int32_t t10 = tmp0 + tmp3, t13 = tmp0 - tmp3, t11 = tmp1 + tmp2, t12 = tmp1 - tmp2;
        const int32_t a0 = v[7], a1 = v[5], a2 = v[3], a3 = v[1];
        const int32_t y3 = w16(a0 + a2), y4 = w16(a1 + a3);
        const int32_t zz3 = y3 * (F1175 - F1961) + y4 * F1175;
        const int32_t zz4 = y3 * F1175 + y4 * (F1175 - F0390);
        const int32_t o0 = a0 * (F0298 - F0899) + a3 * -F0899 + zz3;
        const int32_t o1 = a1 * (F2053 - F2562) + a2 * -F2562 + zz4;
        const int32_t o2 = a1 * -F2562 + a2 * (F3072 - F2562) + zz3;
        const int32_t o3 = a0 * -F0899 + a3 * (F1501 - F0899) + zz4;
        o[0] = t10 + o3; o[7] = t10 - o3;
        o[1] = t11 + o2; o[6] = t11 - o2;
        o[2] = t12 + o1; o[5] = t12 - o1;
        o[3] = t13 + o0; o[4] = t13 - o0;
    };
    int32_t ws[64];
    bool ac_zero = true;
    for (int i = 8; i < 64; ++i) ac_zero &= in[i] == 0;
    for (int c = 0; c < 8; ++c) {
        if (ac_zero) {
            const int32_t dc = w16(w16((int32_t)in[c] * q[c]) * (1 << P1));
            for (int r = 0; r < 8; ++r) ws[8 * r + c] = dc;
            continue;
        }
        int32_t v[8], o[8];
        for (int r = 0; r < 8; ++r) v[r] = w16((int32_t)in[8 * r + c] * q[8 * r + c]);
        pass(v, o);
        constexpr int sh = CB - P1;
        for (int r = 0; r < 8; ++r) ws[8 * r + c] = s16((o[r] + (1 << (sh - 1))) >> sh);
    }
    for (int r = 0; r < 8; ++r) {
        int32_t o[8];
        pass(ws + 8 * r, o);
        constexpr int sh = CB + P1 + 3;
        for (int c = 0; c < 8; ++c) {
            const int32_t x = (o[c] + (1 << (sh - 1))) >> sh;
            out[8 * r + c] = (uint8_t)((x < -128 ? -128 : x > 127 ? 127 : x) + 128);
        }
    }
}

// ---------------------------------------------------------------- upsampling, colour, orientation

// Sample (y, x) of component i's plane; planes hold the image's blocks in decode order, 128 bytes per block with the 64
// samples first
__host__ __device__ inline int plane_at(const Info &I, const uint8_t *blocks, int i, int y, int x) {
    const Comp &C = I.c[i];
    const int by = y >> 3, bx = x >> 3;
    const int64_t mcu = (int64_t)(by / C.lv) * I.mcus_x + bx / C.lh;
    const int64_t b = mcu * I.bpm + C.first + (by % C.lv) * C.lh + bx % C.lh;
    return blocks[b * 128 + (y & 7) * 8 + (x & 7)];
}

// component i upsampled to full resolution at (y, x), as libjpeg-turbo's jdsample.c chooses and computes it
__host__ __device__ inline int upsampled(const Info &I, const uint8_t *blocks, int i, int y, int x) {
    const Comp &C = I.c[i];
    const int rh = I.hmax / C.h, rv = I.vmax / C.v;
    if (rh == 1 && rv == 1) return plane_at(I, blocks, i, y, x);
    auto P = [&](int yy, int xx) { return plane_at(I, blocks, i, yy, xx); };
    if (rh == 2 && rv == 1 && C.dw > 2) {
        const int c = x >> 1, v3 = 3 * P(y, c);
        if (x & 1) return c == C.dw - 1 ? P(y, c) : (v3 + P(y, c + 1) + 2) >> 2;
        return c == 0 ? P(y, c) : (v3 + P(y, c - 1) + 1) >> 2;
    }
    if (rh == 1 && rv == 2) {
        const int r = y >> 1, f = (y & 1) ? (r + 1 < C.dh ? r + 1 : r) : (r > 0 ? r - 1 : 0);
        return (3 * P(r, x) + P(f, x) + ((y & 1) ? 2 : 1)) >> 2;
    }
    if (rh == 2 && rv == 2 && C.dw > 2) {
        const int r = y >> 1, f = (y & 1) ? (r + 1 < C.dh ? r + 1 : r) : (r > 0 ? r - 1 : 0);
        const int c = x >> 1;
        auto cs = [&](int cc) { return 3 * P(r, cc) + P(f, cc); };
        const int t = cs(c);
        if (x & 1) return c == C.dw - 1 ? (t * 4 + 7) >> 4 : (t * 3 + cs(c + 1) + 7) >> 4;
        return c == 0 ? (t * 4 + 8) >> 4 : (t * 3 + cs(c - 1) + 8) >> 4;
    }
    return P(y / rv, x / rh);
}

// source (sy, sx) of output pixel (y, x) under EXIF orientation o of an h x w frame, as OpenCV's ApplyExifOrientation
__host__ __device__ inline void orient_source(int o, int h, int w, int y, int x, int &sy, int &sx) {
    switch (o) {
    case 2: sy = y; sx = w - 1 - x; break;
    case 3: sy = h - 1 - y; sx = w - 1 - x; break;
    case 4: sy = h - 1 - y; sx = x; break;
    case 5: sy = x; sx = y; break;
    case 6: sy = h - 1 - x; sx = y; break;
    case 7: sy = h - 1 - x; sx = w - 1 - y; break;
    case 8: sy = x; sx = w - 1 - y; break;
    default: sy = y; sx = x; break;
    }
}

__host__ __device__ inline uint8_t clamp255(int v) { return (uint8_t)(v < 0 ? 0 : v > 255 ? 255 : v); }

// output pixel (y, x) as B, G, R
__host__ __device__ inline void output_pixel(const Info &I, const uint8_t *blocks, int y, int x, uint8_t *bgr) {
    int sy, sx;
    orient_source(I.orient, I.h, I.w, y, x, sy, sx);
    if (I.cs == kGray) {
        bgr[0] = bgr[1] = bgr[2] = (uint8_t)upsampled(I, blocks, 0, sy, sx);
        return;
    }
    const int a = upsampled(I, blocks, 0, sy, sx), b = upsampled(I, blocks, 1, sy, sx), c = upsampled(I, blocks, 2, sy, sx);
    if (I.cs == kRGB) {
        bgr[0] = (uint8_t)c; bgr[1] = (uint8_t)b; bgr[2] = (uint8_t)a;
        return;
    }
    // jdcolor.c's build_ycc_rgb_table with SCALEBITS 16
    constexpr int64_t half = (int64_t)1 << 15;
    const int cb = b - 128, cr = c - 128;
    const int r_ = (int)((91881 * (int64_t)cr + half) >> 16);
    const int b_ = (int)((116130 * (int64_t)cb + half) >> 16);
    const int g_ = (int)((-46802 * (int64_t)cr + (-22554 * (int64_t)cb + half)) >> 16);
    bgr[0] = clamp255(a + b_);
    bgr[1] = clamp255(a + g_);
    bgr[2] = clamp255(a + r_);
}

}  // namespace mr_jpeg
