// PNG decoding as cv2.imdecode(buf, cv2.IMREAD_COLOR) does it with libpng 1.6 and zlib, shared by the CUDA kernels (png.cu)
// and by a host harness (tests/host_harness/png_core_host.cpp).  Integer arithmetic only.
//
//   parse()          signature, IHDR, the chunk walk to IEND (PLTE, eXIf, the first run of IDAT chunks, acTL / fcTL order),
//                    the CRCs of IHDR, PLTE and eXIf, the zlib header; geometry of the (Adam7) passes; status
//   crc32 helpers    table-driven CRC-32 and zlib's crc32_combine (GF(2) multiplication by x^(8 n) modulo the polynomial)
//   inflate()        RFC 1951 over the gathered zlib stream: literals written, matches handed to a sink (the kernels record
//                    them and resolve them in parallel; the harness copies them); libpng's end-of-data rules
//   unfilter_byte()  the five row filters on one byte
//   output_pixel()   unpacking, palette, grey replication, alpha and 16-bit reduction, BGR, and the eXIf orientation
#pragma once
#include <stdint.h>
#include <string.h>

#include "jpeg_core.cuh"   // tiff_orientation, orient_source: shared with the JPEG decoder

namespace mr_png {

// per-image status bits, as mr_jpeg's
enum Status { kBadHeader = 1, kUnsupportedProcess = 2, kTooLarge = 8, kCorrupt = 16, kBadOffsets = 32 };

constexpr int kMaxSide = 16384;
constexpr int kFast = 11;                // first-level Huffman table bits (longer codes are walked bit by bit)

__host__ __device__ inline bool has_signature(const uint8_t *p, int64_t n) {
    return n >= 8 && p[0] == 0x89 && p[1] == 'P' && p[2] == 'N' && p[3] == 'G' && p[4] == 13 && p[5] == 10 && p[6] == 26 && p[7] == 10;
}

// ---------------------------------------------------------------- CRC-32

__host__ __device__ inline uint32_t crc_table_entry(uint32_t i) {
    uint32_t c = i;
    for (int k = 0; k < 8; ++k) c = c & 1 ? 0xEDB88320u ^ (c >> 1) : c >> 1;
    return c;
}

// the running (pre- and post-inverted) CRC register over p[0, n)
__host__ __device__ inline uint32_t crc_update(const uint32_t *tab, uint32_t c, const uint8_t *p, int64_t n) {
    c = ~c;
    for (int64_t i = 0; i < n; ++i) c = tab[(c ^ p[i]) & 255] ^ (c >> 8);
    return ~c;
}

// a * b modulo the CRC polynomial, bit-reflected (zlib's multmodp)
__host__ __device__ inline uint32_t crc_multmodp(uint32_t a, uint32_t b) {
    uint32_t m = 1u << 31, p = 0;
    for (;;) {
        if (a & m) {
            p ^= b;
            if ((a & (m - 1)) == 0) break;
        }
        m >>= 1;
        b = b & 1 ? (b >> 1) ^ 0xEDB88320u : b >> 1;
    }
    return p;
}

// CRC of A || B from crc(A), crc(B) and the length of B in bytes (zlib's crc32_combine)
__host__ __device__ inline uint32_t crc_combine(uint32_t c1, uint32_t c2, int64_t n2) {
    uint32_t p = 1u << 31;               // x^0
    uint32_t q = 1u << 30;               // x^1, squared to x^8: one byte
    for (int k = 0; k < 3; ++k) q = crc_multmodp(q, q);
    for (uint64_t n = (uint64_t)n2; n; n >>= 1) {
        if (n & 1) p = crc_multmodp(q, p);
        q = crc_multmodp(q, q);
    }
    return crc_multmodp(p, c1) ^ c2;
}

__host__ __device__ inline uint32_t be32(const uint8_t *p) { return ((uint32_t)p[0] << 24) | ((uint32_t)p[1] << 16) | ((uint32_t)p[2] << 8) | p[3]; }

__host__ __device__ inline uint32_t chunk_type(const uint8_t *p) { return be32(p); }
constexpr uint32_t tag(char a, char b, char c, char d) { return ((uint32_t)a << 24) | ((uint32_t)b << 16) | ((uint32_t)c << 8) | (uint32_t)d; }
constexpr uint32_t kIHDR = tag('I', 'H', 'D', 'R'), kPLTE = tag('P', 'L', 'T', 'E'), kIDAT = tag('I', 'D', 'A', 'T'), kIEND = tag('I', 'E', 'N', 'D'),
                   kEXIF = tag('e', 'X', 'I', 'f'), kACTL = tag('a', 'c', 'T', 'L'), kFCTL = tag('f', 'c', 'T', 'L');

// ---------------------------------------------------------------- header

struct Info {
    int status;
    int w, h;                            // IHDR
    int out_h, out_w;                    // after the orientation
    int depth, ctype, interlace;
    int channels, bits;                  // samples and bits per pixel
    int fbpp;                            // bytes per pixel of the row filters (at least 1)
    int orient;
    int npal;
    int npass;                           // 1, or 7 with Adam7
    int pw[7], ph[7];                    // pass sizes (0 x 0 for an empty pass)
    int64_t rb[7];                       // bytes per pass row, without the filter byte
    int64_t poff[8];                     // each pass's first filter byte in the inflated data; poff[npass] = raw
    int64_t idat;                        // the first IDAT chunk's length field (relative to the image's bytes)
    int64_t zbytes;                      // payload bytes of the first run of IDAT chunks
    int split;                           // an IDAT chunk after the first run (the data after the interruption is not read)
    // batch layout (kernels)
    int64_t z;                           // the image's first byte of the gathered stream
    int64_t raw_base;                    // its first inflated byte
    int64_t out;                         // its first output pixel
    int nrec;                            // matches recorded by the inflate
    int check;                           // the stream ended without data past the rows: its Adler-32 is checked
    uint32_t adler;                      // the stream's Adler-32
    uint8_t pal[256 * 3];
};

__host__ __device__ inline bool valid_depth(int ctype, int depth) {
    switch (ctype) {
    case 0: return depth == 1 || depth == 2 || depth == 4 || depth == 8 || depth == 16;
    case 3: return depth == 1 || depth == 2 || depth == 4 || depth == 8;
    case 2: case 4: case 6: return depth == 8 || depth == 16;
    default: return false;
    }
}

// Adam7: origin and step of pass p
__host__ __device__ inline void adam7(int p, int &x0, int &y0, int &dx, int &dy) {
    const int X0[7] = {0, 4, 0, 2, 0, 1, 0}, Y0[7] = {0, 0, 4, 0, 2, 0, 1}, DX[7] = {8, 8, 4, 4, 2, 2, 1}, DY[7] = {8, 8, 8, 4, 4, 2, 2};
    x0 = X0[p]; y0 = Y0[p]; dx = DX[p]; dy = DY[p];
}

__host__ __device__ inline void geometry(Info &I) {
    I.npass = I.interlace ? 7 : 1;
    int64_t o = 0;
    for (int p = 0; p < 7; ++p) {
        I.pw[p] = I.ph[p] = 0;
        I.rb[p] = 0;
        I.poff[p] = o;
        if (p >= I.npass) continue;
        int x0 = 0, y0 = 0, dx = 1, dy = 1;
        if (I.interlace) adam7(p, x0, y0, dx, dy);
        const int pw = I.w > x0 ? (I.w - x0 + dx - 1) / dx : 0, ph = I.h > y0 ? (I.h - y0 + dy - 1) / dy : 0;
        if (pw == 0 || ph == 0) continue;
        I.pw[p] = pw;
        I.ph[p] = ph;
        I.rb[p] = ((int64_t)pw * I.bits + 7) / 8;
        o += (int64_t)ph * (I.rb[p] + 1);
    }
    I.poff[7] = o;
    for (int p = I.npass; p < 8; ++p) I.poff[p] = o;
}

__host__ __device__ inline bool chunk_name_ok(const uint8_t *t) {
    for (int k = 0; k < 4; ++k) {
        const int c = t[k];
        if (!((c >= 'A' && c <= 'Z') || (c >= 'a' && c <= 'z'))) return false;
    }
    return true;
}

// Walks the chunks of one image to IEND and fills I (the first IDAT run's place and size, the palette, the orientation);
// returns I.status.  IDAT CRCs are checked where the payload is gathered (png.cu, the harness), the others here.
__host__ __device__ inline int parse(const uint8_t *p, int64_t n, const uint32_t *crc_tab, Info &I) {
    I.status = 0;
    I.w = I.h = I.out_h = I.out_w = 0;
    I.orient = 1;
    I.npal = 0;
    I.npass = 0;
    I.idat = -1;
    I.zbytes = 0;
    I.split = 0;
    I.nrec = 0;
    I.check = 0;
    I.adler = 0;
    for (int k = 0; k < 8; ++k) I.poff[k] = 0;
    if (!has_signature(p, n)) return I.status = kBadHeader;
    int64_t i = 8;
    bool ihdr = false, plte = false, exif = false, actl = false, fctl_before = false, run_done = false;
    for (int k = 0;; ++k) {
        if (i + 8 > n) return I.status = kBadHeader;               // no IEND: the input is incomplete
        const uint32_t len = be32(p + i);
        const uint8_t *t = p + i + 4;
        if (len > 0x7FFFFFFFu || !chunk_name_ok(t)) return I.status = kBadHeader;
        if (i + 12 + (int64_t)len > n) return I.status = kBadHeader;
        const uint32_t ty = chunk_type(t);
        const uint8_t *d = t + 4;
        // the CRCs libpng acts on here: IHDR and PLTE (an error), eXIf (the chunk is dropped); IEND's and other ancillary
        // chunks' only warn
        const bool crc_ok = !(ty == kIHDR || ty == kPLTE || ty == kEXIF) || crc_update(crc_tab, 0, t, 4 + (int64_t)len) == be32(d + len);
        if (k == 0 && ty != kIHDR) return I.status = kBadHeader;
        if (ty != kIDAT && I.idat >= 0) run_done = true;
        if (ty == kIHDR) {
            if (k != 0 || len != 13 || !crc_ok) return I.status = kBadHeader;
            const uint32_t w = be32(d), h = be32(d + 4);
            I.depth = d[8];
            I.ctype = d[9];
            I.interlace = d[12];
            if (w == 0 || h == 0 || w > 0x7FFFFFFFu || h > 0x7FFFFFFFu || !valid_depth(I.ctype, I.depth) || d[10] != 0 || d[11] != 0 || d[12] > 1)
                return I.status = kBadHeader;
            if (w > (uint32_t)kMaxSide || h > (uint32_t)kMaxSide) I.status = kTooLarge;   // finishes the walk: a malformed file stays 1
            I.w = w > (uint32_t)kMaxSide ? kMaxSide : (int)w;
            I.h = h > (uint32_t)kMaxSide ? kMaxSide : (int)h;
            I.channels = I.ctype == 2 ? 3 : I.ctype == 4 ? 2 : I.ctype == 6 ? 4 : 1;
            I.bits = I.channels * I.depth;
            I.fbpp = I.bits >= 8 ? I.bits / 8 : 1;
            ihdr = true;
        } else if (ty == kPLTE) {
            if (plte || I.idat >= 0 || !crc_ok) return I.status = kBadHeader;
            plte = true;
            if (I.ctype == 3) {
                if (len % 3 || len == 0 || len > 768) return I.status = kBadHeader;
                int np = (int)(len / 3);
                if (np > (1 << I.depth)) np = 1 << I.depth;          // libpng keeps the entries the bit depth can index
                I.npal = np;
                for (int e = 0; e < 3 * np; ++e) I.pal[e] = d[e];
            }
        } else if (ty == kIDAT) {
            if (I.ctype == 3 && !plte) return I.status = kBadHeader;
            if (I.idat < 0) {
                I.idat = i;
                if (actl && !fctl_before) I.status |= kUnsupportedProcess;   // the IDAT image is not the first frame
            }
            if (run_done) I.split = 1;
            else I.zbytes += len;
        } else if (ty == kIEND) {
            break;
        } else if (ty == kEXIF) {
            if (!exif && crc_ok) {
                exif = true;
                I.orient = mr_jpeg::tiff_orientation(d, len);
            }
        } else if (ty == kACTL) {
            if (I.idat < 0) actl = true;
        } else if (ty == kFCTL) {
            if (I.idat < 0) fctl_before = true;
        } else if (!(t[0] & 0x20)) {
            return I.status = kBadHeader;                            // an unknown critical chunk
        }
        i += 12 + (int64_t)len;
    }
    if (!ihdr || I.idat < 0) return I.status = kBadHeader;
    if (I.status) return I.status;
    geometry(I);
    const bool tr = I.orient >= 5;
    I.out_h = tr ? I.w : I.h;
    I.out_w = tr ? I.h : I.w;
    return I.status;
}

// ---------------------------------------------------------------- inflate

struct Huff {
    uint16_t fast[1 << kFast];           // (length << 9) | symbol for codes of up to kFast bits, 0 otherwise
    int16_t count[16];                   // codes per length
    uint16_t sym[288];                   // symbols in canonical order (at most 288 litlen, 32 distance codes)
};

struct Tables {
    Huff lit, dist;
    uint8_t lens[320];                   // code lengths of a dynamic block (or the fixed ones)
};

__host__ __device__ inline uint32_t bitrev(uint32_t c, int l) {
    uint32_t r = 0;
    for (int k = 0; k < l; ++k) { r = (r << 1) | (c & 1); c >>= 1; }
    return r;
}

// zlib's inflate_table rules: -1 over-subscribed or an incomplete set (allowed only for one code of length 1 when
// allow_single; a table with no codes at all is accepted and fails on use), 0 otherwise
__host__ __device__ inline int build(const uint8_t *len, int n, Huff &h, bool allow_single) {
    for (int l = 0; l < 16; ++l) h.count[l] = 0;
    for (int s = 0; s < n; ++s) h.count[len[s]]++;
    int max = 0;
    for (int l = 1; l < 16; ++l)
        if (h.count[l]) max = l;
    for (int k = 0; k < (1 << kFast); ++k) h.fast[k] = 0;
    if (max == 0) { h.count[0] = (int16_t)n; return 0; }
    int left = 1;
    for (int l = 1; l < 16; ++l) {
        left <<= 1;
        left -= h.count[l];
        if (left < 0) return -1;
    }
    if (left > 0 && !(allow_single && max == 1)) return -1;
    int offs[16];
    offs[1] = 0;
    for (int l = 1; l < 15; ++l) offs[l + 1] = offs[l] + h.count[l];
    for (int s = 0; s < n; ++s)
        if (len[s]) h.sym[offs[len[s]]++] = (uint16_t)s;
    uint32_t code = 0;
    int k = 0;
    for (int l = 1; l <= kFast; ++l) {
        for (int j = 0; j < h.count[l]; ++j, ++k, ++code) {
            const uint32_t r = bitrev(code, l);
            for (uint32_t f = r; f < (1u << kFast); f += 1u << l) h.fast[f] = (uint16_t)((l << 9) | h.sym[k]);
        }
        code <<= 1;
    }
    return 0;
}

struct Bits {
    const uint8_t *z;
    int64_t n, i;                        // input bytes and the next byte to load
    uint64_t b;
    int c;                               // bits in b
    __host__ __device__ void fill() {
        while (c <= 56 && i < n) {
            if (c <= 32 && i + 4 <= n && !((uintptr_t)(z + i) & 3)) {   // an aligned word at a time where it can
                uint32_t v;
#ifdef __CUDA_ARCH__
                v = *(const uint32_t *)(z + i);
#else
                memcpy(&v, z + i, 4);
#endif
                b |= (uint64_t)v << c;
                i += 4;
                c += 32;
            } else {
                b |= (uint64_t)z[i++] << c;
                c += 8;
            }
        }
    }
    __host__ __device__ bool need(int k) {
        if (c < k) fill();
        return c >= k;
    }
    __host__ __device__ uint32_t take(int k) {
        const uint32_t v = (uint32_t)(b & ((1ull << k) - 1));
        b >>= k;
        c -= k;
        return v;
    }
};

// one symbol, or -1 for an invalid code, -2 for the end of the input
__host__ __device__ inline int decode_sym(Bits &s, const Huff &h) {
    s.fill();
    const uint16_t f = h.fast[s.b & ((1u << kFast) - 1)];
    if (f) {
        const int l = f >> 9;
        if (l > s.c) return -2;
        s.take(l);
        return f & 511;
    }
    int code = 0, first = 0, index = 0;
    for (int l = 1; l < 16; ++l) {
        if (l > s.c) return -2;
        code |= (int)((s.b >> (l - 1)) & 1);
        const int cnt = h.count[l];
        if (code - cnt < first) {
            s.take(l);
            return h.sym[index + (code - first)];
        }
        index += cnt;
        first += cnt;
        first <<= 1;
        code <<= 1;
    }
    return -1;
}

struct InflateResult {
    int status;                          // 0, kCorrupt, or kBadHeader when the IDAT run was interrupted and ran short
    int64_t written;                     // bytes written (<= raw)
    int check;                           // the stream ended with no byte past raw: adler is to be checked
    uint32_t adler;                      // the stream's stored Adler-32
};

// Inflates the zlib stream z[0, zn) into out[0, raw), raw = I.poff[7] the bytes of I's rows: literals are stored, matches
// go to sink(dst, dist, len) clipped to raw (their bytes are not written here).  As libpng reads it: running short of data
// before raw bytes is an error, so is the end of the input before the stream's end, in every phase; a deflate error once
// a byte past raw has been asked for is only a warning (the rows are complete); the Adler-32 is compared only when the
// stream ends before any byte past raw.
// zlib's "invalid distance too far back" as libpng meets it: libpng inflates one pass row per call, and zlib finds a copy
// source in the bytes of the current call or in its window, the last min(bytes before the call, wsize) bytes.  Only for
// dist > wsize (otherwise the source is always within reach): the match starting at pos is refused when its source lies
// before both, or when it runs on into the next row (whose call sees only the window).
__host__ __device__ inline bool too_far(const Info &I, int64_t pos, int dist, int len, int64_t wsize) {
    int q = 0;
    while (q + 1 < I.npass && pos >= I.poff[q + 1]) ++q;
    const int64_t row = I.rb[q] + 1, cs = I.poff[q] + (pos - I.poff[q]) / row * row;
    const int64_t reach = (pos - cs) + (cs < wsize ? cs : wsize);
    const int64_t next = cs + row;
    return dist > reach || (next < pos + len && next < I.poff[7]);
}

template <class Sink>
__host__ __device__ inline InflateResult inflate(const uint8_t *z, int64_t zn, uint8_t *out, const Info &I, int split, Tables &T, Sink &sink) {
    InflateResult R{0, 0, 0, 0};
    const int64_t raw = I.poff[7];
    const int eof = split ? kBadHeader : kCorrupt;
    if (zn < 2) { R.status = eof; return R; }
    const int cmf = z[0], flg = z[1];
    if ((cmf & 15) != 8 || (cmf >> 4) > 7 || ((cmf << 8) | flg) % 31 != 0 || (flg & 0x20)) { R.status = kCorrupt; return R; }
    const int64_t wsize = (int64_t)1 << ((cmf >> 4) + 8);       // the window the header declares
    Bits s{z, zn, 2, 0, 0};
    int64_t pos = 0;
    bool extra = false;
    // a deflate error: only a warning once the rows are complete and a byte past them was asked for (libpng's check after
    // the last row); running out of input is an error in every phase ("Not enough image data")
#define MR_PNG_FAIL(st)                                     \
    do {                                                    \
        R.written = pos < raw ? pos : raw;                  \
        R.status = extra ? 0 : (st);                        \
        return R;                                           \
    } while (0)
#define MR_PNG_EOF()                                        \
    do {                                                    \
        R.written = pos < raw ? pos : raw;                  \
        R.status = eof;                                     \
        return R;                                           \
    } while (0)
    uint8_t *lens = T.lens;
    for (;;) {
        if (!s.need(3)) MR_PNG_EOF();
        const int last = (int)s.take(1), type = (int)s.take(2);
        if (type == 0) {
            s.take(s.c & 7);
            if (!s.need(32)) MR_PNG_EOF();
            const uint32_t len = s.take(16), nlen = s.take(16);
            if ((len ^ 0xFFFF) != nlen) MR_PNG_FAIL(kCorrupt);
            for (uint32_t k = 0; k < len; ++k) {
                if (!s.need(8)) MR_PNG_EOF();
                const uint8_t v = (uint8_t)s.take(8);
                if (pos < raw) out[pos] = v;
                else extra = true;
                ++pos;
            }
        } else if (type == 1 || type == 2) {
            if (type == 1) {
                for (int k = 0; k < 288; ++k) lens[k] = k < 144 ? 8 : k < 256 ? 9 : k < 280 ? 7 : 8;
                for (int k = 0; k < 32; ++k) lens[288 + k] = 5;    // codes 30 and 31 exist and are invalid
                build(lens, 288, T.lit, false);
                build(lens + 288, 32, T.dist, false);
            } else {
                if (!s.need(14)) MR_PNG_EOF();
                const int nlen = (int)s.take(5) + 257, ndist = (int)s.take(5) + 1, ncode = (int)s.take(4) + 4;
                if (nlen > 286 || ndist > 30) MR_PNG_FAIL(kCorrupt);
                uint8_t cl[19];
                for (int k = 0; k < 19; ++k) cl[k] = 0;
                for (int k = 0; k < ncode; ++k) {
                    if (!s.need(3)) MR_PNG_EOF();
                    // the order 16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15
                    const int j = k - 3, o = k < 3 ? 16 + k : j == 0 ? 0 : (j & 1) ? 8 + (j >> 1) : 8 - (j >> 1);
                    cl[o] = (uint8_t)s.take(3);
                }
                if (build(cl, 19, T.lit, false) < 0 || T.lit.count[0] == 19) MR_PNG_FAIL(kCorrupt);
                int k = 0;
                while (k < nlen + ndist) {
                    const int sym = decode_sym(s, T.lit);
                    if (sym == -2) MR_PNG_EOF();
                    if (sym < 0) MR_PNG_FAIL(kCorrupt);
                    if (sym < 16) { lens[k++] = (uint8_t)sym; continue; }
                    int rep, v = 0;
                    if (sym == 16) {
                        if (k == 0) MR_PNG_FAIL(kCorrupt);
                        if (!s.need(2)) MR_PNG_EOF();
                        v = lens[k - 1];
                        rep = 3 + (int)s.take(2);
                    } else if (sym == 17) {
                        if (!s.need(3)) MR_PNG_EOF();
                        rep = 3 + (int)s.take(3);
                    } else {
                        if (!s.need(7)) MR_PNG_EOF();
                        rep = 11 + (int)s.take(7);
                    }
                    if (k + rep > nlen + ndist) MR_PNG_FAIL(kCorrupt);
                    while (rep--) lens[k++] = (uint8_t)v;
                }
                if (lens[256] == 0) MR_PNG_FAIL(kCorrupt);
                uint8_t dl[30];
                for (int j = 0; j < 30; ++j) dl[j] = j < ndist ? lens[nlen + j] : 0;
                if (build(lens, nlen, T.lit, true) < 0 || build(dl, 30, T.dist, true) < 0) MR_PNG_FAIL(kCorrupt);
            }
            for (;;) {
                const int sym = decode_sym(s, T.lit);
                if (sym == -2) MR_PNG_EOF();
                if (sym < 0) MR_PNG_FAIL(kCorrupt);
                if (sym < 256) {
                    if (pos < raw) out[pos] = (uint8_t)sym;
                    else extra = true;
                    ++pos;
                    continue;
                }
                if (sym == 256) break;
                const int li = sym - 257;
                if (li >= 29) MR_PNG_FAIL(kCorrupt);
                // RFC 1951's length and distance bases, in closed form
                const int le = li < 8 || li == 28 ? 0 : (li - 4) >> 2;
                const int lb = li < 8 ? 3 + li : li == 28 ? 258 : ((4 + (li & 3)) << le) + 3;
                if (!s.need(le)) MR_PNG_EOF();
                const int len = lb + (int)s.take(le);
                const int ds = decode_sym(s, T.dist);
                if (ds == -2) MR_PNG_EOF();
                if (ds < 0 || ds >= 30) MR_PNG_FAIL(kCorrupt);
                const int de = ds < 4 ? 0 : (ds >> 1) - 1, db = ds < 4 ? 1 + ds : ((2 + (ds & 1)) << de) + 1;
                if (!s.need(de)) MR_PNG_EOF();
                const int dist = db + (int)s.take(de);
                if (pos >= raw) extra = true;                            // zlib checks the distance once it has room to copy
                if (dist > pos) MR_PNG_FAIL(kCorrupt);                   // before the start of the output
                if (dist > wsize && pos < raw && too_far(I, pos, dist, len, wsize)) MR_PNG_FAIL(kCorrupt);
                if (pos < raw) sink(pos, dist, (int)(pos + len <= raw ? len : raw - pos));
                if (pos + len > raw) extra = true;
                pos += len;
            }
        } else {
            MR_PNG_FAIL(kCorrupt);
        }
        if (last) break;
    }
    s.take(s.c & 7);
    if (!s.need(32)) MR_PNG_EOF();
    const uint32_t a = s.take(32);
    R.adler = ((a & 0xFF) << 24) | ((a & 0xFF00) << 8) | ((a >> 8) & 0xFF00) | (a >> 24);
    R.written = pos < raw ? pos : raw;
    if (pos < raw) { R.status = split ? kBadHeader : kCorrupt; return R; }     // "Not enough image data"
    R.check = extra ? 0 : 1;
#undef MR_PNG_FAIL
#undef MR_PNG_EOF
    return R;
}

// Adler-32 of d[0, n) (the kernels form the same sums in parallel: A = 1 + sum d, B = n + sum (n - i) d_i)
__host__ __device__ inline uint32_t adler32(const uint8_t *d, int64_t n) {
    uint64_t a = 1, b = 0;
    for (int64_t i = 0; i < n; ++i) {
        a = (a + d[i]) % 65521;
        b = (b + a) % 65521;
    }
    return (uint32_t)((b << 16) | a);
}

// ---------------------------------------------------------------- row filters

__host__ __device__ inline uint8_t unfilter_byte(int type, int x, int a, int b, int c) {
    switch (type) {
    case 1: return (uint8_t)(x + a);
    case 2: return (uint8_t)(x + b);
    case 3: return (uint8_t)(x + ((a + b) >> 1));
    case 4: {
        const int p = a + b - c, pa = p > a ? p - a : a - p, pb = p > b ? p - b : b - p, pc = p > c ? p - c : c - p;
        return (uint8_t)(x + (pa <= pb && pa <= pc ? a : pb <= pc ? b : c));
    }
    default: return (uint8_t)x;
    }
}

// one pass row in place: row[-1] is its filter byte, prev the unfiltered row above (nullptr for the first); false for a
// filter type past 4
__host__ __device__ inline bool unfilter_row(uint8_t *row, const uint8_t *prev, int64_t n, int bpp) {
    const int type = row[-1];
    if (type > 4) return false;
    for (int64_t i = 0; i < n; ++i) {
        const int a = i >= bpp ? row[i - bpp] : 0, b = prev ? prev[i] : 0, c = prev && i >= bpp ? prev[i - bpp] : 0;
        row[i] = unfilter_byte(type, row[i], a, b, c);
    }
    return true;
}

// ---------------------------------------------------------------- output pixel

// the pass of image pixel (y, x) and its place in the pass
__host__ __device__ inline int pass_of(const Info &I, int y, int x, int &py, int &px) {
    if (!I.interlace) { py = y; px = x; return 0; }
    int p;
    if (y & 1) p = 6;
    else if (x & 1) p = 5;
    else if ((y & 3) == 2) p = 4;
    else if ((x & 3) == 2) p = 3;
    else if ((y & 7) == 4) p = 2;
    else if ((x & 7) == 4) p = 1;
    else p = 0;
    int x0, y0, dx, dy;
    adam7(p, x0, y0, dx, dy);
    py = (y - y0) / dy;
    px = (x - x0) / dx;
    return p;
}

// sample k of pass pixel (py, px), reduced to 8 bits (high byte of 16; sub-byte grey scaled as png_set_expand does, a
// palette index as it is)
__host__ __device__ inline int sample(const Info &I, const uint8_t *raw, int p, int py, int px, int k) {
    const uint8_t *row = raw + I.poff[p] + (int64_t)py * (I.rb[p] + 1) + 1;
    if (I.depth == 8) return row[(int64_t)px * I.channels + k];
    if (I.depth == 16) return row[2 * ((int64_t)px * I.channels + k)];
    const int64_t bit = (int64_t)px * I.depth;
    return (row[bit >> 3] >> (8 - I.depth - (int)(bit & 7))) & ((1 << I.depth) - 1);
}

// output pixel (y, x) as B, G, R
__host__ __device__ inline void output_pixel(const Info &I, const uint8_t *raw, int y, int x, uint8_t *bgr) {
    int sy, sx, py, px;
    mr_jpeg::orient_source(I.orient, I.h, I.w, y, x, sy, sx);
    const int p = pass_of(I, sy, sx, py, px);
    if (I.ctype == 3) {
        const int i = sample(I, raw, p, py, px, 0);
        if (i < I.npal) { bgr[0] = I.pal[3 * i + 2]; bgr[1] = I.pal[3 * i + 1]; bgr[2] = I.pal[3 * i]; }
        else bgr[0] = bgr[1] = bgr[2] = 0;
        return;
    }
    if (I.ctype == 2 || I.ctype == 6) {
        bgr[0] = (uint8_t)sample(I, raw, p, py, px, 2);
        bgr[1] = (uint8_t)sample(I, raw, p, py, px, 1);
        bgr[2] = (uint8_t)sample(I, raw, p, py, px, 0);
        return;
    }
    int v = sample(I, raw, p, py, px, 0);
    if (I.depth < 8) v *= I.depth == 1 ? 255 : I.depth == 2 ? 85 : 17;
    bgr[0] = bgr[1] = bgr[2] = (uint8_t)v;
}

}  // namespace mr_png
