// PNG decoding of a batch on the device, equal to cv2.imdecode(buf, cv2.IMREAD_COLOR) (png_core.cuh holds the arithmetic),
// and the decode of a batch mixing JPEG and PNG files.  The output is db_batch's packed layout, as mr_jpeg_decode's.
//   1. png_parse_kernel:    per image (thread) the chunk walk, IHDR / PLTE / eXIf, the first IDAT run, the status;
//   2. png_layout_kernel:   one CTA: overlapping offsets, prefix sums of output pixels (the capacity rule of mr_jpeg_decode),
//                           of inflated bytes (at most 9 per pixel, so they fit when the pixels do) and of zlib bytes;
//   3. png_idat_kernel:     per image (CTA), one warp per IDAT chunk: the chunk's CRC from its lanes' parts combined in GF(2)
//                           (crc_combine), and its payload gathered into one contiguous zlib stream;
//   4. png_inflate_kernel:  per image (warp, tables in shared memory), one lane's serial Huffman decode: literals written,
//                           each match recorded as (dst, dist, len);
//   5. png_expand_kernel:   per image (CTA): src[b] = b, then src[b] = b - dist over every recorded match;
//      png_jump_kernel:     src[b] = src[src[b]] over every inflated byte, rounds_for(pixel capacity) launches that return
//                           at once after a round changed nothing (log2 of the longest copy chain are needed);
//      png_copy_kernel:     every match byte from its literal source, with the Adler-32 sums of the inflated bytes;
//   6. png_unfilter_kernel: per image (warp) a wavefront over bands of 32 rows: lane l owns row r0 + l and reconstructs
//                           pixel s - l at step s, when the lane above has finished the pixels it needs;
//   7. png_finish_kernel:   the Adler-32 check; flagged images get shape (0, 0);
//   8. png_color_kernel:    per output pixel: unpacking, palette, grey, 16 bits, BGR, orientation (Adam7 passes read in place).
// Nothing is read back to the host and nothing is allocated, so the call can be captured in a CUDA graph.
#include <cub/cub.cuh>

#include "common.cuh"
#include "png_core.cuh"

using namespace mr;
using namespace mr_png;

extern "C" int64_t mr_jpeg_workspace_bytes(int64_t N, int64_t byte_capacity, int64_t pixel_capacity);
extern "C" int mr_jpeg_decode(const void *data, int64_t data_bytes, const int64_t *data_offsets, int N, int max_h, int max_w,
                              int64_t pixel_capacity, void *workspace, int64_t workspace_bytes, unsigned char *image_out,
                              int64_t *image_offsets, int *shapes, int *status, void *stream);

namespace {

constexpr int kThreads = 256;
constexpr int kWarpsPerCta = 4;          // images per CTA of the inflate and unfilter kernels
constexpr int kRawPerPixel = 9;          // inflated bytes per pixel at most: 8 (16-bit RGBA) and a filter byte per row

int64_t r256(int64_t b) { return round_up(b, 256); }

struct Layout {
    int64_t o_info, o_z, o_raw, o_src, o_rec, o_acc, o_flags, total;
    int64_t raw_cap, rec_cap;
};

Layout layout(int64_t N, int64_t B, int64_t P) {
    Layout l;
    l.raw_cap = kRawPerPixel * P;
    l.rec_cap = l.raw_cap / 3 + N + 1;             // a recorded match covers at least 3 bytes, except an image's last (cut at the end of its rows)
    int64_t o = 0;
    l.o_info = o; o += r256(N * (int64_t)sizeof(Info));
    l.o_z = o; o += r256(B + 8);
    l.o_raw = o; o += r256(l.raw_cap + 8);
    l.o_src = o; o += r256(4 * l.raw_cap);
    l.o_rec = o; o += r256(8 * l.rec_cap);
    l.o_acc = o; o += r256(16 * N);
    l.o_flags = o; o += 256;
    l.total = o;
    return l;
}

struct Ws {
    Info *info;
    uint8_t *z, *raw;
    uint32_t *src;                             // per inflated byte: the image-relative byte it copies (itself for a literal)
    uint2 *rec;                                // (dst, dist << 9 | len)
    unsigned long long *acc;                   // per image: the two Adler-32 sums
    int *changed;                              // per jump round: a pointer moved
};

Ws carve(void *ws, const Layout &l) {
    char *b = (char *)ws;
    return Ws{(Info *)(b + l.o_info), (uint8_t *)(b + l.o_z), (uint8_t *)(b + l.o_raw), (uint32_t *)(b + l.o_src), (uint2 *)(b + l.o_rec),
              (unsigned long long *)(b + l.o_acc), (int *)(b + l.o_flags)};
}

constexpr int kMaxRounds = 40;

__device__ __forceinline__ void crc_table(uint32_t *tab) {
    for (int i = threadIdx.x; i < 256; i += blockDim.x) tab[i] = crc_table_entry(i);
    __syncthreads();
}

__global__ void __launch_bounds__(64) png_parse_kernel(const uint8_t *__restrict__ data, int64_t data_bytes, const int64_t *__restrict__ off,
                                                        int N, int max_h, int max_w, Ws w, int *status) {
    __shared__ uint32_t tab[256];
    crc_table(tab);
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= N) return;
    Info &I = w.info[n];
    const int64_t a = off[n], b = off[n + 1];
    if (off[0] < 0 || a < off[0] || b < a || b > data_bytes || (n > 0 && off[n - 1] > a)) {
        I.status = kBadOffsets;
        I.poff[7] = 0;
    } else if (parse(data + a, b - a, tab, I) == 0) {
        if (I.out_h > max_h || I.out_w > max_w || I.poff[7] >= ((int64_t)1 << 31)) I.status = kTooLarge;
    }
    status[n] = I.status;
}

// one CTA: offsets (as mr_jpeg_decode: bytes that start before an earlier image's start are flagged), then the prefix sums
constexpr int kScan = 512;               // threads of the one-CTA prefix sums

__global__ void __launch_bounds__(kScan) png_layout_kernel(const int64_t *__restrict__ off, int N, int64_t pixel_cap, Ws w,
                                                          int64_t *image_offsets, int *shapes, int *status) {
    using Scan = cub::BlockScan<int64_t, kScan>;
    __shared__ typename Scan::TempStorage tmp;
    __shared__ int64_t carry, c_px, c_raw, c_z;
    if (threadIdx.x == 0) { carry = off[0]; c_px = c_raw = c_z = 0; }
    for (int i = threadIdx.x; i < kMaxRounds; i += blockDim.x) w.changed[i] = 0;
    __syncthreads();
    for (int n0 = 0; n0 < N; n0 += kScan) {
        const int n = n0 + threadIdx.x;
        const int64_t v = n < N ? off[n] : INT64_MIN;
        int64_t before, top;
        Scan(tmp).ExclusiveScan(v, before, cub::Max(), top);
        const int64_t m = threadIdx.x == 0 ? carry : (before > carry ? before : carry);
        int st = n < N ? status[n] : 0;
        if (n < N && (v < m || off[n + 1] < v)) st |= kBadOffsets;
        int64_t px = 0, raw = 0, zb = 0;
        if (n < N && st == 0) {
            const Info &I = w.info[n];
            px = (int64_t)I.h * I.w;
            raw = I.poff[7];
            zb = I.zbytes;
        }
        int64_t bpx, tpx, braw, traw, bz, tz;
        __syncthreads();
        Scan(tmp).ExclusiveSum(px, bpx, tpx);
        __syncthreads();
        Scan(tmp).ExclusiveSum(raw, braw, traw);
        __syncthreads();
        Scan(tmp).ExclusiveSum(zb, bz, tz);
        if (n < N) {
            bpx += c_px;
            if (st == 0 && bpx + px > pixel_cap) st = kTooLarge;   // then braw + raw <= 9 * pixel_cap as well
            Info &I = w.info[n];
            I.status = st;
            I.out = bpx;
            I.raw_base = c_raw + braw;
            I.z = c_z + bz;
            status[n] = st;
            image_offsets[n] = 3 * bpx;
            shapes[2 * n] = st ? 0 : I.out_h;
            shapes[2 * n + 1] = st ? 0 : I.out_w;
            w.acc[2 * n] = w.acc[2 * n + 1] = 0;
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            if (top > carry) carry = top;
            c_px += tpx;
            c_raw += traw;
            c_z += tz;
        }
        __syncthreads();
    }
}

// one CTA per image, warp k takes IDAT chunks k, k + 8, ... of the first run: CRC over lanes' parts combined, payload copied
__global__ void __launch_bounds__(kThreads) png_idat_kernel(const uint8_t *__restrict__ data, const int64_t *__restrict__ off, Ws w, int *status) {
    __shared__ uint32_t tab[256];
    const int n = blockIdx.x;
    if (status[n]) return;
    crc_table(tab);
    const Info &I = w.info[n];
    const uint8_t *p = data + off[n];
    uint8_t *z = w.z + I.z;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
    int64_t i = I.idat, pos = 0;
    bool bad = false;
    for (int k = 0; be32(p + i + 4) == kIDAT; ++k) {
        const int64_t len = be32(p + i);
        if (k % nw == warp) {
            const uint8_t *t = p + i + 4;
            for (int64_t j = lane; j < len; j += 32) z[pos + j] = t[4 + j];
            const int64_t m = len + 4, per = (m + 31) / 32;
            const int64_t s0 = lane * per < m ? lane * per : m, s1 = s0 + per < m ? s0 + per : m;
            uint32_t c = crc_update(tab, 0, t + s0, s1 - s0);
            for (int s = 1; s < 32; s <<= 1) {           // lane l (l % 2s == 0) appends the parts of lanes l + s .. l + 2s - 1
                const uint32_t right = __shfl_down_sync(0xffffffffu, c, s);
                if ((lane & (2 * s - 1)) == 0) {
                    const int64_t r0 = (lane + s) * per < m ? (lane + s) * per : m, r1 = (lane + 2 * s) * per < m ? (lane + 2 * s) * per : m;
                    c = crc_combine(c, right, r1 - r0);
                }
            }
            if (lane == 0 && c != be32(t + 4 + len)) bad = true;
        }
        pos += len;
        i += 12 + len;
    }
    if (__syncthreads_or(bad) && threadIdx.x == 0) atomicOr(status + n, kBadHeader);
}

struct RecordSink {
    uint2 *rec;
    int n;
    __device__ void operator()(int64_t dst, int dist, int len) { rec[n++] = make_uint2((uint32_t)dst, ((uint32_t)dist << 9) | (uint32_t)len); }
};

__device__ __forceinline__ int64_t rec_base(const Info &I, int n) { return I.raw_base / 3 + n; }

// one warp per image; lane 0 decodes with the tables in shared memory
__global__ void __launch_bounds__(32 * kWarpsPerCta) png_inflate_kernel(int N, Ws w, int *status) {
    __shared__ Tables T[kWarpsPerCta];
    const int n = blockIdx.x * kWarpsPerCta + (threadIdx.x >> 5);
    if (n >= N || (threadIdx.x & 31) || status[n]) return;
    Info &I = w.info[n];
    RecordSink sink{w.rec + rec_base(I, n), 0};
    const InflateResult r = inflate(w.z + I.z, I.zbytes, w.raw + I.raw_base, I, I.split, T[threadIdx.x >> 5], sink);
    I.nrec = sink.n;
    I.check = r.check;
    I.adler = r.adler;
    if (r.status) atomicOr(status + n, r.status);
}

__global__ void __launch_bounds__(kThreads) png_expand_kernel(Ws w, const int *__restrict__ status) {
    const int n = blockIdx.x;
    if (status[n]) return;
    const Info &I = w.info[n];
    uint32_t *src = w.src + I.raw_base;
    const int64_t raw = I.poff[7];
    for (int64_t b = threadIdx.x; b < raw; b += blockDim.x) src[b] = (uint32_t)b;
    __syncthreads();
    const uint2 *rec = w.rec + rec_base(I, n);
    for (int k = threadIdx.x; k < I.nrec; k += blockDim.x) {
        const uint2 r = rec[k];
        const uint32_t dist = r.y >> 9, len = r.y & 511;
        for (uint32_t j = 0; j < len; ++j) src[r.x + j] = r.x + j - dist;
    }
}

// grid (x, image): one round of pointer jumping; returns at once when the previous round moved nothing
__global__ void __launch_bounds__(kThreads) png_jump_kernel(int round, Ws w, const int *__restrict__ status) {
    if (round > 0 && !*(volatile int *)(w.changed + round - 1)) return;
    const int n = blockIdx.y;
    if (status[n]) return;
    const Info &I = w.info[n];
    uint32_t *src = w.src + I.raw_base;
    const int64_t raw = I.poff[7];
    int moved = 0;
    for (int64_t b = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; b < raw; b += (int64_t)gridDim.x * blockDim.x) {
        const uint32_t s = src[b];
        if (s == (uint32_t)b) continue;
        const uint32_t t = src[s];
        if (t != s) { src[b] = t; moved = 1; }
    }
    if (__syncthreads_or(moved) && threadIdx.x == 0) atomicOr(w.changed + round, 1);
}

// grid (x, image): match bytes from their literal sources, and the Adler-32 sums sum d_i and sum (raw - i) d_i mod 65521
__global__ void __launch_bounds__(kThreads) png_copy_kernel(Ws w, const int *__restrict__ status) {
    using Reduce = cub::BlockReduce<unsigned long long, kThreads>;
    __shared__ typename Reduce::TempStorage tmp;
    const int n = blockIdx.y;
    if (status[n]) return;
    const Info &I = w.info[n];
    const uint32_t *src = w.src + I.raw_base;
    uint8_t *raw = w.raw + I.raw_base;
    const int64_t m = I.poff[7];
    unsigned long long sa = 0, sb = 0;
    for (int64_t b = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; b < m; b += (int64_t)gridDim.x * blockDim.x) {
        const uint32_t s = src[b];
        const uint8_t v = raw[s];
        if (s != (uint32_t)b) raw[b] = v;
        sa += v;
        sb = (sb + (unsigned long long)((m - b) % 65521) * v) % 65521;
    }
    sa %= 65521;
    const unsigned long long ta = Reduce(tmp).Sum(sa);
    __syncthreads();
    const unsigned long long tb = Reduce(tmp).Sum(sb);
    if (threadIdx.x == 0) {
        atomicAdd(w.acc + 2 * n, ta);
        atomicAdd(w.acc + 2 * n + 1, tb);
    }
}

// one warp per image: each pass in bands of 32 rows, lane l on row r0 + l, pixel s - l at step s
__global__ void __launch_bounds__(32 * kWarpsPerCta) png_unfilter_kernel(int N, Ws w, int *status) {
    const int n = blockIdx.x * kWarpsPerCta + (threadIdx.x >> 5);
    if (n >= N || status[n]) return;
    const int lane = threadIdx.x & 31;
    const Info &I = w.info[n];
    uint8_t *raw = w.raw + I.raw_base;
    const int bpp = I.fbpp;
    int bad = 0;
    for (int p = 0; p < I.npass; ++p) {
        if (!I.pw[p]) continue;
        const int64_t rb = I.rb[p], units = rb / bpp;
        for (int r0 = 0; r0 < I.ph[p]; r0 += 32) {
            const int row = r0 + lane;
            const bool active = row < I.ph[p];
            uint8_t *cur = raw + I.poff[p] + (int64_t)row * (rb + 1) + 1;
            const uint8_t *prev = row > 0 ? cur - rb - 1 : nullptr;
            const int type = active ? cur[-1] : 0;
            bad |= type > 4;
            for (int64_t s = 0; s < units + 31; ++s) {
                const int64_t x = s - lane;
                if (active && x >= 0 && x < units) {
                    for (int j = 0; j < bpp; ++j) {
                        const int64_t i = x * bpp + j;
                        const int a = x > 0 ? cur[i - bpp] : 0, b = prev ? prev[i] : 0, c = prev && x > 0 ? prev[i - bpp] : 0;
                        cur[i] = unfilter_byte(type, cur[i], a, b, c);
                    }
                }
                __syncwarp();
            }
        }
    }
    if (__any_sync(0xffffffffu, bad) && lane == 0) atomicOr(status + n, kCorrupt);
}

__global__ void png_finish_kernel(int N, Ws w, int *shapes, int *status) {
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= N) return;
    const Info &I = w.info[n];
    if (status[n] == 0 && I.check) {
        const int64_t raw = I.poff[7];
        const uint32_t a = (uint32_t)((w.acc[2 * n] + 1) % 65521), b = (uint32_t)((w.acc[2 * n + 1] + raw % 65521) % 65521);
        if (((b << 16) | a) != I.adler) status[n] |= kCorrupt;
    }
    if (status[n]) shapes[2 * n] = shapes[2 * n + 1] = 0;
}

__global__ void __launch_bounds__(kThreads) png_color_kernel(Ws w, const int *__restrict__ status, uint8_t *image_out) {
    const int n = blockIdx.y;
    if (status[n]) return;
    const Info &I = w.info[n];
    const uint8_t *raw = w.raw + I.raw_base;
    const int64_t np = (int64_t)I.out_h * I.out_w;
    uint8_t *o = image_out + 3 * I.out;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < np; i += (int64_t)gridDim.x * blockDim.x) {
        uint8_t bgr[3];
        output_pixel(I, raw, (int)(i / I.out_w), (int)(i % I.out_w), bgr);
        o[3 * i] = bgr[0];
        o[3 * i + 1] = bgr[1];
        o[3 * i + 2] = bgr[2];
    }
}

// ---------------------------------------------------------------- mixed batches

struct Mixed {
    int64_t o_pass, o_jpix, o_ppix, o_small, total;
};

Mixed mixed_layout(int64_t N, int64_t B, int64_t P) {
    Mixed m;
    const int64_t a = mr_jpeg_workspace_bytes(N, B, P), b = layout(N, B, P).total;
    int64_t o = 0;
    m.o_pass = o; o += r256(a > b ? a : b);    // the two passes run one after the other in the same bytes
    m.o_jpix = o; o += r256(3 * P + 1);
    m.o_ppix = o; o += r256(3 * P + 1);
    m.o_small = o; o += r256(64 * N);           // per pass image_offsets, shapes, status; the merge's sources
    m.total = o;
    return m;
}

struct Pass {
    int64_t *io;
    int *sh, *st;
};

// one CTA: per image the result of the decoder that recognises its signature (JPEG's otherwise, which flags a file with
// neither), then mr_jpeg_decode's capacity rule over the merged pixel sums
__global__ void __launch_bounds__(kScan) image_merge_kernel(const uint8_t *__restrict__ data, int64_t data_bytes, const int64_t *__restrict__ off,
                                                           int N, int64_t pixel_cap, Pass jp, Pass pp, int64_t *src, int64_t *image_offsets,
                                                           int *shapes, int *status) {
    using Scan = cub::BlockScan<int64_t, kScan>;
    __shared__ typename Scan::TempStorage tmp;
    __shared__ int64_t c_px;
    if (threadIdx.x == 0) c_px = 0;
    __syncthreads();
    for (int n0 = 0; n0 < N; n0 += kScan) {
        const int n = n0 + threadIdx.x;
        int st = 0, h = 0, wd = 0;
        int64_t so = 0;
        if (n < N) {
            const int64_t a = off[n], b = off[n + 1];
            const bool png = a >= 0 && b >= a && b <= data_bytes && has_signature(data + a, b - a);
            const Pass &q = png ? pp : jp;
            st = q.st[n];
            h = q.sh[2 * n];
            wd = q.sh[2 * n + 1];
            so = png ? -1 - q.io[n] : q.io[n];  // PNG sources negative
        }
        const int64_t px = st == 0 ? (int64_t)h * wd : 0;
        int64_t bpx, tpx;
        Scan(tmp).ExclusiveSum(px, bpx, tpx);
        if (n < N) {
            bpx += c_px;
            if (st == 0 && bpx + px > pixel_cap) st = kTooLarge;
            status[n] = st;
            image_offsets[n] = 3 * bpx;
            shapes[2 * n] = st ? 0 : h;
            shapes[2 * n + 1] = st ? 0 : wd;
            src[n] = so;
        }
        __syncthreads();
        if (threadIdx.x == 0) c_px += tpx;
        __syncthreads();
    }
}

__global__ void __launch_bounds__(kThreads) image_copy_kernel(const uint8_t *__restrict__ jpix, const uint8_t *__restrict__ ppix,
                                                              const int64_t *__restrict__ src, const int64_t *__restrict__ image_offsets,
                                                              const int *__restrict__ shapes, const int *__restrict__ status, uint8_t *image_out) {
    const int n = blockIdx.y;
    if (status[n]) return;
    const int64_t s = src[n];
    const uint8_t *from = s < 0 ? ppix + (-1 - s) : jpix + s;
    uint8_t *to = image_out + image_offsets[n];
    const int64_t m = 3 * (int64_t)shapes[2 * n] * shapes[2 * n + 1];
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < m; i += (int64_t)gridDim.x * blockDim.x) to[i] = from[i];
}

bool bad_sizes(int64_t N, int64_t B, int64_t P) { return N < 1 || N > 65535 || B < 0 || P < 0 || B > ((int64_t)1 << 40) || P > ((int64_t)1 << 36); }

int rounds_for(int64_t P) {                    // log2 of the longest copy chain (< the image's inflated bytes < 2^31), plus one
    int r = 1;
    while (r < 32 && ((int64_t)1 << r) < kRawPerPixel * P + 1) ++r;
    return r + 1;
}

}  // namespace

extern "C" {

int64_t mr_png_workspace_bytes(int64_t N, int64_t byte_capacity, int64_t pixel_capacity) {
    if (bad_sizes(N, byte_capacity, pixel_capacity)) return 0;
    return layout(N, byte_capacity, pixel_capacity).total;
}

int mr_png_decode(const void *data, int64_t data_bytes, const int64_t *data_offsets, int N, int max_h, int max_w, int64_t pixel_capacity,
                  void *workspace, int64_t workspace_bytes, unsigned char *image_out, int64_t *image_offsets, int *shapes, int *status,
                  void *stream) {
    if (bad_sizes(N, data_bytes, pixel_capacity) || max_h < 1 || max_w < 1 || max_h > kMaxSide || max_w > kMaxSide)
        return MR_ERR_BAD_SHAPE;
    const Layout l = layout(N, data_bytes, pixel_capacity);
    if (workspace_bytes < l.total) return MR_ERR_BAD_SHAPE;
    if (!data || !data_offsets || !workspace || !image_offsets || !shapes || !status) return MR_ERR_NULL_POINTER;
    if (pixel_capacity > 0 && !image_out) return MR_ERR_NULL_POINTER;
    cudaStream_t st = (cudaStream_t)stream;
    const Ws w = carve(workspace, l);
    const uint8_t *d = (const uint8_t *)data;
    const int gx = (int)std::max<int64_t>(1, std::min<int64_t>(64, kRawPerPixel * pixel_capacity / ((int64_t)N * 4 * kThreads)));
    const int wg = (int)ceil_div(N, kWarpsPerCta);
    int rc;
    png_parse_kernel<<<(int)ceil_div(N, 64), 64, 0, st>>>(d, data_bytes, data_offsets, N, max_h, max_w, w, status);
    if ((rc = check_launch("png parse"))) return rc;
    png_layout_kernel<<<1, kScan, 0, st>>>(data_offsets, N, pixel_capacity, w, image_offsets, shapes, status);
    if ((rc = check_launch("png layout"))) return rc;
    png_idat_kernel<<<N, kThreads, 0, st>>>(d, data_offsets, w, status);
    if ((rc = check_launch("png idat"))) return rc;
    png_inflate_kernel<<<wg, 32 * kWarpsPerCta, 0, st>>>(N, w, status);
    if ((rc = check_launch("png inflate"))) return rc;
    png_expand_kernel<<<N, kThreads, 0, st>>>(w, status);
    if ((rc = check_launch("png expand"))) return rc;
    const int rounds = rounds_for(pixel_capacity);
    for (int r = 0; r < rounds; ++r) {
        png_jump_kernel<<<dim3(gx, N), kThreads, 0, st>>>(r, w, status);
        if ((rc = check_launch("png jump"))) return rc;
    }
    png_copy_kernel<<<dim3(gx, N), kThreads, 0, st>>>(w, status);
    if ((rc = check_launch("png copy"))) return rc;
    png_unfilter_kernel<<<wg, 32 * kWarpsPerCta, 0, st>>>(N, w, status);
    if ((rc = check_launch("png unfilter"))) return rc;
    png_finish_kernel<<<(int)ceil_div(N, 256), 256, 0, st>>>(N, w, shapes, status);
    if ((rc = check_launch("png finish"))) return rc;
    const int cx = (int)std::max<int64_t>(1, std::min<int64_t>(64, pixel_capacity / ((int64_t)N * 4 * kThreads)));
    png_color_kernel<<<dim3(cx, N), kThreads, 0, st>>>(w, status, image_out);
    return check_launch("png color");
}

int64_t mr_image_workspace_bytes(int64_t N, int64_t byte_capacity, int64_t pixel_capacity) {
    if (bad_sizes(N, byte_capacity, pixel_capacity)) return 0;
    return mixed_layout(N, byte_capacity, pixel_capacity).total;
}

int mr_image_decode(const void *data, int64_t data_bytes, const int64_t *data_offsets, int N, int max_h, int max_w, int64_t pixel_capacity,
                    void *workspace, int64_t workspace_bytes, unsigned char *image_out, int64_t *image_offsets, int *shapes, int *status,
                    void *stream) {
    if (bad_sizes(N, data_bytes, pixel_capacity) || max_h < 1 || max_w < 1 || max_h > kMaxSide || max_w > kMaxSide)
        return MR_ERR_BAD_SHAPE;
    const Mixed m = mixed_layout(N, data_bytes, pixel_capacity);
    if (workspace_bytes < m.total) return MR_ERR_BAD_SHAPE;
    if (!data || !data_offsets || !workspace || !image_offsets || !shapes || !status) return MR_ERR_NULL_POINTER;
    if (pixel_capacity > 0 && !image_out) return MR_ERR_NULL_POINTER;
    char *b = (char *)workspace;
    void *pass = b + m.o_pass;
    const int64_t pass_bytes = m.o_jpix - m.o_pass;
    uint8_t *jpix = (uint8_t *)(b + m.o_jpix), *ppix = (uint8_t *)(b + m.o_ppix);
    int64_t *small = (int64_t *)(b + m.o_small);
    const Pass jp{small, (int *)(small + 3 * (int64_t)N), (int *)(small + 4 * (int64_t)N)};
    const Pass pp{small + N, (int *)(small + 5 * (int64_t)N), (int *)(small + 6 * (int64_t)N)};
    int64_t *src = small + 2 * (int64_t)N;
    int rc;
    if ((rc = mr_jpeg_decode(data, data_bytes, data_offsets, N, max_h, max_w, pixel_capacity, pass, pass_bytes, jpix, jp.io, jp.sh, jp.st, stream)))
        return rc;
    if ((rc = mr_png_decode(data, data_bytes, data_offsets, N, max_h, max_w, pixel_capacity, pass, pass_bytes, ppix, pp.io, pp.sh, pp.st, stream)))
        return rc;
    cudaStream_t st = (cudaStream_t)stream;
    image_merge_kernel<<<1, kScan, 0, st>>>((const uint8_t *)data, data_bytes, data_offsets, N, pixel_capacity, jp, pp, src, image_offsets,
                                           shapes, status);
    if ((rc = check_launch("image merge"))) return rc;
    const int gx = (int)std::max<int64_t>(1, std::min<int64_t>(64, 3 * pixel_capacity / ((int64_t)N * 4 * kThreads)));
    image_copy_kernel<<<dim3(gx, N), kThreads, 0, st>>>(jpix, ppix, src, image_offsets, shapes, status, image_out);
    return check_launch("image copy");
}

}  // extern "C"
