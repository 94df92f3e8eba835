// Baseline JPEG decoding of a batch on the device, equal to cv2.imdecode(buf, cv2.IMREAD_COLOR) (jpeg_core.cuh holds the
// arithmetic).  The output is db_batch's packed layout: uint8 HWC BGR, image_offsets int64 [N] in elements, shapes int32 [N, 2].
//   1. jpeg_parse_kernel: per image the markers up to SOS (tables, geometry, colour space, orientation) and the status;
//      jpeg_offsets_kernel: images whose bytes start before an earlier image's end are flagged;
//   2. jpeg_split_kernel: per image (one CTA) a parallel pass over the scan bytes that removes the 0xFF00 stuffing, finds
//      RSTn and the end of the scan, records each restart segment's start, and cuts the segments into runs of kRunBits;
//   3. jpeg_layout_kernel: prefix sums over the images of their runs, coefficient blocks and output pixels (image_offsets,
//      shapes, the capacity flags);
//   4. the self-synchronising Huffman decode over every run of the batch (Weissenberger & Schmidt):
//      jpeg_sync_kernel<1>: each run from the assumed state (its first bit, block 0 of an MCU, DC) -- the true state for the
//                           first run of a segment -- to its exit state X;
//      jpeg_sync_kernel<3>: kRelax times, each run again from its predecessor's latest exit (Jacobi passes);
//      jpeg_sync_kernel<2>: each run again from its predecessor's exit X[r - 1], to Y, with its block count and DC sums;
//      jpeg_walk_kernel:    per segment, in order: where the true entry of a run is not X[r - 1] (its predecessor had not
//                           synchronised), the run is decoded again from the true one; the segmented prefix sums of the
//                           block counts and DC differences give each run its first block and DC predictions;
//      jpeg_write_kernel:   each run from its true entry, writing its coefficients in natural order, DC predicted;
//      correctness never depends on synchronisation: a run that never synchronises is decoded by the walker;
//   5. jpeg_finish_kernel: corrupt-scan checks, flagged images get shape (0, 0);
//   6. jpeg_idct_kernel: per block jpeg_idct_islow, in place (the uint8 samples over the block's coefficients);
//   7. jpeg_color_kernel: per output pixel upsampling, colour conversion and orientation into the packed buffer.
// Nothing is read back to the host and nothing is allocated, so the call can be captured in a CUDA graph.
#include <cub/cub.cuh>

#include "common.cuh"
#include "jpeg_core.cuh"

using namespace mr;
using namespace mr_jpeg;

namespace {

// Run size of the synchronising decode.  A run that starts from the assumed state must find both the codeword boundary and
// the block's place in the MCU; with six blocks per 4:2:0 MCU the latter takes long.  On 1280 x 720 scenes at quality 90
// (jpeg_core_host), 59 % of 512-bit runs and 12 % of 2048-bit runs had not synchronised by their end (4:2:0; 7 % and 0 %
// at 4:4:4).  kRelax passes then carry each run's exit one run further, so that the walker, which decodes serially, has
// little left; 2048 bits still gives ~4 k runs per MB.
constexpr int kRunBits = 2048;
constexpr int kRelax = 2;
constexpr int kThreads = 256;
constexpr int kTile = 16;                // bytes per thread per split iteration

int64_t r256(int64_t b) { return round_up(b, 256); }

struct RunCnt {
    int blocks, dc0, dc1, dc2;
};

struct Layout {
    int64_t o_info, o_stream, o_seg_byte, o_seg_run, o_seg_done, o_run_base, o_coef_base, o_totals, o_X, o_Y, o_E, o_Z, o_cnt, o_pre,
        o_run_seg, o_coef, total;
    int64_t slots, runs, blocks;
};

Layout layout(int64_t N, int64_t B, int64_t P) {
    Layout l;
    l.slots = B / 2 + 3 * (int64_t)N + 1;                      // restart segments: an RSTn takes two bytes
    l.runs = B * 8 / kRunBits + l.slots;                       // every segment's bits cut into runs, at least one each
    l.blocks = (6 * P + 3072 * N) / 64;                        // coefficient blocks (DESIGN §7: images past it are flagged)
    int64_t o = 0;
    l.o_info = o; o += r256(N * (int64_t)sizeof(Info));
    l.o_stream = o; o += r256(B + 8);
    l.o_seg_byte = o; o += r256((l.slots + 1) * 8);
    l.o_seg_run = o; o += r256((l.slots + 1) * 4);
    l.o_seg_done = o; o += r256((l.slots + 1) * 4);
    l.o_run_base = o; o += r256((N + 1) * 8);
    l.o_coef_base = o; o += r256((N + 1) * 8);
    l.o_totals = o; o += 256;
    l.o_X = o; o += r256(l.runs * 8);
    l.o_Y = o; o += r256(l.runs * 8);
    l.o_E = o; o += r256(l.runs * 8);
    l.o_Z = o; o += r256(l.runs * 8);
    l.o_cnt = o; o += r256(l.runs * 16);
    l.o_pre = o; o += r256(l.runs * 16);
    l.o_run_seg = o; o += r256(l.runs * 8);
    l.o_coef = o; o += r256(l.blocks * 128);
    l.total = o;
    return l;
}

struct Ws {
    Info *info;
    uint8_t *stream;
    int64_t *seg_byte;
    int *seg_run, *seg_done;
    int64_t *run_base, *coef_base, *totals;    // totals: runs, blocks, pixels
    St *X, *Y, *E, *Z;                        // Z: the other buffer of the relaxation passes
    RunCnt *cnt, *pre;
    int2 *run_seg;                             // (image, segment slot)
    int16_t *coef;
};

Ws carve(void *ws, const Layout &l) {
    char *b = (char *)ws;
    Ws w;
    w.info = (Info *)(b + l.o_info);
    w.stream = (uint8_t *)(b + l.o_stream);
    w.seg_byte = (int64_t *)(b + l.o_seg_byte);
    w.seg_run = (int *)(b + l.o_seg_run);
    w.seg_done = (int *)(b + l.o_seg_done);
    w.run_base = (int64_t *)(b + l.o_run_base);
    w.coef_base = (int64_t *)(b + l.o_coef_base);
    w.totals = (int64_t *)(b + l.o_totals);
    w.X = (St *)(b + l.o_X);
    w.Y = (St *)(b + l.o_Y);
    w.E = (St *)(b + l.o_E);
    w.Z = (St *)(b + l.o_Z);
    w.cnt = (RunCnt *)(b + l.o_cnt);
    w.pre = (RunCnt *)(b + l.o_pre);
    w.run_seg = (int2 *)(b + l.o_run_seg);
    w.coef = (int16_t *)(b + l.o_coef);
    return w;
}

__device__ __forceinline__ int64_t slot_base(const int64_t *off, int n) { return (off[n] - off[0]) / 2 + 3 * (int64_t)n; }

__device__ __forceinline__ int64_t seg_blocks(const Info &I, int64_t k) {
    const int64_t mcus = (int64_t)I.mcus_x * I.mcus_y;
    if (!I.ri) return mcus * I.bpm;
    const int64_t lo = k * I.ri, hi = lo + I.ri < mcus ? lo + I.ri : mcus;
    return (hi - lo) * I.bpm;
}

__global__ void jpeg_parse_kernel(const uint8_t *__restrict__ data, int64_t data_bytes, const int64_t *__restrict__ off, int N, int max_h,
                                  int max_w, Ws w, int *status) {
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= N) return;
    Info &I = w.info[n];
    const int64_t a = off[n], b = off[n + 1];
    if (off[0] < 0 || a < off[0] || b < a || b > data_bytes || (n > 0 && off[n - 1] > a)) {
        I.status = kBadOffsets;
    } else if (parse(data + a, b - a, I) == 0) {
        if (I.out_h > max_h || I.out_w > max_w || b - I.scan - a >= ((int64_t)1 << 27)) I.status = kTooLarge;
    }
    status[n] = I.status;
}

// one CTA: an image whose bytes start before the end of any earlier image's (offsets not non-decreasing over the whole batch)
// is flagged, so that no two images' scans are unstuffed into overlapping parts of the workspace
__global__ void __launch_bounds__(1024) jpeg_offsets_kernel(const int64_t *__restrict__ off, int N, Ws w, int *status) {
    using Scan = cub::BlockScan<int64_t, 1024>;
    __shared__ typename Scan::TempStorage tmp;
    __shared__ int64_t carry;
    if (threadIdx.x == 0) carry = off[0];
    __syncthreads();
    for (int n0 = 0; n0 < N; n0 += 1024) {
        const int n = n0 + threadIdx.x;
        const int64_t v = n < N ? off[n] : INT64_MIN;
        int64_t before, total;
        Scan(tmp).ExclusiveScan(v, before, cub::Max(), total);   // before: max of off[n0 .. n - 1]
        const int64_t m = threadIdx.x == 0 ? carry : (before > carry ? before : carry);
        if (n < N && (v < m || off[n + 1] < v)) {
            status[n] |= kBadOffsets;
            w.info[n].status |= kBadOffsets;
        }
        __syncthreads();
        if (threadIdx.x == 0 && total > carry) carry = total;
        __syncthreads();
    }
}

// one CTA per image: the scan bytes in tiles of kThreads * kTile, each thread classifying kTile consecutive bytes
__global__ void __launch_bounds__(kThreads) jpeg_split_kernel(const uint8_t *__restrict__ data, const int64_t *__restrict__ off, Ws w,
                                                              int *status) {
    using Scan = cub::BlockScan<int, kThreads>;
    using Reduce = cub::BlockReduce<int64_t, kThreads>;
    __shared__ union {
        typename Scan::TempStorage scan;
        typename Reduce::TempStorage red;
    } tmp;
    __shared__ int64_t s_end;
    __shared__ int s_bad, s_carry_data, s_carry_rst;
    const int n = blockIdx.x;
    Info &I = w.info[n];
    if (status[n]) {
        if (threadIdx.x == 0) { I.nseg = 0; I.runs = 0; }
        return;
    }
    const uint8_t *b = data + off[n] + I.scan;
    const int64_t m = off[n + 1] - off[n] - I.scan;
    uint8_t *out = w.stream + (off[n] - off[0]);
    const int64_t sb = slot_base(off, n);
    int64_t *seg_byte = w.seg_byte + sb;
    if (threadIdx.x == 0) { s_bad = 0; s_carry_data = 0; s_carry_rst = 0; seg_byte[0] = 0; }
    __syncthreads();
    for (int64_t t0 = 0; t0 < m; t0 += (int64_t)kThreads * kTile) {
        const int64_t i0 = t0 + (int64_t)threadIdx.x * kTile;
        int kind[kTile];
        int64_t my_end = INT64_MAX;
        for (int j = 0; j < kTile; ++j) {
            kind[j] = i0 + j < m ? classify(b, m, i0 + j) : kDrop;
            if (kind[j] == kEnd && my_end == INT64_MAX) my_end = i0 + j;
        }
        const int64_t tile_end = Reduce(tmp.red).Reduce(my_end, cub::Min());
        if (threadIdx.x == 0) s_end = tile_end;
        __syncthreads();
        const int64_t end = s_end;
        int packed = 0;
        for (int j = 0; j < kTile; ++j)
            if (i0 + j < end) packed += kind[j] == kData ? 1 : kind[j] == kRst ? (1 << 16) : 0;
        int before, total;
        Scan(tmp.scan).ExclusiveSum(packed, before, total);
        int dpos = s_carry_data + (before & 0xFFFF), rpos = s_carry_rst + (before >> 16);
        for (int j = 0; j < kTile; ++j) {
            if (i0 + j >= end) break;
            if (kind[j] == kData) out[dpos++] = b[i0 + j];
            else if (kind[j] == kRst) {
                if (b[i0 + j + 1] - 0xD0 != (rpos & 7)) s_bad = 1;
                ++rpos;
                seg_byte[rpos] = dpos;
            }
        }
        __syncthreads();
        if (threadIdx.x == 0) { s_carry_data += total & 0xFFFF; s_carry_rst += total >> 16; }
        __syncthreads();
        if (end != INT64_MAX) break;
    }
    const int nseg = s_carry_rst + 1;
    const int64_t mcus = (int64_t)I.mcus_x * I.mcus_y;
    const int64_t want = I.ri ? (mcus + I.ri - 1) / I.ri : 1;
    if (threadIdx.x == 0) {
        seg_byte[nseg] = s_carry_data;
        I.nseg = nseg;
        if (s_bad || nseg != want) atomicOr(status + n, kCorrupt);
    }
    __syncthreads();
    // runs per segment and their prefix sum
    int *seg_run = w.seg_run + sb;
    int *seg_done = w.seg_done + sb;
    __shared__ int s_runs;
    if (threadIdx.x == 0) s_runs = 0;
    __syncthreads();
    for (int k0 = 0; k0 < nseg; k0 += kThreads) {
        const int k = k0 + threadIdx.x;
        int nr = 0;
        if (k < nseg) {
            const int64_t bits = 8 * (seg_byte[k + 1] - seg_byte[k]);
            nr = bits > 0 ? (int)((bits + kRunBits - 1) / kRunBits) : 1;
            seg_done[k] = 0;
        }
        int before, total;
        Scan(tmp.scan).ExclusiveSum(nr, before, total);
        if (k < nseg) seg_run[k] = s_runs + before;
        __syncthreads();
        if (threadIdx.x == 0) s_runs += total;
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        seg_run[nseg] = s_runs;
        I.runs = s_runs;
    }
}

// one CTA: prefix sums over the images of output pixels and coefficient blocks (with the capacity flags), then of runs
__global__ void __launch_bounds__(1024) jpeg_layout_kernel(int N, int64_t pixel_cap, int64_t block_cap, Ws w, int64_t *image_offsets,
                                                           int *shapes, int *status) {
    using Scan = cub::BlockScan<int64_t, 1024>;
    __shared__ typename Scan::TempStorage tmp;
    __shared__ int64_t c_px, c_blk, c_run;
    __shared__ unsigned long long used_blk, used_px;   // ends of the accepted images' blocks and pixels (within the capacities)
    if (threadIdx.x == 0) c_px = c_blk = c_run = used_blk = used_px = 0;
    __syncthreads();
    for (int n0 = 0; n0 < N; n0 += 1024) {
        const int n = n0 + threadIdx.x;
        int64_t px = 0, blk = 0;
        if (n < N && status[n] == 0) {
            const Info &I = w.info[n];
            px = (int64_t)I.h * I.w;
            blk = (int64_t)I.mcus_x * I.mcus_y * I.bpm;
        }
        int64_t bpx, tpx, bblk, tblk;
        Scan(tmp).ExclusiveSum(px, bpx, tpx);
        __syncthreads();
        Scan(tmp).ExclusiveSum(blk, bblk, tblk);
        int st = n < N ? status[n] : 0;
        if (n < N) {
            bpx += c_px;
            bblk += c_blk;
            if (st == 0 && (bpx + px > pixel_cap || bblk + blk > block_cap)) st = kTooLarge;
            if (st) status[n] = st;
            else {
                atomicMax(&used_blk, (unsigned long long)(bblk + blk));
                atomicMax(&used_px, (unsigned long long)(bpx + px));
            }
            Info &I = w.info[n];
            I.out = bpx;
            I.coef = bblk;
            w.coef_base[n] = bblk;
            image_offsets[n] = 3 * bpx;
            shapes[2 * n] = st ? 0 : I.out_h;
            shapes[2 * n + 1] = st ? 0 : I.out_w;
        }
        const int64_t runs = n < N && st == 0 ? w.info[n].runs : 0;
        int64_t brun, trun;
        __syncthreads();
        Scan(tmp).ExclusiveSum(runs, brun, trun);
        if (n < N) {
            w.info[n].run_base = c_run + brun;
            w.run_base[n] = c_run + brun;
            if (st) w.info[n].runs = 0;
        }
        __syncthreads();
        if (threadIdx.x == 0) { c_px += tpx; c_blk += tblk; c_run += trun; }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        w.run_base[N] = c_run;
        w.coef_base[N] = c_blk;
        w.totals[0] = c_run;
        w.totals[1] = (int64_t)used_blk;                      // <= block_cap: the zero and IDCT passes stay in the workspace
        w.totals[2] = (int64_t)used_px;
    }
}

__global__ void jpeg_zero_kernel(Ws w) {
    const int64_t n = w.totals[1] * 8;                         // a block is 64 int16 = 8 int4
    int4 *p = (int4 *)w.coef;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) p[i] = make_int4(0, 0, 0, 0);
}

__device__ __forceinline__ int find_le(const int64_t *a, int n, int64_t v) {   // last i in [0, n) with a[i] <= v
    int lo = 0, hi = n - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (a[mid] <= v) lo = mid; else hi = mid - 1;
    }
    return lo;
}

struct RunPos {
    int n, k, j;                          // image, segment, run within the segment
    int64_t slot;                         // the segment's slot
    int64_t b0, b1, rs, re;               // segment bits, run bits
};

__device__ __forceinline__ RunPos run_pos(const Ws &w, const int64_t *off, int N, int64_t r, bool first_time) {
    RunPos p;
    if (first_time) {
        p.n = find_le(w.run_base, N, r);
        const Info &I = w.info[p.n];
        const int64_t sb = slot_base(off, p.n);
        const int rel = (int)(r - w.run_base[p.n]);
        int lo = 0, hi = I.nseg - 1;
        while (lo < hi) {
            const int mid = (lo + hi + 1) >> 1;
            if (w.seg_run[sb + mid] <= rel) lo = mid; else hi = mid - 1;
        }
        p.k = lo;
        p.slot = sb + lo;
        w.run_seg[r] = make_int2(p.n, (int)(p.slot - sb));
    } else {
        const int2 q = w.run_seg[r];
        p.n = q.x;
        p.k = q.y;
        p.slot = slot_base(off, p.n) + p.k;
    }
    p.j = (int)(r - w.run_base[p.n]) - w.seg_run[p.slot];
    p.b0 = 8 * w.seg_byte[p.slot];
    p.b1 = 8 * w.seg_byte[p.slot + 1];
    p.rs = p.b0 + (int64_t)p.j * kRunBits;
    p.re = p.rs + kRunBits < p.b1 ? p.rs + kRunBits : p.b1;
    return p;
}

// PHASE 1: X from the assumed state; 3: dst from src[r - 1]; 2: E = X[r - 1], Y, counts
template <int PHASE>
__global__ void __launch_bounds__(kThreads) jpeg_sync_kernel(const int64_t *__restrict__ off, int N, Ws w, const St *src, St *dst) {
    const int64_t total = w.totals[0];
    for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < total; r += (int64_t)gridDim.x * blockDim.x) {
        const RunPos p = run_pos(w, off, N, r, PHASE == 1);
        const Info &I = w.info[p.n];
        const uint8_t *s = w.stream + (off[p.n] - off[0]);
        const int64_t end = w.seg_byte[slot_base(off, p.n) + I.nseg];
        if (PHASE == 1) {
            St st{(int32_t)p.rs, 0, 0};
            decode_run<false>(I, s, end, p.b1, st, p.re);
            w.X[r] = st;
        } else if (PHASE == 3) {
            St st = p.j ? src[r - 1] : St{(int32_t)p.b0, 0, 0};
            decode_run<false>(I, s, end, p.b1, st, p.re);
            dst[r] = st;
        } else {
            St st = p.j ? w.X[r - 1] : St{(int32_t)p.b0, 0, 0};
            w.E[r] = st;
            const RunOut o = decode_run<false>(I, s, end, p.b1, st, p.re);
            w.Y[r] = st;
            w.cnt[r] = RunCnt{o.blocks, o.dc[0], o.dc[1], o.dc[2]};
        }
    }
}

// per segment (the thread of its first run): the runs in order; a run whose predecessor's true exit Y differs from the
// predecessor's assumed-state exit X is decoded again from Y.  Then the exclusive prefix sums of the block counts and DC sums.
__global__ void __launch_bounds__(kThreads) jpeg_walk_kernel(const int64_t *__restrict__ off, int N, Ws w) {
    const int64_t total = w.totals[0];
    for (int64_t r0 = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r0 < total; r0 += (int64_t)gridDim.x * blockDim.x) {
        const RunPos p = run_pos(w, off, N, r0, false);
        if (p.j != 0) continue;
        const Info &I = w.info[p.n];
        const uint8_t *s = w.stream + (off[p.n] - off[0]);
        const int64_t end = w.seg_byte[slot_base(off, p.n) + I.nseg];
        const int nr = w.seg_run[p.slot + 1] - w.seg_run[p.slot];
        RunCnt acc{0, 0, 0, 0};
        St prev = w.Y[r0];
        for (int j = 0; j < nr; ++j) {
            const int64_t r = r0 + j;
            RunCnt c = w.cnt[r];
            if (j > 0) {
                if (!same(prev, w.X[r - 1])) {
                    St st = prev;
                    w.E[r] = st;
                    const int64_t rs = p.b0 + (int64_t)j * kRunBits, re = rs + kRunBits < p.b1 ? rs + kRunBits : p.b1;
                    const RunOut o = decode_run<false>(I, s, end, p.b1, st, re);
                    c = RunCnt{o.blocks, o.dc[0], o.dc[1], o.dc[2]};
                    prev = st;
                } else {
                    prev = w.Y[r];
                }
            }
            w.pre[r] = acc;
            acc.blocks += c.blocks;
            acc.dc0 += c.dc0;
            acc.dc1 += c.dc1;
            acc.dc2 += c.dc2;
        }
    }
}

__global__ void __launch_bounds__(kThreads) jpeg_write_kernel(const int64_t *__restrict__ off, int N, Ws w, int *status) {
    const int64_t total = w.totals[0];
    for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < total; r += (int64_t)gridDim.x * blockDim.x) {
        const RunPos p = run_pos(w, off, N, r, false);
        const Info &I = w.info[p.n];
        const uint8_t *s = w.stream + (off[p.n] - off[0]);
        const int64_t end = w.seg_byte[slot_base(off, p.n) + I.nseg];
        const int64_t nb = seg_blocks(I, p.k);
        const int64_t seg_first = (I.ri ? (int64_t)p.k * I.ri * I.bpm : 0);
        if (seg_first + nb > (int64_t)I.mcus_x * I.mcus_y * I.bpm) continue;   // more segments than MCUs (flagged by the split)
        const RunCnt pc = w.pre[r];
        const int dc[3] = {pc.dc0, pc.dc1, pc.dc2};
        St st = w.E[r];
        const RunOut o = decode_run<true>(I, s, end, p.b1, st, p.re, w.coef + (w.coef_base[p.n] + seg_first) * 64, pc.blocks, nb, dc);
        if (o.err) atomicOr(status + p.n, kCorrupt);
        if (o.done) w.seg_done[p.slot] = 1;
    }
}

// one CTA per image: every segment completed its blocks; flagged images get shape (0, 0)
__global__ void __launch_bounds__(kThreads) jpeg_finish_kernel(const int64_t *__restrict__ off, Ws w, int *shapes, int *status) {
    const int n = blockIdx.x;
    if (status[n]) {
        if (threadIdx.x == 0) shapes[2 * n] = shapes[2 * n + 1] = 0;
        return;
    }
    const int nseg = w.info[n].nseg;
    const int64_t sb = slot_base(off, n);
    int bad = 0;
    for (int k = threadIdx.x; k < nseg; k += blockDim.x) bad |= !w.seg_done[sb + k];
    bad = __syncthreads_or(bad);
    if (threadIdx.x == 0 && bad) {
        status[n] |= kCorrupt;
        shapes[2 * n] = shapes[2 * n + 1] = 0;
    }
}

__global__ void __launch_bounds__(kThreads) jpeg_idct_kernel(int N, Ws w, const int *__restrict__ status) {
    const int64_t total = w.totals[1];
    for (int64_t b = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; b < total; b += (int64_t)gridDim.x * blockDim.x) {
        const int n = find_le(w.coef_base, N, b);
        if (status[n]) continue;
        const Info &I = w.info[n];
        int16_t *c = w.coef + b * 64;
        int16_t in[64];
        const int4 *c4 = (const int4 *)c;
        for (int i = 0; i < 8; ++i) ((int4 *)in)[i] = c4[i];
        uint8_t out[64];
        idct_islow(in, I.qt[I.mcu_comp[(b - w.coef_base[n]) % I.bpm]], out);
        for (int i = 0; i < 4; ++i) ((int4 *)c)[i] = ((const int4 *)out)[i];
    }
}

// grid (x, image): the image's output pixels
__global__ void __launch_bounds__(kThreads) jpeg_color_kernel(Ws w, const int *__restrict__ status, uint8_t *image_out) {
    const int n = blockIdx.y;
    if (status[n]) return;
    const Info &I = w.info[n];
    const uint8_t *blocks = (const uint8_t *)(w.coef + w.coef_base[n] * 64);
    const int64_t np = (int64_t)I.out_h * I.out_w;
    uint8_t *o = image_out + 3 * I.out;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < np; i += (int64_t)gridDim.x * blockDim.x) {
        uint8_t bgr[3];
        output_pixel(I, blocks, (int)(i / I.out_w), (int)(i % I.out_w), bgr);
        o[3 * i] = bgr[0];
        o[3 * i + 1] = bgr[1];
        o[3 * i + 2] = bgr[2];
    }
}

bool bad_sizes(int64_t N, int64_t B, int64_t P) { return N < 1 || N > 65535 || B < 0 || P < 0 || B > ((int64_t)1 << 40) || P > ((int64_t)1 << 40); }

}  // namespace

extern "C" {

int64_t mr_jpeg_workspace_bytes(int64_t N, int64_t byte_capacity, int64_t pixel_capacity) {
    if (bad_sizes(N, byte_capacity, pixel_capacity)) return 0;
    return layout(N, byte_capacity, pixel_capacity).total;
}

int mr_jpeg_decode(const void *data, int64_t data_bytes, const int64_t *data_offsets, int N, int max_h, int max_w, int64_t pixel_capacity,
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
    const int grid = 4 * sm_count();
    int rc;
    jpeg_parse_kernel<<<(int)ceil_div(N, 64), 64, 0, st>>>(d, data_bytes, data_offsets, N, max_h, max_w, w, status);
    if ((rc = check_launch("jpeg parse"))) return rc;
    jpeg_offsets_kernel<<<1, 1024, 0, st>>>(data_offsets, N, w, status);
    if ((rc = check_launch("jpeg offsets"))) return rc;
    jpeg_split_kernel<<<N, kThreads, 0, st>>>(d, data_offsets, w, status);
    if ((rc = check_launch("jpeg split"))) return rc;
    jpeg_layout_kernel<<<1, 1024, 0, st>>>(N, pixel_capacity, l.blocks, w, image_offsets, shapes, status);
    if ((rc = check_launch("jpeg layout"))) return rc;
    jpeg_zero_kernel<<<grid, kThreads, 0, st>>>(w);
    if ((rc = check_launch("jpeg zero"))) return rc;
    jpeg_sync_kernel<1><<<grid, kThreads, 0, st>>>(data_offsets, N, w, nullptr, nullptr);
    if ((rc = check_launch("jpeg sync 1"))) return rc;
    for (int i = 0; i < kRelax; ++i) {
        jpeg_sync_kernel<3><<<grid, kThreads, 0, st>>>(data_offsets, N, w, i & 1 ? w.Z : w.X, i & 1 ? w.X : w.Z);
        if ((rc = check_launch("jpeg sync relax"))) return rc;
    }
    static_assert(kRelax % 2 == 0, "the relaxation passes end in X");
    jpeg_sync_kernel<2><<<grid, kThreads, 0, st>>>(data_offsets, N, w, nullptr, nullptr);
    if ((rc = check_launch("jpeg sync 2"))) return rc;
    jpeg_walk_kernel<<<grid, kThreads, 0, st>>>(data_offsets, N, w);
    if ((rc = check_launch("jpeg walk"))) return rc;
    jpeg_write_kernel<<<grid, kThreads, 0, st>>>(data_offsets, N, w, status);
    if ((rc = check_launch("jpeg write"))) return rc;
    jpeg_finish_kernel<<<N, kThreads, 0, st>>>(data_offsets, w, shapes, status);
    if ((rc = check_launch("jpeg finish"))) return rc;
    jpeg_idct_kernel<<<grid, kThreads, 0, st>>>(N, w, status);
    if ((rc = check_launch("jpeg idct"))) return rc;
    const int gx = (int)std::max<int64_t>(1, std::min<int64_t>(64, pixel_capacity / ((int64_t)N * 4 * kThreads)));
    jpeg_color_kernel<<<dim3(gx, N), kThreads, 0, st>>>(w, status, image_out);
    return check_launch("jpeg color");
}

}  // extern "C"
