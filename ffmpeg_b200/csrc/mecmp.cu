// mecmp.cu — libavcodec me_cmp SAD/SSE block compare and the exhaustive motion search on sm_90a (C ABI: "me_cmp").
//
// Reference semantics reproduced bit-for-bit (checker: oracle/mecmp_oracle.c):
//   pix_abs16_c / pix_abs8_c, *_x2 / _y2 / _xy2   libavcodec/me_cmp.c:114-385
//   sse16_c / sse8_c / sse4_c                     libavcodec/me_cmp.c:37-103
//   hadamard8_diff8x8_c, hadamard8_diff16_c       libavcodec/me_cmp.c:514-562, 933-950 (SATD)
//   hadamard8_intra8x8_c / 16, vsad, vsse (+ intra), nsse, pix_median_abs, sum_abs_dctelem   libavcodec/me_cmp.c:105-112, 145-183,
//                                                 292-330, 387-437, 564-612, 843-931 (the context-free members of MECmpContext)
//   ff_me_cmp_sad, ff_me_search_esa               libavfilter/motion_estimation.c:60-97 (driver vf_mestimate.c:85-127)
//
// ESA kernel: one CTA per macroblock.  The current block and the clipped search window of the reference frame are
// staged in shared memory once (coalesced row reads); every thread then scores candidates with VABSDIFF4 (4 bytes per
// instruction, unaligned candidate rows are re-assembled from two words with PRMT).  The winner is a 64-bit key
// (cost, not-the-zero-vector, raster index) reduced with warp shuffles: strict '<' in raster order with the zero
// vector tested first is exactly "smallest key".  This search is integer-ALU bound (about 2100 op/byte), not HBM bound.
#include "common.h"
#include "mecmp_dct.h"
#include <cstring>
#include <cstdlib>

namespace {

__device__ __forceinline__ int px_ref(const uint8_t *b, long long stride, int x, int mode)
{
    switch (mode) {
    case 0:  return b[x];
    case 1:  return (b[x] + b[x + 1] + 1) >> 1;
    case 2:  return (b[x] + b[x + stride] + 1) >> 1;
    default: return (b[x] + b[x + 1] + b[x + stride] + b[x + stride + 1] + 2) >> 2;
    }
}

// one warp per comparison; lane = column (w <= 16 -> two rows per pass)
__global__ void __launch_bounds__(256)
me_cmp_kernel(int fn, int w, int mode, const uint8_t *f1, const uint8_t *f2, long long stride, int h,
              const int64_t *off1, const int64_t *off2, long long n, int32_t *out)
{
    const long long i = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (i >= n) return;
    const int lane = threadIdx.x & 31;
    const uint8_t *a = f1 + off1[i], *b = f2 + off2[i];
    const int rows_per_pass = 32 / w, x = lane % w, r0 = lane / w;
    int s = 0;
    for (int y = r0; y < h; y += rows_per_pass) {
        const int pa = a[y * stride + x];
        const int pb = px_ref(b + y * stride, stride, x, mode);
        const int d = pa - pb;
        s += fn == B200_MECMP_SSE ? d * d : abs(d);
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) out[i] = s;
}

// hadamard8_diff (SATD): one warp per comparison, 8 lanes per 8x8 block, lane = one row of differences.  The row transform
// runs in the lane's registers, the column transform across the 8 lanes with xor-shuffles; the sum of absolute values of
// the 64 coefficients does not depend on the butterfly order (exact integers), so this equals the reference's result.
// nblk = 1 (8 wide), 2 (16 wide, h = 8) or 4 (16 wide, h = 16).
__global__ void __launch_bounds__(256)
me_satd_kernel(int nblk, const uint8_t *f1, const uint8_t *f2, long long stride, const int64_t *off1, const int64_t *off2,
               long long n, int32_t *out, int intra = 0)
{
    const long long i = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (i >= n) return;
    const int lane = threadIdx.x & 31, blk = lane >> 3, row = lane & 7;
    int s = 0;
    const bool on = blk < nblk;
    int v[8];
    {
        const long long o = (long long)((blk >> 1) * 8 + row) * stride + (blk & 1) * 8;
        const uint8_t *a = f1 + off1[i] + o, *b = f2 + off2[i] + o;
#pragma unroll
        for (int k = 0; k < 8; k++) v[k] = !on ? 0 : intra ? (int)a[k] : (int)b[k] - (int)a[k];      // src - dst, like the reference; intra: the block itself
    }
#pragma unroll
    for (int span = 1; span < 8; span <<= 1)
#pragma unroll
        for (int k = 0; k < 8; k++)
            if (!(k & span)) { const int x = v[k], y = v[k + span]; v[k] = x + y; v[k + span] = x - y; }
#pragma unroll
    for (int span = 1; span < 8; span <<= 1)
#pragma unroll
        for (int k = 0; k < 8; k++) {
            const int other = __shfl_xor_sync(0xffffffffu, v[k], span);
            v[k] = (row & span) ? other - v[k] : v[k] + other;
        }
#pragma unroll
    for (int k = 0; k < 8; k++) s += abs(v[k]);
    if (intra && row == 0) s -= abs(v[0]);                        // hadamard8_intra: coefficient (0, 0) of each 8x8 block (the mean) is left out
#pragma unroll
    for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) out[i] = s;
}

// vsad / vsse (+ intra), nsse, median_sad: one warp per comparison, a lane per pixel (w * h <= 256 pixels in 8 rounds); every term
// only looks at the pixel itself and its right / lower / upper-left neighbours, read straight from the frames.
__device__ __forceinline__ int mid3(int a, int b, int c)
{
    return max(min(a, b), min(max(a, b), c));
}
__global__ void __launch_bounds__(256)
me_cmp2_kernel(int fn, int w, int intra, int weight, const uint8_t *f1, const uint8_t *f2, long long stride, int h,
               const int64_t *off1, const int64_t *off2, long long n, int32_t *out)
{
    const long long i = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (i >= n) return;
    const int lane = threadIdx.x & 31;
    const uint8_t *a = f1 + off1[i], *b = f2 + off2[i];
    int s1 = 0, s2 = 0;
    for (int p = lane; p < w * h; p += 32) {
        const int y = p / w, x = p - y * w;
        const uint8_t *pa = a + y * stride + x, *pb = b + y * stride + x;
        if (fn == B200_MECMP_VSAD || fn == B200_MECMP_VSSE) {
            if (y + 1 < h) {
                const int d = intra ? (int)pa[0] - (int)pa[stride] : (int)pa[0] - (int)pb[0] - (int)pa[stride] + (int)pb[stride];
                s1 += fn == B200_MECMP_VSSE ? d * d : abs(d);
            }
        } else if (fn == B200_MECMP_NSSE) {
            const int d = (int)pa[0] - (int)pb[0];
            s1 += d * d;
            if (y + 1 < h && x + 1 < w)
                s2 += abs((int)pa[0] - (int)pa[stride] - (int)pa[1] + (int)pa[stride + 1]) -
                      abs((int)pb[0] - (int)pb[stride] - (int)pb[1] + (int)pb[stride + 1]);
        } else {                                                   // median_sad
            const int v = (int)pa[0] - (int)pb[0];
            int pred = 0;
            if (y == 0) pred = x ? (int)pa[-1] - (int)pb[-1] : 0;
            else {
                const int top = (int)pa[-stride] - (int)pb[-stride];
                if (x == 0) pred = top;
                else {
                    const int left = (int)pa[-1] - (int)pb[-1], tl = (int)pa[-stride - 1] - (int)pb[-stride - 1];
                    pred = mid3(top, left, top + left - tl);
                }
            }
            s1 += abs(v - pred);
        }
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) { s1 += __shfl_xor_sync(0xffffffffu, s1, o); s2 += __shfl_xor_sync(0xffffffffu, s2, o); }
    if (lane == 0) out[i] = fn == B200_MECMP_NSSE ? s1 + abs(s2) * weight : s1;
}

// sum_abs_dctelem: one warp per block of 64 coefficients
__global__ void __launch_bounds__(256)
sum_abs_dctelem_kernel(const int16_t *blocks, long long n, int32_t *out)
{
    const long long i = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (i >= n) return;
    const int lane = threadIdx.x & 31;
    const unsigned wv = reinterpret_cast<const unsigned *>(blocks + 64 * i)[lane];
    int s = abs((int)(short)(wv & 0xffff)) + abs((int)wv >> 16);
#pragma unroll
    for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) out[i] = s;
}

// ---------------------------------------------------------------- exhaustive search
constexpr int ESA_THREADS = 256;

template <int MB>
__global__ void __launch_bounds__(ESA_THREADS)
esa_kernel(const uint8_t *cur, const uint8_t *ref, int linesize, long long frame_stride, int b_w, int b_h,
           int search, int win_pitch /* words */, int32_t *out_mv, unsigned long long *out_cost)
{
    extern __shared__ unsigned smem[];
    unsigned *scur = smem;                         // MB rows x MB/4 words
    unsigned *swin = smem + MB * (MB / 4);         // window rows x win_pitch words
    __shared__ unsigned long long best[ESA_THREADS / 32];

    const int bx = blockIdx.x, by = blockIdx.y;
    const long long f = blockIdx.z;
    const int x_mb = bx * MB, y_mb = by * MB;
    const int gx_max = (b_w - 1) * MB, gy_max = (b_h - 1) * MB;
    const int x0 = max(x_mb - search, 0), y0 = max(y_mb - search, 0);
    const int x1 = min(x_mb + search, gx_max), y1 = min(y_mb + search, gy_max);
    const int nx = x1 - x0 + 1, ny = y1 - y0 + 1;
    const int wrows = ny + MB - 1, wcols = nx + MB - 1;            // bytes of the window actually needed
    const uint8_t *c = cur + f * frame_stride + (long long)y_mb * linesize + x_mb;
    const uint8_t *r = ref + f * frame_stride + (long long)y0 * linesize + x0;

    // stage: bytes are written individually into the word arrays (little endian), rows padded to win_pitch words
    uint8_t *scur8 = reinterpret_cast<uint8_t *>(scur), *swin8 = reinterpret_cast<uint8_t *>(swin);
    for (int i = threadIdx.x; i < MB * MB; i += ESA_THREADS) scur8[i] = c[(long long)(i / MB) * linesize + (i % MB)];
    const int wpb = win_pitch * 4;
    for (int i = threadIdx.x; i < wrows * wpb; i += ESA_THREADS) {
        const int yy = i / wpb, xx = i - yy * wpb;
        swin8[i] = xx < wcols ? r[(long long)yy * linesize + xx] : 0;
    }
    __syncthreads();

    // Four horizontally adjacent candidates per thread and pass: they share the window words of every row (5 loads for
    // 4 x 16 pixels) and the current-block words; candidate s is re-aligned with PRMT (s = 0 needs none).
    unsigned long long mine = ~0ull;
    const int ngx = (nx + 3) >> 2, ngroups = ngx * ny;
    for (int g = threadIdx.x; g < ngroups; g += ESA_THREADS) {
        const int cy = g / ngx, gx = g - cy * ngx;
        const int cx0 = gx * 4, wq = gx;
        unsigned sad0 = 0, sad1 = 0, sad2 = 0, sad3 = 0;
#pragma unroll 2
        for (int j = 0; j < MB; j++) {
            const unsigned *row = swin + (cy + j) * win_pitch + wq;
            const unsigned *crow = scur + j * (MB / 4);
            unsigned lo = row[0];
#pragma unroll
            for (int q = 0; q < MB / 4; q++) {
                const unsigned hi = row[q + 1], cw = crow[q];
                sad0 = __vsadu4(lo, cw) + sad0;
                sad1 = __vsadu4(__byte_perm(lo, hi, 0x4321), cw) + sad1;
                sad2 = __vsadu4(__byte_perm(lo, hi, 0x5432), cw) + sad2;
                sad3 = __vsadu4(__byte_perm(lo, hi, 0x6543), cw) + sad3;
                lo = hi;
            }
        }
        const unsigned sads[4] = { sad0, sad1, sad2, sad3 };
#pragma unroll
        for (int sft = 0; sft < 4; sft++) {
            const int cx = cx0 + sft;
            if (cx < nx) {
                const int ax = x0 + cx, ay = y0 + cy;
                const unsigned notzero = (ax == x_mb && ay == y_mb) ? 0u : 1u;
                const unsigned long long key = ((unsigned long long)sads[sft] << 32) | ((unsigned long long)notzero << 31) | (unsigned)(cy * nx + cx);
                mine = key < mine ? key : mine;
            }
        }
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        const unsigned long long other = __shfl_xor_sync(0xffffffffu, mine, o);
        mine = other < mine ? other : mine;
    }
    if ((threadIdx.x & 31) == 0) best[threadIdx.x >> 5] = mine;
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned long long m = best[0];
        for (int i = 1; i < ESA_THREADS / 32; i++) m = best[i] < m ? best[i] : m;
        const int k = (int)(m & 0x7fffffffu);
        const int cy = k / nx, cx = k - cy * nx;
        const long long o = (f * b_h + by) * b_w + bx;
        out_mv[2 * o] = x0 + cx;
        out_mv[2 * o + 1] = y0 + cy;
        out_cost[o] = m >> 32;
    }
}

// ---------------------------------------------------------------- exhaustive search, second kernel
// The first kernel spends 2.3 instructions per VABSDIFF4 in its inner loop: every candidate row is re-assembled from two window words
// with PRMT and every window / current-block word is fetched again for every group of four candidates.  Here
//  * the window is kept in shared memory four times, once per byte phase (copy s holds the window shifted left by s bytes, built from
//    copy 0 with funnel shifts), so a candidate at any column reads aligned words and needs no PRMT at all;
//  * a task is ESA2_NV vertically adjacent candidates of one column: a window row, once loaded, is compared with the ESA2_NV rows of
//    the current block it can face (rows i, i-1, ... of the block for candidates 0, 1, ...), and each row of the current block is
//    loaded once per task (a broadcast LDS.128) and kept in a ring of ESA2_NV rows.  Per window row of a task: 4 + 1 loads, 32
//    VABSDIFF4.U8.ACC: 1.2 instructions per useful one;
//  * a CTA owns MBS horizontally adjacent macroblocks: their windows overlap by all but 16 columns, and 2 x 585 tasks spread over
//    256 threads leave fewer idle slots in the last round than 585 do.
// Key, tie-breaks and outputs are those of esa_kernel.
constexpr int ESA2_THREADS = 256;
constexpr int ESA2_NV = 8;

template <int MB, int MBS>
__global__ void __launch_bounds__(ESA2_THREADS)
esa2_kernel(const uint8_t *cur, const uint8_t *ref, int linesize, long long frame_stride, int b_w, int b_h, int search,
            int pitch /* words per window row */, int copy_words /* words per phase copy */, int32_t *out_mv, unsigned long long *out_cost)
{
    constexpr int WPR = MB / 4;                                    // words per block row
    extern __shared__ unsigned smem[];
    unsigned *scur = smem;                                         // [MBS][MB][WPR]
    unsigned *swin = smem + MBS * MB * WPR;                        // [4][copy_words]
    __shared__ unsigned long long best[MBS][ESA2_THREADS / 32];

    const int bx0 = blockIdx.x * MBS, by = blockIdx.y;
    const long long f = blockIdx.z;
    const int nm = min(MBS, b_w - bx0);
    const int y_mb = by * MB;
    const int gx_max = (b_w - 1) * MB, gy_max = (b_h - 1) * MB;
    const int y0 = max(y_mb - search, 0), y1 = min(y_mb + search, gy_max), ny = y1 - y0 + 1;
    int xmb[MBS], x0[MBS], nx[MBS];
#pragma unroll
    for (int m = 0; m < MBS; m++) {
        xmb[m] = (bx0 + min(m, nm - 1)) * MB;
        x0[m] = max(xmb[m] - search, 0);
        nx[m] = min(xmb[m] + search, gx_max) - x0[m] + 1;
    }
    const int xs = x0[0];
    const int wcols = x0[nm - 1] + nx[nm - 1] - 1 + MB - xs;      // bytes of the joint window
    const int wrows = ny + MB - 1, trows = wrows + ESA2_NV - 1;    // rows a task of the last group may touch (the extra ones are zero)
    const uint8_t *r = ref + f * frame_stride + (long long)y0 * linesize + xs;

    // ---- stage the current blocks and phase 0 of the window
    for (int i = threadIdx.x; i < nm * MB * WPR; i += ESA2_THREADS) {
        const int m = i / (MB * WPR), rem = i - m * (MB * WPR), row = rem / WPR, q = rem - row * WPR;
        const uint8_t *c = cur + f * frame_stride + (long long)(y_mb + row) * linesize + xmb[m] + 4 * q;
        scur[i] = (unsigned)c[0] | (unsigned)c[1] << 8 | (unsigned)c[2] << 16 | (unsigned)c[3] << 24;
    }
    const bool al4 = ((reinterpret_cast<uintptr_t>(r) | (unsigned)linesize) & 3) == 0;
    for (int i = threadIdx.x; i < trows * pitch; i += ESA2_THREADS) {
        const int yy = i / pitch, k = i - yy * pitch;
        unsigned w = 0;
        if (yy < wrows) {
            const uint8_t *p = r + (long long)yy * linesize + 4 * k;
            if (al4 && 4 * k + 3 < wcols) w = __ldg(reinterpret_cast<const unsigned *>(p));
            else
                for (int b = 0; b < 4; b++) if (4 * k + b < wcols) w |= (unsigned)__ldg(p + b) << (8 * b);
        }
        swin[i] = w;
    }
    if (threadIdx.x == 0) swin[trows * pitch] = 0;                  // the word the last funnel shift reads
    __syncthreads();
    for (int i = threadIdx.x; i < trows * pitch; i += ESA2_THREADS) {
        const unsigned w0 = swin[i], w1 = swin[i + 1];
        swin[copy_words + i] = __funnelshift_r(w0, w1, 8);
        swin[2 * copy_words + i] = __funnelshift_r(w0, w1, 16);
        swin[3 * copy_words + i] = __funnelshift_r(w0, w1, 24);
    }
    __syncthreads();

    // ---- tasks: (macroblock m, row group gy, column cx), columns fastest so that a warp reads consecutive words of the four copies
    const int ng = (ny + ESA2_NV - 1) / ESA2_NV;
    const int ntask0 = nx[0] * ng, ntasks = ntask0 + (nm > 1 ? nx[MBS - 1] * ng : 0);
    unsigned long long mine[MBS];
#pragma unroll
    for (int m = 0; m < MBS; m++) mine[m] = ~0ull;
    for (int t = threadIdx.x; t < ntasks; t += ESA2_THREADS) {
        const int m = (MBS > 1 && t >= ntask0) ? 1 : 0;
        const int local = t - (m ? ntask0 : 0);
        const int nxm = m ? nx[MBS - 1] : nx[0], x0m = m ? x0[MBS - 1] : x0[0], xmbm = m ? xmb[MBS - 1] : xmb[0];
        const int gy = local / nxm, cx = local - gy * nxm;
        const int wx = x0m - xs + cx;
        const unsigned *wrow = swin + (wx & 3) * copy_words + gy * ESA2_NV * pitch + (wx >> 2);
        const unsigned *crow = scur + m * (MB * WPR);
        unsigned sad[ESA2_NV], C[ESA2_NV][WPR];
#pragma unroll
        for (int c = 0; c < ESA2_NV; c++) sad[c] = 0;
#pragma unroll
        for (int i = 0; i < MB + ESA2_NV - 1; i++) {
            unsigned W[WPR];
#pragma unroll
            for (int q = 0; q < WPR; q++) W[q] = wrow[q];
            wrow += pitch;
            if (i < MB) {
#pragma unroll
                for (int q = 0; q < WPR; q++) C[i % ESA2_NV][q] = crow[i * WPR + q];
            }
#pragma unroll
            for (int c = 0; c < ESA2_NV; c++) {
                const int j = i - c;
                if (j >= 0 && j < MB) {
#pragma unroll
                    for (int q = 0; q < WPR; q++) sad[c] = __vsadu4(W[q], C[j % ESA2_NV][q]) + sad[c];
                }
            }
        }
        unsigned long long bestk = ~0ull;
#pragma unroll
        for (int c = 0; c < ESA2_NV; c++) {
            const int cy = gy * ESA2_NV + c;
            if (cy < ny) {
                const int ax = x0m + cx, ay = y0 + cy;
                const unsigned notzero = (ax == xmbm && ay == y_mb) ? 0u : 1u;
                const unsigned long long key = ((unsigned long long)sad[c] << 32) | ((unsigned long long)notzero << 31) | (unsigned)(cy * nxm + cx);
                bestk = key < bestk ? key : bestk;
            }
        }
        if (MBS > 1 && m) mine[MBS - 1] = bestk < mine[MBS - 1] ? bestk : mine[MBS - 1];
        else mine[0] = bestk < mine[0] ? bestk : mine[0];
    }
#pragma unroll
    for (int m = 0; m < MBS; m++) {
#pragma unroll
        for (int o = 16; o; o >>= 1) {
            const unsigned long long other = __shfl_xor_sync(0xffffffffu, mine[m], o);
            mine[m] = other < mine[m] ? other : mine[m];
        }
        if ((threadIdx.x & 31) == 0) best[m][threadIdx.x >> 5] = mine[m];
    }
    __syncthreads();
    if (threadIdx.x < nm) {
        const int m = threadIdx.x;
        unsigned long long mm = best[m][0];
        for (int i = 1; i < ESA2_THREADS / 32; i++) mm = best[m][i] < mm ? best[m][i] : mm;
        const int nxm = m ? nx[MBS - 1] : nx[0], x0m = m ? x0[MBS - 1] : x0[0];
        const int k = (int)(mm & 0x7fffffffu);
        const int cy = k / nxm, cx = k - cy * nxm;
        const long long o = (f * b_h + by) * b_w + bx0 + m;
        out_mv[2 * o] = x0m + cx;
        out_mv[2 * o + 1] = y0 + cy;
        out_cost[o] = mm >> 32;
    }
}

template <int MB>
int launch_esa(cudaStream_t st, const uint8_t *cur, const uint8_t *ref, int linesize, long long fs, int b_w, int b_h,
               int nframes, int search, int32_t *mv, unsigned long long *cost)
{
    // the second kernel while its four copies of the joint window fit in 100 KB of shared memory (up to search 64 for 16 x 16
    // blocks), the first one for wider windows
    constexpr int MBS = 2;
    const int wc = 2 * search + MB * MBS;                    // widest joint window in bytes
    const int pitch = (wc + 3) / 4 + 1;
    const int trows = 2 * search + MB + ESA2_NV - 1;
    int copy_words = trows * pitch + 1;
    copy_words += (8 - (copy_words & 31) + 32) & 31;         // copies 8 banks apart: the four phases of 8 neighbouring columns hit 32 banks
    const size_t smem2 = ((size_t)MBS * MB * (MB / 4) + 4 * (size_t)copy_words) * 4;
    if (smem2 <= 100 * 1024) {
        if (smem2 > 48 * 1024)
            B200_CUDA_OK(cudaFuncSetAttribute(esa2_kernel<MB, MBS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem2));
        for (int f0 = 0; f0 < nframes; f0 += 65535) {
            const int nf = nframes - f0 < 65535 ? nframes - f0 : 65535;
            dim3 grid((b_w + MBS - 1) / MBS, b_h, nf);
            esa2_kernel<MB, MBS><<<grid, ESA2_THREADS, smem2, st>>>(cur + (long long)f0 * fs, ref + (long long)f0 * fs, linesize, fs, b_w, b_h,
                                                                    search, pitch, copy_words, mv + 2LL * f0 * b_w * b_h, cost + (long long)f0 * b_w * b_h);
            B200_LAUNCHED();
        }
        B200_CUDA_OK(cudaGetLastError());
        return 0;
    }
    const int wcols = 2 * search + MB;                           // widest window in bytes
    const int win_pitch = (wcols + 3) / 4 + 1;                   // +1 word: the PRMT pair read one past the last needed word
    const size_t smem = ((size_t)MB * (MB / 4) + (size_t)(2 * search + MB) * win_pitch) * 4;
    if (smem > 200 * 1024) return B200_ENOSYS;
    if (smem > 48 * 1024)
        B200_CUDA_OK(cudaFuncSetAttribute(esa_kernel<MB>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    for (int f0 = 0; f0 < nframes; f0 += 65535) {
        const int nf = nframes - f0 < 65535 ? nframes - f0 : 65535;
        dim3 grid(b_w, b_h, nf);
        esa_kernel<MB><<<grid, ESA_THREADS, smem, st>>>(cur + (long long)f0 * fs, ref + (long long)f0 * fs, linesize, fs, b_w, b_h,
                                                        search, win_pitch, mv + 2LL * f0 * b_w * b_h, cost + (long long)f0 * b_w * b_h);
        B200_LAUNCHED();
    }
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

std::atomic<int> g_nsse_weight{8};                               // nsse: the reference's NULL-context weight (me_cmp.c:407-410)

int decode(int fn, int idx, int *w, int *mode)
{
    *mode = 0;
    if (fn == B200_MECMP_SAD) { if (idx < 0 || idx > 1) return B200_EINVAL; *w = 16 >> idx; return 0; }
    if (fn == B200_MECMP_SSE) { if (idx < 0 || idx > 2) return B200_EINVAL; *w = 16 >> idx; return 0; }
    if (fn == B200_MECMP_PIX_ABS) { if (idx < 0 || idx > 7) return B200_EINVAL; *w = idx < 4 ? 16 : 8; *mode = idx & 3; return 0; }
    if (fn == B200_MECMP_HADAMARD8) { if (idx != 0 && idx != 1 && idx != 4 && idx != 5) return B200_EINVAL; *w = 16 >> (idx & 1); *mode = idx >= 4; return 0; }
    if (fn == B200_MECMP_VSAD || fn == B200_MECMP_VSSE) { if (idx != 0 && idx != 1 && idx != 4 && idx != 5) return B200_EINVAL; *w = 16 >> (idx & 1); *mode = idx >= 4; return 0; }
    if (fn == B200_MECMP_NSSE || fn == B200_MECMP_MEDIAN_SAD) { if (idx < 0 || idx > 1) return B200_EINVAL; *w = 16 >> idx; return 0; }
    if (fn == B200_MECMP_DCT_SAD || fn == B200_MECMP_DCT_MAX || fn == B200_MECMP_DCT264_SAD) { if (idx < 0 || idx > 1) return B200_EINVAL; *w = 16 >> idx; return 0; }   // mecmp_dct.cu
    return B200_EINVAL;
}

} // namespace

B200_API int b200_me_cmp_batch_device(B200Device *dev, int fn, int idx, const uint8_t *frame1, const uint8_t *frame2,
                                      ptrdiff_t stride, int h, const int64_t *off1, const int64_t *off2, int64_t n, int32_t *out)
{
    if (!dev || !frame1 || !frame2 || !off1 || !off2 || !out || n < 0 || h < 0) return B200_EINVAL;
    int w, mode;
    int ret = decode(fn, idx, &w, &mode);
    if (ret < 0) return ret;
    if (n == 0) return 0;
    if (int r = b200_use_device(dev)) return r;
    const long long blocks = (n + 7) / 8;
    if (blocks > 0x7fffffffLL) return B200_EINVAL;
    if (fn >= B200_MECMP_DCT_SAD)                                 // 8x8 blocks like hadamard8_diff: two of them, four when h == 16
        mecmp_dct_launch(dev->stream, (unsigned)blocks, 256, fn, w, h, frame1, frame2, stride, off1, off2, n, out);
    else if (fn == B200_MECMP_HADAMARD8)                          // 8 wide ignores h; 16 wide: two blocks, four when h == 16
        me_satd_kernel<<<(unsigned)blocks, 256, 0, dev->stream>>>(w == 8 ? 1 : h == 16 ? 4 : 2, frame1, frame2, stride, off1, off2, n, out, mode);
    else if (fn >= B200_MECMP_VSAD) {
        if (w * h > 256) return B200_EINVAL;
        me_cmp2_kernel<<<(unsigned)blocks, 256, 0, dev->stream>>>(fn, w, mode, g_nsse_weight.load(), frame1, frame2, stride, h, off1, off2, n, out);
    } else
    me_cmp_kernel<<<(unsigned)blocks, 256, 0, dev->stream>>>(fn, w, mode, frame1, frame2, stride, h, off1, off2, n, out);
    B200_LAUNCHED();
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

B200_API int b200_me_esa_device(B200Device *dev, const uint8_t *cur, const uint8_t *ref, int linesize, int width, int height,
                                int64_t frame_stride, int nframes, int mb_size, int search_param, int32_t *out_mv, uint64_t *out_cost)
{
    if (!dev || !cur || !ref || !out_mv || !out_cost || nframes < 0 || search_param < 0 || width <= 0 || height <= 0) return B200_EINVAL;
    if (mb_size != 4 && mb_size != 8 && mb_size != 16) return B200_ENOSYS;
    const int b_w = width / mb_size, b_h = height / mb_size;
    if (b_w == 0 || b_h == 0) return B200_EINVAL;                 // vf_mestimate.c:93-94
    if (b_h > 65535) return B200_ENOSYS;
    if (nframes == 0) return 0;
    if (int r = b200_use_device(dev)) return r;
    unsigned long long *cost = reinterpret_cast<unsigned long long *>(out_cost);
    switch (mb_size) {
    case 4:  return launch_esa<4>(dev->stream, cur, ref, linesize, frame_stride, b_w, b_h, nframes, search_param, out_mv, cost);
    case 8:  return launch_esa<8>(dev->stream, cur, ref, linesize, frame_stride, b_w, b_h, nframes, search_param, out_mv, cost);
    default: return launch_esa<16>(dev->stream, cur, ref, linesize, frame_stride, b_w, b_h, nframes, search_param, out_mv, cost);
    }
}

// HOST buffers: frame pairs are cut into chunks that rotate over the device's three pipeline streams (H2D of the current and the
// reference luma planes, the search kernel, D2H of vectors and costs).
B200_API int b200_me_esa_host(B200Device *dev, const uint8_t *cur, const uint8_t *ref, int linesize, int width, int height,
                              int64_t frame_stride, int nframes, int mb_size, int search_param, int32_t *out_mv, uint64_t *out_cost)
{
    if (!dev || !cur || !ref || !out_mv || !out_cost || nframes < 0 || search_param < 0 || width <= 0 || height <= 0) return B200_EINVAL;
    if (mb_size != 4 && mb_size != 8 && mb_size != 16) return B200_ENOSYS;
    if (linesize < width || frame_stride < (int64_t)linesize * height) return B200_EINVAL;
    const int b_w = width / mb_size, b_h = height / mb_size;
    if (b_w == 0 || b_h == 0) return B200_EINVAL;
    if (b_h > 65535) return B200_ENOSYS;
    if (nframes == 0) return 0;
    B200_CUDA_OK(cudaSetDevice(dev->ordinal));
    const size_t fbytes = (size_t)frame_stride, nmb = (size_t)b_w * b_h;
    const size_t outb = ((nmb * 16) + 255) & ~(size_t)255;          // 2 x int32 + uint64 per block
    const size_t perFrame = 2 * fbytes + outb;
    int chunk = (int)(((size_t)96 << 20) / perFrame);
    if (chunk < 1) chunk = 1;
    if (chunk > nframes) chunk = nframes;
    const int K = B200Device::kPipe;
    B200_LOCK_DEVICE(dev);
    uint8_t *scr = (uint8_t *)b200_scratch(dev, (perFrame * chunk + 256) * K);
    if (!scr) return B200_ENOMEM;
    B200_CUDA_OK(cudaStreamSynchronize(dev->stream));
    int slot = 0;
    for (int f0 = 0; f0 < nframes; f0 += chunk, slot = (slot + 1) % K) {
        const int nf = nframes - f0 < chunk ? nframes - f0 : chunk;
        cudaStream_t st = dev->pipe[slot];
        uint8_t *base = scr + (size_t)slot * (perFrame * chunk + 256);
        uint8_t *dcur = base, *dref = base + fbytes * chunk;
        unsigned long long *dcost = (unsigned long long *)(((uintptr_t)(base + 2 * fbytes * chunk) + 255) & ~(uintptr_t)255);
        int32_t *dmv = (int32_t *)(dcost + nmb * chunk);
        B200_CUDA_OK(cudaMemcpyAsync(dcur, cur + (size_t)f0 * fbytes, (size_t)nf * fbytes, cudaMemcpyHostToDevice, st));
        B200_CUDA_OK(cudaMemcpyAsync(dref, ref + (size_t)f0 * fbytes, (size_t)nf * fbytes, cudaMemcpyHostToDevice, st));
        int ret;
        switch (mb_size) {
        case 4:  ret = launch_esa<4>(st, dcur, dref, linesize, frame_stride, b_w, b_h, nf, search_param, dmv, dcost); break;
        case 8:  ret = launch_esa<8>(st, dcur, dref, linesize, frame_stride, b_w, b_h, nf, search_param, dmv, dcost); break;
        default: ret = launch_esa<16>(st, dcur, dref, linesize, frame_stride, b_w, b_h, nf, search_param, dmv, dcost); break;
        }
        if (ret < 0) return ret;
        B200_CUDA_OK(cudaMemcpyAsync(out_mv + (size_t)f0 * nmb * 2, dmv, (size_t)nf * nmb * 8, cudaMemcpyDeviceToHost, st));
        B200_CUDA_OK(cudaMemcpyAsync(out_cost + (size_t)f0 * nmb, dcost, (size_t)nf * nmb * 8, cudaMemcpyDeviceToHost, st));
    }
    for (int i = 0; i < K; i++) B200_CUDA_OK(cudaStreamSynchronize(dev->pipe[i]));
    return 0;
}

// ------------------------------------------------------------------------------------------------ drop-in pointer table
namespace {

int host_cmp(int fn, int idx, const uint8_t *blk1, const uint8_t *blk2, ptrdiff_t stride, int h)
{
    int w, mode;
    if (decode(fn, idx, &w, &mode) < 0) B200HostCall::fail("me_cmp", "bad index");
    if (fn == B200_MECMP_HADAMARD8 || fn >= B200_MECMP_DCT_SAD) h = (w == 16 && h == 16) ? 16 : 8;   // the reference reads 8 rows unless 16 wide with h == 16
    const int cw = w + 1, ch = h + 1;                             // x2/y2/xy2 read one extra column / row of blk2
    const size_t pitch = 32;
    B200HostCall call("me_cmp", nullptr, 2 * pitch * (ch + 1) + 64);
    uint8_t *d1 = call.scratch, *d2 = call.scratch + pitch * (ch + 1);
    int64_t *offs = (int64_t *)(call.scratch + 2 * pitch * (ch + 1));
    int32_t *dout = (int32_t *)(offs + 2);
    cudaStream_t st = call.stream;
    call.check(b200_h2d_rows(d1, pitch, blk1, stride, w, h, st), "h2d");      // negative strides (flipped frames) are fine
    const int bw = fn == B200_MECMP_PIX_ABS && (mode & 1) ? cw : w, bh = fn == B200_MECMP_PIX_ABS && (mode & 2) ? ch : h;
    call.check(b200_h2d_rows(d2, pitch, blk2, stride, bw, bh, st), "h2d");
    call.check(cudaMemsetAsync(offs, 0, 16, st), "memset");
    if (fn >= B200_MECMP_DCT_SAD) mecmp_dct_launch(st, 1, 32, fn, w, h, d1, d2, (long long)pitch, offs, offs + 1, 1, dout);
    else if (fn == B200_MECMP_HADAMARD8) me_satd_kernel<<<1, 32, 0, st>>>(w == 8 ? 1 : h == 16 ? 4 : 2, d1, d2, (long long)pitch, offs, offs + 1, 1, dout, mode);
    else if (fn >= B200_MECMP_VSAD) me_cmp2_kernel<<<1, 32, 0, st>>>(fn, w, mode, g_nsse_weight.load(), d1, d2, (long long)pitch, h, offs, offs + 1, 1, dout);
    else me_cmp_kernel<<<1, 32, 0, st>>>(fn, w, mode, d1, d2, (long long)pitch, h, offs, offs + 1, 1, dout);
    B200_LAUNCHED();
    call.launched();
    int32_t res = 0;
    call.check(cudaMemcpyAsync(&res, dout, 4, cudaMemcpyDeviceToHost, st), "d2h");
    call.sync();
    return res;
}

template <int FN, int IDX>
int tab_fn(void *, const uint8_t *a, const uint8_t *b, ptrdiff_t stride, int h) { return host_cmp(FN, IDX, a, b, stride, h); }

int host_sum_abs_dctelem(const int16_t *block)
{
    B200HostCall call("sum_abs_dctelem", nullptr, 256);
    cudaStream_t st = call.stream;
    call.check(cudaMemcpyAsync(call.scratch, block, 128, cudaMemcpyHostToDevice, st), "h2d");
    sum_abs_dctelem_kernel<<<1, 32, 0, st>>>((const int16_t *)call.scratch, 1, (int32_t *)(call.scratch + 128));
    B200_LAUNCHED();
    call.launched();
    int32_t res = 0;
    call.check(cudaMemcpyAsync(&res, call.scratch + 128, 4, cudaMemcpyDeviceToHost, st), "d2h");
    call.sync();
    return res;
}

} // namespace

B200_API int b200_me_cmp_init(B200MECmpContext *c, int codec_flags)
{
    (void)codec_flags;
    if (!c) return B200_EINVAL;
    if (!b200_default_device()) return B200_ENODEV;
    memset(c, 0, sizeof(*c));
    c->sad[0] = tab_fn<B200_MECMP_SAD, 0>; c->sad[1] = tab_fn<B200_MECMP_SAD, 1>;
    c->sse[0] = tab_fn<B200_MECMP_SSE, 0>; c->sse[1] = tab_fn<B200_MECMP_SSE, 1>; c->sse[2] = tab_fn<B200_MECMP_SSE, 2>;
    c->pix_abs[0][0] = tab_fn<B200_MECMP_PIX_ABS, 0>; c->pix_abs[0][1] = tab_fn<B200_MECMP_PIX_ABS, 1>;
    c->pix_abs[0][2] = tab_fn<B200_MECMP_PIX_ABS, 2>; c->pix_abs[0][3] = tab_fn<B200_MECMP_PIX_ABS, 3>;
    c->pix_abs[1][0] = tab_fn<B200_MECMP_PIX_ABS, 4>; c->pix_abs[1][1] = tab_fn<B200_MECMP_PIX_ABS, 5>;
    c->pix_abs[1][2] = tab_fn<B200_MECMP_PIX_ABS, 6>; c->pix_abs[1][3] = tab_fn<B200_MECMP_PIX_ABS, 7>;
    c->hadamard8_diff[0] = tab_fn<B200_MECMP_HADAMARD8, 0>; c->hadamard8_diff[1] = tab_fn<B200_MECMP_HADAMARD8, 1>;
    c->hadamard8_diff[4] = tab_fn<B200_MECMP_HADAMARD8, 4>; c->hadamard8_diff[5] = tab_fn<B200_MECMP_HADAMARD8, 5>;
    c->vsad[0] = tab_fn<B200_MECMP_VSAD, 0>; c->vsad[1] = tab_fn<B200_MECMP_VSAD, 1>;
    c->vsad[4] = tab_fn<B200_MECMP_VSAD, 4>; c->vsad[5] = tab_fn<B200_MECMP_VSAD, 5>;
    c->vsse[0] = tab_fn<B200_MECMP_VSSE, 0>; c->vsse[1] = tab_fn<B200_MECMP_VSSE, 1>;
    c->vsse[4] = tab_fn<B200_MECMP_VSSE, 4>; c->vsse[5] = tab_fn<B200_MECMP_VSSE, 5>;
    c->nsse[0] = tab_fn<B200_MECMP_NSSE, 0>; c->nsse[1] = tab_fn<B200_MECMP_NSSE, 1>;
    c->median_sad[0] = tab_fn<B200_MECMP_MEDIAN_SAD, 0>; c->median_sad[1] = tab_fn<B200_MECMP_MEDIAN_SAD, 1>;
    c->dct_sad[0] = tab_fn<B200_MECMP_DCT_SAD, 0>; c->dct_sad[1] = tab_fn<B200_MECMP_DCT_SAD, 1>;
    c->dct_max[0] = tab_fn<B200_MECMP_DCT_MAX, 0>; c->dct_max[1] = tab_fn<B200_MECMP_DCT_MAX, 1>;
    c->dct264_sad[0] = tab_fn<B200_MECMP_DCT264_SAD, 0>; c->dct264_sad[1] = tab_fn<B200_MECMP_DCT264_SAD, 1>;   // upstream: GPL builds only (me_cmp.c:986-988)
    c->sum_abs_dctelem = host_sum_abs_dctelem;
    return 0;
}

B200_API void b200_me_cmp_set_nsse_weight(int weight) { g_nsse_weight.store(weight); }

B200_API int b200_sum_abs_dctelem_batch_device(B200Device *dev, const int16_t *blocks, int64_t n, int32_t *out)
{
    if (!dev || !blocks || !out || n < 0 || ((uintptr_t)blocks & 3)) return B200_EINVAL;
    if (n == 0) return 0;
    if (int r = b200_use_device(dev)) return r;
    const long long ctas = (n + 7) / 8;
    if (ctas > 0x7fffffffLL) return B200_EINVAL;
    sum_abs_dctelem_kernel<<<(unsigned)ctas, 256, 0, dev->stream>>>(blocks, n, out);
    B200_LAUNCHED();
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}
