// hevcdbk.cu — HEVC deblocking on sm_90a: the eight loop-filter members of HEVCDSPContext (libavcodec/hevc/dsp.h:47-125:
// hevc_{h,v}_loop_filter_{luma,chroma} and their _c twins, the same functions, hevc/dsp.c:237-244) as ff_hevc_dsp_init fills them for
// 8, 9, 10 and 12 bit samples, and a one-pass plane entry that deblocks a whole luma or chroma plane from two grids of edge segments.
//
// Reference semantics reproduced bit for bit (checker: oracle/hevcdbk_oracle.c), hevc/dsp_template.c:834-928 with
// h26x/h2656_deblock_template.c; per 4-line segment, beta and tc shifted left by depth - 8:
//   luma    d = dp0 + dq0 + dp3 + dq3 (second differences of lines 0 and 3); nothing when d >= beta.  Strong when both lines 0 and 3
//           pass |P3 - P0| + |Q3 - Q0| < beta >> 3, |P0 - Q0| < (5 tc + 1) >> 1 and 2 (dp + dq) < beta >> 2: P2..Q2 move by at most
//           2 tc.  Else weak, per line: delta0 = (9 (Q0 - P0) - 3 (Q1 - P1) + 8) >> 4, nothing when |delta0| >= 10 tc; P0 / Q0 move by
//           delta0 clipped to tc, P1 / Q1 (when dp0 + dp3 resp. dq0 + dq3 < (beta + beta / 2) >> 3) by tc / 2.  tc <= 0: nothing.
//   chroma  tc > 0 only: delta0 = clip((4 (Q0 - P0) + P1 - Q1 + 4) >> 3, -tc, tc) on P0 / Q0 of every line.
//   no_p / no_q keep the P / Q side as it is.
//
// Plane kernel: every edge lies on the 8x8 grid and reads at most 4 samples on each side, so the vertical edges of a plane are
// independent of one another, as are the horizontal ones, and "all vertical edges, then all horizontal edges" is the decoder's
// CTB-by-CTB result (hevc/filter.c:501-676).  A CTA owns a tile of kTH x kTW samples whose borders lie at rows and columns = 4
// (mod 8): every edge's reads, decisions and writes fall inside one tile.  It loads the tile into shared memory, runs the vertical pass
// (a warp per edge, a lane per line), then the horizontal pass (a lane per column), and stores the tile: each sample is read and
// written once, with no halo and no sample written by two CTAs.  A segment's decision (lines 0 and 3) reaches its four lanes by warp
// shuffles.
#include "common.h"
#include <cstring>

namespace {

constexpr int kTW = 128, kTH = 32;                           // tile: kTH = one warp of lines for a vertical edge
constexpr int kThreads = 256;
constexpr size_t kSmem = sizeof(uint16_t) * kTH * (kTW + 2); // rows padded to an odd number of words: a warp down a column is conflict-free

struct DbkArgs {
    uint8_t *pix;
    long long stride;                                        // bytes
    const B200HevcDbkSeg *vseg, *hseg;
    long long vstride, hstride;                              // records
    int width, height, depth, ntx;
};

__device__ __forceinline__ int clip3(int v, int lo, int hi) { return v < lo ? lo : v > hi ? hi : v; }

// One line across an edge, v[0..7] = P3 P2 P1 P0 Q0 Q1 Q2 Q3, for the segment `s` whose first line is lane (lane & ~3) of the warp.
// Every lane of the warp calls it (the luma decision is shuffled from lines 0 and 3); returns whether v may have changed.
template <bool CHROMA>
__device__ __forceinline__ bool filter_line(int (&v)[8], const B200HevcDbkSeg s, int depth, int lane)
{
    const int sh = depth - 8, maxv = (1 << depth) - 1;
    const int tc = (int)s.tc << sh;
    const bool no_p = s.flags & B200_HEVC_DBK_NO_P, no_q = s.flags & B200_HEVC_DBK_NO_Q;
    if constexpr (CHROMA) {
        if (tc <= 0) return false;
        const int d = clip3((((v[4] - v[3]) * 4) + v[2] - v[5] + 4) >> 3, -tc, tc);
        if (!no_p) v[3] = clip3(v[3] + d, 0, maxv);
        if (!no_q) v[4] = clip3(v[4] - d, 0, maxv);
        return true;
    } else {
        const int beta = (int)s.beta << sh;
        const int dp = abs(v[1] - 2 * v[2] + v[3]), dq = abs(v[6] - 2 * v[5] + v[4]);
        const int tc25 = (tc * 5 + 1) >> 1;
        const int sl = abs(v[0] - v[3]) + abs(v[7] - v[4]) < (beta >> 3) && abs(v[3] - v[4]) < tc25 && ((dp + dq) << 1) < (beta >> 2);
        const int l0 = lane & ~3, l3 = l0 + 3;
        const int dp0 = __shfl_sync(0xFFFFFFFFu, dp, l0), dq0 = __shfl_sync(0xFFFFFFFFu, dq, l0);
        const int dp3 = __shfl_sync(0xFFFFFFFFu, dp, l3), dq3 = __shfl_sync(0xFFFFFFFFu, dq, l3);
        const int strong = __shfl_sync(0xFFFFFFFFu, sl, l0) & __shfl_sync(0xFFFFFFFFu, sl, l3);
        if (tc <= 0 || dp0 + dq0 + dp3 + dq3 >= beta) return false;
        const int p3 = v[0], p2 = v[1], p1 = v[2], p0 = v[3], q0 = v[4], q1 = v[5], q2 = v[6], q3 = v[7];
        if (strong) {
            const int t2 = tc << 1;
            if (!no_p) {
                v[3] = p0 + clip3(((p2 + 2 * p1 + 2 * p0 + 2 * q0 + q1 + 4) >> 3) - p0, -t2, t2);
                v[2] = p1 + clip3(((p2 + p1 + p0 + q0 + 2) >> 2) - p1, -t2, t2);
                v[1] = p2 + clip3(((2 * p3 + 3 * p2 + p1 + p0 + q0 + 4) >> 3) - p2, -t2, t2);
            }
            if (!no_q) {
                v[4] = q0 + clip3(((p1 + 2 * p0 + 2 * q0 + 2 * q1 + q2 + 4) >> 3) - q0, -t2, t2);
                v[5] = q1 + clip3(((p0 + q0 + q1 + q2 + 2) >> 2) - q1, -t2, t2);
                v[6] = q2 + clip3(((2 * q3 + 3 * q2 + q1 + q0 + p0 + 4) >> 3) - q2, -t2, t2);
            }
            return true;
        }
        const int side = (beta + (beta >> 1)) >> 3;
        int d = (9 * (q0 - p0) - 3 * (q1 - p1) + 8) >> 4;
        if (abs(d) >= 10 * tc) return false;
        d = clip3(d, -tc, tc);
        const int tc2 = tc >> 1;
        if (!no_p) v[3] = clip3(p0 + d, 0, maxv);
        if (!no_q) v[4] = clip3(q0 - d, 0, maxv);
        if (!no_p && dp0 + dp3 < side) v[2] = clip3(p1 + clip3((((p2 + p0 + 1) >> 1) - p1 + d) >> 1, -tc2, tc2), 0, maxv);
        if (!no_q && dq0 + dq3 < side) v[5] = clip3(q1 + clip3((((q2 + q0 + 1) >> 1) - q1 - d) >> 1, -tc2, tc2), 0, maxv);
        return true;
    }
}

template <typename P, bool CHROMA>
__global__ void __launch_bounds__(kThreads) hevc_dbk_kernel(DbkArgs a)
{
    extern __shared__ uint16_t dbk_tile[];
    uint16_t (*t)[kTW + 2] = reinterpret_cast<uint16_t (*)[kTW + 2]>(dbk_tile);
    const int tx = (int)(blockIdx.x % (unsigned)a.ntx), ty = (int)(blockIdx.x / (unsigned)a.ntx);
    const int X0 = tx * kTW - 4, Y0 = ty * kTH - 4;          // tile origin in the plane: borders at = 4 (mod 8)
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    for (int i = tid; i < kTH * kTW; i += kThreads) {
        const int r = i / kTW, c = i % kTW, y = Y0 + r, x = X0 + c;
        if (y >= 0 && y < a.height && x >= 0 && x < a.width) t[r][c] = reinterpret_cast<const P *>(a.pix + (long long)y * a.stride)[x];
    }
    __syncthreads();
    const B200HevcDbkSeg none = { 0, 0, 0, 0 };
    // vertical edges at tile columns 4, 12, ..., a warp per edge, a lane per row
    for (int e = warp; e < kTW / 8; e += kThreads / 32) {
        const int c = 4 + 8 * e, x = X0 + c, y = Y0 + lane;
        const bool on = x > 0 && x < a.width && y >= 0 && y < a.height;
        const B200HevcDbkSeg s = on ? a.vseg[(long long)(y >> 2) * a.vstride + (x >> 3)] : none;
        int v[8];
#pragma unroll
        for (int k = 0; k < 8; k++) v[k] = t[lane][c - 4 + k];
        if (filter_line<CHROMA>(v, s, a.depth, lane) && on) {
#pragma unroll
            for (int k = 1; k < 7; k++) t[lane][c - 4 + k] = (uint16_t)v[k];
        }
    }
    __syncthreads();
    // horizontal edges at tile rows 4, 12, 20, 28, a lane per column
    for (int j = warp; j < (kTH / 8) * (kTW / 32); j += kThreads / 32) {
        const int r = 4 + 8 * (j / (kTW / 32)), c = 32 * (j % (kTW / 32)) + lane, x = X0 + c, y = Y0 + r;
        const bool on = y > 0 && y < a.height && x >= 0 && x < a.width;
        const B200HevcDbkSeg s = on ? a.hseg[(long long)(y >> 3) * a.hstride + (x >> 2)] : none;
        int v[8];
#pragma unroll
        for (int k = 0; k < 8; k++) v[k] = t[r - 4 + k][c];
        if (filter_line<CHROMA>(v, s, a.depth, lane) && on) {
#pragma unroll
            for (int k = 1; k < 7; k++) t[r - 4 + k][c] = (uint16_t)v[k];
        }
    }
    __syncthreads();
    for (int i = tid; i < kTH * kTW; i += kThreads) {
        const int r = i / kTW, c = i % kTW, y = Y0 + r, x = X0 + c;
        if (y >= 0 && y < a.height && x >= 0 && x < a.width) reinterpret_cast<P *>(a.pix + (long long)y * a.stride)[x] = (P)t[r][c];
    }
}

bool depth_ok(int d) { return d == 8 || d == 9 || d == 10 || d == 12; }

cudaError_t launch(const DbkArgs &a0, bool chroma, cudaStream_t st)
{
    DbkArgs a = a0;
    a.ntx = (a.width + 4 + kTW - 1) / kTW;
    const int nty = (a.height + 4 + kTH - 1) / kTH;
    const unsigned grid = (unsigned)a.ntx * (unsigned)nty;
    if (a.depth == 8) {
        if (chroma) hevc_dbk_kernel<uint8_t, true><<<grid, kThreads, kSmem, st>>>(a);
        else hevc_dbk_kernel<uint8_t, false><<<grid, kThreads, kSmem, st>>>(a);
    } else {
        if (chroma) hevc_dbk_kernel<uint16_t, true><<<grid, kThreads, kSmem, st>>>(a);
        else hevc_dbk_kernel<uint16_t, false><<<grid, kThreads, kSmem, st>>>(a);
    }
    B200_LAUNCHED();
    return cudaGetLastError();
}

// ---- drop-in members (host pointers): the edge is staged into a 16 x 16 scratch plane with Q0 of line 0 at (8, 0) (vertical edge)
// or (0, 8) (horizontal edge) and run through the plane kernel with its two segments in the grids.  Per segment j with tc[j] > 0 (the
// reference does nothing for the others), the lines 4j..4j+3 of P3..Q3 (luma) or P1..Q1 (chroma) go up, and P2..Q2 / P0..Q0 (what the
// reference can write) come back.
void member_host(int depth, bool chroma, bool horiz, uint8_t *pix, ptrdiff_t stride, int beta, const int32_t *tc, const uint8_t *no_p,
                 const uint8_t *no_q)
{
    if (tc[0] <= 0 && tc[1] <= 0) return;
    const int bps = depth > 8 ? 2 : 1, reach = chroma ? 2 : 4, wr = chroma ? 1 : 3;
    const size_t dpitch = 16 * (size_t)bps;
    B200HostCall call("hevc deblocking", nullptr, 256 + 16 * dpitch);
    uint8_t *scr = call.scratch;
    cudaStream_t st = call.stream;
    B200HevcDbkSeg seg[64];
    memset(seg, 0, sizeof(seg));
    B200HevcDbkSeg *vs = seg, *hs = seg + 32;                // vertical: 16 x 8 plane, vseg 2 x 2; horizontal: 8 x 16 plane, hseg 2 x 2
    for (int j = 0; j < 2; j++) {
        B200HevcDbkSeg s = { (uint8_t)beta, (uint8_t)(tc[j] > 0 ? tc[j] : 0),
                             (uint8_t)((no_p[j] ? B200_HEVC_DBK_NO_P : 0) | (no_q[j] ? B200_HEVC_DBK_NO_Q : 0)), 0 };
        if (horiz) hs[2 + j] = s;
        else vs[2 * j + 1] = s;
    }
    uint8_t *plane = scr + 256;
    const B200HevcDbkSeg *dseg = (const B200HevcDbkSeg *)scr;
    // host sample (column c, line r) of the edge <-> device plane sample
    auto hp = [&](int c, int r) { return pix + (ptrdiff_t)r * stride + (ptrdiff_t)c * bps; };
    auto dp = [&](int c, int r) { return plane + (size_t)(r + (horiz ? 8 : 0)) * dpitch + (size_t)(c + (horiz ? 0 : 8)) * bps; };
    call.check(cudaMemcpyAsync(scr, seg, sizeof(seg), cudaMemcpyHostToDevice, st), "h2d segments");
    for (int j = 0; j < 2; j++) {
        if (tc[j] <= 0) continue;
        cudaError_t e = horiz ? b200_h2d_rows(dp(4 * j, -reach), dpitch, hp(4 * j, -reach), stride, 4 * (size_t)bps, 2 * (size_t)reach, st)
                              : b200_h2d_rows(dp(-reach, 4 * j), dpitch, hp(-reach, 4 * j), stride, 2 * (size_t)reach * bps, 4, st);
        call.check(e, "h2d edge");
    }
    DbkArgs a = { plane, (long long)dpitch, dseg, dseg + 32, 2, 2, horiz ? 8 : 16, horiz ? 16 : 8, depth, 0 };
    call.check(launch(a, chroma, st), "launch");
    for (int j = 0; j < 2; j++) {
        if (tc[j] <= 0) continue;
        cudaError_t e = horiz ? b200_d2h_rows(hp(4 * j, -wr), stride, dp(4 * j, -wr), dpitch, 4 * (size_t)bps, 2 * (size_t)wr, st)
                              : b200_d2h_rows(hp(-wr, 4 * j), stride, dp(-wr, 4 * j), dpitch, 2 * (size_t)wr * bps, 4, st);
        call.check(e, "d2h edge");
    }
    call.sync();
}

// for a vertical edge the member's `pix` is Q0 of line 0 and lines run down the rows; for a horizontal one lines run along the row
template <int D>
void m_h_luma(uint8_t *pix, ptrdiff_t stride, int beta, const int32_t *tc, const uint8_t *no_p, const uint8_t *no_q)
{
    member_host(D, false, true, pix, stride, beta, tc, no_p, no_q);
}
template <int D>
void m_v_luma(uint8_t *pix, ptrdiff_t stride, int beta, const int32_t *tc, const uint8_t *no_p, const uint8_t *no_q)
{
    member_host(D, false, false, pix, stride, beta, tc, no_p, no_q);
}
template <int D>
void m_h_chroma(uint8_t *pix, ptrdiff_t stride, const int32_t *tc, const uint8_t *no_p, const uint8_t *no_q)
{
    member_host(D, true, true, pix, stride, 0, tc, no_p, no_q);
}
template <int D>
void m_v_chroma(uint8_t *pix, ptrdiff_t stride, const int32_t *tc, const uint8_t *no_p, const uint8_t *no_q)
{
    member_host(D, true, false, pix, stride, 0, tc, no_p, no_q);
}

// hevc/dsp.c:237-244: each _c member is the same function as its plain twin
template <int D>
void fill(B200HEVCDSPContext *c)
{
    c->hevc_h_loop_filter_luma = c->hevc_h_loop_filter_luma_c = m_h_luma<D>;
    c->hevc_v_loop_filter_luma = c->hevc_v_loop_filter_luma_c = m_v_luma<D>;
    c->hevc_h_loop_filter_chroma = c->hevc_h_loop_filter_chroma_c = m_h_chroma<D>;
    c->hevc_v_loop_filter_chroma = c->hevc_v_loop_filter_chroma_c = m_v_chroma<D>;
}

} // namespace

B200_API int b200_hevc_dsp_init_deblock(B200HEVCDSPContext *c, int bit_depth)
{
    if (!c) return B200_EINVAL;
    if (!depth_ok(bit_depth)) return B200_ENOSYS;
    if (!b200_default_device()) return B200_ENODEV;
    switch (bit_depth) {
    case 8:  fill<8>(c); break;
    case 9:  fill<9>(c); break;
    case 10: fill<10>(c); break;
    default: fill<12>(c); break;
    }
    return 0;
}

B200_API int b200_hevc_deblock_plane_device(B200Device *dev, int bit_depth, int chroma, uint8_t *pix, ptrdiff_t stride, int width, int height,
                                            const B200HevcDbkSeg *vseg, int64_t vseg_stride, const B200HevcDbkSeg *hseg, int64_t hseg_stride)
{
    if (!pix || !vseg || !hseg) { b200_set_error("hevc deblock plane: NULL pointer"); return B200_EINVAL; }
    if (!depth_ok(bit_depth)) { b200_set_error("hevc deblock plane: bit depth %d is not 8, 9, 10 or 12", bit_depth); return B200_EINVAL; }
    if (chroma != 0 && chroma != 1) { b200_set_error("hevc deblock plane: chroma %d is not 0 or 1", chroma); return B200_EINVAL; }
    if (width < 4 || height < 4 || (width & 3) || (height & 3)) {
        b200_set_error("hevc deblock plane: %dx%d is not a multiple of 4 of at least 4x4", width, height);
        return B200_EINVAL;
    }
    const int bps = bit_depth > 8 ? 2 : 1;
    if (stride < (ptrdiff_t)width * bps || stride % bps || (uintptr_t)pix % bps) {
        b200_set_error("hevc deblock plane: stride shorter than a row, or stride / pix not a whole number of samples");
        return B200_EINVAL;
    }
    if (vseg_stride < (width + 7) / 8 || hseg_stride < width / 4) {
        b200_set_error("hevc deblock plane: grid stride shorter than the grid row");
        return B200_EINVAL;
    }
    if (int r = b200_use_device(dev)) return r;
    const DbkArgs a = { pix, (long long)stride, vseg, hseg, (long long)vseg_stride, (long long)hseg_stride, width, height, bit_depth, 0 };
    B200_CUDA_OK(launch(a, chroma != 0, dev->stream));
    return 0;
}
