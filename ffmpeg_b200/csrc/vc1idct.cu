// vc1idct.cu — VC-1 / WMV3 inverse transforms on sm_90a: the eight vc1_inv_trans_* members of VC1DSPContext (libavcodec/vc1dsp.h:38-45)
// as ff_vc1dsp_init fills them (vc1dsp.c:970-977), and a one-call-per-frame device entry that makes, for every inter 8x8 block, the
// transform calls vc1_decode_p_block makes (vc1_block.c:1124-1240).
//
// Reference semantics reproduced bit for bit (checker: oracle/vc1dsp_oracle.c), vc1dsp.c:240-537:
//   8-point   t1 = 12 (s0 + s4) + b, t2 = 12 (s0 - s4) + b, t3 = 16 s2 + 6 s6, t4 = 6 s2 - 16 s6, odd part 16 15 9 4 / 15 -4 -16 -9 /
//             9 -16 4 15 / 4 -9 15 -16; first pass b = 4, >> 3; second pass b = 64, + 1 on outputs 4..7, >> 7
//   4-point   t1 = 17 (s0 + s2) + b, t2 = 17 (s0 - s2) + b, t3 = 22 s1 + 10 s3, t4 = 22 s3 - 10 s1 -> t1 + t3, t2 - t4, t2 + t4, t1 - t3
//   8x8       column pass into int16 temp (transposed), row pass into int16 block, then add_pixels_clamped
//   8x4 4x8 4x4   row pass written back into int16 block, column pass added to dest and clipped
//   _dc       8x8 (3 dc + 1) >> 1, (3 dc + 16) >> 5; 8x4 (3 dc + 1) >> 1, (17 dc + 64) >> 7; 4x8 (17 dc + 4) >> 3, (12 dc + 64) >> 7;
//             4x4 (17 dc + 4) >> 3, (17 dc + 64) >> 7
// The arithmetic exists once (t8, t4, sub_column, dc_value), used by the members' kernel and by the frame kernel.
//
// Frame kernel: a group of eight threads per 8x8 block, four blocks per warp.  Thread t owns column t of the block's samples: for each
// sub-block that covers it, it loads the sub-block's coefficient rows as 16-byte words, computes the first-pass values of its column
// (the one output of every row / column transform it needs) and the second pass in registers, and adds the result down its column.
// No thread depends on another, so there is no shared memory and no barrier.
#include "common.h"
#include <cstring>

namespace {

constexpr int kGroups = 16;                                               // blocks per 128-thread CTA
constexpr long long kChunkOps = 1LL << 22;                                 // ops per launch

__device__ __forceinline__ void load_row(const int16_t *p, int (&v)[8])   // one 16-byte load, p 16-byte aligned
{
    const int4 q = *reinterpret_cast<const int4 *>(p);
    const int w[4] = { q.x, q.y, q.z, q.w };
#pragma unroll
    for (int k = 0; k < 4; k++) {
        v[2 * k] = (int16_t)(w[k] & 0xFFFF);
        v[2 * k + 1] = (int16_t)((unsigned)w[k] >> 16);
    }
}

// the 8-point transform of v: first pass (second = false) or second pass
__device__ __forceinline__ void t8(const int (&v)[8], bool second, int (&o)[8])
{
    const int b = second ? 64 : 4, sh = second ? 7 : 3, r = second ? 1 : 0;
    const int t1 = 12 * (v[0] + v[4]) + b, t2 = 12 * (v[0] - v[4]) + b, t3 = 16 * v[2] + 6 * v[6], t4 = 6 * v[2] - 16 * v[6];
    const int t5 = t1 + t3, t6 = t2 + t4, t7 = t2 - t4, t8 = t1 - t3;
    const int u1 = 16 * v[1] + 15 * v[3] + 9 * v[5] + 4 * v[7], u2 = 15 * v[1] - 4 * v[3] - 16 * v[5] - 9 * v[7];
    const int u3 = 9 * v[1] - 16 * v[3] + 4 * v[5] + 15 * v[7], u4 = 4 * v[1] - 9 * v[3] + 15 * v[5] - 16 * v[7];
    o[0] = (t5 + u1) >> sh; o[1] = (t6 + u2) >> sh; o[2] = (t7 + u3) >> sh; o[3] = (t8 + u4) >> sh;
    o[4] = (t8 - u4 + r) >> sh; o[5] = (t7 - u3 + r) >> sh; o[6] = (t6 - u2 + r) >> sh; o[7] = (t5 - u1 + r) >> sh;
}

// the 4-point transform of (a0, a1, a2, a3): first pass or second pass
__device__ __forceinline__ void t4(int a0, int a1, int a2, int a3, bool second, int (&o)[4])
{
    const int b = second ? 64 : 4, sh = second ? 7 : 3;
    const int t1 = 17 * (a0 + a2) + b, t2 = 17 * (a0 - a2) + b, t3 = 22 * a1 + 10 * a3, t4v = 22 * a3 - 10 * a1;
    o[0] = (t1 + t3) >> sh; o[1] = (t2 - t4v) >> sh; o[2] = (t2 + t4v) >> sh; o[3] = (t1 - t3) >> sh;
}

__device__ __forceinline__ int pick8(const int (&o)[8], int k)
{
    return k == 0 ? o[0] : k == 1 ? o[1] : k == 2 ? o[2] : k == 3 ? o[3] : k == 4 ? o[4] : k == 5 ? o[5] : k == 6 ? o[6] : o[7];
}
__device__ __forceinline__ int pick4(const int (&o)[4], int k) { return k == 0 ? o[0] : k == 1 ? o[1] : k == 2 ? o[2] : o[3]; }

// Column c of one sub-block transform of type tt (B200_VC1_TT_*).  blk: the sub-block's first coefficient row, 16-byte aligned, rows 8
// int16 apart; half: for a 4-wide sub-block, which half of those rows it is.  w[i]: the first-pass value that the reference stores
// (int16) at row i of column c (8x4 / 4x8 / 4x4: in block; 8x8: temp[c][i]); res[k]: the sample difference at row k, int16 for 8x8 as
// the reference stores it before add_pixels_clamped.  Returns the number of rows.
__device__ __forceinline__ int sub_column(const int16_t *blk, int tt, int half, int c, int16_t (&w)[8], int (&res)[8])
{
    int v[8], o[8], o4[4];
    if (tt == B200_VC1_TT_8X8) {
        int rows[8][8];
#pragma unroll
        for (int r = 0; r < 8; r++) load_row(blk + 8 * r, rows[r]);
#pragma unroll
        for (int col = 0; col < 8; col++) {                               // temp[col][c]: output c of column col's transform
#pragma unroll
            for (int r = 0; r < 8; r++) v[r] = rows[r][col];
            t8(v, false, o);
            w[col] = (int16_t)pick8(o, c);
        }
#pragma unroll
        for (int k = 0; k < 8; k++) v[k] = w[k];
        t8(v, true, o);
#pragma unroll
        for (int k = 0; k < 8; k++) res[k] = (int16_t)o[k];
        return 8;
    }
    if (tt == B200_VC1_TT_8X4) {
#pragma unroll
        for (int r = 0; r < 4; r++) {
            load_row(blk + 8 * r, v);
            t8(v, false, o);
            w[r] = (int16_t)pick8(o, c);
        }
        t4(w[0], w[1], w[2], w[3], true, o4);
#pragma unroll
        for (int k = 0; k < 4; k++) res[k] = o4[k];
        return 4;
    }
    const int nr = tt == B200_VC1_TT_4X8 ? 8 : 4;
#pragma unroll
    for (int r = 0; r < 8; r++) {
        if (r < nr) {
            load_row(blk + 8 * r, v);
            t4(half ? v[4] : v[0], half ? v[5] : v[1], half ? v[6] : v[2], half ? v[7] : v[3], false, o4);
            w[r] = (int16_t)pick4(o4, c);
        }
    }
    if (nr == 8) {
#pragma unroll
        for (int k = 0; k < 8; k++) v[k] = w[k];
        t8(v, true, o);
#pragma unroll
        for (int k = 0; k < 8; k++) res[k] = o[k];
        return 8;
    }
    t4(w[0], w[1], w[2], w[3], true, o4);
#pragma unroll
    for (int k = 0; k < 4; k++) res[k] = o4[k];
    return 4;
}

// vc1_inv_trans_<tt>_dc's value from block[0]
__device__ __forceinline__ int dc_value(int tt, int dc)
{
    if (tt == B200_VC1_TT_8X8) { dc = (3 * dc + 1) >> 1; return (3 * dc + 16) >> 5; }
    if (tt == B200_VC1_TT_8X4) { dc = (3 * dc + 1) >> 1; return (17 * dc + 64) >> 7; }
    dc = (17 * dc + 4) >> 3;
    return tt == B200_VC1_TT_4X8 ? (12 * dc + 64) >> 7 : (17 * dc + 64) >> 7;
}

__device__ __forceinline__ void add_column(uint8_t *d, long long ls, const int (&res)[8], int n)
{
#pragma unroll
    for (int k = 0; k < 8; k++)
        if (k < n) d[k * ls] = (uint8_t)min(max(d[k * ls] + res[k], 0), 255);
}

struct ResArgs {
    const B200Vc1ResidualOp *ops;
    long long nops;
    const int16_t *coef;
    uint8_t *dst[3];
    long long ls_y, ls_uv;
    int mbw, mbh;
};

__global__ void __launch_bounds__(8 * kGroups) vc1_residual_kernel(ResArgs a)
{
    const long long i = (long long)blockIdx.x * kGroups + (threadIdx.x >> 3);
    const int t = threadIdx.x & 7;
    if (i >= a.nops) return;
    const B200Vc1ResidualOp op = a.ops[i];
    const int lim_w = op.plane ? 8 * a.mbw : 16 * a.mbw, lim_h = op.plane ? 8 * a.mbh : 16 * a.mbh;
    if (op.plane > 2 || op.ttblk > B200_VC1_TT_4X4 || op.coef_off < 0 || (op.coef_off & 7) || op.x < 0 || op.y < 0 || (op.x & 7) ||
        (op.y & 7) || op.x + 8 > lim_w || op.y + 8 > lim_h)
        return;
    const int16_t *blk = a.coef + op.coef_off;
    const long long ls = op.plane ? a.ls_uv : a.ls_y;
    uint8_t *col = (op.plane == 0 ? a.dst[0] : op.plane == 1 ? a.dst[1] : a.dst[2]) + (long long)op.y * ls + op.x + t;
    const int tt = op.ttblk;
    // sub-blocks covering column t, top to bottom: (index j, first row, coefficient origin, column within it, half)
    const int nseg = tt == B200_VC1_TT_8X4 || tt == B200_VC1_TT_4X4 ? 2 : 1;
#pragma unroll
    for (int seg = 0; seg < 2; seg++) {
        if (seg >= nseg) break;
        int j, skipbit, row0 = 4 * seg, c = t, half = 0;
        if (tt == B200_VC1_TT_8X8) { j = 0; skipbit = 0; row0 = 0; }
        else if (tt == B200_VC1_TT_8X4) { j = seg; skipbit = 1 << (1 - j); }
        else if (tt == B200_VC1_TT_4X8) { j = t >> 2; skipbit = 1 << (1 - j); row0 = 0; half = j; c = t & 3; }
        else { half = t >> 2; j = 2 * seg + half; skipbit = 1 << (3 - j); c = t & 3; }
        if (op.subblkpat & skipbit) continue;
        const int16_t *sb = blk + 8 * row0;
        int res[8];
        int n;
        if (op.dc & (1 << j)) {
            n = tt == B200_VC1_TT_8X8 || tt == B200_VC1_TT_4X8 ? 8 : 4;
            const int d = dc_value(tt, sb[4 * half]);
#pragma unroll
            for (int k = 0; k < 8; k++) res[k] = d;
        } else {
            int16_t w[8];
            n = sub_column(sb, tt, half, c, w, res);
        }
        add_column(col + row0 * ls, ls, res, n);
    }
}

// ---- drop-in members (host pointers): the coefficients and samples the reference function reads are staged in the device scratch,
// one group of eight threads runs the member with the frame kernel's functions, and what the reference writes comes back.
constexpr int kDstPitch = 8;

// tt's transform on the staged block (64 int16, the sub-block at (0, 0)) and dest (8 x 8, pitch kDstPitch): block rewritten as the
// reference leaves it; dc: the _dc form (block untouched); dest NULL for vc1_inv_trans_8x8, which writes block only
__global__ void vc1_idct_member_kernel(int tt, int dc, int16_t *blk, uint8_t *dest)
{
    const int t = threadIdx.x, cols = tt == B200_VC1_TT_8X8 || tt == B200_VC1_TT_8X4 ? 8 : 4;
    const bool on = t < cols;
    int res[8];
    int16_t w[8];
    int n = 0;
    if (on && dc) {
        n = tt == B200_VC1_TT_8X8 || tt == B200_VC1_TT_4X8 ? 8 : 4;
        const int d = dc_value(tt, blk[0]);
#pragma unroll
        for (int k = 0; k < 8; k++) res[k] = d;
    } else if (on) {
        n = sub_column(blk, tt, 0, t, w, res);
    }
    __syncwarp();                                                          // every thread has read block before any writes it back
    if (!on) return;
    if (!dc)
#pragma unroll
        for (int k = 0; k < 8; k++)
            if (k < n) blk[8 * k + t] = tt == B200_VC1_TT_8X8 ? (int16_t)res[k] : w[k];
    if (dest) add_column(dest + t, kDstPitch, res, n);
}

void member_host(int tt, int dc, uint8_t *dest, ptrdiff_t stride, int16_t *block)
{
    const int cols = tt == B200_VC1_TT_8X8 || tt == B200_VC1_TT_8X4 ? 8 : 4;
    const int rows = tt == B200_VC1_TT_8X8 || tt == B200_VC1_TT_4X8 ? 8 : 4;
    B200HostCall call("vc1 transform member", nullptr, 256);
    cudaStream_t st = call.stream;
    int16_t *dblk = (int16_t *)call.scratch;
    uint8_t *ddst = call.scratch + 128;
    const size_t bpitch = 8 * sizeof(int16_t);
    // the reference reads block[0] (_dc) or the rows x cols coefficients at pitch 8
    call.check(b200_h2d_rows(dblk, bpitch, block, (ptrdiff_t)bpitch, dc ? sizeof(int16_t) : cols * sizeof(int16_t), dc ? 1 : rows, st), "h2d block");
    if (dest) call.check(b200_h2d_rows(ddst, kDstPitch, dest, stride, (size_t)cols, (size_t)rows, st), "h2d dest");
    vc1_idct_member_kernel<<<1, 32, 0, st>>>(tt, dc, dblk, dest ? ddst : nullptr);
    B200_LAUNCHED();
    call.launched();
    if (dest) call.check(b200_d2h_rows(dest, stride, ddst, kDstPitch, (size_t)cols, (size_t)rows, st), "d2h dest");
    if (!dc) call.check(b200_d2h_rows(block, (ptrdiff_t)bpitch, dblk, bpitch, cols * sizeof(int16_t), rows, st), "d2h block");
    call.sync();
}

void m_8x8(int16_t *b) { member_host(B200_VC1_TT_8X8, 0, nullptr, 0, b); }
template <int TT, int DC>
void m_tx(uint8_t *dest, ptrdiff_t stride, int16_t *block) { member_host(TT, DC, dest, stride, block); }

} // namespace

// vc1mc.cu's b200_vc1_dsp_init calls this after it has cleared the context and filled the MC tables
void b200_vc1_fill_transforms(B200VC1DSPContext *c)
{
    c->vc1_inv_trans_8x8 = m_8x8;
    c->vc1_inv_trans_8x4 = m_tx<B200_VC1_TT_8X4, 0>;
    c->vc1_inv_trans_4x8 = m_tx<B200_VC1_TT_4X8, 0>;
    c->vc1_inv_trans_4x4 = m_tx<B200_VC1_TT_4X4, 0>;
    c->vc1_inv_trans_8x8_dc = m_tx<B200_VC1_TT_8X8, 1>;
    c->vc1_inv_trans_8x4_dc = m_tx<B200_VC1_TT_8X4, 1>;
    c->vc1_inv_trans_4x8_dc = m_tx<B200_VC1_TT_4X8, 1>;
    c->vc1_inv_trans_4x4_dc = m_tx<B200_VC1_TT_4X4, 1>;
}

B200_API int b200_vc1_residual_frame_device(B200Device *dev, uint8_t *const dst[3], ptrdiff_t ls_y, ptrdiff_t ls_uv, int mb_width,
                                            int mb_height, const int16_t *coef, int64_t nops, const B200Vc1ResidualOp *ops)
{
    if (nops < 0 || mb_width < 1 || mb_height < 1 || mb_width > 2047 || mb_height > 2047) {
        b200_set_error("vc1 residual frame: negative nops or a macroblock count outside 1..2047");
        return B200_EINVAL;
    }
    if (nops == 0) return 0;
    if (!ops || !coef || !dst || ((uintptr_t)ops & 7) || ((uintptr_t)coef & 15)) {
        b200_set_error("vc1 residual frame: NULL or misaligned ops / coef");
        return B200_EINVAL;
    }
    if ((ls_y & 3) || (ls_uv & 3)) { b200_set_error("vc1 residual frame: line size not a multiple of 4"); return B200_EINVAL; }
    for (int p = 0; p < 3; p++)
        if (!dst[p] || ((uintptr_t)dst[p] & 3)) { b200_set_error("vc1 residual frame: plane %d NULL or not 4-byte aligned", p); return B200_EINVAL; }
    if (int r = b200_use_device(dev)) return r;
    ResArgs a;
    memset(&a, 0, sizeof(a));
    a.coef = coef;
    for (int p = 0; p < 3; p++) a.dst[p] = dst[p];
    a.ls_y = (long long)ls_y;
    a.ls_uv = (long long)ls_uv;
    a.mbw = mb_width;
    a.mbh = mb_height;
    for (long long b = 0; b < (long long)nops; b += kChunkOps) {
        a.ops = ops + b;
        a.nops = (long long)nops - b < kChunkOps ? (long long)nops - b : kChunkOps;
        const unsigned grid = (unsigned)((a.nops + kGroups - 1) / kGroups);
        vc1_residual_kernel<<<grid, 8 * kGroups, 0, dev->stream>>>(a);
        B200_LAUNCHED();
        B200_CUDA_OK(cudaGetLastError());
    }
    return 0;
}
