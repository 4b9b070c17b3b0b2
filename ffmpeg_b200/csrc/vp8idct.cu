// vp8idct.cu — VP8 / VP7 residual reconstruction on sm_90a: the six residual members of VP8DSPContext (libavcodec/vp8dsp.h:37-45) as
// ff_vp8dsp_init / ff_vp7dsp_init fill them (vp8dsp.c:693-760), and a one-call-per-frame device entry that runs, for every macroblock,
// the luma DC transform of decode_mb_coeffs (vp8.c:1517-1524) and then idct_mb (vp8.c:2085-2146).
//
// Reference semantics reproduced bit for bit (checker: oracle/vp8dsp_oracle.c), vp8dsp.c:56-247:
//   VP8 WHT    column pass t0 = a + d, t1 = b + c, t2 = b - c, t3 = a - d -> (t0 + t1, t3 + t2, t0 - t1, t3 - t2) stored in int16 dc[]
//              (truncated), then the same butterfly along each row with + 3 and >> 3 into block[row][col][0]
//   VP8 IDCT   MUL_20091(a) = ((a * 20091) >> 16) + a, MUL_35468(a) = (a * 35468) >> 16 in int; column pass into int16 tmp, row
//              pass (x + 4) >> 3 added to dst and clipped; DC only (block[0] + 4) >> 3
//   VP7        row pass first, products in unsigned, (int) >> 14 into int16 tmp, column pass (int)(x + 0x20000) >> 18; DC only
//              (23170 * (23170 * b0 >> 14) + 0x20000) >> 18, for the WHT's DC too
// The arithmetic exists once (wht_value, residual4x4, dc_value), used by the members' kernel and by the frame kernel.
//
// Frame kernel: one warp per macroblock, four per CTA.  Lanes 0..15 own the luma blocks (raster order), lanes 16..23 the chroma blocks
// (U then V, 2 x 2 each); each lane's 16 coefficients lie at coef_off + 16 * lane.  A luma lane with Y2 coefficients computes its own WHT
// output in closed form from the 16 Y2 values (every lane of the MB loads the same two 16-byte words), then applies idct_mb's decision
// for its block: the row's (plane's) four nnz bytes all <= 1 and not all 0 -> its DC added (dc_add4y / dc_add4uv, nnz-0 blocks
// included); else nnz 1 -> dc_add, nnz > 1 -> the full transform in registers from two 16-byte loads, 0 -> nothing.  Each lane updates
// its block's four rows as 4-byte words.  No lane depends on another, so there is no shared memory and no barrier.
#include "common.h"
#include <cstring>

namespace {

constexpr int kWarps = 4;
constexpr long long kChunkOps = 1LL << 20;                                 // ops per launch

// butterfly output k of the VP8 WHT on (a, b, c, d): t0 + t1, t3 + t2, t0 - t1, t3 - t2
__device__ __forceinline__ int wht_bfly(int a, int b, int c, int d, int k)
{
    const int t0 = a + d, t1 = b + c, t2 = b - c, t3 = a - d;
    return k == 0 ? t0 + t1 : k == 1 ? t3 + t2 : k == 2 ? t0 - t1 : t3 - t2;
}

// output k of the VP7 1-D transform of (v0, v1, v2, v3) before its shift, in unsigned as the reference keeps it: a1 + d1, b1 + c1,
// b1 - c1, a1 - d1 (the reference's positions 0, 1, 2, 3)
__device__ __forceinline__ unsigned vp7_1d(int v0, int v1, int v2, int v3, int k)
{
    const unsigned a1 = (unsigned)((v0 + v2) * 23170), b1 = (unsigned)((v0 - v2) * 23170);
    const unsigned c1 = (unsigned)(v1 * 12540 - v3 * 30274), d1 = (unsigned)(v1 * 30274 + v3 * 12540);
    return k == 0 ? a1 + d1 : k == 1 ? b1 + c1 : k == 2 ? b1 - c1 : a1 - d1;
}

// the VP8 1-D IDCT of (v0, v1, v2, v3)
__device__ __forceinline__ void vp8_1d(int v0, int v1, int v2, int v3, int (&o)[4])
{
    const int t0 = v0 + v2, t1 = v0 - v2;
    const int t2 = ((v1 * 35468) >> 16) - (((v3 * 20091) >> 16) + v3);
    const int t3 = (((v1 * 20091) >> 16) + v1) + ((v3 * 35468) >> 16);
    o[0] = t0 + t3; o[1] = t1 + t2; o[2] = t1 - t2; o[3] = t0 - t3;
}

// luma_dc_wht: the value written to block[b >> 2][b & 3][0], b = 0..15, from dc[16]
__device__ __forceinline__ int16_t wht_value(const int16_t (&dc)[16], int b, bool vp7)
{
    const int y = b >> 2, x = b & 3;
    int t[4];
    if (vp7) {
#pragma unroll
        for (int r = 0; r < 4; r++) t[r] = (int16_t)((int)vp7_1d(dc[4 * r], dc[4 * r + 1], dc[4 * r + 2], dc[4 * r + 3], x) >> 14);
        return (int16_t)((int)(vp7_1d(t[0], t[1], t[2], t[3], y) + 0x20000u) >> 18);
    }
#pragma unroll
    for (int c = 0; c < 4; c++) t[c] = (int16_t)wht_bfly(dc[c], dc[4 + c], dc[8 + c], dc[12 + c], y);
    return (int16_t)((wht_bfly(t[0], t[1], t[2], t[3], x) + 3) >> 3);
}

// the DC-only value: dc_add's from block[0], and (VP7) luma_dc_wht_dc's from dc[0]; VP8's wht_dc is (dc0 + 3) >> 3, see wht_dc_value
__device__ __forceinline__ int dc_value(int b0, bool vp7) { return vp7 ? (23170 * (23170 * b0 >> 14) + 0x20000) >> 18 : (b0 + 4) >> 3; }
__device__ __forceinline__ int16_t wht_dc_value(int dc0, bool vp7) { return (int16_t)(vp7 ? (23170 * (23170 * dc0 >> 14) + 0x20000) >> 18 : (dc0 + 3) >> 3); }

// idct_add's residual of a 4x4 block, res[row * 4 + col]
__device__ __forceinline__ void residual4x4(const int16_t (&b)[16], bool vp7, int (&res)[16])
{
    int16_t tmp[16];
    if (vp7) {
#pragma unroll
        for (int r = 0; r < 4; r++)
#pragma unroll
            for (int k = 0; k < 4; k++) tmp[4 * r + k] = (int16_t)((int)vp7_1d(b[4 * r], b[4 * r + 1], b[4 * r + 2], b[4 * r + 3], k) >> 14);
#pragma unroll
        for (int i = 0; i < 4; i++)
#pragma unroll
            for (int k = 0; k < 4; k++) res[4 * k + i] = (int)(vp7_1d(tmp[i], tmp[4 + i], tmp[8 + i], tmp[12 + i], k) + 0x20000u) >> 18;
        return;
    }
    int o[4];
#pragma unroll
    for (int i = 0; i < 4; i++) {
        vp8_1d(b[i], b[4 + i], b[8 + i], b[12 + i], o);
#pragma unroll
        for (int k = 0; k < 4; k++) tmp[4 * i + k] = (int16_t)o[k];
    }
#pragma unroll
    for (int i = 0; i < 4; i++) {
        vp8_1d(tmp[i], tmp[4 + i], tmp[8 + i], tmp[12 + i], o);
#pragma unroll
        for (int k = 0; k < 4; k++) res[4 * i + k] = (o[k] + 4) >> 3;
    }
}

__device__ __forceinline__ uint32_t add_word(uint32_t w, int r0, int r1, int r2, int r3)
{
    const int r[4] = { r0, r1, r2, r3 };
    uint32_t o = 0;
#pragma unroll
    for (int k = 0; k < 4; k++) o |= (uint32_t)min(max((int)((w >> (8 * k)) & 0xFF) + r[k], 0), 255) << (8 * k);
    return o;
}

// the four rows of a 4x4 block at dst (4-byte aligned), as 4-byte words
__device__ __forceinline__ void add_residual(uint8_t *dst, long long stride, const int (&res)[16])
{
#pragma unroll
    for (int r = 0; r < 4; r++) {
        uint32_t *p = reinterpret_cast<uint32_t *>(dst + r * stride);
        *p = add_word(*p, res[4 * r], res[4 * r + 1], res[4 * r + 2], res[4 * r + 3]);
    }
}
__device__ __forceinline__ void add_dc(uint8_t *dst, long long stride, int dc)
{
#pragma unroll
    for (int r = 0; r < 4; r++) {
        uint32_t *p = reinterpret_cast<uint32_t *>(dst + r * stride);
        *p = add_word(*p, dc, dc, dc, dc);
    }
}

__device__ __forceinline__ void load16(const int16_t *p, int16_t (&v)[16])          // two 16-byte loads (p 16-byte aligned)
{
    const int4 a = reinterpret_cast<const int4 *>(p)[0], b = reinterpret_cast<const int4 *>(p)[1];
    const int w[8] = { a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w };
#pragma unroll
    for (int k = 0; k < 8; k++) {
        v[2 * k] = (int16_t)(w[k] & 0xFFFF);
        v[2 * k + 1] = (int16_t)((unsigned)w[k] >> 16);
    }
}

struct ResArgs {
    const B200Vp8ResidualOp *ops;
    long long nops;
    const int16_t *coef;
    uint8_t *dst[3];
    long long ls_y, ls_uv;
    int is_vp7;
};

__global__ void __launch_bounds__(32 * kWarps) vp8_residual_kernel(ResArgs a)
{
    const long long i = (long long)blockIdx.x * kWarps + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (i >= a.nops || lane >= 24) return;
    const B200Vp8ResidualOp &op = a.ops[i];
    const long long off = op.coef_off;
    if (op.mb_x < 0 || op.mb_y < 0 || off < 0 || (off & 7)) return;
    const bool luma = lane < 16, vp7 = a.is_vp7 != 0;
    if (luma && !(op.flags & B200_VP8_RESIDUAL_LUMA)) return;
    const int row = luma ? lane >> 2 : 4 + ((lane - 16) >> 2), k = lane & 3;
    const uint8_t *nz = op.nnz[row];
    const int n0 = nz[0], n1 = nz[1], n2 = nz[2], n3 = nz[3];
    if (!(n0 | n1 | n2 | n3)) return;
    const bool all_dc = n0 <= 1 && n1 <= 1 && n2 <= 1 && n3 <= 1;      // idct_mb: !(nnz4 & ~0x01010101) -> dc_add4y / dc_add4uv
    const int nnz = nz[k];
    if (!all_dc && nnz == 0) return;
    const int16_t *mb = a.coef + off;
    int16_t dc0 = 0;                                                     // the block's coefficient 0 after the WHT
    bool have_dc0 = false;
    if (luma && op.y2_nnz) {
        if (op.y2_nnz == 1) {
            dc0 = wht_dc_value(mb[384], vp7);
        } else {
            int16_t y2[16];
            load16(mb + 384, y2);
            dc0 = wht_value(y2, lane, vp7);
        }
        have_dc0 = true;
    }
    uint8_t *dst;
    long long ls;
    if (luma) {
        ls = a.ls_y;
        dst = a.dst[0] + ((long long)op.mb_y * 16 + 4 * (lane >> 2)) * ls + (long long)op.mb_x * 16 + 4 * k;
    } else {
        ls = a.ls_uv;
        dst = a.dst[row - 3] + ((long long)op.mb_y * 8 + 4 * (k >> 1)) * ls + (long long)op.mb_x * 8 + 4 * (k & 1);
    }
    const int16_t *blk = mb + 16 * lane;
    if (all_dc || nnz == 1) {                                           // dc_add: coefficient 0 only
        add_dc(dst, ls, dc_value(have_dc0 ? dc0 : blk[0], vp7));
        return;
    }
    int16_t b[16];
    load16(blk, b);
    if (have_dc0) b[0] = dc0;
    int res[16];
    residual4x4(b, vp7, res);
    add_residual(dst, ls, res);
}

// ---- drop-in members (host pointers): the coefficients and samples the reference function reads are staged in the device scratch,
// one warp of the members' kernel runs the member, and what the reference writes comes back.
enum { M_WHT, M_WHT_DC, M_IDCT, M_DC, M_DC4Y, M_DC4UV };
constexpr int kMemberPitch = 16;                                          // bytes per staged dst row

// blocks: 16 coefficients per block, dense; M_WHT / M_WHT_DC write coefficient 0 of blocks 0..15 from dc; the others update the
// staged dst (pitch kMemberPitch) and clear what the reference clears
__global__ void vp8_idct_member_kernel(int kind, int is_vp7, int16_t *blocks, const int16_t *dc, uint8_t *dst)
{
    const int lane = threadIdx.x;
    const bool vp7 = is_vp7 != 0;
    if (kind == M_WHT || kind == M_WHT_DC) {
        if (lane >= 16) return;
        int16_t v[16];
#pragma unroll
        for (int k = 0; k < 16; k++) v[k] = kind == M_WHT ? dc[k] : 0;
        blocks[16 * lane] = kind == M_WHT ? wht_value(v, lane, vp7) : wht_dc_value(dc[0], vp7);
        return;
    }
    const int nblk = kind == M_IDCT || kind == M_DC ? 1 : 4;
    if (lane >= nblk) return;
    int16_t *blk = blocks + 16 * lane;
    uint8_t *d = dst + (kind == M_DC4UV ? 4 * (lane >> 1) * kMemberPitch + 4 * (lane & 1) : 4 * lane);
    if (kind != M_IDCT) {
        add_dc(d, kMemberPitch, dc_value(blk[0], vp7));
        blk[0] = 0;
        return;
    }
    int16_t b[16];
#pragma unroll
    for (int k = 0; k < 16; k++) b[k] = blk[k];
    int res[16];
    residual4x4(b, vp7, res);
    add_residual(d, kMemberPitch, res);
#pragma unroll
    for (int k = 0; k < 16; k++) blk[k] = 0;
}

// kind's member on host memory: dst rows x cols (0 for the WHT members), the coefficients it reads (`coef`, 16 per block, nblk blocks,
// only coefficient 0 of each where dc0_only), dc (the WHT members)
void member_host(int kind, int is_vp7, uint8_t *dst, ptrdiff_t stride, int16_t *coef, int16_t *dc)
{
    const int rows = kind == M_DC4UV ? 8 : 4, cols = kind == M_DC4Y ? 16 : kind == M_DC4UV ? 8 : 4;
    const int nblk = kind == M_WHT || kind == M_WHT_DC ? 16 : kind == M_DC4Y || kind == M_DC4UV ? 4 : 1;
    const bool wht = kind == M_WHT || kind == M_WHT_DC, dc0_only = kind != M_IDCT;
    B200HostCall call("vp8 residual member", nullptr, 1024);
    uint8_t *scr = call.scratch;
    cudaStream_t st = call.stream;
    int16_t *dblk = (int16_t *)scr, *ddc = (int16_t *)(scr + 512);
    uint8_t *ddst = scr + 576;
    const size_t bpitch = 16 * sizeof(int16_t);
    if (!wht) {
        call.check(b200_h2d_rows(ddst, kMemberPitch, dst, stride, (size_t)cols, (size_t)rows, st), "h2d dst");
        call.check(b200_h2d_rows(dblk, bpitch, coef, (ptrdiff_t)bpitch, dc0_only ? sizeof(int16_t) : bpitch, (size_t)nblk, st), "h2d coef");
    } else {
        call.check(cudaMemcpyAsync(ddc, dc, (kind == M_WHT ? 16 : 1) * sizeof(int16_t), cudaMemcpyHostToDevice, st), "h2d dc");
    }
    vp8_idct_member_kernel<<<1, 32, 0, st>>>(kind, is_vp7, dblk, ddc, ddst);
    B200_LAUNCHED();
    call.launched();
    if (!wht) call.check(b200_d2h_rows(dst, stride, ddst, kMemberPitch, (size_t)cols, (size_t)rows, st), "d2h dst");
    call.check(b200_d2h_rows(coef, (ptrdiff_t)bpitch, dblk, bpitch, dc0_only ? sizeof(int16_t) : bpitch, (size_t)nblk, st), "d2h coef");
    call.sync();
    if (kind == M_WHT) memset(dc, 0, 16 * sizeof(int16_t));                // the reference clears dc[0..15] (wht) / dc[0] (wht_dc)
    if (kind == M_WHT_DC) dc[0] = 0;
}

template <int V7> void m_wht(int16_t block[4][4][16], int16_t dc[16]) { member_host(M_WHT, V7, nullptr, 0, &block[0][0][0], dc); }
template <int V7> void m_wht_dc(int16_t block[4][4][16], int16_t dc[16]) { member_host(M_WHT_DC, V7, nullptr, 0, &block[0][0][0], dc); }
template <int V7> void m_idct(uint8_t *dst, int16_t block[16], ptrdiff_t stride) { member_host(M_IDCT, V7, dst, stride, block, nullptr); }
template <int V7> void m_dc(uint8_t *dst, int16_t block[16], ptrdiff_t stride) { member_host(M_DC, V7, dst, stride, block, nullptr); }
template <int V7> void m_dc4y(uint8_t *dst, int16_t block[4][16], ptrdiff_t stride) { member_host(M_DC4Y, V7, dst, stride, block[0], nullptr); }
template <int V7> void m_dc4uv(uint8_t *dst, int16_t block[4][16], ptrdiff_t stride) { member_host(M_DC4UV, V7, dst, stride, block[0], nullptr); }

template <int V7> void fill(B200VP8DSPContext *c)
{
    c->vp8_luma_dc_wht = m_wht<V7>;
    c->vp8_luma_dc_wht_dc = m_wht_dc<V7>;
    c->vp8_idct_add = m_idct<V7>;
    c->vp8_idct_dc_add = m_dc<V7>;
    c->vp8_idct_dc_add4y = m_dc4y<V7>;
    c->vp8_idct_dc_add4uv = m_dc4uv<V7>;
}

} // namespace

// vp8mc.cu's b200_vp8_dsp_init calls this after it has cleared the context and filled the MC tables
void b200_vp8_fill_residual(B200VP8DSPContext *c, int is_vp7)
{
    if (is_vp7) fill<1>(c);
    else fill<0>(c);
}

B200_API int b200_vp8_residual_frame_device(B200Device *dev, int is_vp7, int64_t nops, const B200Vp8ResidualOp *ops, const int16_t *coef,
                                            uint8_t *const dst[3], ptrdiff_t ls_y, ptrdiff_t ls_uv)
{
    if (nops < 0 || (is_vp7 != 0 && is_vp7 != 1)) { b200_set_error("vp8 residual frame: negative nops or is_vp7 not 0 / 1"); return B200_EINVAL; }
    if (nops == 0) return 0;
    if (!ops || !coef || !dst || ((uintptr_t)ops & 7) || ((uintptr_t)coef & 15)) {
        b200_set_error("vp8 residual frame: NULL or misaligned ops / coef");
        return B200_EINVAL;
    }
    if ((ls_y & 3) || (ls_uv & 3)) { b200_set_error("vp8 residual frame: line size not a multiple of 4"); return B200_EINVAL; }
    for (int p = 0; p < 3; p++)
        if (!dst[p] || ((uintptr_t)dst[p] & 3)) { b200_set_error("vp8 residual frame: plane %d NULL or not 4-byte aligned", p); return B200_EINVAL; }
    if (int r = b200_use_device(dev)) return r;
    ResArgs a;
    memset(&a, 0, sizeof(a));
    a.coef = coef;
    for (int p = 0; p < 3; p++) a.dst[p] = dst[p];
    a.ls_y = (long long)ls_y;
    a.ls_uv = (long long)ls_uv;
    a.is_vp7 = is_vp7;
    for (long long b = 0; b < (long long)nops; b += kChunkOps) {
        a.ops = ops + b;
        a.nops = (long long)nops - b < kChunkOps ? (long long)nops - b : kChunkOps;
        const unsigned grid = (unsigned)((a.nops + kWarps - 1) / kWarps);
        vp8_residual_kernel<<<grid, 32 * kWarps, 0, dev->stream>>>(a);
        B200_LAUNCHED();
        B200_CUDA_OK(cudaGetLastError());
    }
    return 0;
}
