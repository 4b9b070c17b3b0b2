// vp8mc.cu — VP8 / VP7 inter prediction on sm_90a: put_vp8_epel_pixels_tab[3][3][3] and put_vp8_bilinear_pixels_tab[3][3][3] of
// VP8DSPContext (libavcodec/vp8dsp.h:72-81) as ff_vp78dsp_init fills them (vp8dsp.c:641-688), and a one-call-per-frame device entry
// that runs the decoder's per-block sequence (vp8_mc_luma / vp8_mc_chroma, vp8.c:1831-1929) with edge emulation fused into the reads.
//
// Reference semantics reproduced bit for bit (checker: oracle/vp8dsp_oracle.c), vp8dsp.c:459-639:
//   6-tap     clip((F0 s[-2] - F1 s[-1] + F2 s[0] + F3 s[1] - F4 s[2] + F5 s[3] + 64) >> 7), F = subpel_filters[phase - 1]
//   4-tap     the same row with F0 and F5 left out, whatever the phase's parity (the decoder only uses odd phases here, whose outer
//             taps are 0; a drop-in member may be handed an even one)
//   bilinear  ((8 - m) s[0] + m s[1] + 4) >> 3 == (16 ((8 - m) s[0] + m s[1]) + 64) >> 7: the 6-tap form with the row
//             { 0, 0, 128 - 16 m, 16 m, 0, 0 }, whose result never leaves 0..255, so the clip changes nothing
//   2-D       the horizontal pass is clipped to uint8 before the vertical pass filters it
// One filter path: phase 0 is the identity row { 0, 0, 128, 0, 0, 0 } in every bank, so the 1-D and full-pel entries are the 2-D path
// with an identity pass.  The horizontal pass covers rows -2 .. h + 2 and stores clipped uint8, the vertical pass follows.
//
// Kernel: one warp per op, four per CTA, each warp with its own shared memory and no CTA-wide barrier.  The warp stages the op's
// (w + 5) x (h + 5) window from (src_x - 2, src_y - 2) through clamped coordinates (edge replication), for a CHROMA op the U and the V
// window in the same pass, runs the horizontal pass four output columns per item into a second shared array, then the vertical pass,
// and stores each output row as 4-byte words.  The drop-in members stage what the reference function reads in the device scratch and
// run the same kernel on it, one op, with the table position's filter banks forced.
#include "common.h"
#include <cstring>

namespace {

constexpr int kWarps = 4;
constexpr int kWinRows = 21;                              // h + 5 for h <= 16
constexpr int kWinPitch = 24;                             // bytes per window row: w + 5 <= 21, rounded up to 4-byte words
constexpr int kTmpPitch = 16;                             // bytes per row of the horizontal pass
constexpr int kPlaneSmem = kWinRows * (kWinPitch + kTmpPitch);
constexpr int kWarpSmem = 2 * kPlaneSmem;                 // U and V of a CHROMA op
constexpr int kMaxRefs = 3;
constexpr long long kChunkOps = 1LL << 20;                // ops per launch

// [bank: 0 6-tap, 1 4-tap, 2 bilinear][phase 0..7][tap at -2 .. +3]: subpel_filters (vp8dsp.c:459-467, the sixtap_filters of RFC 6386)
// with the reference's signs applied; the 4-tap bank is the 6-tap one with its outer taps zeroed
__constant__ int16_t c_vp8_filters[3][8][6] = {
    { { 0, 0, 128, 0, 0, 0 }, { 0, -6, 123, 12, -1, 0 }, { 2, -11, 108, 36, -8, 1 }, { 0, -9, 93, 50, -6, 0 },
      { 3, -16, 77, 77, -16, 3 }, { 0, -6, 50, 93, -9, 0 }, { 1, -8, 36, 108, -11, 2 }, { 0, -1, 12, 123, -6, 0 } },
    { { 0, 0, 128, 0, 0, 0 }, { 0, -6, 123, 12, -1, 0 }, { 0, -11, 108, 36, -8, 0 }, { 0, -9, 93, 50, -6, 0 },
      { 0, -16, 77, 77, -16, 0 }, { 0, -6, 50, 93, -9, 0 }, { 0, -8, 36, 108, -11, 0 }, { 0, -1, 12, 123, -6, 0 } },
    { { 0, 0, 128, 0, 0, 0 }, { 0, 0, 112, 16, 0, 0 }, { 0, 0, 96, 32, 0, 0 }, { 0, 0, 80, 48, 0, 0 },
      { 0, 0, 64, 64, 0, 0 }, { 0, 0, 48, 80, 0, 0 }, { 0, 0, 32, 96, 0, 0 }, { 0, 0, 16, 112, 0, 0 } },
};

struct McArgs {
    const B200Vp8McOp *ops;
    long long nops;
    uint8_t *dst[3];
    long long ls_y, ls_uv;
    int rw[2], rh[2];          // [luma, chroma]: reads clamp to [0, rw) x [0, rh)
    int dw[2], dh[2];          // blocks must lie inside [0, dw) x [0, dh)
    int nrefs, bilinear;
    int bank_h, bank_v;        // drop-in members: the table position's bank per direction; -1: from the phase (the decoder's subpel_idx)
    B200Vp8McRef refs[kMaxRefs];
};

__device__ __forceinline__ int bank_of(int phase, int forced, int bilinear)
{
    return bilinear ? 2 : forced >= 0 ? forced : (phase & 1) ? 1 : 0;
}

// the device-side guard: an op it refuses writes nothing
__device__ __forceinline__ bool op_ok(const B200Vp8McOp &op, const McArgs &a)
{
    const int w = op.w, c = op.plane;
    if (c > 1 || (w != 4 && w != 8 && w != 16) || op.h < 1 || op.h > 16 || op.mx > 7 || op.my > 7 || op.ref >= a.nrefs) return false;
    if (!a.bilinear && a.bank_h < 0 && w == 16 && ((op.mx | op.my) & 1)) return false;     // put_vp8_epel_pixels_tab[0][1][*] / [0][*][1]
    return (op.dst_x & 3) == 0 && op.dst_x >= 0 && op.dst_y >= 0 && op.dst_x <= a.dw[c] - w && op.dst_y <= a.dh[c] - op.h;
}

__global__ void __launch_bounds__(32 * kWarps) vp8_mc_kernel(McArgs a)
{
    extern __shared__ uint32_t vp8_smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long i = (long long)blockIdx.x * kWarps + warp;
    if (i >= a.nops) return;
    const B200Vp8McOp op = a.ops[i];
    if (!op_ok(op, a)) return;                                            // warp-uniform
    const int c = op.plane, np = c ? 2 : 1, w = op.w, h = op.h, q = w >> 2, wc = w + 5, wr = h + 5;
    uint8_t *smem = reinterpret_cast<uint8_t *>(vp8_smem) + warp * kWarpSmem;
    const B200Vp8McRef &ref = a.refs[op.ref];
    const long long X = (long long)op.src_x - 2, Y = (long long)op.src_y - 2;
    const int rw = a.rw[c], rh = a.rh[c];
    for (int e = lane; e < np * wr * wc; e += 32) {
        const int p = e >= wr * wc, r = e - p * wr * wc, wi = r / wc, wj = r - wi * wc;
        long long yy = Y + wi, xx = X + wj;
        yy = yy < 0 ? 0 : yy >= rh ? rh - 1 : yy;
        xx = xx < 0 ? 0 : xx >= rw ? rw - 1 : xx;
        const uint8_t *base = c == 0 ? ref.y : p ? ref.v : ref.u;
        smem[p * kPlaneSmem + wi * kWinPitch + wj] = base[yy * (c ? ref.ls_uv : ref.ls_y) + xx];
    }
    __syncwarp();
    int f[6];
    const int16_t *fh = c_vp8_filters[bank_of(op.mx, a.bank_h, a.bilinear)][op.mx];
#pragma unroll
    for (int t = 0; t < 6; t++) f[t] = fh[t];
    for (int e = lane; e < np * wr * q; e += 32) {                        // window row wi, output columns x0 .. x0 + 3
        const int p = e >= wr * q, r = e - p * wr * q, wi = r / q, x0 = (r - wi * q) * 4;
        const uint8_t *s = smem + p * kPlaneSmem + wi * kWinPitch + x0;  // window column x0 is source column x0 - 2
        uint32_t word = 0;
#pragma unroll
        for (int k = 0; k < 4; k++) {
            int acc = 64;
#pragma unroll
            for (int t = 0; t < 6; t++) acc += f[t] * s[k + t];
            word |= (uint32_t)min(max(acc >> 7, 0), 255) << (8 * k);
        }
        *reinterpret_cast<uint32_t *>(smem + p * kPlaneSmem + kWinRows * kWinPitch + wi * kTmpPitch + x0) = word;
    }
    __syncwarp();
    const int16_t *fv = c_vp8_filters[bank_of(op.my, a.bank_v, a.bilinear)][op.my];
#pragma unroll
    for (int t = 0; t < 6; t++) f[t] = fv[t];
    const long long ls = c ? a.ls_uv : a.ls_y;
    for (int e = lane; e < np * h * q; e += 32) {                         // output row y, columns x0 .. x0 + 3: tmp rows y .. y + 5
        const int p = e >= h * q, r = e - p * h * q, y = r / q, x0 = (r - y * q) * 4;
        const uint8_t *s = smem + p * kPlaneSmem + kWinRows * kWinPitch + y * kTmpPitch + x0;
        uint32_t word = 0;
#pragma unroll
        for (int k = 0; k < 4; k++) {
            int acc = 64;
#pragma unroll
            for (int t = 0; t < 6; t++) acc += f[t] * s[t * kTmpPitch + k];
            word |= (uint32_t)min(max(acc >> 7, 0), 255) << (8 * k);
        }
        uint8_t *d = a.dst[c ? 1 + p : 0] + (long long)(op.dst_y + y) * ls + op.dst_x + x0;
        *reinterpret_cast<uint32_t *>(d) = word;
    }
}

cudaError_t launch(McArgs a, cudaStream_t st)
{
    const long long nops = a.nops;
    const B200Vp8McOp *ops = a.ops;
    for (long long b = 0; b < nops; b += kChunkOps) {
        a.ops = ops + b;
        a.nops = nops - b < kChunkOps ? nops - b : kChunkOps;
        const unsigned grid = (unsigned)((a.nops + kWarps - 1) / kWarps);
        vp8_mc_kernel<<<grid, 32 * kWarps, kWarps * kWarpSmem, st>>>(a);
        B200_LAUNCHED();
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
}

// ---- drop-in members (host pointers).  vt / ht: 0 no filter, 4 / 6 taps (epel), 1 bilinear.  The samples the reference function
// reads are copied into a dense device window that is the op's whole reference plane (the kernel's other reads clamp into it and
// meet zero taps), the block is predicted into a dense device buffer and copied back.
void member_host(int W, int vt, int ht, uint8_t *dst, ptrdiff_t dststride, const uint8_t *src, ptrdiff_t srcstride, int h, int mx, int my)
{
    const bool bil = vt == 1 || ht == 1;
    if (!ht) mx = 0;
    if (!vt) my = 0;
    if (h < 1 || h > 2 * W || mx < 0 || mx > 7 || my < 0 || my > 7 || (!bil && ((ht && !mx) || (vt && !my)))) {
        b200_set_error("vp8 mc member: h %d outside 1..%d, or phase (%d, %d) outside 0..7 or 0 where an epel member filters", h, 2 * W, mx, my);
        return;
    }
    const int left = ht == 6 ? 2 : ht == 4 ? 1 : 0, right = ht == 6 ? 3 : ht == 4 ? 2 : ht == 1 ? 1 : 0;
    const int top = vt == 6 ? 2 : vt == 4 ? 1 : 0, bottom = vt == 6 ? 3 : vt == 4 ? 2 : vt == 1 ? 1 : 0;
    const int wc = left + W + right, wr = top + h + bottom;
    const size_t wpitch = 32, wbytes = (wpitch * wr + 255) & ~(size_t)255;
    B200HostCall call("vp8 motion compensation", nullptr, wbytes + 256 + 16 * 32);
    uint8_t *scr = call.scratch;
    cudaStream_t st = call.stream;
    uint8_t *dwin = scr, *dop = scr + wbytes, *ddst = dop + 256;
    call.check(b200_h2d_rows(dwin, wpitch, src - top * srcstride - left, srcstride, (size_t)wc, (size_t)wr, st), "h2d window");
    B200Vp8McOp op[2];                                                   // ops take h <= 16: a taller call is two ops
    memset(op, 0, sizeof(op));
    const int nops = h > 16 ? 2 : 1;
    for (int k = 0; k < nops; k++) {
        op[k].src_x = left;
        op[k].src_y = top + 16 * k;
        op[k].dst_y = 16 * k;
        op[k].plane = B200_VP8_MC_LUMA;
        op[k].w = (uint8_t)W;
        op[k].h = (uint8_t)(k ? h - 16 : h > 16 ? 16 : h);
        op[k].mx = (uint8_t)mx;
        op[k].my = (uint8_t)my;
    }
    call.check(cudaMemcpyAsync(dop, op, sizeof(op), cudaMemcpyHostToDevice, st), "h2d op");
    McArgs a;
    memset(&a, 0, sizeof(a));
    a.ops = (const B200Vp8McOp *)dop;
    a.nops = nops;
    a.dst[0] = ddst;
    a.ls_y = 16;
    a.rw[0] = wc;
    a.rh[0] = wr;
    a.dw[0] = W;
    a.dh[0] = h;
    a.nrefs = 1;
    a.bilinear = bil;
    a.bank_h = ht == 4 ? 1 : 0;
    a.bank_v = vt == 4 ? 1 : 0;
    a.refs[0].y = dwin;
    a.refs[0].ls_y = (ptrdiff_t)wpitch;
    call.check(launch(a, st), "launch");
    call.check(b200_d2h_rows(dst, dststride, ddst, 16, (size_t)W, (size_t)h, st), "d2h");
    call.sync();
}

template <int W, int VT, int HT>
void m_mc(uint8_t *dst, ptrdiff_t dststride, const uint8_t *src, ptrdiff_t srcstride, int h, int mx, int my)
{
    member_host(W, VT, HT, dst, dststride, src, srcstride, h, mx, my);
}

// VP78_MC_FUNC / VP78_BILINEAR_MC_FUNC (vp8dsp.c:641-661): [v][h] = 0 none, 1 4-tap, 2 6-tap; the full-pel function is shared by both
// tables, and the bilinear functions by the positions that filter in the same directions
template <int I, int W>
void fill_size(B200VP8DSPContext *c)
{
    c->put_vp8_epel_pixels_tab[I][0][0] = m_mc<W, 0, 0>;
    if (W != 16) {
        c->put_vp8_epel_pixels_tab[I][0][1] = m_mc<W, 0, 4>;
        c->put_vp8_epel_pixels_tab[I][1][0] = m_mc<W, 4, 0>;
        c->put_vp8_epel_pixels_tab[I][1][1] = m_mc<W, 4, 4>;
        c->put_vp8_epel_pixels_tab[I][1][2] = m_mc<W, 4, 6>;
        c->put_vp8_epel_pixels_tab[I][2][1] = m_mc<W, 6, 4>;
    }
    c->put_vp8_epel_pixels_tab[I][0][2] = m_mc<W, 0, 6>;
    c->put_vp8_epel_pixels_tab[I][2][0] = m_mc<W, 6, 0>;
    c->put_vp8_epel_pixels_tab[I][2][2] = m_mc<W, 6, 6>;
    c->put_vp8_bilinear_pixels_tab[I][0][0] = m_mc<W, 0, 0>;
    c->put_vp8_bilinear_pixels_tab[I][0][1] = c->put_vp8_bilinear_pixels_tab[I][0][2] = m_mc<W, 0, 1>;
    c->put_vp8_bilinear_pixels_tab[I][1][0] = c->put_vp8_bilinear_pixels_tab[I][2][0] = m_mc<W, 1, 0>;
    c->put_vp8_bilinear_pixels_tab[I][1][1] = c->put_vp8_bilinear_pixels_tab[I][1][2] = m_mc<W, 1, 1>;
    c->put_vp8_bilinear_pixels_tab[I][2][1] = c->put_vp8_bilinear_pixels_tab[I][2][2] = m_mc<W, 1, 1>;
}

} // namespace

void b200_vp8_fill_residual(B200VP8DSPContext *c, int is_vp7);           // vp8idct.cu

B200_API int b200_vp8_dsp_init(B200VP8DSPContext *c, int is_vp7)
{
    if (!c || (is_vp7 != 0 && is_vp7 != 1)) { b200_set_error("vp8 dsp init: NULL context or is_vp7 not 0 / 1"); return B200_EINVAL; }
    if (!b200_default_device()) return B200_ENODEV;
    memset(c, 0, sizeof(*c));                                            // the loop-filter members: NULL (b200_vp8_dsp_init_loopfilter fills them)
    fill_size<0, 16>(c);
    fill_size<1, 8>(c);
    fill_size<2, 4>(c);
    b200_vp8_fill_residual(c, is_vp7);
    return 0;
}

B200_API int b200_vp8_mc_frame_device(B200Device *dev, int bilinear, int mb_width, int mb_height, int nrefs, const B200Vp8McRef *refs,
                                      int64_t nops, const B200Vp8McOp *ops, uint8_t *const dst[3], ptrdiff_t ls_y, ptrdiff_t ls_uv)
{
    if (nops < 0 || nrefs < 1 || nrefs > kMaxRefs || mb_width < 1 || mb_height < 1 || mb_width > (1 << 20) / 16 || mb_height > (1 << 20) / 16) {
        b200_set_error("vp8 mc frame: negative nops, nrefs outside 1..3 or a macroblock count outside 1..65536");
        return B200_EINVAL;
    }
    if (nops == 0) return 0;
    if (!refs || !ops || !dst || ((uintptr_t)ops & 3)) { b200_set_error("vp8 mc frame: NULL or misaligned refs / ops / dst"); return B200_EINVAL; }
    if ((ls_y & 3) || (ls_uv & 3)) { b200_set_error("vp8 mc frame: line size not a multiple of 4"); return B200_EINVAL; }
    for (int p = 0; p < 3; p++)
        if (!dst[p] || ((uintptr_t)dst[p] & 3)) { b200_set_error("vp8 mc frame: plane %d NULL or not 4-byte aligned", p); return B200_EINVAL; }
    McArgs a;
    memset(&a, 0, sizeof(a));
    for (int r = 0; r < nrefs; r++) {
        if (!refs[r].y || !refs[r].u || !refs[r].v) { b200_set_error("vp8 mc frame: reference %d has a NULL plane", r); return B200_EINVAL; }
        a.refs[r] = refs[r];
    }
    if (int r = b200_use_device(dev)) return r;
    a.ops = ops;
    a.nops = (long long)nops;
    for (int p = 0; p < 3; p++) a.dst[p] = dst[p];
    a.ls_y = (long long)ls_y;
    a.ls_uv = (long long)ls_uv;
    a.rw[0] = a.dw[0] = 16 * mb_width;
    a.rh[0] = a.dh[0] = 16 * mb_height;
    a.rw[1] = a.dw[1] = 8 * mb_width;
    a.rh[1] = a.dh[1] = 8 * mb_height;
    a.nrefs = nrefs;
    a.bilinear = bilinear != 0;
    a.bank_h = a.bank_v = -1;
    B200_CUDA_OK(launch(a, dev->stream));
    return 0;
}
