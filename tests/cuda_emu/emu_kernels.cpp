// emu_kernels.cpp — TEST INFRASTRUCTURE ONLY.  Includes the [device-code ...] blocks that tests/test_cuda_emu.py cuts out of
// ffmpeg_b200/csrc/*.cu (into tests/cuda_emu/_gen/) and exposes one C entry per kernel that launches it with the same grid
// arithmetic as the library's host code.
#include "emu.h"
#include "b200dsp.h"

static inline int ceil_div(long long a, long long b) { return (int)((a + b - 1) / b); }

namespace sws {
#include "_gen/sws_new.inc"
#include "_gen/sws_nvout.inc"
}
namespace fdsp {
#include "_gen/fdsp.inc"
}
namespace hbd {
#include "_gen/idct_hbd.inc"
}
namespace unq {
constexpr int WARPS = 4;
#include "_gen/unquant.inc"
}

namespace pfa {
#include "_gen/tx_pfa.inc"
}
namespace txi {
#include "_gen/tx_int32.inc"         // likewise
}
namespace dct {
#include "_gen/tx_dct.inc"           // exercised through the library's entry points in test_tx_whole_path_on_emulated_device
}

extern "C" {

// tables = what b200_tx_pfa_tables() of the library returns (host-only), layout8 as it reports it; after the cosine tables the words
// hold 12 level starts, 12 level counts and the block offsets of the m-point split-radix transform.  One CTA per transform
// (block-synchronous emulation: an OS thread per CUDA thread, dynamic shared memory = nfac sub-transforms).
int emu_tx_pfa(int inv, int len, const int32_t *words, const int32_t *lay, float *out, const float *in, long long stride_floats, long long out_step,
               long long in_step, long long count, float2 *)
{
    pfa::PfaDev P;
    P.in_map = words + lay[0]; P.out_map = words + lay[1]; P.sub_map = words + lay[2];
    P.exp = (const float2 *)(words + lay[3]); P.tab53 = (const float *)(words + lay[4]);
    const float *c = (const float *)(words + lay[5]);
    for (int k = 0; k < 12; k++) P.tabs[k] = nullptr;
    for (int k = 3; k <= (lay[7] & 255); k++) { P.tabs[k] = c; c += (1 << k) / 4 + 1; }
    const int32_t *lv = (const int32_t *)c;
    for (int L = 0; L < 12; L++) { P.lvl_start[L] = lv[L]; P.lvl_cnt[L] = lv[12 + L]; }
    P.blk = lv + 24;
    P.m = lay[6]; P.log2m = lay[7] & 255; P.nfac = lay[7] >> 8; P.len = len;
    P.ms = P.m + (P.m >> 4) + 1;
    const size_t smem = (size_t)P.nfac * P.ms * sizeof(float2);
    const dim3 g((unsigned)(count < 3 ? count : 3)), t(pfa::PFA_THREADS);            // fewer CTAs than transforms: the batch loop runs too
    if (inv) emu_launch_blocks(g, t, smem, [&] { pfa::tx_mdct_pfa_inv_kernel(P, out, in, stride_floats, out_step, in_step, count); });
    else     emu_launch_blocks(g, t, smem, [&] { pfa::tx_mdct_pfa_fwd_kernel(P, out, in, stride_floats, out_step, in_step, count); });
    return 0;
}

void emu_sws_range(int16_t *mid, int w, int rows, int frames, long long dfs, int coeff, int offset, int clip)
{
    emu_launch(dim3(ceil_div(w, 256), rows, frames), dim3(256), [&] { sws::sws_range_kernel(mid, w, dfs, coeff, offset, clip); });
}

static sws::RgbIn mk(const int *r) { sws::RgbIn R; R.bpp = r[0]; R.ro = r[1]; R.go = r[2]; R.bo = r[3]; R.half = r[4]; for (int i = 0; i < 9; i++) R.c[i] = r[5 + i]; return R; }

void emu_sws_rgbin_y(const uint8_t *src, long long sstride, long long sfs, int16_t *dst, int dstW, long long dfs, const int16_t *filter,
                     const int32_t *pos, int fs, const int *rgbin, int lines, int frames)
{
    const sws::RgbIn R = mk(rgbin);
    emu_launch(dim3(ceil_div(dstW, 256), lines, frames), dim3(256),
               [&] { sws::sws_rgbin_hscale_y_kernel(src, sstride, sfs, dst, dstW, dfs, filter, pos, fs, R); });
}

void emu_sws_rgbin_a(const uint8_t *src, long long sstride, long long sfs, int16_t *dst, int dstW, long long dfs, const int16_t *filter,
                     const int32_t *pos, int fs, int sao, int lines, int frames)
{
    emu_launch(dim3(ceil_div(dstW, 256), lines, frames), dim3(256),
               [&] { sws::sws_rgbin_hscale_a_kernel(src, sstride, sfs, dst, dstW, dfs, filter, pos, fs, sao); });
}

void emu_sws_alpha(const int16_t *al, long long alfs, int srcH, uint8_t *dst, long long ds, long long dfs, int dstW, int dstH, int bpp, int ao,
                   const int16_t *vLum, const int32_t *vLumPos, int lfs, const int32_t *rowMode, int full, int frames)
{
    emu_launch(dim3(ceil_div(dstW, 256), dstH, frames), dim3(256),
               [&] { sws::sws_vscale_alpha_kernel(al, alfs, srcH, dst, ds, dfs, dstW, bpp, ao, vLum, vLumPos, lfs, rowMode, full, 0); });
}

void emu_sws_rgbin_uv(const uint8_t *src, long long sstride, long long sfs, int16_t *dstU, int16_t *dstV, int dstW, long long dfs,
                      const int16_t *filter, const int32_t *pos, int fs, const int *rgbin, int lines, int frames)
{
    const sws::RgbIn R = mk(rgbin);
    emu_launch(dim3(ceil_div(dstW, 256), lines, frames), dim3(256),
               [&] { sws::sws_rgbin_hscale_uv_kernel(src, sstride, sfs, dstU, dstV, dstW, dfs, filter, pos, fs, R); });
}

void emu_sws_bgr24_yv12(const uint8_t *src, long long sstride, uint8_t *dy, long long dys, uint8_t *du, long long dus, uint8_t *dv,
                        long long dvs, int w, int h, const int *rgbin)
{
    const sws::RgbIn R = mk(rgbin);
    emu_launch(dim3(ceil_div(w >> 1, 256), (h + 1) / 2, 1), dim3(256),
               [&] { sws::sws_bgr24_yv12_kernel(src, sstride, 0, dy, dys, 0, du, dus, 0, dv, dvs, 0, w, h, R); });
}

void emu_sws_nv_interleave(const uint8_t *u, const uint8_t *v, long long cs, uint8_t *dst, long long ds, int cw, int ch)
{
    emu_launch(dim3(ceil_div(cw, 256), ch, 1), dim3(256), [&] { sws::sws_nv_interleave_kernel(u, v, cs, 0, dst, ds, 0, cw); });
}

int emu_fdsp(int op, long long nvec, int len, void *dst, long long dstS, const void *s0, long long s0S, const void *s1, long long s1S,
             const void *s2, long long s2S, double mul)
{
    fdsp::Operands o = { dst, s0, s1 ? s1 : s0, s2 ? s2 : s0, dstS, s0S, s1S, s2S };
    const dim3 g(ceil_div(len, 256), (unsigned)nvec), t(256);
    switch (op) {
#define EL(OPC, T) case OPC: emu_launch(g, t, [&] { fdsp::fdsp_kernel<T, OPC>(o, 0, len, (T)mul); }); return 0;
    EL(B200_FDSP_VECTOR_FMUL, float) EL(B200_FDSP_VECTOR_FMAC_SCALAR, float) EL(B200_FDSP_VECTOR_DMAC_SCALAR, double)
    EL(B200_FDSP_VECTOR_FMUL_SCALAR, float) EL(B200_FDSP_VECTOR_DMUL_SCALAR, double) EL(B200_FDSP_VECTOR_FMUL_WINDOW, float)
    EL(B200_FDSP_VECTOR_FMUL_ADD, float) EL(B200_FDSP_VECTOR_FMUL_REVERSE, float) EL(B200_FDSP_BUTTERFLIES_FLOAT, float)
    EL(B200_FDSP_VECTOR_DMUL, double)
#undef EL
    case B200_FDSP_SCALARPRODUCT_FLOAT:  emu_launch(dim3(ceil_div(nvec, 128)), dim3(128), [&] { fdsp::fdsp_dot_kernel<float>(o, nvec, len); }); return 0;
    case B200_FDSP_SCALARPRODUCT_DOUBLE: emu_launch(dim3(ceil_div(nvec, 128)), dim3(128), [&] { fdsp::fdsp_dot_kernel<double>(o, nvec, len); }); return 0;
    }
    return -1;
}

int emu_idct_hbd(int depth, int kind, int16_t *blocks, long long n, uint8_t *dest, const int64_t *off, int uls)
{
    const dim3 g(ceil_div(n, 128)), t(128);
#define RUN(D, K) emu_launch(g, t, [&] { hbd::idct_hbd_kernel<D, K>(blocks, n, dest, off, nullptr, uls); })
    if (depth == 10) { if (kind == 0) RUN(10, 0); else if (kind == 1) RUN(10, 1); else RUN(10, 2); }
    else if (depth == 12) { if (kind == 0) RUN(12, 0); else if (kind == 1) RUN(12, 1); else RUN(12, 2); }
    else return -1;
#undef RUN
    return 0;
}

int emu_unquant(int variant, const B200MpvUnquant *p, int16_t *blocks, long long nblocks, const uint8_t *blk_n, const uint8_t *qscale,
                const int8_t *last_index)
{
    unq::UnquantDev P;
    if (!unq::mpv_unquant_params(p, &P)) return -1;
    const dim3 g(ceil_div(nblocks, unq::WARPS)), t(32 * unq::WARPS);
    switch (variant) {
#define CASE(V) case V: emu_launch_warps(g, t, [&] { unq::mpv_unquant_kernel<V>(P, blocks, nblocks, blk_n, qscale, last_index); }); return 0;
    CASE(B200_UNQUANT_MPEG1_INTRA) CASE(B200_UNQUANT_MPEG1_INTER) CASE(B200_UNQUANT_MPEG2_INTRA) CASE(B200_UNQUANT_MPEG2_INTRA_BITEXACT)
    CASE(B200_UNQUANT_MPEG2_INTER) CASE(B200_UNQUANT_H263_INTRA) CASE(B200_UNQUANT_H263_INTER)
#undef CASE
    }
    return -1;
}

}
