// sws.cu — libswscale yuv420p -> packed 8-bit RGB (rgb24, bgr24, rgba, bgra, argb, abgr) on sm_90a: kernels + the C ABI (include/b200dsp.h, "libswscale" section).
//
// Reference semantics reproduced bit-for-bit (see oracle/sws_oracle.c for the CPU restatement used as checker):
//   unscaled LUT converter  yuv2rgb_c_24_rgb          libswscale/yuv2rgb.c:137-236,530   -> sws_unscaled_kernel
//   horizontal FIR          hScale8To15_c             libswscale/swscale.c:128-142       -> sws_hscale_kernel (IDP.2A)
//   vertical FIR + writers  yuv2rgb24_{X,2,1}_c       libswscale/output.c:1789-1939      -> sws_vscale_rgb24_kernel
//   full-chroma writers     yuv2rgb24_full_{X,2,1}_c  libswscale/output.c:2161-2310      -> sws_vscale_rgb24_full_kernel
// The reference's pointer LUTs (table_rV/gU/gV/bU into a clipped luma ramp) are evaluated in closed form, which is
// exact because the ramp is clip_u8((yb0 + k*cy) >> 16) for every k (yuv2rgb.c:901-914).
//
// Data layout in HBM: planar u8 Y/U/V exactly as the caller's AVFrame planes (any stride), packed rgb24 rows out.
// The kernels are HBM-bound byte movers: each thread owns 16 horizontally adjacent pixels so that luma moves as one
// 128-bit load, chroma as 64-bit loads and rgb24 as three 128-bit stores (48 B = 16 px).
#include "common.h"
#include "sws_plan.h"
#include <vector>
#include <cstring>
#include <new>
#include <cstdlib>
#include <algorithm>

// ------------------------------------------------------------------------------------------------ device helpers
struct SwsDevTables {            // device copies of the vertical banks and the per-line writer choice
    const int16_t *vLum; const int32_t *vLumPos; int vLumSize;
    const int16_t *vChr; const int32_t *vChrPos; int vChrSize;
    const int32_t *rowMode;
    const int32_t *vLum2, *vChr2;     // vertical banks with tap pairs packed (lo16 = tap 2j, hi16 = tap 2j+1 or 0)
    const int16_t *hLum; const int32_t *hLumPos; int hLumSize;
    const int16_t *hChr; const int32_t *hChrPos; int hChrSize;
    const int32_t *hLum2, *hChr2;     // horizontal banks, tap pairs packed the same way
};

struct SwsMmaBank {                  // one horizontal filter bank in tensor-core form (device pointers)
    const int2 *ginfo;               // per group of 8 output columns: { first source column of the group's window (multiple of 4), index of its first chunk };
                                     // entry [ngroups] closes the chunk count
    const uint4 *bfrag;              // per chunk: 32 lanes x { hi b0, hi b1, lo b0, lo b1 }
    int ngroups;
};

struct SwsFrameArgs {
    const uint8_t *y, *u, *v;         // u8 source planes (or int16 planes reinterpret_cast for the scaled path)
    long long ys, us, vs;             // strides in BYTES (may be negative for u8 planes)
    long long yfs, ufs, vfs;          // frame strides in bytes
    uint8_t *dst; long long ds, dfs;
    int srcH, chrSrcH, dstW, dstH, chrDstW;
    int y0;                           // first output line of this launch (slice calls), 0 for whole frames
    int bpp, ro, go, bo, ao;          // output pixel: bytes and channel byte positions (scalar writers; ao < 0: no alpha)
};


__device__ __forceinline__ int clamp_u8(int v) { return __vimin_s32_relu(v, 255); }   // one VIMNMX.RELU

__device__ __forceinline__ int dp2a_lo_su(int a, unsigned b, int c)   // c + a.h0*b.b0 + a.h1*b.b1 (s16 x u8)
{ int d; asm("dp2a.lo.s32.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c)); return d; }
__device__ __forceinline__ int dp2a_hi_su(int a, unsigned b, int c)   // c + a.h0*b.b2 + a.h1*b.b3
{ int d; asm("dp2a.hi.s32.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c)); return d; }

// colour constants per chroma sample: A_c such that channel = clip_u8((A_c + Y*cy) >> 16)
struct ChromaBase { int r, g, b; };
__device__ __forceinline__ ChromaBase chroma_base(const SwsColorConst &c, int U, int V)
{
    const int u8 = clamp_u8(U), v8 = clamp_u8(V);
    ChromaBase o;
    o.r = c.yb0 + (c.baseR + ((v8 * c.crv) >> 16)) * c.cy;
    o.g = c.yb0 + (c.baseG + ((u8 * c.cgu) >> 16) + ((v8 * c.cgv) >> 16)) * c.cy;
    o.b = c.yb0 + (c.baseB + ((u8 * c.cbu) >> 16)) * c.cy;
    return o;
}

// (Folding the ">> 16, add base" pairs into IMAD.HI — hi32((u8 << 12) * (coef << 4)) + base — would remove 64 ALU-pipe shift-adds per
// 32 pixels, but IMAD.HI is not a full-rate instruction.  The plain form below is kept.)
// Two pixels sharing one chroma sample -> three words holding (r0,g0) (b0,r1) (g1,b1) as clamped s16x2 (bytes 0 and 2).
// (A + Y*cy) >> 16 is the high half of the 32-bit sum: PRMT picks the high halves, VIMNMX.S16x2.RELU clamps both to 0..255.
__device__ __forceinline__ void pair_rgb_packed(int cy, const ChromaBase &cb, int Y0, int Y1, unsigned *m)
{
    const int r0 = Y0 * cy + cb.r, g0 = Y0 * cy + cb.g, b0 = Y0 * cy + cb.b;
    const int r1 = Y1 * cy + cb.r, g1 = Y1 * cy + cb.g, b1 = Y1 * cy + cb.b;
    m[0] = __vimin_s16x2_relu(__byte_perm(r0, g0, 0x7632), 0x00ff00ffu);
    m[1] = __vimin_s16x2_relu(__byte_perm(b0, r1, 0x7632), 0x00ff00ffu);
    m[2] = __vimin_s16x2_relu(__byte_perm(g1, b1, 0x7632), 0x00ff00ffu);
}
// 32-bit outputs: one pixel -> one word.  (r,g) and (b,255) are clamped as s16x2, then one PRMT orders the four bytes.
template <int KIND>
__device__ __forceinline__ void pair_rgb32(int cy, const ChromaBase &cb, int Y0, int Y1, unsigned *m)
{
    constexpr unsigned SEL = KIND == SWS_OUT_RGBA ? 0x6420 : KIND == SWS_OUT_BGRA ? 0x6024 : KIND == SWS_OUT_ARGB ? 0x4206 : 0x0246;
    const int r0 = Y0 * cy + cb.r, g0 = Y0 * cy + cb.g, b0 = Y0 * cy + cb.b;
    const int r1 = Y1 * cy + cb.r, g1 = Y1 * cy + cb.g, b1 = Y1 * cy + cb.b;
    const unsigned p0 = __vimin_s16x2_relu(__byte_perm(r0, g0, 0x7632), 0x00ff00ffu), q0 = __vimin_s16x2_relu(__byte_perm(b0, 0xffu, 0x5432), 0x00ff00ffu);
    const unsigned p1 = __vimin_s16x2_relu(__byte_perm(r1, g1, 0x7632), 0x00ff00ffu), q1 = __vimin_s16x2_relu(__byte_perm(b1, 0xffu, 0x5432), 0x00ff00ffu);
    m[0] = __byte_perm(p0, q0, SEL);
    m[1] = __byte_perm(p1, q1, SEL);
}
// words one pixel pair occupies in the per-thread staging array
template <int KIND> struct OutWords { static constexpr int per_pair = KIND <= SWS_OUT_BGR24 ? 3 : 2, bpp = KIND <= SWS_OUT_BGR24 ? 3 : 4; };
template <int KIND>
__device__ __forceinline__ void pair_out(int cy, ChromaBase cb, int Y0, int Y1, unsigned *m)
{
    if (KIND == SWS_OUT_RGB24) pair_rgb_packed(cy, cb, Y0, Y1, m);
    else if (KIND == SWS_OUT_BGR24) { const int t = cb.r; cb.r = cb.b; cb.b = t; pair_rgb_packed(cy, cb, Y0, Y1, m); }
    else pair_rgb32<KIND>(cy, cb, Y0, Y1, m);
}
__device__ __forceinline__ void store_packed48(uint8_t *dst, const unsigned *m);
// 16 px of one line: 48 bytes (three 128-bit stores) or 64 bytes (four)
template <int KIND>
__device__ __forceinline__ void store_out(uint8_t *dst, const unsigned *m)
{
    if (KIND <= SWS_OUT_BGR24) store_packed48(dst, m);
    else {
        uint4 *d4 = reinterpret_cast<uint4 *>(dst);
#pragma unroll
        for (int k = 0; k < 4; k++) d4[k] = make_uint4(m[4 * k], m[4 * k + 1], m[4 * k + 2], m[4 * k + 3]);
    }
}
// 16 px = 8 pairs = 24 packed words -> 12 output words (48 bytes), stored as three 128-bit words
__device__ __forceinline__ void store_packed48(uint8_t *dst, const unsigned *m)
{
    uint4 *d4 = reinterpret_cast<uint4 *>(dst);
#pragma unroll
    for (int k = 0; k < 3; k++) {
        uint4 v;
        v.x = __byte_perm(m[8 * k + 0], m[8 * k + 1], 0x6420);
        v.y = __byte_perm(m[8 * k + 2], m[8 * k + 3], 0x6420);
        v.z = __byte_perm(m[8 * k + 4], m[8 * k + 5], 0x6420);
        v.w = __byte_perm(m[8 * k + 6], m[8 * k + 7], 0x6420);
        d4[k] = v;
    }
}
__device__ __forceinline__ int byte_of(unsigned w, int k) { return (int)__byte_perm(w, 0, 0x4440 | k); }

// scalar writer used by the slow (edge / unaligned / int16-source) kernels
__device__ __forceinline__ void put_pair_bytes(uint8_t *d, const SwsFrameArgs &a, const SwsColorConst &c, const ChromaBase &cb, int Y0, int Y1, bool second)
{
    const int t0 = Y0 * c.cy;
    d[a.ro] = (uint8_t)clamp_u8((cb.r + t0) >> 16); d[a.go] = (uint8_t)clamp_u8((cb.g + t0) >> 16); d[a.bo] = (uint8_t)clamp_u8((cb.b + t0) >> 16);
    if (a.ao >= 0) d[a.ao] = 255;
    if (second) {
        const int t1 = Y1 * c.cy;
        d += a.bpp;
        d[a.ro] = (uint8_t)clamp_u8((cb.r + t1) >> 16); d[a.go] = (uint8_t)clamp_u8((cb.g + t1) >> 16); d[a.bo] = (uint8_t)clamp_u8((cb.b + t1) >> 16);
        if (a.ao >= 0) d[a.ao] = 255;
    }
}

// ------------------------------------------------------------------------------------------------ kernel: unscaled LUT path (fast)
// yuv2rgb_c_24_rgb: chroma sample (x>>1, y>>1), no interpolation.  One thread = 16 px x 2 lines (one chroma line):
// 2 x LDG.128 luma + 2 x LDG.64 chroma in, 6 x STG.128 out.  Grid: x over 16-px groups, y over line pairs, z over frames.
template <int KIND>
__global__ void __launch_bounds__(128)
sws_unscaled_kernel(SwsFrameArgs a, SwsColorConst c, int ngroups)
{
    constexpr int PW = OutWords<KIND>::per_pair;
    const int xg = blockIdx.x * blockDim.x + threadIdx.x;
    if (xg >= ngroups) return;
    const int row = blockIdx.y * 2 + a.y0;
    const long long f = blockIdx.z;
    const uint8_t *py = a.y + f * a.yfs + (long long)row * a.ys + xg * 16;
    const uint2 u = __ldg(reinterpret_cast<const uint2 *>(a.u + f * a.ufs + (long long)(row >> 1) * a.us + xg * 8));
    const uint2 v = __ldg(reinterpret_cast<const uint2 *>(a.v + f * a.vfs + (long long)(row >> 1) * a.vs + xg * 8));
    const uint4 y0 = __ldg(reinterpret_cast<const uint4 *>(py));
    const uint4 y1 = __ldg(reinterpret_cast<const uint4 *>(py + a.ys));
    const unsigned uw[2] = { u.x, u.y }, vw[2] = { v.x, v.y };
    const unsigned y0w[4] = { y0.x, y0.y, y0.z, y0.w }, y1w[4] = { y1.x, y1.y, y1.z, y1.w };
    unsigned m0[8 * PW], m1[8 * PW];
#pragma unroll
    for (int i = 0; i < 8; i++) {
        const ChromaBase cb = chroma_base(c, byte_of(uw[i >> 2], i & 3), byte_of(vw[i >> 2], i & 3));
        const int w = i >> 1, k = (i & 1) * 2;
        pair_out<KIND>(c.cy, cb, byte_of(y0w[w], k), byte_of(y0w[w], k + 1), m0 + PW * i);
        pair_out<KIND>(c.cy, cb, byte_of(y1w[w], k), byte_of(y1w[w], k + 1), m1 + PW * i);
    }
    uint8_t *d0 = a.dst + f * a.dfs + (long long)row * a.ds + (long long)xg * (16 * OutWords<KIND>::bpp);
    store_out<KIND>(d0, m0);
    store_out<KIND>(d0 + a.ds, m1);
}

// slow variant: one thread = one pixel pair x 2 lines, any alignment; covers pairs [p0, p1)
__global__ void __launch_bounds__(128)
sws_unscaled_slow_kernel(SwsFrameArgs a, SwsColorConst c, int p0, int p1)
{
    const int p = p0 + blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= p1) return;
    const int row = blockIdx.y * 2 + a.y0;
    const long long f = blockIdx.z;
    const uint8_t *py = a.y + f * a.yfs + (long long)row * a.ys + 2 * p;
    const int U = a.u[f * a.ufs + (long long)(row >> 1) * a.us + p], V = a.v[f * a.vfs + (long long)(row >> 1) * a.vs + p];
    const ChromaBase cb = chroma_base(c, U, V);
    uint8_t *d = a.dst + f * a.dfs + (long long)row * a.ds + (long long)p * (2 * a.bpp);
    put_pair_bytes(d, a, c, cb, py[0], py[1], true);
    put_pair_bytes(d + a.ds, a, c, cb, py[a.ys], py[a.ys + 1], true);
}

// ------------------------------------------------------------------------------------------------ kernel: horizontal FIR
// dst[i] = min((sum_j src[pos[i]+j] * coef[i*fs+j]) >> 7, 32767); one thread per output sample, grid y = lines, z = frames.
// The source window is fetched as aligned 32-bit words (only words that hold a needed byte), shifted to tap 0 with a funnel
// shift, and each word feeds two IDP.2A (s16 tap pair x u8 sample pair); coef2 holds the taps packed in pairs.
__global__ void __launch_bounds__(256)
sws_hscale_kernel(const uint8_t *src, long long sstride, long long sfs, int16_t *dst, int dstW, long long dfs,
                     const int32_t *coef2, const int32_t *pos, int fs, int line0)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= dstW) return;
    const int line = blockIdx.y + line0;
    const uint8_t *s = src + (long long)blockIdx.z * sfs + (long long)line * sstride + __ldg(pos + i);
    const unsigned sh = (unsigned)(reinterpret_cast<uintptr_t>(s) & 3);
    const unsigned *w = reinterpret_cast<const unsigned *>(s - sh);
    const int need = (int)sh + fs, np = (fs + 1) >> 1;
    const int32_t *k = coef2 + (long long)i * np;
    unsigned prev = __ldg(w);
    int acc = 0;
    for (int q = 0; q * 4 < fs; q++) {                       // window word q = taps 4q .. 4q+3
        const unsigned next = ((q + 1) * 4 < need) ? __ldg(w + q + 1) : 0u;
        const unsigned win = __funnelshift_r(prev, next, sh * 8);
        prev = next;
        acc = dp2a_lo_su(__ldg(k + 2 * q), win, acc);
        if (2 * q + 1 < np) acc = dp2a_hi_su(__ldg(k + 2 * q + 1), win, acc);
    }
    dst[(long long)blockIdx.z * dfs + (long long)line * dstW + i] = (int16_t)min(acc >> 7, 32767);
}

// Same filter, one thread = one output column over HROWS consecutive lines: position and tap pairs of a column are the same
// on every line, so they are fetched once and held in registers (NP pairs, filter sizes up to 2*NP); per line only the
// source words are loaded.  Adjacent threads read adjacent source bytes and write adjacent int16 samples.
constexpr int HROWS = 8;
template <int NP>
__global__ void __launch_bounds__(256)
sws_hscale_rows_kernel(const uint8_t *src, long long sstride, long long sfs, int16_t *dst, int dstW, long long dfs,
                       const int32_t *coef2, const int32_t *pos, int fs, int line0, int nlines)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= dstW) return;
    const int np = (fs + 1) >> 1, p0 = __ldg(pos + i);
    int k[NP];
#pragma unroll
    for (int j = 0; j < NP; j++) k[j] = j < np ? __ldg(coef2 + (long long)i * np + j) : 0;
    const int r0 = blockIdx.y * HROWS, r1 = min(r0 + HROWS, nlines);
    const uint8_t *base = src + (long long)blockIdx.z * sfs + p0;
    int16_t *out = dst + (long long)blockIdx.z * dfs + i;
    for (int r = r0; r < r1; r++) {
        const int line = r + line0;
        const uint8_t *s = base + (long long)line * sstride;
        const unsigned sh = (unsigned)(reinterpret_cast<uintptr_t>(s) & 3);
        const unsigned *w = reinterpret_cast<const unsigned *>(s - sh);
        const int need = (int)sh + fs;
        unsigned prev = __ldg(w);
        int acc = 0;
#pragma unroll
        for (int q = 0; q < (NP + 1) / 2; q++) {               // window word q = taps 4q .. 4q+3 (zero pairs beyond the filter)
            if (q * 4 < fs) {
                const unsigned next = ((q + 1) * 4 < need) ? __ldg(w + q + 1) : 0u;
                const unsigned win = __funnelshift_r(prev, next, sh * 8);
                prev = next;
                acc = dp2a_lo_su(k[2 * q], win, acc);
                if (2 * q + 1 < NP) acc = dp2a_hi_su(k[2 * q + 1], win, acc);
            }
        }
        out[(long long)line * dstW] = (int16_t)min(acc >> 7, 32767);
    }
}

// SWS_FAST_BILINEAR horizontal pass (ff_hyscale_fast_c / ff_hcscale_fast_c, hscale_fast_bilinear.c:27-67): 16.16 stepping with
// 7-bit blend weights; outputs whose left sample is the last source sample (or beyond) are src[srcW-1] * 128, which is what
// the fix-up loop at the end of both reference functions leaves (so the sample right of the row end is never read).
template <bool CHROMA>
__global__ void __launch_bounds__(256)
sws_hscale_fast_kernel(const uint8_t *src, long long sstride, long long sfs, int16_t *dst, int dstW, long long dfs,
                       int srcW, int xInc, int line0)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= dstW) return;
    const int line = blockIdx.y + line0;
    const uint8_t *s = src + (long long)blockIdx.z * sfs + (long long)line * sstride;
    const unsigned xpos = (unsigned)i * (unsigned)xInc;             // the reference accumulates in 32 bits
    const unsigned xx = xpos >> 16, xalpha = (xpos & 0xFFFF) >> 9;
    int v;
    if ((((long long)i * xInc) >> 16) >= srcW - 1) v = (int)__ldg(s + srcW - 1) * 128;
    else {
        const int a = __ldg(s + xx), b = __ldg(s + xx + 1);
        v = CHROMA ? a * (int)(xalpha ^ 127) + b * (int)xalpha : (a << 7) + (b - a) * (int)xalpha;
    }
    dst[(long long)blockIdx.z * dfs + (long long)line * dstW + i] = (int16_t)v;
}

// ------------------------------------------------------------------------------------------------ kernel: vertical FIR + rgb24 (fast)
// Same-size conversion with the reference's scaler flags (the FATE path): the horizontal pass is the identity, so the
// vertical taps are read straight from the u8 planes.  Only the general `_X` writer (yuv2rgb_X_c_template,
// output.c:1789-1840) is handled here; lines that the reference sends to the `_1`/`_2` writers go to the slow kernel.
//   Y = (2^18 + sum_j (y_j << 7) * lf_j) >> 19  ==  (2^11 + sum_j y_j * lf_j) >> 12   (same for U, V)
// which holds while the 32-bit sum does not wrap (the host checks sum |coef| per line).  Two taps are folded per
// IDP.2A (s16 coefficient pair x u8 sample pair) after interleaving two source lines with PRMT.
// LUMID: the luma bank is a single tap of 4096 on every line, so Y is the source byte itself.
// One thread = 16 px of one output line.  Grid: x over 16-px groups, y over lines, z over frames.
// chroma taps of two source lines folded into 8 accumulators (4 PRMT + 8 IDP.2A per plane)
__device__ __forceinline__ void fold2(int k2, const uint2 &r0, const uint2 &r1, int *acc)
{
    unsigned lo = __byte_perm(r0.x, r1.x, 0x5140), hi = __byte_perm(r0.x, r1.x, 0x7362);
    acc[0] = dp2a_lo_su(k2, lo, acc[0]); acc[1] = dp2a_hi_su(k2, lo, acc[1]); acc[2] = dp2a_lo_su(k2, hi, acc[2]); acc[3] = dp2a_hi_su(k2, hi, acc[3]);
    lo = __byte_perm(r0.y, r1.y, 0x5140); hi = __byte_perm(r0.y, r1.y, 0x7362);
    acc[4] = dp2a_lo_su(k2, lo, acc[4]); acc[5] = dp2a_hi_su(k2, lo, acc[5]); acc[6] = dp2a_lo_su(k2, hi, acc[6]); acc[7] = dp2a_hi_su(k2, hi, acc[7]);
}

// nv12 / nv21 chroma: the two source lines come as 16 interleaved bytes (U,V pairs; V,U for nv21); PRMT picks the U (or V)
// bytes of both lines at once, so de-interleaving costs nothing over the planar case (same 8 PRMT + 16 IDP.2A per tap pair).
template <int NV>
__device__ __forceinline__ void fold2_nv(int k2, const uint4 &r0, const uint4 &r1, int *aU, int *aV)
{
    constexpr unsigned SU = NV == 1 ? 0x6240 : 0x7351, SV = NV == 1 ? 0x7351 : 0x6240;
    const unsigned w0[4] = { r0.x, r0.y, r0.z, r0.w }, w1[4] = { r1.x, r1.y, r1.z, r1.w };
#pragma unroll
    for (int j = 0; j < 4; j++) {
        const unsigned wu = __byte_perm(w0[j], w1[j], SU), wv = __byte_perm(w0[j], w1[j], SV);
        aU[2 * j] = dp2a_lo_su(k2, wu, aU[2 * j]); aU[2 * j + 1] = dp2a_hi_su(k2, wu, aU[2 * j + 1]);
        aV[2 * j] = dp2a_lo_su(k2, wv, aV[2 * j]); aV[2 * j + 1] = dp2a_hi_su(k2, wv, aV[2 * j + 1]);
    }
}

// CFS4: the chroma bank has exactly 4 taps (bicubic 2x vertical chroma up-sampling, the BASELINE case): fully unrolled.
// Line offsets are 32-bit (the host guarantees |stride| * lines < 2^31); coefficient pairs come pre-packed (t.vChr2/vLum2).
// NV: 0 planar chroma (a.u, a.v), 1 nv12 / 2 nv21 (a.u = interleaved plane; only instantiated with CFS4)
template <bool LUMID, bool CFS4, int KIND, int NV = 0>
__global__ void __launch_bounds__(128, LUMID ? (KIND <= SWS_OUT_BGR24 ? 12 : 10) : 8)
sws_vscale_rgb24_fast_kernel(SwsFrameArgs a, SwsDevTables t, SwsColorConst c, int ngroups)
{
    constexpr int PW = OutWords<KIND>::per_pair;
    const int xg = blockIdx.x * blockDim.x + threadIdx.x;
    if (xg >= ngroups) return;
    const int dy = blockIdx.y + a.y0;
    const long long f = blockIdx.z;
    const int lfs = t.vLumSize, cfs = CFS4 ? 4 : t.vChrSize;
    const int lp = (lfs + 1) >> 1, cp = (cfs + 1) >> 1;
    const int firstLum = max(1 - lfs, __ldg(t.vLumPos + dy));
    const int firstChr = max(1 - cfs, __ldg(t.vChrPos + dy));
    const uint8_t *ub = a.u + f * a.ufs + xg * 8, *vb = a.v + f * a.vfs + xg * 8, *yb = a.y + f * a.yfs + xg * 16;
    const int us = (int)a.us, vs = (int)a.vs, ys = (int)a.ys, chmax = a.chrSrcH - 1;

    int aU[8], aV[8];
#pragma unroll
    for (int i = 0; i < 8; i++) aU[i] = aV[i] = 1 << 11;
    if (CFS4 && NV) {
        const int2 k = __ldg(reinterpret_cast<const int2 *>(t.vChr2 + 2 * dy));
        const int l0 = min(max(firstChr, 0), chmax), l1 = min(max(firstChr + 1, 0), chmax);
        const int l2 = min(max(firstChr + 2, 0), chmax), l3 = min(max(firstChr + 3, 0), chmax);
        const uint8_t *uvb = a.u + f * a.ufs + xg * 16;
        const uint4 q0 = __ldg(reinterpret_cast<const uint4 *>(uvb + l0 * us)), q1 = __ldg(reinterpret_cast<const uint4 *>(uvb + l1 * us));
        const uint4 q2 = __ldg(reinterpret_cast<const uint4 *>(uvb + l2 * us)), q3 = __ldg(reinterpret_cast<const uint4 *>(uvb + l3 * us));
        fold2_nv<NV ? NV : 1>(k.x, q0, q1, aU, aV); fold2_nv<NV ? NV : 1>(k.y, q2, q3, aU, aV);
    } else if (CFS4) {
        const int2 k = __ldg(reinterpret_cast<const int2 *>(t.vChr2 + 2 * dy));
        const int l0 = min(max(firstChr, 0), chmax), l1 = min(max(firstChr + 1, 0), chmax);
        const int l2 = min(max(firstChr + 2, 0), chmax), l3 = min(max(firstChr + 3, 0), chmax);
        const uint2 u0 = __ldg(reinterpret_cast<const uint2 *>(ub + l0 * us)), u1 = __ldg(reinterpret_cast<const uint2 *>(ub + l1 * us));
        const uint2 u2 = __ldg(reinterpret_cast<const uint2 *>(ub + l2 * us)), u3 = __ldg(reinterpret_cast<const uint2 *>(ub + l3 * us));
        const uint2 v0 = __ldg(reinterpret_cast<const uint2 *>(vb + l0 * vs)), v1 = __ldg(reinterpret_cast<const uint2 *>(vb + l1 * vs));
        const uint2 v2 = __ldg(reinterpret_cast<const uint2 *>(vb + l2 * vs)), v3 = __ldg(reinterpret_cast<const uint2 *>(vb + l3 * vs));
        fold2(k.x, u0, u1, aU); fold2(k.y, u2, u3, aU);
        fold2(k.x, v0, v1, aV); fold2(k.y, v2, v3, aV);
    } else {
        for (int j = 0; j < cp; j++) {
            const int k2 = __ldg(t.vChr2 + (long long)dy * cp + j);
            const int l0 = min(max(firstChr + 2 * j, 0), chmax), l1 = min(max(firstChr + 2 * j + 1, 0), chmax);
            const uint2 u0 = __ldg(reinterpret_cast<const uint2 *>(ub + l0 * us)), u1 = __ldg(reinterpret_cast<const uint2 *>(ub + l1 * us));
            const uint2 v0 = __ldg(reinterpret_cast<const uint2 *>(vb + l0 * vs)), v1 = __ldg(reinterpret_cast<const uint2 *>(vb + l1 * vs));
            fold2(k2, u0, u1, aU);
            fold2(k2, v0, v1, aV);
        }
    }

    int Y[16];
    if (LUMID) {
        const uint4 q = __ldg(reinterpret_cast<const uint4 *>(yb + min(max(firstLum, 0), a.srcH - 1) * ys));
        const unsigned w[4] = { q.x, q.y, q.z, q.w };
#pragma unroll
        for (int i = 0; i < 16; i++) Y[i] = byte_of(w[i >> 2], i & 3);
    } else {
#pragma unroll
        for (int i = 0; i < 16; i++) Y[i] = 1 << 11;
        for (int j = 0; j < lp; j++) {
            const int k2 = __ldg(t.vLum2 + (long long)dy * lp + j);
            const int l0 = min(max(firstLum + 2 * j, 0), a.srcH - 1), l1 = min(max(firstLum + 2 * j + 1, 0), a.srcH - 1);
            const uint4 q0 = __ldg(reinterpret_cast<const uint4 *>(yb + l0 * ys)), q1 = __ldg(reinterpret_cast<const uint4 *>(yb + l1 * ys));
            const uint2 a0 = make_uint2(q0.x, q0.y), a1 = make_uint2(q1.x, q1.y), b0 = make_uint2(q0.z, q0.w), b1 = make_uint2(q1.z, q1.w);
            fold2(k2, a0, a1, Y);
            fold2(k2, b0, b1, Y + 8);
        }
#pragma unroll
        for (int i = 0; i < 16; i++) Y[i] >>= 12;
    }

    unsigned m[8 * PW];
#pragma unroll
    for (int i = 0; i < 8; i++) {
        const ChromaBase cb = chroma_base(c, aU[i] >> 12, aV[i] >> 12);
        pair_out<KIND>(c.cy, cb, Y[2 * i], Y[2 * i + 1], m + PW * i);
    }
    store_out<KIND>(a.dst + f * a.dfs + (long long)dy * (int)a.ds + xg * (16 * OutWords<KIND>::bpp), m);
}

// ------------------------------------------------------------------------------------------------ kernel: line pairs, streamed down bands
// Same arithmetic as sws_vscale_rgb24_fast_kernel<true, true, KIND, NV> (identity luma bank, 4 chroma taps), for pairs of output lines
// whose chroma windows coincide.  With 2x vertical chroma up-sampling the bicubic window of output lines 2k+1 and 2k+2 starts at the same
// chroma line (vChrFilterPos equal, only the coefficients differ; the host checks this for the whole bank), so the four chroma lines are
// interleaved once (PRMT) and both lines are evaluated from the same registers.
// One thread walks a band of up to PairShape<KIND>::band consecutive pairs of one frame, top to bottom:
//  - the chroma tap lines stay in registers as a sliding window: when the next pair's window starts one line lower (2x up-sampling)
//    only the line it gains is loaded (one line per plane per pair instead of four); any other step reloads the window;
//  - the next pair's luma rows, gained chroma line and coefficients are loaded before the current pair is computed, and the positions
//    two pairs ahead, so that no load waits for another load issued in the same step.
// What a thread writes depends on the row width:
//  - 24-bit rows: one 16-byte chunk of each line (pair_chunks).  Adjacent lanes write adjacent chunks in the same instruction, so one
//    warp store covers 512 contiguous bytes and fills whole 32-byte sectors when dst and ds are 32-byte aligned (16-byte alignment
//    stays correct, only with a half sector at each end of a warp's span).  A chunk is not a whole number of pixels, so three lanes
//    read the same 16-px group's luma and chroma (served by L1 as a broadcast) and each computes the 8 pixels under its chunk.
//  - 32-bit rows: 16 px, four 128-bit stores per line at a 64-byte lane stride.
// Threads do not share data (no shared memory, no shuffles).  Grid: x over chunks (24-bit) or 16-px groups (32-bit), y over bands, z
// over frames.  Band length and CTAs per SM as measured on the H100 (DESIGN.md §5).  24-bit rows: bands of 32 pairs at 8 CTAs per SM
// (64 registers) from planar chroma, 7 (72 registers) from nv12 / nv21: each source ran about 7 % slower at the other's count.
// 32-bit rows: one pair per thread at 5 CTAs per SM (96 registers): with their 64-byte stores, bands of 4 or 16 pairs
// were slower than one pair, whatever the occupancy; with one pair the steps ahead reload the same pair's rows (L1 hits) and the
// window never slides.
constexpr int PAIR_THREADS = 128;
template <int KIND, int NV = 0> struct PairShape { static constexpr int band = KIND <= SWS_OUT_BGR24 ? 32 : 1, ctas = KIND <= SWS_OUT_BGR24 ? (NV ? 7 : 8) : 5; };
__device__ __forceinline__ void interleave2(const uint2 &r0, const uint2 &r1, unsigned *w)
{
    w[0] = __byte_perm(r0.x, r1.x, 0x5140); w[1] = __byte_perm(r0.x, r1.x, 0x7362);
    w[2] = __byte_perm(r0.y, r1.y, 0x5140); w[3] = __byte_perm(r0.y, r1.y, 0x7362);
}
template <int NV>
__device__ __forceinline__ void interleave2_nv(const uint4 &r0, const uint4 &r1, unsigned *wu, unsigned *wv)
{
    constexpr unsigned SU = NV == 1 ? 0x6240 : 0x7351, SV = NV == 1 ? 0x7351 : 0x6240;
    wu[0] = __byte_perm(r0.x, r1.x, SU); wv[0] = __byte_perm(r0.x, r1.x, SV);
    wu[1] = __byte_perm(r0.y, r1.y, SU); wv[1] = __byte_perm(r0.y, r1.y, SV);
    wu[2] = __byte_perm(r0.z, r1.z, SU); wv[2] = __byte_perm(r0.z, r1.z, SV);
    wu[3] = __byte_perm(r0.w, r1.w, SU); wv[3] = __byte_perm(r0.w, r1.w, SV);
}
// one chroma tap line of a thread's 16 px: 8 U bytes in .x/.y and 8 V bytes in .z/.w (planar), or the 16 interleaved bytes (nv12 / nv21)
template <int NV>
__device__ __forceinline__ uint4 pair_chroma_line(const uint8_t *ub, const uint8_t *vb, int us, int vs, int l)
{
    if (NV) return __ldg(reinterpret_cast<const uint4 *>(ub + l * us));
    const uint2 u = __ldg(reinterpret_cast<const uint2 *>(ub + l * us)), v = __ldg(reinterpret_cast<const uint2 *>(vb + l * vs));
    return make_uint4(u.x, u.y, v.x, v.y);
}
// two tap lines -> two chroma samples x two lines per word, U in iu[0..3], V in iv[0..3]
template <int NV>
__device__ __forceinline__ void pair_interleave(const uint4 &r0, const uint4 &r1, unsigned *iu, unsigned *iv)
{
    if (NV) interleave2_nv<NV>(r0, r1, iu, iv);
    else {
        interleave2(make_uint2(r0.x, r0.y), make_uint2(r1.x, r1.y), iu);
        interleave2(make_uint2(r0.z, r0.w), make_uint2(r1.z, r1.w), iv);
    }
}

// x, y or z for r = 0, 1 or 2: two SELs, the same instructions in every lane
__device__ __forceinline__ unsigned sel3(unsigned x, unsigned y, unsigned z, int r) { return r == 0 ? x : r == 1 ? y : z; }
// 24-bit rows, one thread = one 16-byte chunk: chroma samples 2r .. 2r+3 of one tap line of the chunk's group (r = chunk % 3), U in .x and
// V in .y.  The lanes of a warp have all three phases, so the selection is by lane-dependent PRMT selectors and SELs, not by branches.
template <int NV>
__device__ __forceinline__ uint2 chunk_chroma_line(const uint8_t *ub, const uint8_t *vb, int us, int vs, int l, int r, unsigned sel)
{
    if (NV) {                                                           // 16 interleaved bytes: samples 2r .. 2r+3 are words r, r + 1
        const uint4 q = __ldg(reinterpret_cast<const uint4 *>(ub + l * us));
        const unsigned w0 = sel3(q.x, q.y, q.z, r), w1 = sel3(q.y, q.z, q.w, r);
        return NV == 1 ? make_uint2(__byte_perm(w0, w1, 0x6420), __byte_perm(w0, w1, 0x7531))
                       : make_uint2(__byte_perm(w0, w1, 0x7531), __byte_perm(w0, w1, 0x6420));
    }
    const uint2 u = __ldg(reinterpret_cast<const uint2 *>(ub + l * us)), v = __ldg(reinterpret_cast<const uint2 *>(vb + l * vs));
    return make_uint2(__byte_perm(u.x, u.y, sel), __byte_perm(v.x, v.y, sel));
}
// words r, r + 1 of a 16-px luma row: the chunk's pixels 4r .. 4r+7
__device__ __forceinline__ uint2 chunk_luma(const uint4 &q, int r) { return make_uint2(sel3(q.x, q.y, q.z, r), sel3(q.y, q.z, q.w, r)); }

// 24-bit rows.  Chunk r of a 16-px group (bytes 16r .. 16r+15 of its 48) starts r bytes into pixel 5r and ends in pixel 5r+5.  The thread
// computes the 8 pixels 4r .. 4r+7 (chroma samples 2r .. 2r+3, 24 bytes from byte 12r of the group): the chunk is their words r .. r+3.
template <int KIND, int NV>
__device__ __forceinline__ void pair_chunks(const SwsFrameArgs &a, const SwsDevTables &t, const SwsColorConst &c, int ngroups, int npairs)
{
    constexpr int BAND = PairShape<KIND>::band;
    const int xc = blockIdx.x * blockDim.x + threadIdx.x;
    if (xc >= 3 * ngroups) return;
    const int xg = xc / 3, r = xc - 3 * xg;
    const unsigned csel = 0x3210u + 0x2222u * r;                        // bytes 2r .. 2r+3 of a chroma uint2
    const int dA0 = a.y0 + 2 * blockIdx.y * BAND, np = min(BAND, npairs - (int)blockIdx.y * BAND);
    const long long f = blockIdx.z;
    const int ys = (int)a.ys, us = (int)a.us, vs = (int)a.vs, chmax = a.chrSrcH - 1, lmax = a.srcH - 1;
    const uint8_t *yb = a.y + f * a.yfs + xg * 16;
    const uint8_t *ub = a.u + f * a.ufs + xg * (NV ? 16 : 8), *vb = NV ? nullptr : a.v + f * a.vfs + xg * 8;
    uint8_t *d = a.dst + f * a.dfs + (long long)dA0 * a.ds + xc * 16;                    // line 2i of the band
    auto line = [&](int l) { return chunk_chroma_line<NV>(ub, vb, us, vs, min(max(l, 0), chmax), r, csel); };
    auto luma = [&](int dy) { return chunk_luma(__ldg(reinterpret_cast<const uint4 *>(yb + min(max(__ldg(t.vLumPos + dy), 0), lmax) * ys)), r); };
    auto first_chr = [&](int p) { return max(-3, __ldg(t.vChrPos + dA0 + 2 * p)); };          // == vChrPos[dA + 1]

    // pair 0: the whole window; pair 1: its positions
    int fc = first_chr(0);
    uint2 W0 = line(fc), W1 = line(fc + 1), W2 = line(fc + 2), W3 = line(fc + 3);
    uint2 YA = luma(dA0), YB = luma(dA0 + 1);
    int2 kA = __ldg(reinterpret_cast<const int2 *>(t.vChr2 + 2 * dA0)), kB = __ldg(reinterpret_cast<const int2 *>(t.vChr2 + 2 * dA0 + 2));
    const int p1 = min(1, np - 1);
    int fcN = first_chr(p1);
    int lyNA = min(max(__ldg(t.vLumPos + dA0 + 2 * p1), 0), lmax) * ys, lyNB = min(max(__ldg(t.vLumPos + dA0 + 2 * p1 + 1), 0), lmax) * ys;
    for (int i = 0; i < np; i++) {
        // pair i + 1 (the last pair repeats itself): the line its window gains, its luma rows and coefficients; pair i + 2: positions
        const int in = min(i + 1, np - 1), i2 = min(i + 2, np - 1), dN = dA0 + 2 * in, d2 = dA0 + 2 * i2;
        const bool slide = fcN == fc + 1;
        const uint2 G = slide ? line(fcN + 3) : W3;
        const uint2 NA = chunk_luma(__ldg(reinterpret_cast<const uint4 *>(yb + lyNA)), r), NB = chunk_luma(__ldg(reinterpret_cast<const uint4 *>(yb + lyNB)), r);
        const int2 kNA = __ldg(reinterpret_cast<const int2 *>(t.vChr2 + 2 * dN)), kNB = __ldg(reinterpret_cast<const int2 *>(t.vChr2 + 2 * dN + 2));
        const int fc2 = first_chr(i2);
        const int ly2A = min(max(__ldg(t.vLumPos + d2), 0), lmax) * ys, ly2B = min(max(__ldg(t.vLumPos + d2 + 1), 0), lmax) * ys;

        unsigned IU[2][2], IV[2][2];                                        // [tap pair][word]: two chroma samples x two lines each
        interleave2(make_uint2(W0.x, W2.x), make_uint2(W1.x, W3.x), &IU[0][0]);   // IU[0] = taps 0 / 1, IU[1] = taps 2 / 3
        interleave2(make_uint2(W0.y, W2.y), make_uint2(W1.y, W3.y), &IV[0][0]);
#pragma unroll
        for (int L = 0; L < 2; L++) {
            const int kx = L ? kB.x : kA.x, ky = L ? kB.y : kA.y;
            int aU[4], aV[4];
#pragma unroll
            for (int w = 0; w < 2; w++) {
                aU[2 * w]     = dp2a_lo_su(ky, IU[1][w], dp2a_lo_su(kx, IU[0][w], 1 << 11));
                aU[2 * w + 1] = dp2a_hi_su(ky, IU[1][w], dp2a_hi_su(kx, IU[0][w], 1 << 11));
                aV[2 * w]     = dp2a_lo_su(ky, IV[1][w], dp2a_lo_su(kx, IV[0][w], 1 << 11));
                aV[2 * w + 1] = dp2a_hi_su(ky, IV[1][w], dp2a_hi_su(kx, IV[0][w], 1 << 11));
            }
            const uint2 q = L ? YB : YA;
            const unsigned yw[2] = { q.x, q.y };
            unsigned m[12], o[6];
#pragma unroll
            for (int j = 0; j < 4; j++) {
                const ChromaBase cb = chroma_base(c, aU[j] >> 12, aV[j] >> 12);
                pair_out<KIND>(c.cy, cb, byte_of(yw[j >> 1], 2 * (j & 1)), byte_of(yw[j >> 1], 2 * (j & 1) + 1), m + 3 * j);
            }
#pragma unroll
            for (int k = 0; k < 6; k++) o[k] = __byte_perm(m[2 * k], m[2 * k + 1], 0x6420);
            *reinterpret_cast<uint4 *>(L ? d + a.ds : d) = make_uint4(sel3(o[0], o[1], o[2], r), sel3(o[1], o[2], o[3], r),
                                                                     sel3(o[2], o[3], o[4], r), sel3(o[3], o[4], o[5], r));
        }

        if (slide) { W0 = W1; W1 = W2; W2 = W3; W3 = G; }
        else if (fcN != fc) { W0 = line(fcN); W1 = line(fcN + 1); W2 = line(fcN + 2); W3 = line(fcN + 3); }
        d += 2 * a.ds;
        YA = NA; YB = NB; kA = kNA; kB = kNB;
        fc = fcN; fcN = fc2; lyNA = ly2A; lyNB = ly2B;
    }
}

// pairs [0, npairs) of output lines (a.y0 + 2p, a.y0 + 2p + 1), a.y0 odd; ngroups 16-px groups per line (24-bit rows: 3 * ngroups threads)
template <int KIND, int NV>
__global__ void __launch_bounds__(PAIR_THREADS, PairShape<KIND, NV>::ctas)
sws_vscale_rgb24_pair_kernel(SwsFrameArgs a, SwsDevTables t, SwsColorConst c, int ngroups, int npairs)
{
    if (KIND <= SWS_OUT_BGR24) { pair_chunks<KIND, NV>(a, t, c, ngroups, npairs); return; }
    constexpr int PW = OutWords<KIND>::per_pair, BAND = PairShape<KIND>::band;
    const int xg = blockIdx.x * blockDim.x + threadIdx.x;
    if (xg >= ngroups) return;
    const int dA0 = a.y0 + 2 * blockIdx.y * BAND, np = min(BAND, npairs - (int)blockIdx.y * BAND);
    const long long f = blockIdx.z;
    const int ys = (int)a.ys, us = (int)a.us, vs = (int)a.vs, chmax = a.chrSrcH - 1, lmax = a.srcH - 1;
    const uint8_t *yb = a.y + f * a.yfs + xg * 16;
    const uint8_t *ub = a.u + f * a.ufs + xg * (NV ? 16 : 8), *vb = NV ? nullptr : a.v + f * a.vfs + xg * 8;
    uint8_t *drow = a.dst + f * a.dfs + (long long)dA0 * a.ds + xg * (16 * OutWords<KIND>::bpp);
    auto line = [&](int l) { return pair_chroma_line<NV>(ub, vb, us, vs, min(max(l, 0), chmax)); };
    auto luma = [&](int dy) { return __ldg(reinterpret_cast<const uint4 *>(yb + min(max(__ldg(t.vLumPos + dy), 0), lmax) * ys)); };
    auto first_chr = [&](int p) { return max(-3, __ldg(t.vChrPos + dA0 + 2 * p)); };          // == vChrPos[dA + 1]

    // pair 0: the whole window; pair 1: its positions
    int fc = first_chr(0);
    uint4 W0 = line(fc), W1 = line(fc + 1), W2 = line(fc + 2), W3 = line(fc + 3);
    uint4 YA = luma(dA0), YB = luma(dA0 + 1);
    int2 kA = __ldg(reinterpret_cast<const int2 *>(t.vChr2 + 2 * dA0)), kB = __ldg(reinterpret_cast<const int2 *>(t.vChr2 + 2 * dA0 + 2));
    const int p1 = min(1, np - 1);
    int fcN = first_chr(p1);
    int lyNA = min(max(__ldg(t.vLumPos + dA0 + 2 * p1), 0), lmax) * ys, lyNB = min(max(__ldg(t.vLumPos + dA0 + 2 * p1 + 1), 0), lmax) * ys;
    for (int i = 0; i < np; i++) {
        // pair i + 1 (the last pair repeats itself): the line its window gains, its luma rows and coefficients; pair i + 2: positions
        const int in = min(i + 1, np - 1), i2 = min(i + 2, np - 1), dN = dA0 + 2 * in, d2 = dA0 + 2 * i2;
        const bool slide = fcN == fc + 1;
        const uint4 G = slide ? line(fcN + 3) : W3;
        const uint4 NA = __ldg(reinterpret_cast<const uint4 *>(yb + lyNA)), NB = __ldg(reinterpret_cast<const uint4 *>(yb + lyNB));
        const int2 kNA = __ldg(reinterpret_cast<const int2 *>(t.vChr2 + 2 * dN)), kNB = __ldg(reinterpret_cast<const int2 *>(t.vChr2 + 2 * dN + 2));
        const int fc2 = first_chr(i2);
        const int ly2A = min(max(__ldg(t.vLumPos + d2), 0), lmax) * ys, ly2B = min(max(__ldg(t.vLumPos + d2 + 1), 0), lmax) * ys;

        unsigned IU[2][4], IV[2][4];                                        // [tap pair][word]: two chroma samples x two lines each
        pair_interleave<NV>(W0, W1, IU[0], IV[0]);
        pair_interleave<NV>(W2, W3, IU[1], IV[1]);
        uint8_t *d = drow + (long long)(2 * i) * a.ds;
#pragma unroll 1
        for (int L = 0; L < 2; L++) {
            const int kx = L ? kB.x : kA.x, ky = L ? kB.y : kA.y;
            int aU[8], aV[8];
#pragma unroll
            for (int w = 0; w < 4; w++) {
                aU[2 * w]     = dp2a_lo_su(ky, IU[1][w], dp2a_lo_su(kx, IU[0][w], 1 << 11));
                aU[2 * w + 1] = dp2a_hi_su(ky, IU[1][w], dp2a_hi_su(kx, IU[0][w], 1 << 11));
                aV[2 * w]     = dp2a_lo_su(ky, IV[1][w], dp2a_lo_su(kx, IV[0][w], 1 << 11));
                aV[2 * w + 1] = dp2a_hi_su(ky, IV[1][w], dp2a_hi_su(kx, IV[0][w], 1 << 11));
            }
            const uint4 q = L ? YB : YA;
            const unsigned yw[4] = { q.x, q.y, q.z, q.w };
            unsigned m[8 * PW];
#pragma unroll
            for (int j = 0; j < 8; j++) {
                const ChromaBase cb = chroma_base(c, aU[j] >> 12, aV[j] >> 12);
                pair_out<KIND>(c.cy, cb, byte_of(yw[(2 * j) >> 2], (2 * j) & 3), byte_of(yw[(2 * j + 1) >> 2], (2 * j + 1) & 3), m + PW * j);
            }
            store_out<KIND>(L ? d + a.ds : d, m);
        }

        if (slide) { W0 = W1; W1 = W2; W2 = W3; W3 = G; }
        else if (fcN != fc) { W0 = line(fcN); W1 = line(fcN + 1); W2 = line(fcN + 2); W3 = line(fcN + 3); }
        YA = NA; YB = NB; kA = kNA; kB = kNB;
        fc = fcN; fcN = fc2; lyNA = ly2A; lyNB = ly2B;
    }
}

// ------------------------------------------------------------------------------------------------ kernel: vertical FIR + rgb24 (slow, general)
// All three writers (_X, _1, _2), u8 (identity horizontal pass) or int16 line-plane sources, any alignment.
// One thread = one pixel pair of one output line; covers pairs [p0, p1).  Grid: x over pairs, y over lines, z over frames.
template <bool SRC8>
__global__ void __launch_bounds__(128)
sws_vscale_rgb24_slow_kernel(SwsFrameArgs a, SwsDevTables t, SwsColorConst c, int p0, int p1)
{
    const int p = p0 + blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= p1) return;
    const int dy = blockIdx.y + a.y0;
    const long long f = blockIdx.z;
    const int lfs = t.vLumSize, cfs = t.vChrSize;
    const int16_t *lf = t.vLum + (long long)dy * lfs, *cf = t.vChr + (long long)dy * cfs;
    const int firstLum = max(1 - lfs, __ldg(t.vLumPos + dy));
    const int firstChr = max(1 - cfs, __ldg(t.vChrPos + dy));
    const int mode = __ldg(t.rowMode + 4 * dy), yalpha = __ldg(t.rowMode + 4 * dy + 1), uvalpha = __ldg(t.rowMode + 4 * dy + 2);
    const bool second = 2 * p + 1 < a.dstW;
    auto lum = [&](int line, int x) -> int {
        line = min(max(line, 0), a.srcH - 1);
        const uint8_t *b = a.y + f * a.yfs + (long long)line * a.ys;
        return SRC8 ? ((int)b[x] << 7) : (int)reinterpret_cast<const int16_t *>(b)[x];
    };
    auto chr = [&](const uint8_t *base, long long fs_, long long stride, int line) -> int {
        line = min(max(line, 0), a.chrSrcH - 1);
        const uint8_t *b = base + f * fs_ + (long long)line * stride;
        return SRC8 ? ((int)b[p] << 7) : (int)reinterpret_cast<const int16_t *>(b)[p];
    };
    const int x0 = 2 * p, x1 = second ? 2 * p + 1 : 2 * p;
    int Y0, Y1, U, V;
    if (mode == 1) {                                   // yuv2rgb_1_c_template, output.c:1883-1939
        Y0 = (lum(firstLum, x0) + 64) >> 7; Y1 = (lum(firstLum, x1) + 64) >> 7;
        if (!uvalpha) {
            U = (chr(a.u, a.ufs, a.us, firstChr) + 64) >> 7; V = (chr(a.v, a.vfs, a.vs, firstChr) + 64) >> 7;
        } else {
            const int a1 = 4096 - uvalpha;
            U = (chr(a.u, a.ufs, a.us, firstChr) * a1 + chr(a.u, a.ufs, a.us, firstChr + 1) * uvalpha + (128 << 11)) >> 19;
            V = (chr(a.v, a.vfs, a.vs, firstChr) * a1 + chr(a.v, a.vfs, a.vs, firstChr + 1) * uvalpha + (128 << 11)) >> 19;
        }
    } else if (mode == 2) {                            // yuv2rgb_2_c_template, output.c:1843-1880
        const int ya1 = 4096 - yalpha, ua1 = 4096 - uvalpha;
        Y0 = (lum(firstLum, x0) * ya1 + lum(firstLum + 1, x0) * yalpha) >> 19;
        Y1 = (lum(firstLum, x1) * ya1 + lum(firstLum + 1, x1) * yalpha) >> 19;
        U = (chr(a.u, a.ufs, a.us, firstChr) * ua1 + chr(a.u, a.ufs, a.us, firstChr + 1) * uvalpha) >> 19;
        V = (chr(a.v, a.vfs, a.vs, firstChr) * ua1 + chr(a.v, a.vfs, a.vs, firstChr + 1) * uvalpha) >> 19;
    } else {                                           // yuv2rgb_X_c_template, output.c:1789-1840 (unsigned wrap-around sums)
        unsigned s0 = 1u << 18, s1 = 1u << 18, su = 1u << 18, sv = 1u << 18;
        for (int j = 0; j < lfs; j++) {
            const unsigned k = (unsigned)(int)__ldg(lf + j);
            s0 += (unsigned)lum(firstLum + j, x0) * k; s1 += (unsigned)lum(firstLum + j, x1) * k;
        }
        for (int j = 0; j < cfs; j++) {
            const unsigned k = (unsigned)(int)__ldg(cf + j);
            su += (unsigned)chr(a.u, a.ufs, a.us, firstChr + j) * k; sv += (unsigned)chr(a.v, a.vfs, a.vs, firstChr + j) * k;
        }
        Y0 = (int)s0 >> 19; Y1 = (int)s1 >> 19; U = (int)su >> 19; V = (int)sv >> 19;
    }
    const ChromaBase cb = chroma_base(c, U, V);
    put_pair_bytes(a.dst + f * a.dfs + (long long)dy * a.ds + (long long)p * (2 * a.bpp), a, c, cb, Y0, Y1, second);
}

// ------------------------------------------------------------------------------------------------ kernel: vertical FIR + packed RGB from int16 lines (vector)
// The scaled path's `_X` writer (yuv2rgb_X_c_template) on the int16 line planes the horizontal pass leaves: one thread = 8
// pixels (4 chroma pairs) of one output line, 128-bit luma and 64-bit chroma line loads, sums mod 2^32 like the reference.
// Used when every line takes the `_X` writer, dstW % 8 == 0 and everything is aligned; other cases stay on the scalar kernel.
template <int KIND>
__global__ void __launch_bounds__(128)
sws_vscale_rgb24_x8_kernel(SwsFrameArgs a, SwsDevTables t, SwsColorConst c, int ngroups)
{
    constexpr int PW = OutWords<KIND>::per_pair, BPP = OutWords<KIND>::bpp;
    const int xg = blockIdx.x * blockDim.x + threadIdx.x;
    if (xg >= ngroups) return;
    const int dy = blockIdx.y + a.y0;
    const long long f = blockIdx.z;
    const int lfs = t.vLumSize, cfs = t.vChrSize;
    const int16_t *lf = t.vLum + (long long)dy * lfs, *cf = t.vChr + (long long)dy * cfs;
    const int firstLum = max(1 - lfs, __ldg(t.vLumPos + dy));
    const int firstChr = max(1 - cfs, __ldg(t.vChrPos + dy));
    const uint8_t *yb = a.y + f * a.yfs + xg * 16, *ub = a.u + f * a.ufs + xg * 8, *vb = a.v + f * a.vfs + xg * 8;
    unsigned sY[8], sU[4], sV[4];
#pragma unroll
    for (int i = 0; i < 8; i++) sY[i] = 1u << 18;
#pragma unroll
    for (int i = 0; i < 4; i++) sU[i] = sV[i] = 1u << 18;
    for (int j = 0; j < lfs; j++) {
        const int line = min(max(firstLum + j, 0), a.srcH - 1);
        const uint4 q = __ldg(reinterpret_cast<const uint4 *>(yb + (long long)line * a.ys));
        const unsigned k = (unsigned)(int)__ldg(lf + j);
        const unsigned w[4] = { q.x, q.y, q.z, q.w };
#pragma unroll
        for (int i = 0; i < 4; i++) { sY[2 * i] += (unsigned)(int)(short)(w[i] & 0xffff) * k; sY[2 * i + 1] += (unsigned)((int)w[i] >> 16) * k; }
    }
    for (int j = 0; j < cfs; j++) {
        const int line = min(max(firstChr + j, 0), a.chrSrcH - 1);
        const uint2 qu = __ldg(reinterpret_cast<const uint2 *>(ub + (long long)line * a.us));
        const uint2 qv = __ldg(reinterpret_cast<const uint2 *>(vb + (long long)line * a.vs));
        const unsigned k = (unsigned)(int)__ldg(cf + j);
        sU[0] += (unsigned)(int)(short)(qu.x & 0xffff) * k; sU[1] += (unsigned)((int)qu.x >> 16) * k;
        sU[2] += (unsigned)(int)(short)(qu.y & 0xffff) * k; sU[3] += (unsigned)((int)qu.y >> 16) * k;
        sV[0] += (unsigned)(int)(short)(qv.x & 0xffff) * k; sV[1] += (unsigned)((int)qv.x >> 16) * k;
        sV[2] += (unsigned)(int)(short)(qv.y & 0xffff) * k; sV[3] += (unsigned)((int)qv.y >> 16) * k;
    }
    unsigned m[4 * PW];
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const ChromaBase cb = chroma_base(c, (int)sU[i] >> 19, (int)sV[i] >> 19);
        pair_out<KIND>(c.cy, cb, (int)sY[2 * i] >> 19, (int)sY[2 * i + 1] >> 19, m + PW * i);
    }
    uint8_t *d = a.dst + f * a.dfs + (long long)dy * a.ds + (long long)xg * (8 * BPP);
    if (KIND <= SWS_OUT_BGR24) {                              // 4 pairs = 12 packed words -> 6 output words (24 bytes)
        uint2 *d2 = reinterpret_cast<uint2 *>(d);
#pragma unroll
        for (int k2 = 0; k2 < 3; k2++)
            d2[k2] = make_uint2(__byte_perm(m[4 * k2], m[4 * k2 + 1], 0x6420), __byte_perm(m[4 * k2 + 2], m[4 * k2 + 3], 0x6420));
    } else {
        uint4 *d4 = reinterpret_cast<uint4 *>(d);
        d4[0] = make_uint4(m[0], m[1], m[2], m[3]); d4[1] = make_uint4(m[4], m[5], m[6], m[7]);
    }
}

// ------------------------------------------------------------------------------------------------ kernel: full-chroma writer
// chrDstW == dstW (SWS_FULL_CHR_H_INT, forced for odd widths).  One thread per pixel; taps always from int16 planes.
__global__ void __launch_bounds__(256)
sws_vscale_rgb24_full_kernel(SwsFrameArgs a, SwsDevTables t, SwsColorConst c)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int dy = blockIdx.y + a.y0;
    if (x >= a.dstW) return;
    const long long f = blockIdx.z;
    const int lfs = t.vLumSize, cfs = t.vChrSize;
    const int16_t *lf = t.vLum + (long long)dy * lfs, *cf = t.vChr + (long long)dy * cfs;
    const int firstLum = max(1 - lfs, __ldg(t.vLumPos + dy));
    const int firstChr = max(1 - cfs, __ldg(t.vChrPos + dy));
    const int mode = __ldg(t.rowMode + 4 * dy), yalpha = __ldg(t.rowMode + 4 * dy + 1), uvalpha = __ldg(t.rowMode + 4 * dy + 2);
    auto L = [&](int line) { line = min(max(line, 0), a.srcH - 1);
        return (int)__ldg(reinterpret_cast<const int16_t *>(a.y + f * a.yfs + line * a.ys) + x); };
    auto Uu = [&](int line) { line = min(max(line, 0), a.chrSrcH - 1);
        return (int)__ldg(reinterpret_cast<const int16_t *>(a.u + f * a.ufs + line * a.us) + x); };
    auto Vv = [&](int line) { line = min(max(line, 0), a.chrSrcH - 1);
        return (int)__ldg(reinterpret_cast<const int16_t *>(a.v + f * a.vfs + line * a.vs) + x); };
    int Y, U, V;
    if (mode == 1) {                                   // output.c:2257-2310
        Y = L(firstLum) * 4;
        if (!uvalpha) { U = (Uu(firstChr) - (128 << 7)) * 4; V = (Vv(firstChr) - (128 << 7)) * 4; }
        else {
            const int a1 = 4096 - uvalpha;
            U = (Uu(firstChr) * a1 + Uu(firstChr + 1) * uvalpha - (128 << 19)) >> 10;
            V = (Vv(firstChr) * a1 + Vv(firstChr + 1) * uvalpha - (128 << 19)) >> 10;
        }
    } else if (mode == 2) {                            // output.c:2211-2254
        const int ya1 = 4096 - yalpha, ua1 = 4096 - uvalpha;
        Y = (L(firstLum) * ya1 + L(firstLum + 1) * yalpha) >> 10;
        U = (Uu(firstChr) * ua1 + Uu(firstChr + 1) * uvalpha - (128 << 19)) >> 10;
        V = (Vv(firstChr) * ua1 + Vv(firstChr + 1) * uvalpha - (128 << 19)) >> 10;
    } else {                                           // output.c:2161-2208
        unsigned ay = 1u << 9, au = (unsigned)((1 << 9) - (128 << 19)), av = au;
        for (int j = 0; j < lfs; j++) ay += (unsigned)L(firstLum + j) * (unsigned)(int)__ldg(lf + j);
        for (int j = 0; j < cfs; j++) {
            const unsigned k = (unsigned)(int)__ldg(cf + j);
            au += (unsigned)Uu(firstChr + j) * k;
            av += (unsigned)Vv(firstChr + j) * k;
        }
        Y = (int)ay >> 10; U = (int)au >> 10; V = (int)av >> 10;
    }
    // yuv2rgb_write_full, output.c:1998-2030
    const unsigned yy = (unsigned)(Y - c.y_offset) * (unsigned)c.y_coeff + (1u << 21);
    int R = (int)(yy + (unsigned)V * (unsigned)c.v2r);
    int G = (int)(yy + (unsigned)V * (unsigned)c.v2g + (unsigned)U * (unsigned)c.u2g);
    int B = (int)(yy + (unsigned)U * (unsigned)c.u2b);
    if ((R | G | B) & 0xC0000000) {
        R = (R & 0xC0000000) ? ((~R) >> 31 & 0x3FFFFFFF) : R;
        G = (G & 0xC0000000) ? ((~G) >> 31 & 0x3FFFFFFF) : G;
        B = (B & 0xC0000000) ? ((~B) >> 31 & 0x3FFFFFFF) : B;
    }
    uint8_t *d = a.dst + f * a.dfs + (long long)dy * a.ds + (long long)x * a.bpp;
    d[a.ro] = (uint8_t)(R >> 22); d[a.go] = (uint8_t)(G >> 22); d[a.bo] = (uint8_t)(B >> 22);
    if (a.ao >= 0) d[a.ao] = 255;
}

// ------------------------------------------------------------------------------------------------ kernels: planar destination
// yuv2planeX_8_c / yuv2plane1_8_c (output.c:468-493) with the flat dither of the 8-bit path (sws_pb_64, swscale.c:385-387):
//   fs > 1: clip_u8(((64 << 12) + sum_j line[first+j][x] * coef[j]) >> 19)      fs == 1: clip_u8((line[first][x] + 64) >> 7)
// One thread per output sample of one plane; lines outside the plane replicate the border line like the reference's ring.
__global__ void __launch_bounds__(256)
sws_vscale_planar_kernel(const int16_t *src, int sls, long long sfs, int nlines, uint8_t *dst, long long ds, long long dfs,
                         int w, const int16_t *coef, const int32_t *pos, int fs, int line0)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    if (x >= w) return;
    const int dy = blockIdx.y + line0;
    const long long f = blockIdx.z;
    const int16_t *p = reinterpret_cast<const int16_t *>(reinterpret_cast<const char *>(src) + f * sfs) + x;
    const int first = max(1 - fs, __ldg(pos + dy));
    int val;
    if (fs == 1) {
        val = ((int)__ldg(p + (long long)min(max(first, 0), nlines - 1) * sls) + 64) >> 7;
    } else {
        unsigned acc = 64u << 12;
        const int16_t *k = coef + (long long)dy * fs;
        for (int j = 0; j < fs; j++)
            acc += (unsigned)((int)__ldg(p + (long long)min(max(first + j, 0), nlines - 1) * sls) * (int)__ldg(k + j));
        val = (int)acc >> 19;
    }
    dst[f * dfs + (long long)dy * ds + x] = (uint8_t)clamp_u8(val);
}

// [device-code sws_new] (tests/cuda_emu runs this block on the CPU against the checker; comment markers only)
// ------------------------------------------------------------------------------------------------ kernels: packed RGB source
// Input readers fused into the horizontal pass.  The reference converts every source line to a 16-bit line first
// (rgb24ToY_c / bgr24ToY_c / the 32-bit templates, input.c:264-393,1068-1134: identical values for all six byte orders; chroma
// rgb24ToUV_c or, when the scaler samples chroma from every other pixel, rgb24ToUV_half_c on the sum of two pixels,
// input.c:1083-1172) and then runs hScale16To15_c (swscale.c:99-125: taps read as uint16, sum >> 13, clamp to 2^15-1).
// Here each thread produces one output sample and evaluates the reader for the taps it needs; first version, not tuned
// (neighbouring threads re-read overlapping source pixels from L1).
struct RgbIn { int bpp, ro, go, bo, half; int c[9]; };

__global__ void __launch_bounds__(256)
sws_rgbin_hscale_y_kernel(const uint8_t *src, long long sstride, long long sfs, int16_t *dst, int dstW, long long dfs,
                          const int16_t *filter, const int32_t *pos, int fs, const RgbIn R)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= dstW) return;
    const int line = blockIdx.y;
    const uint8_t *s = src + (long long)blockIdx.z * sfs + (long long)line * sstride;
    const int p0 = __ldg(pos + i);
    const int16_t *f = filter + (long long)i * fs;
    int acc = 0;
    for (int j = 0; j < fs; j++) {
        const uint8_t *px = s + (long long)(p0 + j) * R.bpp;
        const int v = (R.c[0] * (int)__ldg(px + R.ro) + R.c[1] * (int)__ldg(px + R.go) + R.c[2] * (int)__ldg(px + R.bo) + (32 << 14) + (1 << 8)) >> 9;
        acc += (int)(uint16_t)(int16_t)v * (int)__ldg(f + j);
    }
    dst[(long long)blockIdx.z * dfs + (long long)line * dstW + i] = (int16_t)min(acc >> 13, 32767);
}

// the alpha plane of a 32-bit source when the destination carries alpha too (c->needAlpha): rgbaToA_c / abgrToA_c (input.c:455-475) widen
// the byte to 14 bits, then the luma filter like any other line (hscale.c:103-160; hScale16To15_c, shift 13 for RGB sources)
__global__ void __launch_bounds__(256)
sws_rgbin_hscale_a_kernel(const uint8_t *src, long long sstride, long long sfs, int16_t *dst, int dstW, long long dfs,
                          const int16_t *filter, const int32_t *pos, int fs, int sao)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= dstW) return;
    const int line = blockIdx.y;
    const uint8_t *s = src + (long long)blockIdx.z * sfs + (long long)line * sstride;
    const int p0 = __ldg(pos + i);
    const int16_t *f = filter + (long long)i * fs;
    int acc = 0;
    for (int j = 0; j < fs; j++) {
        const int a = (int)__ldg(s + (long long)(p0 + j) * 4 + sao);
        acc += (a << 6 | a >> 2) * (int)__ldg(f + j);
    }
    dst[(long long)blockIdx.z * dfs + (long long)line * dstW + i] = (int16_t)min(acc >> 13, 32767);
}

// Alpha of the packed writers, run after the RGB writer has stored 255: the vertical luma filter on the alpha lines.
//   full-chroma writers (output.c:2191-2199 _X, :2240-2244 _2, :2282-2286 _1): (1 << 18 + sum) >> 19, (a0 ya1 + a1 ya + (1 << 18)) >> 19,
//   (a0 + 64) >> 7, each clipped only when bit 8 is set;
//   two-pixel writers (:1818-1830 _X: both clipped when either has bit 8 set; :1867-1872 _2: no rounding term; :1903-1908 / :1928-1933 _1:
//   (a0 * 255 + 16384) >> 15 below uvalpha 2048, else (a0 + 64) >> 7), always clipped.
// mode / yalpha / uvalpha per output line as packed_vscale picks them (rowMode, vscale.c:144-169).  One thread per pixel.
__global__ void __launch_bounds__(256)
sws_vscale_alpha_kernel(const int16_t *al, long long alfs, int srcH, uint8_t *dst, long long ds, long long dfs, int dstW, int bpp, int ao,
                        const int16_t *vLum, const int32_t *vLumPos, int lfs, const int32_t *rowMode, int full, int y0)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    if (x >= dstW) return;
    const int dy = blockIdx.y + y0;
    const int16_t *plane = al + (long long)blockIdx.z * alfs;
    const int16_t *lf = vLum + (long long)dy * lfs;
    const int firstLum = max(1 - lfs, __ldg(vLumPos + dy));
    const int mode = __ldg(rowMode + 4 * dy), yalpha = __ldg(rowMode + 4 * dy + 1), uvalpha = __ldg(rowMode + 4 * dy + 2);
    auto A_ = [&](int line, int xx) { line = min(max(line, 0), srcH - 1); return (int)__ldg(plane + (long long)line * dstW + xx); };
    auto sumX = [&](int xx) { unsigned s = 1u << 18; for (int j = 0; j < lfs; j++) s += (unsigned)A_(firstLum + j, xx) * (unsigned)(int)__ldg(lf + j); return (int)s >> 19; };
    int A;
    if (full) {
        if (mode == 1) A = (A_(firstLum, x) + 64) >> 7;
        else if (mode == 2) A = (A_(firstLum, x) * (4096 - yalpha) + A_(firstLum + 1, x) * yalpha + (1 << 18)) >> 19;
        else A = sumX(x);
        if (A & 0x100) A = min(max(A, 0), 255);
    } else {
        if (mode == 1) A = min(max(uvalpha < 2048 ? (A_(firstLum, x) * 255 + 16384) >> 15 : (A_(firstLum, x) + 64) >> 7, 0), 255);
        else if (mode == 2) A = min(max((A_(firstLum, x) * (4096 - yalpha) + A_(firstLum + 1, x) * yalpha) >> 19, 0), 255);
        else {
            A = sumX(x);
            const int B = (x ^ 1) < dstW ? sumX(x ^ 1) : A;
            if ((A | B) & 0x100) A = min(max(A, 0), 255);
        }
    }
    dst[(long long)blockIdx.z * dfs + (long long)dy * ds + (long long)x * bpp + ao] = (uint8_t)A;
}

__global__ void __launch_bounds__(256)
sws_rgbin_hscale_uv_kernel(const uint8_t *src, long long sstride, long long sfs, int16_t *dstU, int16_t *dstV, int dstW, long long dfs,
                           const int16_t *filter, const int32_t *pos, int fs, const RgbIn R)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= dstW) return;
    const int line = blockIdx.y;
    const uint8_t *s = src + (long long)blockIdx.z * sfs + (long long)line * sstride;
    const int p0 = __ldg(pos + i);
    const int16_t *f = filter + (long long)i * fs;
    int accU = 0, accV = 0;
    for (int j = 0; j < fs; j++) {
        int r, g, b, u, v;
        if (R.half) {
            const uint8_t *px = s + (long long)(p0 + j) * 2 * R.bpp, *q = px + R.bpp;
            r = (int)__ldg(px + R.ro) + (int)__ldg(q + R.ro); g = (int)__ldg(px + R.go) + (int)__ldg(q + R.go); b = (int)__ldg(px + R.bo) + (int)__ldg(q + R.bo);
            u = (R.c[3] * r + R.c[4] * g + R.c[5] * b + (256 << 15) + (1 << 9)) >> 10;
            v = (R.c[6] * r + R.c[7] * g + R.c[8] * b + (256 << 15) + (1 << 9)) >> 10;
        } else {
            const uint8_t *px = s + (long long)(p0 + j) * R.bpp;
            r = __ldg(px + R.ro); g = __ldg(px + R.go); b = __ldg(px + R.bo);
            u = (R.c[3] * r + R.c[4] * g + R.c[5] * b + (256 << 14) + (1 << 8)) >> 9;
            v = (R.c[6] * r + R.c[7] * g + R.c[8] * b + (256 << 14) + (1 << 8)) >> 9;
        }
        const int k = __ldg(f + j);
        accU += (int)(uint16_t)(int16_t)u * k;
        accV += (int)(uint16_t)(int16_t)v * k;
    }
    const long long o = (long long)blockIdx.z * dfs + (long long)line * dstW + i;
    dstU[o] = (int16_t)min(accU >> 13, 32767);
    dstV[o] = (int16_t)min(accV >> 13, 32767);
}

// bgr24 -> yuv420p, same size, without accurate_rnd: the reference's special converter ff_rgb24toyv12_c
// (rgb2rgb_template.c:580-641): Y = (dot >> 15) + 16 (truncating), U / V from the 2x2 box average of each channel; sums are
// formed in unsigned arithmetic and the byte store keeps the low 8 bits.  One thread per 2x2 pixel block.
__global__ void __launch_bounds__(256)
sws_bgr24_yv12_kernel(const uint8_t *src, long long sstride, long long sfs, uint8_t *dy, long long dys, long long dyf,
                      uint8_t *du, long long dus, long long duf, uint8_t *dv, long long dvs, long long dvf, int w, int h, const RgbIn R)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (w >> 1)) return;
    const int y = 2 * blockIdx.y;
    const long long f = blockIdx.z;
    const bool last = y + 1 == h;                                           // odd height: the last line pairs with itself
    const uint8_t *s1 = src + f * sfs + (long long)y * sstride + 6 * i, *s2 = last ? s1 : s1 + sstride;
    unsigned px[4][3];
#pragma unroll
    for (int k = 0; k < 3; k++) { px[0][k] = __ldg(s1 + k); px[1][k] = __ldg(s1 + 3 + k); px[2][k] = __ldg(s2 + k); px[3][k] = __ldg(s2 + 3 + k); }
    unsigned Y[4];
#pragma unroll
    for (int k = 0; k < 4; k++) Y[k] = (((unsigned)R.c[0] * px[k][2] + (unsigned)R.c[1] * px[k][1] + (unsigned)R.c[2] * px[k][0]) >> 15) + 16;
    uint8_t *y1 = dy + f * dyf + (long long)y * dys + 2 * i;
    y1[0] = (uint8_t)Y[0]; y1[1] = (uint8_t)Y[1];
    if (!last) { y1[dys] = (uint8_t)Y[2]; y1[dys + 1] = (uint8_t)Y[3]; }
    const unsigned bx = (px[0][0] + px[1][0] + px[2][0] + px[3][0]) >> 2, gx = (px[0][1] + px[1][1] + px[2][1] + px[3][1]) >> 2,
                   rx = (px[0][2] + px[1][2] + px[2][2] + px[3][2]) >> 2;
    du[f * duf + (long long)blockIdx.y * dus + i] = (uint8_t)((((unsigned)R.c[3] * rx + (unsigned)R.c[4] * gx + (unsigned)R.c[5] * bx) >> 15) + 128);
    dv[f * dvf + (long long)blockIdx.y * dvs + i] = (uint8_t)((((unsigned)R.c[6] * rx + (unsigned)R.c[7] * gx + (unsigned)R.c[8] * bx) >> 15) + 128);
}

// lumRangeToJpeg_c / lumRangeFromJpeg_c / chrRange*_c (swscale.c:163-209) applied in place to the horizontally scaled lines,
// where the reference calls them (hscale.c:61-63, :195-197): v = (v * coeff + offset) >> 14, limited -> full clips at 2^15-1.
// One thread per sample; grid x over the line, y over lines, z over frames (dfs in int16 elements).
__global__ void __launch_bounds__(256)
sws_range_kernel(int16_t *mid, int w, long long dfs, int coeff, int offset, int clip)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    if (x >= w) return;
    int16_t *p = mid + (long long)blockIdx.z * dfs + (long long)blockIdx.y * w + x;
    int v = ((int)*p * coeff + offset) >> 14;
    if (clip) v = min(v, 32767);
    *p = (int16_t)v;
}

// [/device-code sws_new]
// four adjacent samples per thread: 64-bit loads of the int16 lines, one 32-bit store (w % 4 == 0, 4-aligned destination)
__global__ void __launch_bounds__(256)
sws_vscale_planar4_kernel(const int16_t *src, int sls, long long sfs, int nlines, uint8_t *dst, long long ds, long long dfs,
                          int w, const int16_t *coef, const int32_t *pos, int fs, int line0)
{
    const int x = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
    if (x >= w) return;
    const int dy = blockIdx.y + line0;
    const long long f = blockIdx.z;
    const int16_t *p = reinterpret_cast<const int16_t *>(reinterpret_cast<const char *>(src) + f * sfs) + x;
    const int first = max(1 - fs, __ldg(pos + dy));
    int v0, v1, v2, v3;
    if (fs == 1) {
        const uint2 q = __ldg(reinterpret_cast<const uint2 *>(p + (long long)min(max(first, 0), nlines - 1) * sls));
        v0 = ((int)(short)(q.x & 0xffff) + 64) >> 7; v1 = (((int)q.x >> 16) + 64) >> 7;
        v2 = ((int)(short)(q.y & 0xffff) + 64) >> 7; v3 = (((int)q.y >> 16) + 64) >> 7;
    } else {
        unsigned a0 = 64u << 12, a1 = a0, a2 = a0, a3 = a0;
        const int16_t *k = coef + (long long)dy * fs;
        for (int j = 0; j < fs; j++) {
            const uint2 q = __ldg(reinterpret_cast<const uint2 *>(p + (long long)min(max(first + j, 0), nlines - 1) * sls));
            const int c = (int)__ldg(k + j);
            a0 += (unsigned)((int)(short)(q.x & 0xffff) * c); a1 += (unsigned)(((int)q.x >> 16) * c);
            a2 += (unsigned)((int)(short)(q.y & 0xffff) * c); a3 += (unsigned)(((int)q.y >> 16) * c);
        }
        v0 = (int)a0 >> 19; v1 = (int)a1 >> 19; v2 = (int)a2 >> 19; v3 = (int)a3 >> 19;
    }
    const unsigned lo = __vimin_s16x2_relu(__byte_perm((unsigned)v0, (unsigned)v1, 0x5410), 0x00ff00ffu);
    const unsigned hi = __vimin_s16x2_relu(__byte_perm((unsigned)v2, (unsigned)v3, 0x5410), 0x00ff00ffu);
    *reinterpret_cast<unsigned *>(dst + f * dfs + (long long)dy * ds + x) = __byte_perm(lo, hi, 0x6420);
}

// eight adjacent samples per thread: 128-bit loads of the int16 lines, one 64-bit store (w % 8 == 0, 8-aligned destination)
__global__ void __launch_bounds__(256)
sws_vscale_planar8_kernel(const int16_t *src, int sls, long long sfs, int nlines, uint8_t *dst, long long ds, long long dfs,
                          int w, const int16_t *coef, const int32_t *pos, int fs, int line0)
{
    const int x = (blockIdx.x * blockDim.x + threadIdx.x) * 8;
    if (x >= w) return;
    const int dy = blockIdx.y + line0;
    const long long f = blockIdx.z;
    const int16_t *p = reinterpret_cast<const int16_t *>(reinterpret_cast<const char *>(src) + f * sfs) + x;
    const int first = max(1 - fs, __ldg(pos + dy));
    int v[8];
    if (fs == 1) {
        const uint4 q = __ldg(reinterpret_cast<const uint4 *>(p + (long long)min(max(first, 0), nlines - 1) * sls));
        const unsigned ww[4] = { q.x, q.y, q.z, q.w };
#pragma unroll
        for (int j = 0; j < 4; j++) { v[2 * j] = ((int)(short)(ww[j] & 0xffff) + 64) >> 7; v[2 * j + 1] = (((int)ww[j] >> 16) + 64) >> 7; }
    } else {
        unsigned a[8];
#pragma unroll
        for (int j = 0; j < 8; j++) a[j] = 64u << 12;
        const int16_t *k = coef + (long long)dy * fs;
        for (int t = 0; t < fs; t++) {
            const uint4 q = __ldg(reinterpret_cast<const uint4 *>(p + (long long)min(max(first + t, 0), nlines - 1) * sls));
            const unsigned ww[4] = { q.x, q.y, q.z, q.w };
            const int c = (int)__ldg(k + t);
#pragma unroll
            for (int j = 0; j < 4; j++) { a[2 * j] += (unsigned)((int)(short)(ww[j] & 0xffff) * c); a[2 * j + 1] += (unsigned)(((int)ww[j] >> 16) * c); }
        }
#pragma unroll
        for (int j = 0; j < 8; j++) v[j] = (int)a[j] >> 19;
    }
    unsigned o[2];
#pragma unroll
    for (int h = 0; h < 2; h++) {
        const unsigned lo = __vimin_s16x2_relu(__byte_perm((unsigned)v[4 * h], (unsigned)v[4 * h + 1], 0x5410), 0x00ff00ffu);
        const unsigned hi = __vimin_s16x2_relu(__byte_perm((unsigned)v[4 * h + 2], (unsigned)v[4 * h + 3], 0x5410), 0x00ff00ffu);
        o[h] = __byte_perm(lo, hi, 0x6420);
    }
    *reinterpret_cast<uint2 *>(dst + f * dfs + (long long)dy * ds + x) = make_uint2(o[0], o[1]);
}

// planarCopyWrapper (swscale_unscaled.c:2220-2333, 8-bit planes): row copies, 16 bytes per thread when everything is aligned
__global__ void __launch_bounds__(256)
sws_plane_copy_kernel(const uint8_t *src, long long ss, long long sfs, uint8_t *dst, long long ds, long long dfs, int w, int vec)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const uint8_t *s = src + blockIdx.z * sfs + (long long)blockIdx.y * ss;
    uint8_t *d = dst + blockIdx.z * dfs + (long long)blockIdx.y * ds;
    if (vec) {
        if (i * 16 + 16 <= w) reinterpret_cast<uint4 *>(d)[i] = __ldg(reinterpret_cast<const uint4 *>(s) + i);
        else for (int k = i * 16; k < w; k++) d[k] = s[k];
    } else if (i < w) d[i] = s[i];
}

// nv12 / nv21 source: plane 1 -> separate U and V planes (nvXXtoUV_c, input.c:921-948).  One thread per chroma sample pair.
__global__ void __launch_bounds__(256)
sws_nv_split_kernel(const uint8_t *uv, long long uvs, long long uvfs, uint8_t *u, uint8_t *v, long long pitch, long long fs,
                    int cw, int row0)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= cw) return;
    const int r = blockIdx.y + row0;
    const uint8_t *s = uv + blockIdx.z * uvfs + (long long)r * uvs + 2 * i;
    const long long o = blockIdx.z * fs + (long long)r * pitch + i;
    u[o] = __ldg(s); v[o] = __ldg(s + 1);
}

// ------------------------------------------------------------------------------------------------ host side
struct B200SwsContext {
    B200Device *dev = nullptr;
    SwsPlan plan;
    void *tables = nullptr;          // one device allocation holding all banks
    SwsDevTables dt{};
    void *mma_tables = nullptr;      // horizontal banks as tensor-core operands (sws_mma.cuh)
    SwsMmaBank mmaL{}, mmaC{};
    int last_path = 0;               // kernels the last launches used: 1 two passes, 2 fused CUDA-core, 4 fused tensor-core (scaled path),
                                     // 8 same-size line-pair kernel (b200_sws_last_path)
    int mma_pitchL = 0, mma_pitchC = 0, mma_pitchC8 = 0;   // staged-line pitches: luma / chroma tiles of 16 groups, chroma tiles of 8 groups
    bool h_identity = false;         // both horizontal banks are the identity -> u8-source kernels
    bool fast_x = false;             // every line uses the _X writer and no 32-bit sum can wrap -> vector kernel
    bool lum_identity = false;       // vertical luma bank is a single tap of 4096 on every line
    bool all_x = false;              // every output line takes the `_X` writer (rowMode 0)
    bool pair_ok = false;            // identity luma bank, 4 chroma taps, and output lines 2k+1 / 2k+2 share their chroma window
    // intermediate int16 line planes for the scaled path (grown on demand, per batch)
    void *mid = nullptr; size_t mid_bytes = 0;
    // de-interleaved chroma of an nv12 / nv21 source (persistent: slice calls keep earlier bands here)
    void *nv_buf = nullptr; size_t nv_bytes = 0;
    // chroma planes of an nv12 / nv21 destination before they are interleaved
    void *nvout_buf = nullptr; size_t nvout_bytes = 0;
    // slice calls (sws_scale with srcSliceH < srcH): device copies of the source planes and of the picture being built,
    // plus the next output line (SwsInternal.dstY, swscale.c:297,551)
    void *slice_buf = nullptr;
    int next_dst_y = 0;
    bool slice_open = false;
    int slice_dir = 1;               // SwsInternal.sliceDir: 1 top-down, -1 bottom-up (the picture is flipped internally, swscale.c:1096-1159)
    // yuv -> yuv with two different matrices: the reference cascades two contexts through a bgr24 picture (utils.c:914-989)
    B200SwsContext *casc[2] = { nullptr, nullptr };
    void *casc_tmp = nullptr;        // the intermediate picture on the device (zeroed once: the unscaled converter of context 0
                                     // leaves an odd last column unwritten, the reference reads uninitialised memory there)
    size_t casc_pitch = 0;
    int casc_w = 0, casc_h = 0;
    int open_src_fmt = 0, open_dst_fmt = 0, open_flags = 0;      // as given to sws_getContext
    bool has_param = false;
    double open_param[2] = { 0, 0 };
};

static int upload_mma_tables(B200SwsContext *c);
static int upload_tables(B200SwsContext *c)
{
    const SwsPlan &p = c->plan;
    if (c->tables) { cudaFree(c->tables); c->tables = nullptr; }
    if (c->mma_tables) { cudaFree(c->mma_tables); c->mma_tables = nullptr; c->mmaL = SwsMmaBank{}; c->mmaC = SwsMmaBank{}; }
    if (p.unscaled_lut || p.planar_copy || p.bgr24_yv12 || p.rgb_shuffle) return 0;
    auto al = [](size_t v) { return (v + 255) & ~(size_t)255; };
    size_t off = 0;
    size_t o_vl = off;  off += al(p.vLum.coef.size() * 2);
    size_t o_vlp = off; off += al(p.vLum.pos.size() * 4);
    size_t o_vc = off;  off += al(p.vChr.coef.size() * 2);
    size_t o_vcp = off; off += al(p.vChr.pos.size() * 4);
    size_t o_rm = off;  off += al(p.rowMode.size() * 4);
    auto pack_pairs = [](const SwsFilterBank &b) {
        const int np = (b.size + 1) / 2;
        std::vector<int32_t> o((size_t)b.n * np);
        for (int i = 0; i < b.n; i++)
            for (int j = 0; j < np; j++) {
                const uint32_t lo = (uint16_t)b.coef[(size_t)i * b.size + 2 * j];
                const uint32_t hi = 2 * j + 1 < b.size ? (uint16_t)b.coef[(size_t)i * b.size + 2 * j + 1] : 0;
                o[(size_t)i * np + j] = (int32_t)(lo | (hi << 16));
            }
        return o;
    };
    const std::vector<int32_t> vl2 = pack_pairs(p.vLum), vc2 = pack_pairs(p.vChr);
    size_t o_vl2 = off; off += al(vl2.size() * 4);
    size_t o_vc2 = off; off += al(vc2.size() * 4);
    const std::vector<int32_t> hl2 = pack_pairs(p.hLum), hc2 = pack_pairs(p.hChr);
    size_t o_hl2 = off; off += al(hl2.size() * 4);
    size_t o_hc2 = off; off += al(hc2.size() * 4);
    size_t o_hl = off;  off += al(p.hLum.coef.size() * 2);
    size_t o_hlp = off; off += al(p.hLum.pos.size() * 4);
    size_t o_hc = off;  off += al(p.hChr.coef.size() * 2);
    size_t o_hcp = off; off += al(p.hChr.pos.size() * 4);
    std::vector<uint8_t> host(off, 0);
    memcpy(&host[o_vl], p.vLum.coef.data(), p.vLum.coef.size() * 2);
    memcpy(&host[o_vlp], p.vLum.pos.data(), p.vLum.pos.size() * 4);
    memcpy(&host[o_vc], p.vChr.coef.data(), p.vChr.coef.size() * 2);
    memcpy(&host[o_vcp], p.vChr.pos.data(), p.vChr.pos.size() * 4);
    memcpy(&host[o_rm], p.rowMode.data(), p.rowMode.size() * 4);
    memcpy(&host[o_vl2], vl2.data(), vl2.size() * 4);
    memcpy(&host[o_vc2], vc2.data(), vc2.size() * 4);
    memcpy(&host[o_hl2], hl2.data(), hl2.size() * 4);
    memcpy(&host[o_hc2], hc2.data(), hc2.size() * 4);
    memcpy(&host[o_hl], p.hLum.coef.data(), p.hLum.coef.size() * 2);
    memcpy(&host[o_hlp], p.hLum.pos.data(), p.hLum.pos.size() * 4);
    memcpy(&host[o_hc], p.hChr.coef.data(), p.hChr.coef.size() * 2);
    memcpy(&host[o_hcp], p.hChr.pos.data(), p.hChr.pos.size() * 4);
    B200_CUDA_OK(cudaMalloc(&c->tables, off));
    B200_CUDA_OK(cudaMemcpy(c->tables, host.data(), off, cudaMemcpyHostToDevice));
    uint8_t *b = (uint8_t *)c->tables;
    c->dt.vLum = (const int16_t *)(b + o_vl); c->dt.vLumPos = (const int32_t *)(b + o_vlp); c->dt.vLumSize = p.vLum.size;
    c->dt.vChr = (const int16_t *)(b + o_vc); c->dt.vChrPos = (const int32_t *)(b + o_vcp); c->dt.vChrSize = p.vChr.size;
    c->dt.rowMode = (const int32_t *)(b + o_rm);
    c->dt.vLum2 = (const int32_t *)(b + o_vl2); c->dt.vChr2 = (const int32_t *)(b + o_vc2);
    c->dt.hLum2 = (const int32_t *)(b + o_hl2); c->dt.hChr2 = (const int32_t *)(b + o_hc2);
    c->dt.hLum = (const int16_t *)(b + o_hl); c->dt.hLumPos = (const int32_t *)(b + o_hlp); c->dt.hLumSize = p.hLum.size;
    c->dt.hChr = (const int16_t *)(b + o_hc); c->dt.hChrPos = (const int32_t *)(b + o_hcp); c->dt.hChrSize = p.hChr.size;
    c->h_identity = !p.fast_bilinear && p.chrDstHSub == 1 && p.hLum.identity() && p.hChr.identity();
    c->all_x = !p.planar;
    for (int y = 0; y < p.dstH && c->all_x; y++) if (p.rowMode[(size_t)y * 4] != 0) c->all_x = false;
    c->fast_x = c->h_identity && !p.planar;
    c->lum_identity = p.vLum.size == 1;
    for (int y = 0; y < p.dstH && c->fast_x; y++) {
        if (p.rowMode[(size_t)y * 4] != 0) c->fast_x = false;
        long long sl = 0, sc = 0;
        for (int j = 0; j < p.vLum.size; j++) sl += std::abs((int)p.vLum.coef[(size_t)y * p.vLum.size + j]);
        for (int j = 0; j < p.vChr.size; j++) sc += std::abs((int)p.vChr.coef[(size_t)y * p.vChr.size + j]);
        if (sl > 60000 || sc > 60000) c->fast_x = false;         // (2^18 + 32640 * sum|coef|) must stay below 2^31
        if (p.vLum.size != 1 || p.vLum.coef[y] != 4096) c->lum_identity = false;
    }
    c->pair_ok = c->fast_x && c->lum_identity && p.vChr.size == 4 && p.dstH >= 4;
    for (int y = 1; y + 1 < p.dstH && c->pair_ok; y += 2)
        if (p.vChr.pos[y] != p.vChr.pos[y + 1]) c->pair_ok = false;
    return upload_mma_tables(c);
}

// source side of a plan: yuv420p, nv12 / nv21, or packed 8-bit RGB (input readers); false = not a source this path reads
static bool set_source_format(SwsPlan &p, int srcFormat)
{
    p.src_nv = srcFormat == B200_PIX_FMT_NV12 ? 1 : srcFormat == B200_PIX_FMT_NV21 ? 2 : 0;
    p.src_rgb = 0;
    if (srcFormat == B200_PIX_FMT_YUV420P || p.src_nv) return true;
    SwsOutFmt f;
    if (!sws_out_format(srcFormat, f) || sws_out_is_yuv(f.kind)) return false;
    p.src_rgb = f.bpp; p.sro = f.ro; p.sgo = f.go; p.sbo = f.bo;
    return true;
}

B200_API B200SwsContext *b200_sws_getContext(B200Device *dev, int srcW, int srcH, int srcFormat,
                                             int dstW, int dstH, int dstFormat, int flags)
{
    return b200_sws_getContext_range(dev, srcW, srcH, srcFormat, 0, dstW, dstH, dstFormat, 0, flags);
}

B200_API B200SwsContext *b200_sws_getContext_range(B200Device *dev, int srcW, int srcH, int srcFormat, int srcRange,
                                                   int dstW, int dstH, int dstFormat, int dstRange, int flags)
{
    return b200_sws_getContext_params(dev, srcW, srcH, srcFormat, srcRange, dstW, dstH, dstFormat, dstRange, flags, nullptr);
}

B200_API B200SwsContext *b200_sws_getContext_params(B200Device *dev, int srcW, int srcH, int srcFormat, int srcRange,
                                                    int dstW, int dstH, int dstFormat, int dstRange, int flags, const double *param)
{
    return b200_sws_getContext_filters(dev, srcW, srcH, srcFormat, srcRange, dstW, dstH, dstFormat, dstRange, flags, nullptr, nullptr, param);
}

B200_API B200SwsContext *b200_sws_getContext_filters(B200Device *dev, int srcW, int srcH, int srcFormat, int srcRange, int dstW, int dstH, int dstFormat,
                                                     int dstRange, int flags, const B200SwsFilter *srcFilter, const B200SwsFilter *dstFilter,
                                                     const double *param)
{
    if (!dev) { b200_set_error("b200_sws_getContext: no device"); return nullptr; }
    SwsOutFmt out;
    B200SwsContext *c = new (std::nothrow) B200SwsContext();
    if (!c) return nullptr;
    if (!set_source_format(c->plan, srcFormat) || !sws_out_format(dstFormat, out)) {
        b200_set_error("b200_sws_getContext: only yuv420p / nv12 / nv21 -> rgb24 / bgr24 / rgba / bgra / argb / abgr / yuv420p and "
                       "packed 8-bit RGB -> yuv420p are implemented");
        delete c;
        return nullptr;
    }
    c->dev = dev;
    c->plan.out = out;
    {
        const B200SwsVector *sv[4] = { srcFilter ? srcFilter->lumH : nullptr, srcFilter ? srcFilter->lumV : nullptr, srcFilter ? srcFilter->chrH : nullptr, srcFilter ? srcFilter->chrV : nullptr };
        const B200SwsVector *dv[4] = { dstFilter ? dstFilter->lumH : nullptr, dstFilter ? dstFilter->lumV : nullptr, dstFilter ? dstFilter->chrH : nullptr, dstFilter ? dstFilter->chrV : nullptr };
        for (int k = 0; k < 4; k++) {
            if (sv[k] && sv[k]->coeff && sv[k]->length > 0) c->plan.srcFilt[k].assign(sv[k]->coeff, sv[k]->coeff + sv[k]->length);
            if (dv[k] && dv[k]->length > 0) c->plan.dstFiltLen[k] = dv[k]->length;
        }
    }
    c->open_src_fmt = srcFormat; c->open_dst_fmt = dstFormat; c->open_flags = flags;
    if (param) { c->plan.param[0] = param[0]; c->plan.param[1] = param[1]; c->has_param = true; c->open_param[0] = param[0]; c->open_param[1] = param[1]; }
    int ret = sws_plan_build(c->plan, srcW, srcH, dstW, dstH, flags, srcRange, dstRange);
    if (ret < 0) { b200_set_error("b200_sws_getContext: unsupported configuration (%d)", ret); delete c; return nullptr; }
    cudaSetDevice(dev->ordinal);
    if (upload_tables(c) < 0) { delete c; return nullptr; }
    return c;
}

B200_API void b200_sws_freeContext(B200SwsContext *c)
{
    if (!c) return;
    cudaSetDevice(c->dev->ordinal);
    cudaStreamSynchronize(c->dev->stream);
    if (c->tables) cudaFree(c->tables);
    if (c->mma_tables) cudaFree(c->mma_tables);
    if (c->mid) cudaFree(c->mid);
    if (c->nv_buf) cudaFree(c->nv_buf);
    if (c->nvout_buf) cudaFree(c->nvout_buf);
    if (c->slice_buf) cudaFree(c->slice_buf);
    if (c->casc_tmp) cudaFree(c->casc_tmp);
    b200_sws_freeContext(c->casc[0]);
    b200_sws_freeContext(c->casc[1]);
    delete c;
}

B200_API int b200_sws_setColorspaceDetails(B200SwsContext *c, const int inv_table[4], int srcRange,
                                           const int table[4], int dstRange, int brightness, int contrast, int saturation)
{
    if (!c || !inv_table || !table) return B200_EINVAL;
    if (c->casc[0])                                              // utils.c:908-909: a cascaded context hands the call to its main child
        return b200_sws_setColorspaceDetails(c->casc[0], inv_table, srcRange, table, dstRange, brightness, contrast, saturation);
    const int ret = sws_plan_colorspace_details(c->plan, inv_table, srcRange, table, dstRange, brightness, contrast, saturation);
    if (ret != B200_ENOSYS) return ret;
    // yuv -> yuv with different matrices (utils.c:914-989): context 0 = source -> bgr24 at the smaller of the two sizes with these details
    // (its RGB side ignores the destination half), context 1 = bgr24 -> destination with the ranges set before its initialisation and
    // the details again without brightness / contrast / saturation; sws_scale then runs whole frames through both (scale_cascaded)
    const SwsPlan &p = c->plan;
    const bool big = (long long)p.srcW * p.srcH > (long long)p.dstW * p.dstH;
    c->casc_w = big ? p.dstW : p.srcW; c->casc_h = big ? p.dstH : p.srcH;
    const double *pr = c->has_param ? c->open_param : nullptr;
    c->casc[0] = b200_sws_getContext_params(c->dev, p.srcW, p.srcH, c->open_src_fmt, 0, c->casc_w, c->casc_h, B200_PIX_FMT_BGR24, 0, c->open_flags, pr);
    c->casc[1] = b200_sws_getContext_params(c->dev, c->casc_w, c->casc_h, B200_PIX_FMT_BGR24, srcRange, p.dstW, p.dstH, c->open_dst_fmt, dstRange, c->open_flags, pr);
    c->casc_pitch = ((size_t)c->casc_w * 3 + 255) & ~(size_t)255;
    if (!c->casc[0] || !c->casc[1] || cudaSetDevice(c->dev->ordinal) != cudaSuccess ||
        cudaMalloc(&c->casc_tmp, c->casc_pitch * c->casc_h) != cudaSuccess || cudaMemsetAsync(c->casc_tmp, 0, c->casc_pitch * c->casc_h, c->dev->stream) != cudaSuccess) {
        b200_sws_freeContext(c->casc[0]); b200_sws_freeContext(c->casc[1]);
        c->casc[0] = c->casc[1] = nullptr;
        if (c->casc_tmp) { cudaFree(c->casc_tmp); c->casc_tmp = nullptr; }
        b200_set_error("sws_setColorspaceDetails: could not set up the yuv -> bgr24 -> yuv cascade for two different matrices");
        return B200_ENOSYS;
    }
    b200_sws_setColorspaceDetails(c->casc[0], inv_table, srcRange, table, dstRange, brightness, contrast, saturation);
    b200_sws_setColorspaceDetails(c->casc[1], inv_table, srcRange, table, dstRange, 0, 1 << 16, 1 << 16);
    return 0;
}

B200_API int b200_sws_info(const B200SwsContext *c, int *o)
{
    if (!c || !o) return B200_EINVAL;
    const SwsPlan &p = c->plan;
    o[0] = p.hLum.size; o[1] = p.hChr.size; o[2] = p.vLum.size; o[3] = p.vChr.size;
    o[4] = p.chrSrcW; o[5] = p.chrSrcH; o[6] = p.chrDstW; o[7] = p.chrDstH;
    o[8] = p.unscaled_lut; o[9] = 1; o[10] = 1; o[11] = p.chrDstHSub; o[12] = 0;
    o[13] = p.dstW; o[14] = p.dstH; o[15] = 0;
    return 0;
}

B200_API int b200_sws_last_path(B200SwsContext *c)
{
    if (!c) return B200_EINVAL;
    const int v = c->last_path;
    c->last_path = 0;
    return v;
}

B200_API int b200_sws_get_filter(const B200SwsContext *c, int which, int16_t *filter, int32_t *pos, int cap)
{
    if (!c) return B200_EINVAL;
    const SwsFilterBank &b = which == 0 ? c->plan.hLum : which == 1 ? c->plan.hChr : which == 2 ? c->plan.vLum : c->plan.vChr;
    int n = b.n < cap ? b.n : cap;
    if (filter) memcpy(filter, b.coef.data(), (size_t)n * b.size * 2);
    if (pos) memcpy(pos, b.pos.data(), (size_t)n * 4);
    return n;
}

B200_API int b200_sws_plan_probe(int srcW, int srcH, int dstW, int dstH, int flags, int which,
                                 int16_t *filter, int32_t *pos, int cap, int *o)
{
    SwsPlan p;
    int ret = sws_plan_build(p, srcW, srcH, dstW, dstH, flags);
    if (ret < 0) return ret;
    if (o) {
        o[0] = p.hLum.size; o[1] = p.hChr.size; o[2] = p.vLum.size; o[3] = p.vChr.size;
        o[4] = p.chrSrcW; o[5] = p.chrSrcH; o[6] = p.chrDstW; o[7] = p.chrDstH;
        o[8] = p.unscaled_lut; o[9] = 1; o[10] = 1; o[11] = p.chrDstHSub; o[12] = 0;
        o[13] = p.dstW; o[14] = p.dstH; o[15] = 0;
    }
    const SwsFilterBank &b = which == 0 ? p.hLum : which == 1 ? p.hChr : which == 2 ? p.vLum : p.vChr;
    int n = b.n < cap ? b.n : cap;
    if (filter && n) memcpy(filter, b.coef.data(), (size_t)n * b.size * 2);
    if (pos && n) memcpy(pos, b.pos.data(), (size_t)n * 4);
    return n;
}

// The general form: any source / destination format and ranges this path takes, plus an optional sws_setColorspaceDetails()
// call after the build.  cfg = { srcW, srcH, srcFormat, srcRange, dstW, dstH, dstFormat, dstRange, flags };
// details = NULL or { inv_table[4], srcRange, table[4], dstRange, brightness, contrast, saturation } (13 ints);
// info32: [0..15] as b200_sws_info, [16] plain copy, [17] range conversion (0 none, 1 limited->full, 2 full->limited),
// [18..21] luma coefficient, luma offset, chroma coefficient, chroma offset, [22] fast-bilinear horizontal pass,
// [23] semi-planar source kind, [24] what the details call returned, [25] src_range, [26] dst_range, [27] packed RGB source
// (bytes per pixel), [28] / [29] horizontal / vertical chroma shift of the source as scaled, [30] bgr24 -> yv12 converter, [31] nv12 / nv21 destination,
// [32..40] the rgb -> yuv table (needs room for 48 ints).
B200_API int b200_sws_plan_probe2(const int cfg[9], const int *details, int which, int16_t *filter, int32_t *pos, int cap, int *o)
{
    if (!cfg) return B200_EINVAL;
    SwsPlan p;
    if (!set_source_format(p, cfg[2]) || !sws_out_format(cfg[6], p.out)) return B200_ENOSYS;
    int ret = sws_plan_build(p, cfg[0], cfg[1], cfg[4], cfg[5], cfg[8], cfg[3], cfg[7]);
    if (ret < 0) return ret;
    int dret = 0;
    if (details)
        dret = sws_plan_colorspace_details(p, details, details[4], details + 5, details[9], details[10], details[11], details[12]);
    if (o) {
        o[0] = p.hLum.size; o[1] = p.hChr.size; o[2] = p.vLum.size; o[3] = p.vChr.size;
        o[4] = p.chrSrcW; o[5] = p.chrSrcH; o[6] = p.chrDstW; o[7] = p.chrDstH;
        o[8] = p.unscaled_lut; o[9] = 1; o[10] = 1; o[11] = p.chrDstHSub; o[12] = p.planar ? 1 : 0;
        o[13] = p.dstW; o[14] = p.dstH; o[15] = 0;
        o[16] = p.planar_copy; o[17] = p.range_conv;
        o[18] = p.lumRangeCoeff; o[19] = p.lumRangeOffset; o[20] = p.chrRangeCoeff; o[21] = p.chrRangeOffset;
        o[22] = p.fast_bilinear; o[23] = p.src_nv; o[24] = dret; o[25] = p.src_range; o[26] = p.dst_range;
        o[27] = p.src_rgb; o[28] = p.chrSrcHSub; o[29] = p.chrSrcVSub; o[30] = p.bgr24_yv12; o[31] = p.dst_nv;
        for (int i = 0; i < 9; i++) o[32 + i] = p.rgb2yuv[i];
        o[41] = p.rgb_shuffle; o[42] = (int)p.shuffle_sel;
    }
    const SwsFilterBank &b = which == 0 ? p.hLum : which == 1 ? p.hChr : which == 2 ? p.vLum : p.vChr;
    int n = b.n < cap ? b.n : cap;
    if (filter && n) memcpy(filter, b.coef.data(), (size_t)n * b.size * 2);
    if (pos && n) memcpy(pos, b.pos.data(), (size_t)n * 4);
    return n;
}

// ------------------------------------------------------------------------------------------------ kernels: fused horizontal + vertical scaler
// The two-pass scaler writes every horizontally scaled line to HBM as int16 and the vertical pass reads each of them back once per
// tap (through L2 mostly): about 2.6 x the algorithmic traffic, and both passes are load-bound.  Here a CTA owns a tile of FT_W output
// columns x TR output lines: it runs the horizontal FIR (same code and arithmetic as sws_hscale_rows_kernel) over exactly the source
// lines the tile's vertical taps reach — the reference's ring buffer of scaled lines (swscale.c:412-535), tile-sized, in shared
// memory — and then the vertical FIR + writer (same arithmetic as sws_vscale_planar8_kernel / sws_vscale_rgb24_x8_kernel) out of
// shared memory.  Source bytes are read from HBM once (plus the vertical halo, 8 lines in 72 for 4K -> 1080p), nothing else moves.
constexpr int FT_W = 128;               // output columns per CTA = threads per CTA

// horizontal FIR of output column `col` over source lines ra .. rb into lines[(r - ra) * FT_W + slot]
template <int NP, int PITCH>
__device__ __forceinline__ void fused_hstage(const uint8_t *plane, long long sstride, const int32_t *coef2, const int32_t *pos, int fs,
                                             int col, int ra, int rb, int16_t *lines, int slot)
{
    const int np = (fs + 1) >> 1, p0 = __ldg(pos + col);
    int k[NP];
#pragma unroll
    for (int j = 0; j < NP; j++) k[j] = j < np ? __ldg(coef2 + (long long)col * np + j) : 0;
    const uint8_t *base = plane + p0;
    for (int r = ra; r <= rb; r++) {
        const uint8_t *s = base + (long long)r * sstride;
        const unsigned sh = (unsigned)(reinterpret_cast<uintptr_t>(s) & 3);
        const unsigned *w = reinterpret_cast<const unsigned *>(s - sh);
        const int need = (int)sh + fs;
        unsigned prev = __ldg(w);
        int acc = 0;
#pragma unroll
        for (int q = 0; q < (NP + 1) / 2; q++) {
            if (q * 4 < fs) {
                const unsigned next = ((q + 1) * 4 < need) ? __ldg(w + q + 1) : 0u;
                const unsigned win = __funnelshift_r(prev, next, sh * 8);
                prev = next;
                acc = dp2a_lo_su(k[2 * q], win, acc);
                if (2 * q + 1 < NP) acc = dp2a_hi_su(k[2 * q + 1], win, acc);
            }
        }
        lines[(r - ra) * PITCH + slot] = (int16_t)min(acc >> 7, 32767);
    }
}

// one 8-bit plane -> one 8-bit plane (yuv2planeX_8_c / yuv2plane1_8_c with the flat dither of SWS_BITEXACT, output.c:468-493)
template <int NP>
__global__ void __launch_bounds__(FT_W)
sws_fused_plane_kernel(const uint8_t *src, long long sstride, long long sfs, int srcH, uint8_t *dst, long long ds, long long dfs,
                       int dstW, int dstH, const int32_t *hcoef2, const int32_t *hpos, int hfs, const int16_t *vcoef,
                       const int32_t *vpos, int vfs, int TR)
{
    extern __shared__ __align__(16) int16_t fused_lines[];
    const int tid = threadIdx.x, x0 = blockIdx.x * FT_W, dy0 = blockIdx.y * TR, dy1 = min(dy0 + TR, dstH) - 1;
    const long long f = blockIdx.z;
    const int ra = min(max(max(1 - vfs, __ldg(vpos + dy0)), 0), srcH - 1);
    const int rb = min(max(max(1 - vfs, __ldg(vpos + dy1)) + vfs - 1, 0), srcH - 1);
    if (x0 + tid < dstW) fused_hstage<NP, FT_W>(src + f * sfs, sstride, hcoef2, hpos, hfs, x0 + tid, ra, rb, fused_lines, tid);
    __syncthreads();
    const int nrows = dy1 - dy0 + 1;
    for (int it = tid; it < nrows * (FT_W / 8); it += FT_W) {
        const int row = it / (FT_W / 8), g = it - row * (FT_W / 8), x = x0 + g * 8;
        if (x >= dstW) continue;
        const int dy = dy0 + row;
        const int first = max(1 - vfs, __ldg(vpos + dy));
        int v[8];
        if (vfs == 1) {
            const uint4 q = *reinterpret_cast<const uint4 *>(fused_lines + (min(max(first, 0), srcH - 1) - ra) * FT_W + g * 8);
            const unsigned ww[4] = { q.x, q.y, q.z, q.w };
#pragma unroll
            for (int j = 0; j < 4; j++) { v[2 * j] = ((int)(short)(ww[j] & 0xffff) + 64) >> 7; v[2 * j + 1] = (((int)ww[j] >> 16) + 64) >> 7; }
        } else {
            unsigned a[8];
#pragma unroll
            for (int j = 0; j < 8; j++) a[j] = 64u << 12;
            const int16_t *k = vcoef + (long long)dy * vfs;
            for (int t = 0; t < vfs; t++) {
                const uint4 q = *reinterpret_cast<const uint4 *>(fused_lines + (min(max(first + t, 0), srcH - 1) - ra) * FT_W + g * 8);
                const unsigned ww[4] = { q.x, q.y, q.z, q.w };
                const int c = (int)__ldg(k + t);
#pragma unroll
                for (int j = 0; j < 4; j++) { a[2 * j] += (unsigned)((int)(short)(ww[j] & 0xffff) * c); a[2 * j + 1] += (unsigned)(((int)ww[j] >> 16) * c); }
            }
#pragma unroll
            for (int j = 0; j < 8; j++) v[j] = (int)a[j] >> 19;
        }
        unsigned o[2];
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const unsigned lo = __vimin_s16x2_relu(__byte_perm((unsigned)v[4 * h], (unsigned)v[4 * h + 1], 0x5410), 0x00ff00ffu);
            const unsigned hi = __vimin_s16x2_relu(__byte_perm((unsigned)v[4 * h + 2], (unsigned)v[4 * h + 3], 0x5410), 0x00ff00ffu);
            o[h] = __byte_perm(lo, hi, 0x6420);
        }
        *reinterpret_cast<uint2 *>(dst + f * dfs + (long long)dy * ds + x) = make_uint2(o[0], o[1]);
    }
}

// yuv420p -> packed RGB through the `_X` writer (yuv2rgb_X_c_template, output.c:1789-1840): luma tile FT_W x TR, chroma FT_W/2 columns
// of both planes; smem = luma lines (pitch FT_W), then U lines, then V lines (pitch FT_W/2); rowsL, rowsC: the largest tile's need
template <int KIND, int NP>
__global__ void __launch_bounds__(FT_W)
sws_fused_rgb_kernel(SwsFrameArgs a, SwsDevTables t, SwsColorConst c, int TR, int rowsL, int rowsC)
{
    constexpr int PW = OutWords<KIND>::per_pair, BPP = OutWords<KIND>::bpp, CW = FT_W / 2;
    extern __shared__ __align__(16) int16_t fused_lines[];
    int16_t *lumL = fused_lines, *chrU = lumL + rowsL * FT_W, *chrV = chrU + rowsC * CW;
    const int tid = threadIdx.x, x0 = blockIdx.x * FT_W, dy0 = blockIdx.y * TR, dy1 = min(dy0 + TR, a.dstH) - 1;
    const long long f = blockIdx.z;
    const int lfs = t.vLumSize, cfs = t.vChrSize;
    const int la = min(max(max(1 - lfs, __ldg(t.vLumPos + dy0)), 0), a.srcH - 1);
    const int lb = min(max(max(1 - lfs, __ldg(t.vLumPos + dy1)) + lfs - 1, 0), a.srcH - 1);
    const int ca = min(max(max(1 - cfs, __ldg(t.vChrPos + dy0)), 0), a.chrSrcH - 1);
    const int cb_ = min(max(max(1 - cfs, __ldg(t.vChrPos + dy1)) + cfs - 1, 0), a.chrSrcH - 1);
    if (x0 + tid < a.dstW) fused_hstage<NP, FT_W>(a.y + f * a.yfs, a.ys, t.hLum2, t.hLumPos, t.hLumSize, x0 + tid, la, lb, lumL, tid);
    {
        const int cc = tid & (CW - 1), ccol = x0 / 2 + cc;
        if (ccol < a.chrDstW) {
            if (tid < CW) fused_hstage<NP, CW>(a.u + f * a.ufs, a.us, t.hChr2, t.hChrPos, t.hChrSize, ccol, ca, cb_, chrU, cc);
            else          fused_hstage<NP, CW>(a.v + f * a.vfs, a.vs, t.hChr2, t.hChrPos, t.hChrSize, ccol, ca, cb_, chrV, cc);
        }
    }
    __syncthreads();
    const int nrows = dy1 - dy0 + 1;
    for (int it = tid; it < nrows * (FT_W / 8); it += FT_W) {
        const int row = it / (FT_W / 8), g = it - row * (FT_W / 8), x = x0 + g * 8;
        if (x >= a.dstW) continue;
        const int dy = dy0 + row;
        const int16_t *lf = t.vLum + (long long)dy * lfs, *cf = t.vChr + (long long)dy * cfs;
        const int firstLum = max(1 - lfs, __ldg(t.vLumPos + dy));
        const int firstChr = max(1 - cfs, __ldg(t.vChrPos + dy));
        unsigned sY[8], sU[4], sV[4];
#pragma unroll
        for (int i = 0; i < 8; i++) sY[i] = 1u << 18;
#pragma unroll
        for (int i = 0; i < 4; i++) sU[i] = sV[i] = 1u << 18;
        for (int j = 0; j < lfs; j++) {
            const int line = min(max(firstLum + j, 0), a.srcH - 1) - la;
            const uint4 q = *reinterpret_cast<const uint4 *>(lumL + line * FT_W + g * 8);
            const unsigned k = (unsigned)(int)__ldg(lf + j);
            const unsigned w[4] = { q.x, q.y, q.z, q.w };
#pragma unroll
            for (int i = 0; i < 4; i++) { sY[2 * i] += (unsigned)(int)(short)(w[i] & 0xffff) * k; sY[2 * i + 1] += (unsigned)((int)w[i] >> 16) * k; }
        }
        for (int j = 0; j < cfs; j++) {
            const int line = min(max(firstChr + j, 0), a.chrSrcH - 1) - ca;
            const uint2 qu = *reinterpret_cast<const uint2 *>(chrU + line * CW + g * 4);
            const uint2 qv = *reinterpret_cast<const uint2 *>(chrV + line * CW + g * 4);
            const unsigned k = (unsigned)(int)__ldg(cf + j);
            sU[0] += (unsigned)(int)(short)(qu.x & 0xffff) * k; sU[1] += (unsigned)((int)qu.x >> 16) * k;
            sU[2] += (unsigned)(int)(short)(qu.y & 0xffff) * k; sU[3] += (unsigned)((int)qu.y >> 16) * k;
            sV[0] += (unsigned)(int)(short)(qv.x & 0xffff) * k; sV[1] += (unsigned)((int)qv.x >> 16) * k;
            sV[2] += (unsigned)(int)(short)(qv.y & 0xffff) * k; sV[3] += (unsigned)((int)qv.y >> 16) * k;
        }
        unsigned m[4 * PW];
#pragma unroll
        for (int i = 0; i < 4; i++) {
            const ChromaBase cb = chroma_base(c, (int)sU[i] >> 19, (int)sV[i] >> 19);
            pair_out<KIND>(c.cy, cb, (int)sY[2 * i] >> 19, (int)sY[2 * i + 1] >> 19, m + PW * i);
        }
        uint8_t *d = a.dst + f * a.dfs + (long long)dy * a.ds + (long long)x * BPP;
        if (KIND <= SWS_OUT_BGR24) {
            uint2 *d2 = reinterpret_cast<uint2 *>(d);
#pragma unroll
            for (int k2 = 0; k2 < 3; k2++)
                d2[k2] = make_uint2(__byte_perm(m[4 * k2], m[4 * k2 + 1], 0x6420), __byte_perm(m[4 * k2 + 2], m[4 * k2 + 3], 0x6420));
        } else {
            uint4 *d4 = reinterpret_cast<uint4 *>(d);
            d4[0] = make_uint4(m[0], m[1], m[2], m[3]); d4[1] = make_uint4(m[4], m[5], m[6], m[7]);
        }
    }
}

#include "sws_mma.cuh"

// Host side of the tensor-core horizontal pass: a filter bank regrouped into the B operands of mma.m16n8k32 (see sws_mma.cuh).
struct SwsMmaHost { std::vector<int32_t> ginfo; std::vector<uint32_t> bfrag; int ngroups = 0; };
static void sws_mma_build(const SwsFilterBank &b, SwsMmaHost &o)
{
    const int ng = (b.n + 7) / 8;
    o.ngroups = ng;
    o.ginfo.assign((size_t)(ng + 1) * 2, 0);
    o.bfrag.clear();
    int chunk = 0;
    for (int G = 0; G < ng; G++) {
        int lo = 0x7fffffff, hi = 0;
        for (int i = 8 * G; i < std::min(8 * G + 8, b.n); i++) { lo = std::min(lo, (int)b.pos[i]); hi = std::max(hi, (int)b.pos[i] + b.size); }
        const int kstart = lo & ~3, nch = (hi - kstart + 31) / 32;
        o.ginfo[2 * G] = kstart;
        o.ginfo[2 * G + 1] = chunk;
        o.bfrag.resize((size_t)(chunk + nch) * 128, 0);
        for (int c = 0; c < nch; c++)
            for (int lane = 0; lane < 32; lane++) {
                const int g = lane >> 2, t = lane & 3, i = 8 * G + g;      // B fragment: column n = lane / 4, rows k = 4 * (lane % 4) .. + 3 (b0) and 16 + the same (b1)
                uint32_t w[4] = { 0, 0, 0, 0 };
                if (i < b.n)
                    for (int half = 0; half < 2; half++)
                        for (int bb = 0; bb < 4; bb++) {
                            const int k = 32 * c + 16 * half + 4 * t + bb, j = kstart + k - b.pos[i];
                            if (j < 0 || j >= b.size) continue;
                            const int cf = b.coef[(size_t)i * b.size + j];
                            w[half] |= (uint32_t)((cf >> 8) & 0xff) << (8 * bb);         // signed high byte
                            w[2 + half] |= (uint32_t)(cf & 0xff) << (8 * bb);            // unsigned low byte
                        }
                memcpy(&o.bfrag[((size_t)(chunk + c) * 32 + lane) * 4], w, 16);
            }
        chunk += nch;
    }
    o.ginfo[2 * ng] = 0;
    o.ginfo[2 * ng + 1] = chunk;
}
// byte pitch of the staged source lines for tiles of `tile_groups` groups: the widest tile's span in 16-byte segments, made odd
static int sws_mma_pitch(const SwsMmaHost &m, int tile_groups)
{
    int mx = 1;
    for (int G0 = 0; G0 < m.ngroups; G0 += tile_groups) {
        int s = 0x7fffffff, e = 0;
        for (int G = G0; G < std::min(G0 + tile_groups, m.ngroups); G++) {
            s = std::min(s, (int)m.ginfo[2 * G]);
            e = std::max(e, (int)m.ginfo[2 * G] + 32 * (int)(m.ginfo[2 * G + 3] - m.ginfo[2 * G + 1]));
        }
        mx = std::max(mx, (e - (s & ~15) + 15) >> 4);
    }
    return (mx | 1) * 16;
}

static int upload_mma_tables(B200SwsContext *c)
{
    const SwsPlan &p = c->plan;
    if (c->h_identity || p.fast_bilinear || p.src_rgb || p.hLum.n <= 0 || p.hChr.n <= 0) return 0;
    SwsMmaHost L, C;
    sws_mma_build(p.hLum, L);
    sws_mma_build(p.hChr, C);
    auto al = [](size_t v) { return (v + 255) & ~(size_t)255; };
    const size_t o_lg = 0, o_lb = o_lg + al(L.ginfo.size() * 4), o_cg = o_lb + al(L.bfrag.size() * 4), o_cb = o_cg + al(C.ginfo.size() * 4),
                 total = o_cb + al(C.bfrag.size() * 4);
    std::vector<uint8_t> host(total, 0);
    memcpy(&host[o_lg], L.ginfo.data(), L.ginfo.size() * 4); memcpy(&host[o_lb], L.bfrag.data(), L.bfrag.size() * 4);
    memcpy(&host[o_cg], C.ginfo.data(), C.ginfo.size() * 4); memcpy(&host[o_cb], C.bfrag.data(), C.bfrag.size() * 4);
    B200_CUDA_OK(cudaMalloc(&c->mma_tables, total));
    B200_CUDA_OK(cudaMemcpy(c->mma_tables, host.data(), total, cudaMemcpyHostToDevice));
    const uint8_t *b = (const uint8_t *)c->mma_tables;
    c->mmaL = SwsMmaBank{ (const int2 *)(b + o_lg), (const uint4 *)(b + o_lb), L.ngroups };
    c->mmaC = SwsMmaBank{ (const int2 *)(b + o_cg), (const uint4 *)(b + o_cb), C.ngroups };
    c->mma_pitchL = sws_mma_pitch(L, MT_W / 8);
    c->mma_pitchC = sws_mma_pitch(C, MT_W / 8);
    c->mma_pitchC8 = sws_mma_pitch(C, MT_W / 16);
    return 0;
}

// host-only: the tensor-core operand tables of an arbitrary filter bank (CPU test tier: replayed lane by lane against hScale8To15_c)
B200_API int b200_sws_mma_probe(const int16_t *coef, const int32_t *pos, int n, int size, int32_t *ginfo, int ginfo_cap,
                                uint32_t *bfrag, int bfrag_cap, int *pitch)
{
    if (!coef || !pos || n <= 0 || size <= 0) return B200_EINVAL;
    SwsFilterBank b;
    b.coef.assign(coef, coef + (size_t)n * size);
    b.pos.assign(pos, pos + n);
    b.size = size; b.n = n;
    SwsMmaHost m;
    sws_mma_build(b, m);
    if (ginfo) { if ((int)m.ginfo.size() > ginfo_cap) return B200_EINVAL; memcpy(ginfo, m.ginfo.data(), m.ginfo.size() * 4); }
    if (bfrag) { if ((int)m.bfrag.size() > bfrag_cap) return B200_EINVAL; memcpy(bfrag, m.bfrag.data(), m.bfrag.size() * 4); }
    if (pitch) { pitch[0] = sws_mma_pitch(m, MT_W / 8); pitch[1] = sws_mma_pitch(m, MT_W / 16); }
    return (int)m.bfrag.size();                       // words of B fragments (128 per chunk)
}

// rows of the horizontally scaled plane the vertical taps of output lines [dy0, dy1] reach (the kernels compute the same range)
static int fused_rows_needed(const SwsFilterBank &v, int srcH, int dstH, int TR)
{
    int mx = 0;
    for (int dy0 = 0; dy0 < dstH; dy0 += TR) {
        const int dy1 = std::min(dy0 + TR, dstH) - 1;
        const int ra = std::min(std::max(std::max(1 - v.size, v.pos[dy0]), 0), srcH - 1);
        const int rb = std::min(std::max(std::max(1 - v.size, v.pos[dy1]) + v.size - 1, 0), srcH - 1);
        if (rb < ra) return -1;                      // not monotone: leave it to the two-pass path
        mx = std::max(mx, rb - ra + 1);
        for (int dy = dy0; dy <= dy1; dy++) {         // every line of the tile must stay inside [ra, rb]
            const int fa = std::min(std::max(std::max(1 - v.size, v.pos[dy]), 0), srcH - 1);
            const int fb = std::min(std::max(std::max(1 - v.size, v.pos[dy]) + v.size - 1, 0), srcH - 1);
            if (fa < ra || fb > rb) return -1;
        }
    }
    return mx;
}
static bool aligned16(const void *p, long long stride, long long fstride)
{
    return (((uintptr_t)p) & 15) == 0 && (stride & 15) == 0 && (fstride & 15) == 0;
}
static bool aligned8(const void *p, long long stride, long long fstride)
{
    return (((uintptr_t)p) & 7) == 0 && (stride & 7) == 0 && (fstride & 7) == 0;
}

// nv12 / nv21: split plane 1 of `nframes` frames (chroma rows [row0, row0 + nrows)) into U and V planes and redirect the
// plane pointers.  `scratch` (per-call) or the context's persistent buffer holds them: per frame U then V, pitch nv_pitch().
static size_t nv_pitch(const SwsPlan &p) { return ((size_t)p.chrSrcW + 255) & ~(size_t)255; }
static size_t nv_frame_bytes(const SwsPlan &p) { return 2 * nv_pitch(p) * p.chrSrcH; }
static int nv_split(B200SwsContext *c, cudaStream_t stream, uint8_t *scratch, int nframes, int row0, int nrows,
                    const uint8_t *s3[3], long long st3[3], long long fs3[3])
{
    const SwsPlan &p = c->plan;
    const size_t pitch = nv_pitch(p), fb = nv_frame_bytes(p);
    uint8_t *buf = scratch;
    if (!buf) {
        if (c->nv_bytes < fb * nframes) {
            if (c->nv_buf) { cudaStreamSynchronize(stream); cudaFree(c->nv_buf); c->nv_buf = nullptr; c->nv_bytes = 0; }
            B200_CUDA_OK(cudaMalloc(&c->nv_buf, fb * nframes));
            c->nv_bytes = fb * nframes;
        }
        buf = (uint8_t *)c->nv_buf;
    }
    uint8_t *pu = buf, *pv = buf + pitch * p.chrSrcH;
    if (p.src_nv == 2) { uint8_t *t = pu; pu = pv; pv = t; }               // nv21: first byte of a pair is V
    for (int f0 = 0; f0 < nframes && nrows > 0; f0 += 65535) {
        const int nf = nframes - f0 < 65535 ? nframes - f0 : 65535;
        dim3 block(256), grid(b200_ceil_div(p.chrSrcW, 256), nrows, nf);
        sws_nv_split_kernel<<<grid, block, 0, stream>>>(s3[1] + (long long)f0 * fs3[1], st3[1], fs3[1], pu + (size_t)f0 * fb, pv + (size_t)f0 * fb,
                                                        (long long)pitch, (long long)fb, p.chrSrcW, row0);
        B200_LAUNCHED();
    }
    s3[1] = buf; s3[2] = buf + pitch * p.chrSrcH;                          // [1] = U plane, [2] = V plane
    st3[1] = st3[2] = (long long)pitch;
    fs3[1] = fs3[2] = (long long)fb;
    return 0;
}

template <int KIND>
static void launch_vscale_fast(bool lumid, bool c4, dim3 grid, dim3 block, cudaStream_t stream, const SwsFrameArgs &b,
                               const SwsDevTables &dt, const SwsColorConst &col, int ngroups)
{
    if (lumid && c4)  sws_vscale_rgb24_fast_kernel<true, true, KIND><<<grid, block, 0, stream>>>(b, dt, col, ngroups);
    else if (lumid)   sws_vscale_rgb24_fast_kernel<true, false, KIND><<<grid, block, 0, stream>>>(b, dt, col, ngroups);
    else if (c4)      sws_vscale_rgb24_fast_kernel<false, true, KIND><<<grid, block, 0, stream>>>(b, dt, col, ngroups);
    else              sws_vscale_rgb24_fast_kernel<false, false, KIND><<<grid, block, 0, stream>>>(b, dt, col, ngroups);
}

// horizontal pass of `nlines` lines starting at line0 (filter sizes up to 16 take the register-resident variant)
static void launch_hscale(cudaStream_t stream, const uint8_t *src, long long sstride, long long sfs, int16_t *dst, int dstW, long long dfs,
                          const int32_t *coef2, const int32_t *pos, int fs, int line0, int nlines, int nf)
{
    dim3 block(256);
    if (fs <= 16) {
        dim3 grid(b200_ceil_div(dstW, 256), b200_ceil_div(nlines, HROWS), nf);
        if (fs <= 2)      sws_hscale_rows_kernel<1><<<grid, block, 0, stream>>>(src, sstride, sfs, dst, dstW, dfs, coef2, pos, fs, line0, nlines);
        else if (fs <= 4) sws_hscale_rows_kernel<2><<<grid, block, 0, stream>>>(src, sstride, sfs, dst, dstW, dfs, coef2, pos, fs, line0, nlines);
        else if (fs <= 8) sws_hscale_rows_kernel<4><<<grid, block, 0, stream>>>(src, sstride, sfs, dst, dstW, dfs, coef2, pos, fs, line0, nlines);
        else              sws_hscale_rows_kernel<8><<<grid, block, 0, stream>>>(src, sstride, sfs, dst, dstW, dfs, coef2, pos, fs, line0, nlines);
    } else {
        dim3 grid(b200_ceil_div(dstW, 256), nlines, nf);
        sws_hscale_kernel<<<grid, block, 0, stream>>>(src, sstride, sfs, dst, dstW, dfs, coef2, pos, fs, line0);
    }
}

template <int KIND>
static void launch_vscale_fast_nv_k(int nv, dim3 grid, dim3 block, cudaStream_t stream, const SwsFrameArgs &b, const SwsDevTables &dt,
                                    const SwsColorConst &col, int ngroups)
{
    if (nv == 1) sws_vscale_rgb24_fast_kernel<true, true, KIND, 1><<<grid, block, 0, stream>>>(b, dt, col, ngroups);
    else         sws_vscale_rgb24_fast_kernel<true, true, KIND, 2><<<grid, block, 0, stream>>>(b, dt, col, ngroups);
}
static void launch_vscale_fast_nv(int kind, int nv, dim3 grid, dim3 block, cudaStream_t stream, const SwsFrameArgs &b,
                                  const SwsDevTables &dt, const SwsColorConst &col, int ngroups)
{
    switch (kind) {
    case SWS_OUT_RGB24: launch_vscale_fast_nv_k<SWS_OUT_RGB24>(nv, grid, block, stream, b, dt, col, ngroups); break;
    case SWS_OUT_BGR24: launch_vscale_fast_nv_k<SWS_OUT_BGR24>(nv, grid, block, stream, b, dt, col, ngroups); break;
    case SWS_OUT_RGBA:  launch_vscale_fast_nv_k<SWS_OUT_RGBA>(nv, grid, block, stream, b, dt, col, ngroups); break;
    case SWS_OUT_BGRA:  launch_vscale_fast_nv_k<SWS_OUT_BGRA>(nv, grid, block, stream, b, dt, col, ngroups); break;
    case SWS_OUT_ARGB:  launch_vscale_fast_nv_k<SWS_OUT_ARGB>(nv, grid, block, stream, b, dt, col, ngroups); break;
    default:            launch_vscale_fast_nv_k<SWS_OUT_ABGR>(nv, grid, block, stream, b, dt, col, ngroups); break;
    }
}

// enqueue the conversion of nframes frames on `stream`
// Which lines a launch covers.  Whole frames: everything.  Slice calls: the output lines that became computable and the
// source lines that were just uploaded (only those need the horizontal pass).
struct SwsRows { int dy0, ndy, ly0, nly, cy0, ncy; };


// the line-pair kernel over output lines [b.y0, b.y0 + 2 * npairs), b.y0 odd, for ngroups 16-px groups of each line
template <int NV>
static void launch_vscale_pair(int kind, int ngroups, int npairs, int nf, cudaStream_t stream, const SwsFrameArgs &b, const SwsDevTables &dt,
                               const SwsColorConst &col)
{
    const dim3 block(PAIR_THREADS);
    // x: one thread per 16-byte chunk of a line (24-bit rows: three per 16-px group) or per 16-px group (32-bit rows)
    auto grid = [&](int band) { return dim3(b200_ceil_div((kind <= SWS_OUT_BGR24 ? 3 : 1) * ngroups, PAIR_THREADS), b200_ceil_div(npairs, band), nf); };
    switch (kind) {
    case SWS_OUT_RGB24: sws_vscale_rgb24_pair_kernel<SWS_OUT_RGB24, NV><<<grid(PairShape<SWS_OUT_RGB24>::band), block, 0, stream>>>(b, dt, col, ngroups, npairs); break;
    case SWS_OUT_BGR24: sws_vscale_rgb24_pair_kernel<SWS_OUT_BGR24, NV><<<grid(PairShape<SWS_OUT_BGR24>::band), block, 0, stream>>>(b, dt, col, ngroups, npairs); break;
    case SWS_OUT_RGBA:  sws_vscale_rgb24_pair_kernel<SWS_OUT_RGBA, NV><<<grid(PairShape<SWS_OUT_RGBA>::band), block, 0, stream>>>(b, dt, col, ngroups, npairs); break;
    case SWS_OUT_BGRA:  sws_vscale_rgb24_pair_kernel<SWS_OUT_BGRA, NV><<<grid(PairShape<SWS_OUT_BGRA>::band), block, 0, stream>>>(b, dt, col, ngroups, npairs); break;
    case SWS_OUT_ARGB:  sws_vscale_rgb24_pair_kernel<SWS_OUT_ARGB, NV><<<grid(PairShape<SWS_OUT_ARGB>::band), block, 0, stream>>>(b, dt, col, ngroups, npairs); break;
    default:            sws_vscale_rgb24_pair_kernel<SWS_OUT_ABGR, NV><<<grid(PairShape<SWS_OUT_ABGR>::band), block, 0, stream>>>(b, dt, col, ngroups, npairs); break;
    }
}

static int launch_batch(B200SwsContext *c, cudaStream_t stream, const uint8_t *const src_in[3], const long long sstr_in[3],
                        const long long sfs_in[3], uint8_t *dst, long long ds, long long dfs, int nframes,
                        const SwsRows *rows = nullptr, uint8_t *nv_scratch = nullptr)
{
    const SwsPlan &p = c->plan;
    if (nframes <= 0) return 0;
    const SwsRows full = { 0, p.dstH, 0, p.srcH, 0, p.chrSrcH };
    const SwsRows R = rows ? *rows : full;
    if (R.ndy <= 0 && R.nly <= 0 && R.ncy <= 0) return 0;
    const uint8_t *src[3] = { src_in[0], src_in[1], src_in[2] };
    long long sstr[3] = { sstr_in[0], sstr_in[1], sstr_in[2] }, sfs[3] = { sfs_in[0], sfs_in[1], sfs_in[2] };
    // nv12 / nv21 straight into the vector kernel (no split pass) when the whole line is covered by 16-pixel groups
    auto fits32_ = [](long long stride, long long lines) { return (stride < 0 ? -stride : stride) * (lines + 1) < (1LL << 31); };
    const bool nv_direct = p.src_nv && !p.unscaled_lut && c->h_identity && c->fast_x && c->lum_identity && p.vChr.size == 4 &&
                           p.dstW % 16 == 0 && R.ndy > 0 && aligned16(src[0], sstr[0], sfs[0]) && aligned16(src[1], sstr[1], sfs[1]) &&
                           aligned16(dst, ds, dfs) && fits32_(sstr[0], p.srcH) && fits32_(sstr[1], p.chrSrcH) && fits32_(ds, p.dstH);
    if (p.src_nv && !nv_direct) {
        int ret = nv_split(c, stream, nv_scratch, nframes, R.cy0, R.ncy, src, sstr, sfs);
        if (ret < 0) return ret;
    }
    SwsFrameArgs a{};
    a.y = src[0]; a.u = src[1]; a.v = src[2];
    a.ys = sstr[0]; a.us = sstr[1]; a.vs = sstr[2];
    a.yfs = sfs[0]; a.ufs = sfs[1]; a.vfs = sfs[2];
    a.dst = dst; a.ds = ds; a.dfs = dfs;
    a.srcH = p.srcH; a.chrSrcH = p.chrSrcH; a.dstW = p.dstW; a.dstH = p.dstH; a.chrDstW = p.chrDstW;
    a.y0 = R.dy0;
    a.bpp = p.out.bpp; a.ro = p.out.ro; a.go = p.out.go; a.bo = p.out.bo; a.ao = p.out.ao;
    const int vecSrc = aligned16(src[0], sstr[0], sfs[0]) && aligned8(src[1], sstr[1], sfs[1]) && aligned8(src[2], sstr[2], sfs[2]);
    const int vecOK = vecSrc && aligned16(dst, ds, dfs);
    for (int f0 = 0; f0 < nframes; f0 += 65535) {            // gridDim.z limit
        const int nf = nframes - f0 < 65535 ? nframes - f0 : 65535;
        SwsFrameArgs b = a;
        b.y += (long long)f0 * a.yfs; b.u += (long long)f0 * a.ufs; b.v += (long long)f0 * a.vfs; b.dst += (long long)f0 * a.dfs;
        if (p.unscaled_lut) {
            const int wpix = ((p.dstW >> 3) << 3) + (p.dstW & 4) + (p.dstW & 2);
            if (wpix == 0 || R.ndy < 2) continue;
            const int ngroups = vecOK ? wpix / 16 : 0;
            if (ngroups) {
                dim3 block(128), grid(b200_ceil_div(ngroups, 128), R.ndy / 2, nf);
                switch (p.out.kind) {
                case SWS_OUT_RGB24: sws_unscaled_kernel<SWS_OUT_RGB24><<<grid, block, 0, stream>>>(b, p.color, ngroups); break;
                case SWS_OUT_BGR24: sws_unscaled_kernel<SWS_OUT_BGR24><<<grid, block, 0, stream>>>(b, p.color, ngroups); break;
                case SWS_OUT_RGBA:  sws_unscaled_kernel<SWS_OUT_RGBA><<<grid, block, 0, stream>>>(b, p.color, ngroups); break;
                case SWS_OUT_BGRA:  sws_unscaled_kernel<SWS_OUT_BGRA><<<grid, block, 0, stream>>>(b, p.color, ngroups); break;
                case SWS_OUT_ARGB:  sws_unscaled_kernel<SWS_OUT_ARGB><<<grid, block, 0, stream>>>(b, p.color, ngroups); break;
                default:            sws_unscaled_kernel<SWS_OUT_ABGR><<<grid, block, 0, stream>>>(b, p.color, ngroups); break;
                }
                B200_LAUNCHED();
            }
            const int p0 = ngroups * 8, p1 = wpix / 2;
            if (p1 > p0) {
                dim3 block(128), grid(b200_ceil_div(p1 - p0, 128), R.ndy / 2, nf);
                sws_unscaled_slow_kernel<<<grid, block, 0, stream>>>(b, p.color, p0, p1);
                B200_LAUNCHED();
            }
        } else if (c->h_identity) {
            auto fits32 = [](long long stride, long long lines) { return (stride < 0 ? -stride : stride) * (lines + 1) < (1LL << 31); };
            const bool off32 = fits32(b.ys, p.srcH) && fits32(b.us, p.chrSrcH) && fits32(b.vs, p.chrSrcH) && fits32(b.ds, p.dstH);
            const int ngroups = (vecOK && c->fast_x && off32 && R.ndy > 0) ? p.dstW / 16 : 0;
            // lines [R.dy0, R.dy0 + R.ndy) = at most one leading line, pairs (odd, even) for the two-line kernel, at most one trailing line
            const bool pairs_on = c->pair_ok && R.ndy >= 3 && (nv_direct || ngroups);
            const int pfirst = pairs_on ? (R.dy0 | 1) : R.dy0, npairs = pairs_on ? (R.dy0 + R.ndy - pfirst) / 2 : 0;
            if (npairs > 0) {
                const int ng = nv_direct ? p.dstW / 16 : ngroups;
                SwsFrameArgs bp = b;
                bp.y0 = pfirst;
                if (!nv_direct) launch_vscale_pair<0>(p.out.kind, ng, npairs, nf, stream, bp, c->dt, p.color);
                else if (p.src_nv == 1) launch_vscale_pair<1>(p.out.kind, ng, npairs, nf, stream, bp, c->dt, p.color);
                else launch_vscale_pair<2>(p.out.kind, ng, npairs, nf, stream, bp, c->dt, p.color);
                B200_LAUNCHED();
                c->last_path |= 8;
            }
            // the one-line kernel: everything when no pairs were formed, else the lines left over at either end
            const int seg0[2] = { R.dy0, pfirst + 2 * npairs }, segn[2] = { npairs > 0 ? pfirst - R.dy0 : R.ndy, npairs > 0 ? R.dy0 + R.ndy - (pfirst + 2 * npairs) : 0 };
            for (int sg = 0; sg < 2; sg++) {
            if (segn[sg] <= 0) continue;
            SwsFrameArgs b1 = b;
            b1.y0 = seg0[sg];
            const SwsFrameArgs &b = b1;
            if (nv_direct) {
                dim3 block(128), grid(b200_ceil_div(p.dstW / 16, 128), segn[sg], nf);
                launch_vscale_fast_nv(p.out.kind, p.src_nv, grid, block, stream, b, c->dt, p.color, p.dstW / 16);
                B200_LAUNCHED();
                continue;
            }
            if (ngroups) {
                dim3 block(128), grid(b200_ceil_div(ngroups, 128), segn[sg], nf);
                const bool c4 = p.vChr.size == 4;
                switch (p.out.kind) {
                case SWS_OUT_RGB24: launch_vscale_fast<SWS_OUT_RGB24>(c->lum_identity, c4, grid, block, stream, b, c->dt, p.color, ngroups); break;
                case SWS_OUT_BGR24: launch_vscale_fast<SWS_OUT_BGR24>(c->lum_identity, c4, grid, block, stream, b, c->dt, p.color, ngroups); break;
                case SWS_OUT_RGBA:  launch_vscale_fast<SWS_OUT_RGBA>(c->lum_identity, c4, grid, block, stream, b, c->dt, p.color, ngroups); break;
                case SWS_OUT_BGRA:  launch_vscale_fast<SWS_OUT_BGRA>(c->lum_identity, c4, grid, block, stream, b, c->dt, p.color, ngroups); break;
                case SWS_OUT_ARGB:  launch_vscale_fast<SWS_OUT_ARGB>(c->lum_identity, c4, grid, block, stream, b, c->dt, p.color, ngroups); break;
                default:            launch_vscale_fast<SWS_OUT_ABGR>(c->lum_identity, c4, grid, block, stream, b, c->dt, p.color, ngroups); break;
                }
                B200_LAUNCHED();
            }
            }
            if (nv_direct) continue;
            const int p0 = ngroups * 8, p1 = (p.dstW + 1) / 2;
            if (p1 > p0 && R.ndy > 0) {
                dim3 block(128), grid(b200_ceil_div(p1 - p0, 128), R.ndy, nf);
                sws_vscale_rgb24_slow_kernel<true><<<grid, block, 0, stream>>>(b, c->dt, p.color, p0, p1);
                B200_LAUNCHED();
            }
        } else {
            // scaled path.  Whole frames through the `_X` writer: one fused kernel (no int16 planes in HBM)
            if (!rows && c->mma_tables && p.chrDstHSub && c->all_x && p.dstW % 16 == 0 && p.chrDstW * 2 == p.dstW &&
                aligned16(dst, ds, dfs) && aligned16(b.y, b.ys, b.yfs) && aligned16(b.u, b.us, b.ufs) && aligned16(b.v, b.vs, b.vfs)) {
                auto need = [&](int rl_, int rc_) {
                    const size_t RL = (size_t)((rl_ + 15) & ~15), RC = (size_t)((rc_ + 15) & ~15);
                    return MT_HDR + RL * (c->mma_pitchL + MT_TPB) + 2 * RC * (c->mma_pitchC8 + MT_CPB);
                };
                // output lines per tile: the horizontal pass works in blocks of 16 staged lines, so pick the height whose windows waste the
                // fewest of them (e.g. 29 lines at 2:1 with 8 taps = exactly 64 source lines) among those that leave room for 4 CTAs per SM
                // (measured, 4K -> 1080p rgb24: 16 lines 0.197 of the HBM roofline, 29 lines 0.179 — three planes' tiles leave 2 CTAs per SM —
                // 13 lines 0.172: 16 is tried first, the search below only runs when 16 does not fit)
                int TR = 16, rl = -1, rc = -1;
                rl = fused_rows_needed(p.vLum, p.srcH, p.dstH, TR); rc = fused_rows_needed(p.vChr, p.chrSrcH, p.dstH, TR);
                if (rl <= 0 || rc <= 0 || need(rl, rc) > 80 * 1024) {
                    TR = 0; rl = rc = -1;
                    double best = 1e30;
                    for (int cand = 32; cand >= 8; cand--) {
                        const int a_ = fused_rows_needed(p.vLum, p.srcH, p.dstH, cand), b_ = fused_rows_needed(p.vChr, p.chrSrcH, p.dstH, cand);
                        if (a_ <= 0 || b_ <= 0) continue;
                        const size_t sm_ = need(a_, b_);
                        if (sm_ > 112 * 1024) continue;
                        const double cost = (double)(((a_ + 15) >> 4) + ((b_ + 15) >> 4)) / cand * (1.0 + (sm_ > 56 * 1024 ? 0.15 : 0.0) + (sm_ > 75 * 1024 ? 0.15 : 0.0));
                        if (cost < best - 1e-9) { best = cost; TR = cand; rl = a_; rc = b_; }
                    }
                }
                const size_t smem = rl > 0 && rc > 0 ? need(rl, rc) : 0;
                if (smem && smem <= 112 * 1024) {
                    dim3 gf(b200_ceil_div(p.dstW, MT_W), b200_ceil_div(p.dstH, TR), nf);
                    const int RL = (rl + 15) & ~15, RC = (rc + 15) & ~15;
#define B200_MMA_RGB(K)                                                                                                           \
                    do {                                                                                                          \
                        if (smem > 48 * 1024) B200_CUDA_OK(cudaFuncSetAttribute(sws_mma_rgb_kernel<K>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
                        sws_mma_rgb_kernel<K><<<gf, MT_THREADS, smem, stream>>>(b, c->dt, p.color, c->mmaL, c->mmaC, p.srcW, p.chrSrcW, TR, RL, RC,   \
                                                                                c->mma_pitchL, c->mma_pitchC8);                  \
                    } while (0)
                    switch (p.out.kind) {
                    case SWS_OUT_RGB24: B200_MMA_RGB(SWS_OUT_RGB24); break;
                    case SWS_OUT_BGR24: B200_MMA_RGB(SWS_OUT_BGR24); break;
                    case SWS_OUT_RGBA:  B200_MMA_RGB(SWS_OUT_RGBA); break;
                    case SWS_OUT_BGRA:  B200_MMA_RGB(SWS_OUT_BGRA); break;
                    case SWS_OUT_ARGB:  B200_MMA_RGB(SWS_OUT_ARGB); break;
                    default:            B200_MMA_RGB(SWS_OUT_ABGR); break;
                    }
#undef B200_MMA_RGB
                    B200_LAUNCHED();
                    c->last_path |= 4;
                    continue;
                }
            }
            if (!rows && !p.fast_bilinear && p.chrDstHSub && c->all_x && p.dstW % 8 == 0 && aligned16(dst, ds, dfs) &&
                p.hLum.size <= 16 && p.hChr.size <= 16) {
                int TR = 32;
                int rl = fused_rows_needed(p.vLum, p.srcH, p.dstH, TR), rc = fused_rows_needed(p.vChr, p.chrSrcH, p.dstH, TR);
                if (rl > 0 && rc > 0 && (size_t)(rl * FT_W + rc * FT_W) * 2 > 64 * 1024) {
                    TR = 16;
                    rl = fused_rows_needed(p.vLum, p.srcH, p.dstH, TR); rc = fused_rows_needed(p.vChr, p.chrSrcH, p.dstH, TR);
                }
                const size_t smem = rl > 0 && rc > 0 ? (size_t)(rl * FT_W + rc * FT_W) * 2 : 0;
                if (smem && smem <= 64 * 1024) {
                    dim3 gf(b200_ceil_div(p.dstW, FT_W), b200_ceil_div(p.dstH, TR), nf);
                    const bool np4 = p.hLum.size <= 8 && p.hChr.size <= 8;
#define B200_FUSED_RGB(K)                                                                                                         \
                    do {                                                                                                          \
                        if (np4) {                                                                                                \
                            if (smem > 48 * 1024) B200_CUDA_OK(cudaFuncSetAttribute(sws_fused_rgb_kernel<K, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
                            sws_fused_rgb_kernel<K, 4><<<gf, FT_W, smem, stream>>>(b, c->dt, p.color, TR, rl, rc);                   \
                        } else {                                                                                                  \
                            if (smem > 48 * 1024) B200_CUDA_OK(cudaFuncSetAttribute(sws_fused_rgb_kernel<K, 8>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
                            sws_fused_rgb_kernel<K, 8><<<gf, FT_W, smem, stream>>>(b, c->dt, p.color, TR, rl, rc);                   \
                        }                                                                                                         \
                    } while (0)
                    switch (p.out.kind) {
                    case SWS_OUT_RGB24: B200_FUSED_RGB(SWS_OUT_RGB24); break;
                    case SWS_OUT_BGR24: B200_FUSED_RGB(SWS_OUT_BGR24); break;
                    case SWS_OUT_RGBA:  B200_FUSED_RGB(SWS_OUT_RGBA); break;
                    case SWS_OUT_BGRA:  B200_FUSED_RGB(SWS_OUT_BGRA); break;
                    case SWS_OUT_ARGB:  B200_FUSED_RGB(SWS_OUT_ARGB); break;
                    default:            B200_FUSED_RGB(SWS_OUT_ABGR); break;
                    }
#undef B200_FUSED_RGB
                    B200_LAUNCHED();
                    c->last_path |= 2;
                    continue;
                }
            }
            // two passes: horizontal pass into int16 line planes, then the vertical pass
            c->last_path |= 1;
            const size_t lumPlane = (size_t)p.srcH * p.dstW * 2, chrPlane = (size_t)p.chrSrcH * p.chrDstW * 2;
            const size_t perFrame = ((lumPlane + 2 * chrPlane) + 255) & ~(size_t)255;
            const size_t need = perFrame * nf;
            if (c->mid_bytes < need) {
                if (c->mid) { cudaStreamSynchronize(stream); cudaFree(c->mid); c->mid = nullptr; c->mid_bytes = 0; }
                B200_CUDA_OK(cudaMalloc(&c->mid, need));
                c->mid_bytes = need;
            }
            int16_t *mY = (int16_t *)c->mid;
            int16_t *mU = (int16_t *)((uint8_t *)c->mid + lumPlane);
            int16_t *mV = (int16_t *)((uint8_t *)c->mid + lumPlane + chrPlane);
            const long long mfs = (long long)(perFrame / 2);
            dim3 block(256);
            if (R.nly > 0) {
                dim3 grid(b200_ceil_div(p.dstW, 256), R.nly, nf);
                if (p.fast_bilinear) sws_hscale_fast_kernel<false><<<grid, block, 0, stream>>>(b.y, b.ys, b.yfs, mY, p.dstW, mfs, p.srcW, p.lumXInc, R.ly0);
                else launch_hscale(stream, b.y, b.ys, b.yfs, mY, p.dstW, mfs, c->dt.hLum2, c->dt.hLumPos, c->dt.hLumSize, R.ly0, R.nly, nf);
                B200_LAUNCHED();
            }
            if (R.ncy > 0) {
                dim3 gridc(b200_ceil_div(p.chrDstW, 256), R.ncy, nf);
                if (p.fast_bilinear) sws_hscale_fast_kernel<true><<<gridc, block, 0, stream>>>(b.u, b.us, b.ufs, mU, p.chrDstW, mfs, p.chrSrcW, p.chrXInc, R.cy0);
                else launch_hscale(stream, b.u, b.us, b.ufs, mU, p.chrDstW, mfs, c->dt.hChr2, c->dt.hChrPos, c->dt.hChrSize, R.cy0, R.ncy, nf);
                B200_LAUNCHED();
                if (p.fast_bilinear) sws_hscale_fast_kernel<true><<<gridc, block, 0, stream>>>(b.v, b.vs, b.vfs, mV, p.chrDstW, mfs, p.chrSrcW, p.chrXInc, R.cy0);
                else launch_hscale(stream, b.v, b.vs, b.vfs, mV, p.chrDstW, mfs, c->dt.hChr2, c->dt.hChrPos, c->dt.hChrSize, R.cy0, R.ncy, nf);
                B200_LAUNCHED();
            }
            if (R.ndy <= 0) continue;
            SwsFrameArgs m = b;
            m.y = (const uint8_t *)mY; m.u = (const uint8_t *)mU; m.v = (const uint8_t *)mV;
            m.ys = (long long)p.dstW * 2; m.us = m.vs = (long long)p.chrDstW * 2;
            m.yfs = m.ufs = m.vfs = (long long)perFrame;
            if (p.chrDstHSub && c->all_x && p.dstW % 8 == 0 && aligned16(dst, ds, dfs) && lumPlane % 16 == 0 && chrPlane % 8 == 0) {
                const int ng = p.dstW / 8;
                dim3 block2(128), grid(b200_ceil_div(ng, 128), R.ndy, nf);
                switch (p.out.kind) {
                case SWS_OUT_RGB24: sws_vscale_rgb24_x8_kernel<SWS_OUT_RGB24><<<grid, block2, 0, stream>>>(m, c->dt, p.color, ng); break;
                case SWS_OUT_BGR24: sws_vscale_rgb24_x8_kernel<SWS_OUT_BGR24><<<grid, block2, 0, stream>>>(m, c->dt, p.color, ng); break;
                case SWS_OUT_RGBA:  sws_vscale_rgb24_x8_kernel<SWS_OUT_RGBA><<<grid, block2, 0, stream>>>(m, c->dt, p.color, ng); break;
                case SWS_OUT_BGRA:  sws_vscale_rgb24_x8_kernel<SWS_OUT_BGRA><<<grid, block2, 0, stream>>>(m, c->dt, p.color, ng); break;
                case SWS_OUT_ARGB:  sws_vscale_rgb24_x8_kernel<SWS_OUT_ARGB><<<grid, block2, 0, stream>>>(m, c->dt, p.color, ng); break;
                default:            sws_vscale_rgb24_x8_kernel<SWS_OUT_ABGR><<<grid, block2, 0, stream>>>(m, c->dt, p.color, ng); break;
                }
            } else if (p.chrDstHSub) {
                const int np = (p.dstW + 1) / 2;
                dim3 block2(128), grid(b200_ceil_div(np, 128), R.ndy, nf);
                sws_vscale_rgb24_slow_kernel<false><<<grid, block2, 0, stream>>>(m, c->dt, p.color, 0, np);
            } else {
                dim3 block2(256), grid(b200_ceil_div(p.dstW, 256), R.ndy, nf);
                sws_vscale_rgb24_full_kernel<<<grid, block2, 0, stream>>>(m, c->dt, p.color);
            }
            B200_LAUNCHED();
        }
    }
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

// packed RGB source -> packed RGB destination (always through the scaler: the same-size case is the reference's rgb2rgb shuffle and
// is refused at context creation): input readers + 16-bit horizontal pass into the int16 line planes, then the same vertical
// writers as the yuv-source scaled path (the stage after the horizontal pass in launch_batch)
// Same-size packed RGB -> packed RGB (rgbToRgbWrapper's byte shuffles / packedCopyWrapper, swscale_unscaled.c:2001-2060,2138-2170): every
// destination byte is one source byte of the same pixel or the constant 255 (alpha of a 24-bit source).  A thread takes four pixels as
// whole 32-bit words when both lines are 4-byte aligned, else (and for the last pixels of a line) one pixel byte by byte.
template <int SB, int DB>
__global__ void __launch_bounds__(128)
sws_rgb_shuffle_kernel(const uint8_t *__restrict__ src, long long sstride, long long sfs, uint8_t *__restrict__ dst, long long dstride, long long dfs,
                       int W, unsigned sel, int vec)
{
    const int q = blockIdx.x * blockDim.x + threadIdx.x;           // group of four pixels
    const uint8_t *s = src + (long long)blockIdx.z * sfs + (long long)blockIdx.y * sstride;
    uint8_t *d = dst + (long long)blockIdx.z * dfs + (long long)blockIdx.y * dstride;
    const int x0 = 4 * q;
    if (x0 >= W) return;
    if (vec && x0 + 4 <= W) {
        unsigned px[4], o[4];
        if (SB == 4) {
            const uint4 v = *reinterpret_cast<const uint4 *>(s + 16LL * q);
            px[0] = v.x; px[1] = v.y; px[2] = v.z; px[3] = v.w;
        } else {
            const unsigned *w = reinterpret_cast<const unsigned *>(s + 12LL * q);
            const unsigned w0 = w[0], w1 = w[1], w2 = w[2];
            px[0] = w0; px[1] = __funnelshift_r(w0, w1, 24); px[2] = __funnelshift_r(w1, w2, 16); px[3] = w2 >> 8;
        }
#pragma unroll
        for (int k = 0; k < 4; k++) o[k] = __byte_perm(px[k], 0xffu, sel);
        if (DB == 4) {
            *reinterpret_cast<uint4 *>(d + 16LL * q) = make_uint4(o[0], o[1], o[2], o[3]);
        } else {
            unsigned *w = reinterpret_cast<unsigned *>(d + 12LL * q);
            w[0] = __byte_perm(o[0], o[1], 0x4210); w[1] = __byte_perm(o[1], o[2], 0x5421); w[2] = __byte_perm(o[2], o[3], 0x6542);
        }
        return;
    }
    for (int x = x0; x < min(x0 + 4, W); x++) {
        unsigned px = 0;
#pragma unroll
        for (int b = 0; b < SB; b++) px |= (unsigned)s[(long long)x * SB + b] << (8 * b);
        const unsigned o = __byte_perm(px, 0xffu, sel);
#pragma unroll
        for (int b = 0; b < DB; b++) d[(long long)x * DB + b] = (uint8_t)(o >> (8 * b));
    }
}

static void launch_rgb_shuffle(const SwsPlan &p, cudaStream_t stream, const uint8_t *src, long long sstr, long long sfs, uint8_t *dst, long long ds,
                               long long dfs, int lines, int nframes)
{
    // 16-byte accesses for 4-byte pixels, 4-byte accesses for 3-byte pixels
    auto al = [](const void *ptr, long long a, long long b, int n) { return ((reinterpret_cast<uintptr_t>(ptr) | (uintptr_t)a | (uintptr_t)b) & (uintptr_t)(n - 1)) == 0; };
    const int vec = al(src, sstr, sfs, p.src_rgb == 4 ? 16 : 4) && al(dst, ds, dfs, p.out.bpp == 4 ? 16 : 4);
    for (int f0 = 0; f0 < nframes; f0 += 65535) {
        const int nf = nframes - f0 < 65535 ? nframes - f0 : 65535;
        const uint8_t *s = src + (long long)f0 * sfs;
        uint8_t *d = dst + (long long)f0 * dfs;
        for (int l0 = 0; l0 < lines; l0 += 65535) {
            const int nl = lines - l0 < 65535 ? lines - l0 : 65535;
            dim3 block(128), grid(b200_ceil_div(b200_ceil_div(p.srcW, 4), 128), nl, nf);
            const uint8_t *sl = s + (long long)l0 * sstr;
            uint8_t *dl = d + (long long)l0 * ds;
            if (p.src_rgb == 4 && p.out.bpp == 4)      sws_rgb_shuffle_kernel<4, 4><<<grid, block, 0, stream>>>(sl, sstr, sfs, dl, ds, dfs, p.srcW, p.shuffle_sel, vec);
            else if (p.src_rgb == 4)                   sws_rgb_shuffle_kernel<4, 3><<<grid, block, 0, stream>>>(sl, sstr, sfs, dl, ds, dfs, p.srcW, p.shuffle_sel, vec);
            else if (p.out.bpp == 4)                   sws_rgb_shuffle_kernel<3, 4><<<grid, block, 0, stream>>>(sl, sstr, sfs, dl, ds, dfs, p.srcW, p.shuffle_sel, vec);
            else                                       sws_rgb_shuffle_kernel<3, 3><<<grid, block, 0, stream>>>(sl, sstr, sfs, dl, ds, dfs, p.srcW, p.shuffle_sel, vec);
            B200_LAUNCHED();
        }
    }
}

static int launch_rgbsrc_packed(B200SwsContext *c, cudaStream_t stream, const uint8_t *src, long long sstr, long long sfs,
                                uint8_t *dst, long long ds, long long dfs, int nframes)
{
    const SwsPlan &p = c->plan;
    if (nframes <= 0) return 0;
    if (p.rgb_shuffle) {
        launch_rgb_shuffle(p, stream, src, sstr, sfs, dst, ds, dfs, p.srcH, nframes);
        B200_CUDA_OK(cudaGetLastError());
        return 0;
    }
    RgbIn Rg;
    Rg.bpp = p.src_rgb; Rg.ro = p.sro; Rg.go = p.sgo; Rg.bo = p.sbo; Rg.half = p.chrSrcHSub;
    for (int i = 0; i < 9; i++) Rg.c[i] = p.rgb2yuv[i];
    const size_t lumPlane = (size_t)p.srcH * p.dstW * 2, chrPlane = (size_t)p.chrSrcH * p.chrDstW * 2;
    const size_t perFrame = ((lumPlane + 2 * chrPlane + (p.need_alpha ? lumPlane : 0)) + 255) & ~(size_t)255;
    long long chunk = (long long)((size_t)(512u << 20) / perFrame);
    if (chunk < 1) chunk = 1;
    if (chunk > nframes) chunk = nframes;
    if (chunk > 65535) chunk = 65535;
    const size_t need = perFrame * (size_t)chunk;
    if (c->mid_bytes < need) {
        if (c->mid) { cudaStreamSynchronize(stream); cudaFree(c->mid); c->mid = nullptr; c->mid_bytes = 0; }
        B200_CUDA_OK(cudaMalloc(&c->mid, need));
        c->mid_bytes = need;
    }
    int16_t *mY = (int16_t *)c->mid;
    int16_t *mU = (int16_t *)((uint8_t *)c->mid + lumPlane);
    int16_t *mV = (int16_t *)((uint8_t *)c->mid + lumPlane + chrPlane);
    int16_t *mA = (int16_t *)((uint8_t *)c->mid + lumPlane + 2 * chrPlane);           // alpha lines (need_alpha only)
    const long long mfs = (long long)(perFrame / 2);
    for (long long f0 = 0; f0 < nframes; f0 += chunk) {
        const int nf = (int)(nframes - f0 < chunk ? nframes - f0 : chunk);
        const uint8_t *s = src + f0 * sfs;
        uint8_t *d = dst + f0 * dfs;
        dim3 block(256);
        sws_rgbin_hscale_y_kernel<<<dim3(b200_ceil_div(p.dstW, 256), p.srcH, nf), block, 0, stream>>>(s, sstr, sfs, mY, p.dstW, mfs, c->dt.hLum, c->dt.hLumPos,
                                                                                                        c->dt.hLumSize, Rg);
        B200_LAUNCHED();
        sws_rgbin_hscale_uv_kernel<<<dim3(b200_ceil_div(p.chrDstW, 256), p.chrSrcH, nf), block, 0, stream>>>(s, sstr, sfs, mU, mV, p.chrDstW, mfs, c->dt.hChr,
                                                                                                               c->dt.hChrPos, c->dt.hChrSize, Rg);
        B200_LAUNCHED();
        if (p.need_alpha) {
            sws_rgbin_hscale_a_kernel<<<dim3(b200_ceil_div(p.dstW, 256), p.srcH, nf), block, 0, stream>>>(s, sstr, sfs, mA, p.dstW, mfs, c->dt.hLum, c->dt.hLumPos,
                                                                                                            c->dt.hLumSize, 6 - p.sro - p.sgo - p.sbo);
            B200_LAUNCHED();
        }
        SwsFrameArgs m{};
        m.y = (const uint8_t *)mY; m.u = (const uint8_t *)mU; m.v = (const uint8_t *)mV;
        m.ys = (long long)p.dstW * 2; m.us = m.vs = (long long)p.chrDstW * 2;
        m.yfs = m.ufs = m.vfs = (long long)perFrame;
        m.dst = d; m.ds = ds; m.dfs = dfs;
        m.srcH = p.srcH; m.chrSrcH = p.chrSrcH; m.dstW = p.dstW; m.dstH = p.dstH; m.chrDstW = p.chrDstW;
        m.y0 = 0;
        m.bpp = p.out.bpp; m.ro = p.out.ro; m.go = p.out.go; m.bo = p.out.bo; m.ao = p.out.ao;
        if (p.chrDstHSub && c->all_x && p.dstW % 8 == 0 && aligned16(d, ds, dfs) && lumPlane % 16 == 0 && chrPlane % 8 == 0) {
            const int ng = p.dstW / 8;
            dim3 block2(128), grid(b200_ceil_div(ng, 128), p.dstH, nf);
            switch (p.out.kind) {
            case SWS_OUT_RGB24: sws_vscale_rgb24_x8_kernel<SWS_OUT_RGB24><<<grid, block2, 0, stream>>>(m, c->dt, p.color, ng); break;
            case SWS_OUT_BGR24: sws_vscale_rgb24_x8_kernel<SWS_OUT_BGR24><<<grid, block2, 0, stream>>>(m, c->dt, p.color, ng); break;
            case SWS_OUT_RGBA:  sws_vscale_rgb24_x8_kernel<SWS_OUT_RGBA><<<grid, block2, 0, stream>>>(m, c->dt, p.color, ng); break;
            case SWS_OUT_BGRA:  sws_vscale_rgb24_x8_kernel<SWS_OUT_BGRA><<<grid, block2, 0, stream>>>(m, c->dt, p.color, ng); break;
            case SWS_OUT_ARGB:  sws_vscale_rgb24_x8_kernel<SWS_OUT_ARGB><<<grid, block2, 0, stream>>>(m, c->dt, p.color, ng); break;
            default:            sws_vscale_rgb24_x8_kernel<SWS_OUT_ABGR><<<grid, block2, 0, stream>>>(m, c->dt, p.color, ng); break;
            }
        } else if (p.chrDstHSub) {
            const int np = (p.dstW + 1) / 2;
            dim3 block2(128), grid(b200_ceil_div(np, 128), p.dstH, nf);
            sws_vscale_rgb24_slow_kernel<false><<<grid, block2, 0, stream>>>(m, c->dt, p.color, 0, np);
        } else {
            dim3 block2(256), grid(b200_ceil_div(p.dstW, 256), p.dstH, nf);
            sws_vscale_rgb24_full_kernel<<<grid, block2, 0, stream>>>(m, c->dt, p.color);
        }
        B200_LAUNCHED();
        if (p.need_alpha) {                                    // the writers stored 255: the scaled alpha goes on top
            sws_vscale_alpha_kernel<<<dim3(b200_ceil_div(p.dstW, 256), p.dstH, nf), dim3(256), 0, stream>>>(mA, mfs, p.srcH, d, ds, dfs, p.dstW, p.out.bpp, p.out.ao,
                c->dt.vLum, c->dt.vLumPos, c->dt.vLumSize, c->dt.rowMode, p.chrDstHSub ? 0 : 1, 0);
            B200_LAUNCHED();
        }
    }
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

B200_API int b200_sws_scale_batch_device(B200SwsContext *c, const uint8_t *const src[3], const int srcStride[3],
                                         const int64_t srcFrameStride[3], uint8_t *dst, int dstStride,
                                         int64_t dstFrameStride, int nframes)
{
    if (!c || !src || !srcStride || !srcFrameStride || !dst) return B200_EINVAL;
    if (c->plan.planar) return B200_EINVAL;                   // three destination planes: b200_sws_scale_batch_device_planar
    B200_CUDA_OK(cudaSetDevice(c->dev->ordinal));
    if (c->plan.src_rgb) {                                    // packed source: plane 0 only
        if (!src[0] || srcStride[0] < 0 || dstStride < 0) return B200_EINVAL;
        return launch_rgbsrc_packed(c, c->dev->stream, src[0], srcStride[0], srcFrameStride[0], dst, dstStride, dstFrameStride, nframes);
    }
    const bool nv = c->plan.src_nv != 0;                      // nv12 / nv21: src[2] and its strides are not read
    const long long ss[3] = { srcStride[0], srcStride[1], nv ? 0 : srcStride[2] };
    const long long fs[3] = { srcFrameStride[0], srcFrameStride[1], nv ? 0 : srcFrameStride[2] };
    return launch_batch(c, c->dev->stream, src, ss, fs, dst, dstStride, dstFrameStride, nframes);
}

// yuv420p -> yuv420p: horizontal pass of the three planes into int16 line planes, then one vertical pass per plane
static int launch_planar3(B200SwsContext *c, cudaStream_t stream, const uint8_t *const src_in[3], const long long sstr_in[3],
                          const long long sfs_in[3], uint8_t *const dst[3], const long long dstr[3], const long long dfs[3], int nframes)
{
    const SwsPlan &p = c->plan;
    if (nframes <= 0) return 0;
    const uint8_t *src[3] = { src_in[0], src_in[1], src_in[2] };
    long long sstr[3] = { sstr_in[0], sstr_in[1], sstr_in[2] }, sfs[3] = { sfs_in[0], sfs_in[1], sfs_in[2] };
    if (p.src_nv) {
        int ret = nv_split(c, stream, nullptr, nframes, 0, p.chrSrcH, src, sstr, sfs);
        if (ret < 0) return ret;
    }
    const int sw[3] = { p.srcW, p.chrSrcW, p.chrSrcW }, sh[3] = { p.srcH, p.chrSrcH, p.chrSrcH };
    const int dw[3] = { p.dstW, p.chrDstW, p.chrDstW }, dh[3] = { p.dstH, p.chrDstH, p.chrDstH };
    RgbIn R;
    R.bpp = p.src_rgb; R.ro = p.sro; R.go = p.sgo; R.bo = p.sbo; R.half = p.chrSrcHSub;
    for (int i = 0; i < 9; i++) R.c[i] = p.rgb2yuv[i];
    for (int f0 = 0; f0 < nframes; f0 += 65535) {
        const int nf = nframes - f0 < 65535 ? nframes - f0 : 65535;
        if (p.bgr24_yv12) {
            dim3 block(256), grid(b200_ceil_div(p.srcW >> 1, 256), (p.srcH + 1) / 2, nf);
            sws_bgr24_yv12_kernel<<<grid, block, 0, stream>>>(src[0] + (long long)f0 * sfs[0], sstr[0], sfs[0],
                                                               dst[0] + (long long)f0 * dfs[0], dstr[0], dfs[0],
                                                               dst[1] + (long long)f0 * dfs[1], dstr[1], dfs[1],
                                                               dst[2] + (long long)f0 * dfs[2], dstr[2], dfs[2], p.srcW, p.srcH, R);
            B200_LAUNCHED();
            continue;
        }
        if (p.planar_copy) {
            for (int pl = 0; pl < 3; pl++) {
                const uint8_t *s = src[pl] + (long long)f0 * sfs[pl];
                uint8_t *d = dst[pl] + (long long)f0 * dfs[pl];
                const int vec = aligned16(s, sstr[pl], sfs[pl]) && aligned16(d, dstr[pl], dfs[pl]);
                dim3 block(256), grid(b200_ceil_div(vec ? b200_ceil_div(sw[pl], 16) : sw[pl], 256), sh[pl], nf);
                sws_plane_copy_kernel<<<grid, block, 0, stream>>>(s, sstr[pl], sfs[pl], d, dstr[pl], dfs[pl], sw[pl], vec);
                B200_LAUNCHED();
            }
            continue;
        }
        const size_t plane[3] = { (size_t)p.srcH * p.dstW * 2, (size_t)p.chrSrcH * p.chrDstW * 2, (size_t)p.chrSrcH * p.chrDstW * 2 };
        const size_t perFrame = ((plane[0] + plane[1] + plane[2]) + 255) & ~(size_t)255;
        const size_t need = perFrame * nf;
        if (c->mid_bytes < need) {
            if (c->mid) { cudaStreamSynchronize(stream); cudaFree(c->mid); c->mid = nullptr; c->mid_bytes = 0; }
            B200_CUDA_OK(cudaMalloc(&c->mid, need));
            c->mid_bytes = need;
        }
        int16_t *m[3] = { (int16_t *)c->mid, (int16_t *)((uint8_t *)c->mid + plane[0]), (int16_t *)((uint8_t *)c->mid + plane[0] + plane[1]) };
        const int32_t *hc[3] = { c->dt.hLum2, c->dt.hChr2, c->dt.hChr2 };
        const int32_t *hp[3] = { c->dt.hLumPos, c->dt.hChrPos, c->dt.hChrPos };
        const int hs[3] = { c->dt.hLumSize, c->dt.hChrSize, c->dt.hChrSize };
        const int16_t *vc[3] = { c->dt.vLum, c->dt.vChr, c->dt.vChr };
        const int32_t *vp[3] = { c->dt.vLumPos, c->dt.vChrPos, c->dt.vChrPos };
        const int vs[3] = { c->dt.vLumSize, c->dt.vChrSize, c->dt.vChrSize };
        for (int pl = 0; pl < 3; pl++) {
            dim3 block(256), gh(b200_ceil_div(dw[pl], 256), sh[pl], nf), gv(b200_ceil_div(dw[pl], 256), dh[pl], nf);
            if (p.src_rgb) {                    // packed source in src[0]: luma lines, then both chroma planes in one launch
                if (pl == 0)
                    sws_rgbin_hscale_y_kernel<<<gh, block, 0, stream>>>(src[0] + (long long)f0 * sfs[0], sstr[0], sfs[0], m[0], dw[0],
                                                                        (long long)(perFrame / 2), c->dt.hLum, c->dt.hLumPos, c->dt.hLumSize, R);
                else if (pl == 1)
                    sws_rgbin_hscale_uv_kernel<<<gh, block, 0, stream>>>(src[0] + (long long)f0 * sfs[0], sstr[0], sfs[0], m[1], m[2], dw[1],
                                                                         (long long)(perFrame / 2), c->dt.hChr, c->dt.hChrPos, c->dt.hChrSize, R);
            }
            else if (p.fast_bilinear && pl == 0)
                sws_hscale_fast_kernel<false><<<gh, block, 0, stream>>>(src[pl] + (long long)f0 * sfs[pl], sstr[pl], sfs[pl], m[pl], dw[pl],
                                                                        (long long)(perFrame / 2), sw[pl], p.lumXInc, 0);
            else if (p.fast_bilinear)
                sws_hscale_fast_kernel<true><<<gh, block, 0, stream>>>(src[pl] + (long long)f0 * sfs[pl], sstr[pl], sfs[pl], m[pl], dw[pl],
                                                                       (long long)(perFrame / 2), sw[pl], p.chrXInc, 0);
            else {
                // fused horizontal + vertical pass for this plane when the writer below would be the 8-sample one
                uint8_t *dplf = dst[pl] + (long long)f0 * dfs[pl];
                const SwsFilterBank &vb = pl ? p.vChr : p.vLum;
                const bool m8 = c->mma_tables && !p.range_conv && dw[pl] % 8 == 0 &&
                                (((uintptr_t)dplf | (uintptr_t)dstr[pl] | (uintptr_t)dfs[pl]) & 7) == 0 &&
                                aligned16(src[pl] + (long long)f0 * sfs[pl], sstr[pl], sfs[pl]);
                if (m8) {
                    const SwsFilterBank &vbm = pl ? p.vChr : p.vLum;
                    const int SP = pl ? c->mma_pitchC : c->mma_pitchL;
                    auto needb = [&](int r) { return MT_HDR + (size_t)((r + 15) & ~15) * (SP + MT_TPB); };
                    int TRm = 0, nr = -1;
                    double best = 1e30;
                    for (int cand = 32; cand >= 8; cand--) {                       // see the packed-RGB launch: fewest wasted 16-line blocks
                        const int a_ = fused_rows_needed(vbm, sh[pl], dh[pl], cand);
                        if (a_ <= 0 || needb(a_) > 112 * 1024) continue;
                        const double cost = (double)((a_ + 15) >> 4) / cand * (1.0 + (needb(a_) > 56 * 1024 ? 0.15 : 0.0) + (needb(a_) > 75 * 1024 ? 0.15 : 0.0));
                        if (cost < best - 1e-9) { best = cost; TRm = cand; nr = a_; }
                    }
                    if (nr > 0 && needb(nr) <= 112 * 1024) {
                        const size_t smem = needb(nr);
                        dim3 gm(b200_ceil_div(dw[pl], MT_W), b200_ceil_div(dh[pl], TRm), nf);
                        if (smem > 48 * 1024) B200_CUDA_OK(cudaFuncSetAttribute(sws_mma_plane_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
                        sws_mma_plane_kernel<<<gm, MT_THREADS, smem, stream>>>(src[pl] + (long long)f0 * sfs[pl], sstr[pl], sfs[pl], sw[pl], sh[pl], dplf,
                                                                              dstr[pl], dfs[pl], dw[pl], dh[pl], pl ? c->mmaC : c->mmaL, pl ? c->dt.vChr2 : c->dt.vLum2, vp[pl], vs[pl],
                                                                              TRm, (nr + 15) & ~15, SP);
                        B200_LAUNCHED();
                        c->last_path |= 4;
                        continue;
                    }
                }
                const bool f8 = !p.range_conv && hs[pl] <= 16 && dw[pl] % 8 == 0 &&
                                (((uintptr_t)dplf | (uintptr_t)dstr[pl] | (uintptr_t)dfs[pl]) & 7) == 0;
                int TR = 32, need_rows = f8 ? fused_rows_needed(vb, sh[pl], dh[pl], TR) : -1;
                if (need_rows > 96) { TR = 16; need_rows = fused_rows_needed(vb, sh[pl], dh[pl], TR); }
                if (need_rows > 0 && need_rows <= 96) {
                    const size_t smem = (size_t)need_rows * FT_W * 2;
                    dim3 gf(b200_ceil_div(dw[pl], FT_W), b200_ceil_div(dh[pl], TR), nf);
                    const uint8_t *sp = src[pl] + (long long)f0 * sfs[pl];
                    if (hs[pl] <= 8) {
                        if (smem > 48 * 1024) B200_CUDA_OK(cudaFuncSetAttribute(sws_fused_plane_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
                        sws_fused_plane_kernel<4><<<gf, FT_W, smem, stream>>>(sp, sstr[pl], sfs[pl], sh[pl], dplf, dstr[pl], dfs[pl], dw[pl], dh[pl],
                                                                              hc[pl], hp[pl], hs[pl], vc[pl], vp[pl], vs[pl], TR);
                    } else {
                        if (smem > 48 * 1024) B200_CUDA_OK(cudaFuncSetAttribute(sws_fused_plane_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
                        sws_fused_plane_kernel<8><<<gf, FT_W, smem, stream>>>(sp, sstr[pl], sfs[pl], sh[pl], dplf, dstr[pl], dfs[pl], dw[pl], dh[pl],
                                                                              hc[pl], hp[pl], hs[pl], vc[pl], vp[pl], vs[pl], TR);
                    }
                    B200_LAUNCHED();
                    c->last_path |= 2;
                    continue;
                }
                c->last_path |= 1;
                launch_hscale(stream, src[pl] + (long long)f0 * sfs[pl], sstr[pl], sfs[pl], m[pl], dw[pl], (long long)(perFrame / 2),
                              hc[pl], hp[pl], hs[pl], 0, sh[pl], nf);
            }
            if (!(p.src_rgb && pl == 2)) B200_LAUNCHED();
            if (p.range_conv) {
                sws_range_kernel<<<gh, block, 0, stream>>>(m[pl], dw[pl], (long long)(perFrame / 2), pl ? p.chrRangeCoeff : p.lumRangeCoeff,
                                                           pl ? p.chrRangeOffset : p.lumRangeOffset, p.range_conv == 1);
                B200_LAUNCHED();
            }
            uint8_t *dpl = dst[pl] + (long long)f0 * dfs[pl];
            const bool v4 = dw[pl] % 4 == 0 && (plane[0] % 8 == 0) && (plane[1] % 8 == 0) &&
                            (((uintptr_t)dpl | (uintptr_t)dstr[pl] | (uintptr_t)dfs[pl]) & 3) == 0;
            const bool v8 = v4 && dw[pl] % 8 == 0 && (plane[0] % 16 == 0) && (plane[1] % 16 == 0) &&
                            (((uintptr_t)dpl | (uintptr_t)dstr[pl] | (uintptr_t)dfs[pl]) & 7) == 0;
            if (v8) {
                dim3 g8(b200_ceil_div(dw[pl] / 8, 256), dh[pl], nf);
                sws_vscale_planar8_kernel<<<g8, block, 0, stream>>>(m[pl], dw[pl], (long long)perFrame, sh[pl], dpl, dstr[pl], dfs[pl],
                                                                    dw[pl], vc[pl], vp[pl], vs[pl], 0);
            } else if (v4) {
                dim3 g4(b200_ceil_div(dw[pl] / 4, 256), dh[pl], nf);
                sws_vscale_planar4_kernel<<<g4, block, 0, stream>>>(m[pl], dw[pl], (long long)perFrame, sh[pl], dpl, dstr[pl], dfs[pl],
                                                                    dw[pl], vc[pl], vp[pl], vs[pl], 0);
            } else {
                sws_vscale_planar_kernel<<<gv, block, 0, stream>>>(m[pl], dw[pl], (long long)perFrame, sh[pl], dpl, dstr[pl], dfs[pl],
                                                                   dw[pl], vc[pl], vp[pl], vs[pl], 0);
            }
            B200_LAUNCHED();
        }
    }
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

// [device-code sws_nvout]
// nv12 / nv21 destination: U and V of planarToNv12Wrapper / yuv2nv12cX_c are what the three-plane writers produce (same sums, same
// flat dither), stored side by side (V first for nv21): one byte pair per thread
__global__ void __launch_bounds__(256)
sws_nv_interleave_kernel(const uint8_t *u, const uint8_t *v, long long cs, long long cfs, uint8_t *dst, long long ds, long long dfs, int cw)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= cw) return;
    const long long o = (long long)blockIdx.z * cfs + (long long)blockIdx.y * cs + i;
    uint8_t *d = dst + (long long)blockIdx.z * dfs + (long long)blockIdx.y * ds + 2 * i;
    d[0] = __ldg(u + o);
    d[1] = __ldg(v + o);
}

// [/device-code sws_nvout]
// yuv destinations: three planes, or (nv12 / nv21) the same into scratch chroma planes followed by the interleave
static int launch_planar(B200SwsContext *c, cudaStream_t stream, const uint8_t *const src[3], const long long sstr[3],
                         const long long sfs[3], uint8_t *const dst[3], const long long dstr[3], const long long dfs[3], int nframes)
{
    const SwsPlan &p = c->plan;
    if (!p.dst_nv) return launch_planar3(c, stream, src, sstr, sfs, dst, dstr, dfs, nframes);
    if (nframes <= 0) return 0;
    const size_t cplane = (size_t)p.chrDstW * p.chrDstH;
    long long chunk = (long long)((size_t)(64u << 20) / (2 * cplane ? 2 * cplane : 1));
    if (chunk < 1) chunk = 1;
    if (chunk > nframes) chunk = nframes;
    const size_t need = 2 * cplane * (size_t)chunk;
    if (c->nvout_bytes < need) {
        if (c->nvout_buf) { cudaStreamSynchronize(stream); cudaFree(c->nvout_buf); c->nvout_buf = nullptr; c->nvout_bytes = 0; }
        B200_CUDA_OK(cudaMalloc(&c->nvout_buf, need));
        c->nvout_bytes = need;
    }
    uint8_t *buf = (uint8_t *)c->nvout_buf;
    for (long long f0 = 0; f0 < nframes; f0 += chunk) {
        const int nf = (int)(nframes - f0 < chunk ? nframes - f0 : chunk);
        const uint8_t *s3[3] = { src[0] ? src[0] + f0 * sfs[0] : nullptr, src[1] ? src[1] + f0 * sfs[1] : nullptr, src[2] ? src[2] + f0 * sfs[2] : nullptr };
        uint8_t *d3[3] = { dst[0] + f0 * dfs[0], buf, buf + cplane };
        const long long ds3[3] = { dstr[0], p.chrDstW, p.chrDstW }, df3[3] = { dfs[0], (long long)(2 * cplane), (long long)(2 * cplane) };
        const int ret = launch_planar3(c, stream, s3, sstr, sfs, d3, ds3, df3, nf);
        if (ret < 0) return ret;
        dim3 block(256), grid(b200_ceil_div(p.chrDstW, 256), p.chrDstH, nf);
        sws_nv_interleave_kernel<<<grid, block, 0, stream>>>(p.dst_nv == 1 ? d3[1] : d3[2], p.dst_nv == 1 ? d3[2] : d3[1], p.chrDstW,
                                                             (long long)(2 * cplane), dst[1] + f0 * dfs[1], dstr[1], dfs[1], p.chrDstW);
        B200_LAUNCHED();
    }
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

B200_API int b200_sws_scale_batch_device_planar(B200SwsContext *c, const uint8_t *const src[3], const int srcStride[3],
                                                const int64_t srcFrameStride[3], uint8_t *const dst[3], const int dstStride[3],
                                                const int64_t dstFrameStride[3], int nframes)
{
    if (!c || !src || !srcStride || !srcFrameStride || !dst || !dstStride || !dstFrameStride) return B200_EINVAL;
    if (!c->plan.planar) return B200_EINVAL;
    if (c->casc[0]) {                                                       // two matrices: frame by frame through the bgr24 picture
        const int nsp0 = c->plan.src_nv ? 2 : 3, ndp0 = c->plan.dst_nv ? 2 : 3;
        for (int f = 0; f < nframes; f++) {
            const uint8_t *s3[3] = { nullptr, nullptr, nullptr }; uint8_t *d3[3] = { nullptr, nullptr, nullptr };
            for (int i = 0; i < nsp0; i++) s3[i] = src[i] + (long long)f * srcFrameStride[i];
            for (int i = 0; i < ndp0; i++) d3[i] = dst[i] + (long long)f * dstFrameStride[i];
            int r = b200_sws_scale_batch_device(c->casc[0], s3, srcStride, srcFrameStride, (uint8_t *)c->casc_tmp, (int)c->casc_pitch, 0, 1);
            if (r < 0) return r;
            const uint8_t *t3[3] = { (const uint8_t *)c->casc_tmp, nullptr, nullptr };
            const int ts[3] = { (int)c->casc_pitch, 0, 0 };
            const int64_t tf[3] = { 0, 0, 0 };
            r = b200_sws_scale_batch_device_planar(c->casc[1], t3, ts, tf, d3, dstStride, dstFrameStride, 1);
            if (r < 0) return r;
        }
        return 0;
    }
    const int nsp = c->plan.src_rgb ? 1 : c->plan.src_nv ? 2 : 3;           // packed RGB: plane 0 only; nv12 / nv21: planes 0 and 1
    const int ndp = c->plan.dst_nv ? 2 : 3;                                 // nv12 / nv21 destination: dst[1] is the interleaved plane
    for (int i = 0; i < 3; i++) if ((i < nsp && (!src[i] || srcStride[i] < 0)) || (i < ndp && (!dst[i] || dstStride[i] < 0))) return B200_EINVAL;
    B200_CUDA_OK(cudaSetDevice(c->dev->ordinal));
    const long long ss[3] = { srcStride[0], nsp >= 2 ? srcStride[1] : 0, nsp == 3 ? srcStride[2] : 0 };
    const long long fs[3] = { srcFrameStride[0], nsp >= 2 ? srcFrameStride[1] : 0, nsp == 3 ? srcFrameStride[2] : 0 };
    const long long ds[3] = { dstStride[0], dstStride[1], ndp == 3 ? dstStride[2] : 0 };
    const long long df[3] = { dstFrameStride[0], dstFrameStride[1], ndp == 3 ? dstFrameStride[2] : 0 };
    return launch_planar(c, c->dev->stream, src, ss, fs, dst, ds, df, nframes);
}

// sws_scale() with a yuv420p destination: whole frames, host pointers
static int sws_scale_planar_host(B200SwsContext *c, const uint8_t *const srcSlice[], const int srcStride[],
                                 int srcSliceY, int srcSliceH, uint8_t *const dst[], const int dstStride[])
{
    const SwsPlan &p = c->plan;
    if (c->casc[0]) {                                            // scale_cascaded (swscale.c:1001-1030; whole frames only, :1084-1086)
        if (srcSliceY != 0 || srcSliceH != p.srcH) {
            b200_set_error("sws_scale: a context cascaded for two yuv matrices converts whole frames only");
            return B200_ENOSYS;
        }
        std::vector<uint8_t> tmp(((size_t)c->casc_w * 3 + 63 & ~(size_t)63) * c->casc_h, 0);
        const int tstride = (int)(((size_t)c->casc_w * 3 + 63) & ~(size_t)63);
        uint8_t *td[4] = { tmp.data(), nullptr, nullptr, nullptr };
        const int tds[4] = { tstride, 0, 0, 0 };
        int r = b200_sws_scale(c->casc[0], srcSlice, srcStride, 0, p.srcH, td, tds);
        if (r < 0) return r;
        const uint8_t *ts[4] = { tmp.data(), nullptr, nullptr, nullptr };
        return b200_sws_scale(c->casc[1], ts, tds, 0, c->casc_h, dst, dstStride);
    }
    const bool whole = srcSliceY == 0 && srcSliceH == p.srcH && !c->slice_open;
    const int macro = p.src_rgb ? 1 : 2;                         // macro_height_src: 1 for packed RGB, 2 for 4:2:0 sources (swscale.c:1063-1071)
    if (!whole && p.bgr24_yv12 && ((srcSliceY | srcSliceH) & 1)) {
        b200_set_error("bgr24 -> yuv420p converter: slices must cover whole line pairs");      // ff_rgb24toyv12 works on line pairs of the band it is given
        return B200_ENOSYS;
    }
    if (!whole) {
        // parameter checks of scale_internal, as in the packed-RGB slice path below
        if ((srcSliceY & (macro - 1)) || ((srcSliceH & (macro - 1)) && srcSliceY + srcSliceH != p.srcH) || srcSliceY + srcSliceH > p.srcH || srcSliceY < 0 || srcSliceH < 0) {
            b200_set_error("Slice parameters %d, %d are invalid", srcSliceY, srcSliceH);
            return B200_EINVAL;
        }
        if (srcSliceH == 0) return 0;
        if (!c->slice_open && srcSliceY != 0) {
            b200_set_error("Slices start in the middle!");
            return B200_EINVAL;
        }
    }
    const int nsp = p.src_rgb ? 1 : p.src_nv ? 2 : 3;             // packed RGB: one plane; nv12 / nv21: plane 1 carries both chroma components
    const int ndp = p.dst_nv ? 2 : 3;                             // nv12 / nv21 destination: two planes
    for (int i = 0; i < 3; i++) {
        if ((i < ndp && !dst[i]) || (i < nsp && !srcSlice[i])) return B200_EINVAL;
        if (whole && ((i < ndp && dstStride[i] < 0) || (i < nsp && srcStride[i] < 0))) return B200_ENOSYS;
    }
    B200Device *d = c->dev;
    B200_CUDA_OK(cudaSetDevice(d->ordinal));
    const int sw[3] = { p.src_rgb ? p.srcW * p.src_rgb : p.srcW, p.src_rgb ? 0 : p.src_nv ? 2 * p.chrSrcW : p.chrSrcW, (p.src_nv || p.src_rgb) ? 0 : p.chrSrcW },
              sh[3] = { p.srcH, p.src_rgb ? 0 : p.chrSrcH, p.src_rgb ? 0 : p.chrSrcH };
    const int dw[3] = { p.dstW, p.dst_nv ? 2 * p.chrDstW : p.chrDstW, p.dst_nv ? 0 : p.chrDstW }, dh[3] = { p.dstH, p.chrDstH, p.dst_nv ? 0 : p.chrDstH };
    size_t spitch[3], dpitch[3], soff[3], doff[3], total = 0;
    for (int i = 0; i < 3; i++) { spitch[i] = ((size_t)sw[i] + 255) & ~(size_t)255; soff[i] = total; total += spitch[i] * sh[i]; }
    for (int i = 0; i < 3; i++) { dpitch[i] = ((size_t)dw[i] + 255) & ~(size_t)255; doff[i] = total; total += dpitch[i] * dh[i]; }
    cudaStream_t st = d->stream;
    const uint8_t *sp[3]; uint8_t *dp[3]; long long ss[3], ds[3];
    const long long zero[3] = { 0, 0, 0 };
    if (!whole) {
        // Slice sequence (top-down): the bands accumulate in a device copy of the picture that lives in the context; after each band
        // the whole picture is converted again — an output line only depends on source lines that have arrived once ff_swscale's
        // "enough lines" test (swscale.c:463-465) passes for it — and the lines that became complete are copied back: the return
        // value and the lines written per call are the reference's.
        if (!c->slice_buf) {                                // cleared once: the whole-picture passes below read lines that have not arrived yet
            B200_CUDA_OK(cudaMalloc(&c->slice_buf, total));
            B200_CUDA_OK(cudaMemsetAsync(c->slice_buf, 0, total, d->stream));
        }
        uint8_t *sb = (uint8_t *)c->slice_buf;
        if (srcSliceY == 0) { c->next_dst_y = 0; c->slice_open = true; }
        const int chrY = srcSliceY >> 1, chrH = -((-srcSliceH) >> 1);
        const int by[3] = { srcSliceY, chrY, chrY }, bh[3] = { srcSliceH, chrH, chrH };
        for (int i = 0; i < 3; i++) {
            if (i < nsp)
                B200_CUDA_OK(b200_h2d_rows(sb + soff[i] + (size_t)by[i] * spitch[i], spitch[i], srcSlice[i], srcStride[i], sw[i], bh[i], st));
            sp[i] = sb + soff[i]; dp[i] = sb + doff[i]; ss[i] = (long long)spitch[i]; ds[i] = (long long)dpitch[i];
        }
        int y0, y1;
        if (p.planar_copy || p.bgr24_yv12) {                   // the unscaled wrappers handle exactly the band they are given
            y0 = srcSliceY; y1 = srcSliceY + srcSliceH;
        } else {
            y0 = c->next_dst_y;
            // chroma lines of the source that have arrived: one per luma line for packed RGB sources (chrSrcVSubSample = 0, utils.c:1366-1396)
            const int avail_l = srcSliceY + srcSliceH, avail_c = p.src_rgb ? avail_l : -((-(srcSliceY + srcSliceH)) >> 1);
            for (y1 = y0; y1 < p.dstH; y1++) {
                // luma availability is tested for the last luma line of the chroma line's pair: firstLumSrcY2 (swscale.c:419-421)
                const int firstLum = std::max(1 - p.vLum.size, p.vLum.pos[std::min(y1 | 1, p.dstH - 1)]);
                const int firstChr = std::max(1 - p.vChr.size, p.vChr.pos[y1 >> 1]);      // chrDstY = dstY >> 1 (swscale.c:414)
                const int lastLum = std::min(p.srcH, firstLum + p.vLum.size) - 1;
                const int lastChr = std::min(p.chrSrcH, firstChr + p.vChr.size) - 1;
                if (!(lastLum < avail_l && lastChr < avail_c)) break;
            }
            c->next_dst_y = y1;
        }
        if (y1 > y0) {
            int ret = launch_planar(c, st, sp, ss, zero, dp, ds, zero, 1);
            if (ret < 0) return ret;
            const int c0 = (y0 + 1) >> 1, c1 = (y1 + 1) >> 1;           // chroma lines are written with the even luma lines (vscale.c:34-107)
            B200_CUDA_OK(b200_d2h_rows(dst[0] + (long long)y0 * dstStride[0], dstStride[0], dp[0] + (size_t)y0 * dpitch[0], dpitch[0], dw[0], y1 - y0, st));
            for (int i = 1; i < ndp && c1 > c0; i++)
                B200_CUDA_OK(b200_d2h_rows(dst[i] + (long long)c0 * dstStride[i], dstStride[i], dp[i] + (size_t)c0 * dpitch[i], dpitch[i], dw[i], c1 - c0, st));
        }
        B200_CUDA_OK(cudaStreamSynchronize(st));
        if (srcSliceY + srcSliceH == p.srcH) c->slice_open = false;
        return y1 - y0;
    }
    B200_LOCK_DEVICE(d);      // scratch + stream are per device: one host-pointer call at a time (released on return)
    uint8_t *scr = (uint8_t *)b200_scratch(d, total);
    if (!scr) return B200_ENOMEM;
    for (int i = 0; i < 3; i++) {
        if (i < nsp)
            B200_CUDA_OK(cudaMemcpy2DAsync(scr + soff[i], spitch[i], srcSlice[i], (size_t)srcStride[i], sw[i], sh[i], cudaMemcpyHostToDevice, st));
        sp[i] = scr + soff[i]; dp[i] = scr + doff[i]; ss[i] = (long long)spitch[i]; ds[i] = (long long)dpitch[i];
    }
    int ret = launch_planar(c, st, sp, ss, zero, dp, ds, zero, 1);
    if (ret < 0) return ret;
    for (int i = 0; i < ndp; i++)
        B200_CUDA_OK(cudaMemcpy2DAsync(dst[i], (size_t)dstStride[i], dp[i], dpitch[i], dw[i], dh[i], cudaMemcpyDeviceToHost, st));
    B200_CUDA_OK(cudaStreamSynchronize(st));
    return p.dstH;
}

// device-side packed layout used by the host-pointer entry points
struct PackedLayout {
    size_t yPitch, cPitch, dPitch, yOff, uOff, vOff, srcBytes, dstBytes;
};
static PackedLayout packed_layout(const SwsPlan &p)
{
    PackedLayout L;
    L.yPitch = ((size_t)p.srcW + 255) & ~(size_t)255;
    L.cPitch = ((size_t)p.chrSrcW + 255) & ~(size_t)255;
    L.dPitch = ((size_t)p.dstW * p.out.bpp + 255) & ~(size_t)255;
    L.yOff = 0; L.uOff = L.yPitch * p.srcH; L.vOff = L.uOff + L.cPitch * p.chrSrcH;
    L.srcBytes = L.vOff + L.cPitch * p.chrSrcH;
    L.dstBytes = L.dPitch * p.dstH;
    return L;
}


// bytes of a destination row the reference writes: its unscaled LUT converters work on pixel pairs and never touch an odd last
// column (yuv2rgb.c:137-236: (dstW >> 3) * 8 + (dstW & 4) + (dstW & 2) pixels per line), so the host entry points must not either
static inline size_t sws_written_row_bytes(const SwsPlan &p)
{
    return (size_t)(p.unscaled_lut ? (p.dstW & ~1) : p.dstW) * p.out.bpp;
}

B200_API int b200_sws_scale_batch_host(B200SwsContext *c, const uint8_t *const src[3], const int srcStride[3],
                                       const int64_t srcFrameStride[3], uint8_t *dst, int dstStride,
                                       int64_t dstFrameStride, int nframes)
{
    if (!c || !src || !srcStride || !srcFrameStride || !dst || nframes < 0) return B200_EINVAL;
    if (c->plan.planar) return B200_EINVAL;
    if (c->plan.src_rgb) { b200_set_error("b200_sws_scale_batch_host: packed RGB sources are not wired into this entry point"); return B200_ENOSYS; }
    B200Device *d = c->dev;
    B200_CUDA_OK(cudaSetDevice(d->ordinal));
    const SwsPlan &p = c->plan;
    const PackedLayout L = packed_layout(p);
    // Chunks of at most 8 frames: the device-to-host copies are the bottleneck of this entry point (PCIe), and they can
    // only start once the first chunk has been uploaded and converted, so short chunks keep the pipeline fill short;
    // the three in-flight chunks stay within ~0.8 GB of scratch at 4K.
    const size_t nvBytes = p.src_nv ? nv_frame_bytes(p) : 0;     // per-slot room for the de-interleaved chroma of nv12 / nv21
    const size_t perFrame = L.srcBytes + L.dstBytes + nvBytes;
    int chunk = (int)((size_t)256 << 20) / (int)(perFrame ? perFrame : 1);
    if (chunk < 1) chunk = 1;
    if (chunk > 8) chunk = 8;
    if (chunk > nframes) chunk = nframes > 0 ? nframes : 1;
    const int K = B200Device::kPipe;
    B200_LOCK_DEVICE(d);      // scratch + stream are per device: one host-pointer call at a time (released on return)
    uint8_t *scr = (uint8_t *)b200_scratch(d, perFrame * chunk * K);
    if (!scr) return B200_ENOMEM;
    B200_CUDA_OK(cudaStreamSynchronize(d->stream));
    const int nsp = p.src_nv ? 2 : 3;
    const int wbytes[3] = { p.srcW, p.src_nv ? 2 * p.chrSrcW : p.chrSrcW, p.chrSrcW }, rows[3] = { p.srcH, p.chrSrcH, p.chrSrcH };
    const size_t pitch[3] = { L.yPitch, p.src_nv ? 2 * L.cPitch : L.cPitch, L.cPitch }, poff[3] = { L.yOff, L.uOff, L.vOff };
    int slot = 0;
    for (int f0 = 0; f0 < nframes; f0 += chunk, slot = (slot + 1) % K) {
        const int nf = nframes - f0 < chunk ? nframes - f0 : chunk;
        cudaStream_t st = d->pipe[slot];
        uint8_t *sbase = scr + (size_t)slot * perFrame * chunk;
        uint8_t *dbase = sbase + L.srcBytes * chunk;
        for (int pl = 0; pl < nsp; pl++) {
            if (srcStride[pl] < 0) return B200_ENOSYS;                    // bottom-up pictures: use b200_sws_scale()
            for (int f = 0; f < nf; f++) {
                const uint8_t *hp = src[pl] + (int64_t)(f0 + f) * srcFrameStride[pl];
                uint8_t *dp = sbase + (size_t)f * L.srcBytes + poff[pl];
                B200_CUDA_OK(cudaMemcpy2DAsync(dp, pitch[pl], hp, (size_t)srcStride[pl], wbytes[pl], rows[pl], cudaMemcpyHostToDevice, st));
            }
        }
        const uint8_t *sp[3] = { sbase + L.yOff, sbase + L.uOff, sbase + L.vOff };
        const long long ss[3] = { (long long)pitch[0], (long long)pitch[1], (long long)pitch[2] };
        const long long fs[3] = { (long long)L.srcBytes, (long long)L.srcBytes, (long long)L.srcBytes };
        int ret = launch_batch(c, st, sp, ss, fs, dbase, (long long)L.dPitch, (long long)L.dstBytes, nf, nullptr,
                               p.src_nv ? dbase + L.dstBytes * chunk : nullptr);
        if (ret < 0) return ret;
        const size_t rowBytes = sws_written_row_bytes(p);
        if (rowBytes == (size_t)p.dstW * p.out.bpp && (size_t)dstStride == rowBytes && L.dPitch == rowBytes && dstFrameStride == (int64_t)(rowBytes * p.dstH)) {
            // contiguous on both sides: the whole chunk comes back as one linear copy
            B200_CUDA_OK(cudaMemcpyAsync(dst + (int64_t)f0 * dstFrameStride, dbase, L.dstBytes * nf, cudaMemcpyDeviceToHost, st));
        } else {
            for (int f = 0; f < nf && rowBytes; f++)
                B200_CUDA_OK(cudaMemcpy2DAsync(dst + (int64_t)(f0 + f) * dstFrameStride, (size_t)dstStride,
                                               dbase + (size_t)f * L.dstBytes, L.dPitch, rowBytes, p.dstH, cudaMemcpyDeviceToHost, st));
        }
    }
    for (int i = 0; i < K; i++) B200_CUDA_OK(cudaStreamSynchronize(d->pipe[i]));
    return 0;
}

// sws_scale() called with a horizontal band of the source (top-down slices, like slice-threaded decoders feed it).
// Mirrors scale_internal() (swscale.c:1022-1200) and the line scheduling of ff_swscale() (swscale.c:412-535): the band
// is uploaded into a device copy of the source picture, the horizontal pass runs on the new lines only, and every
// output line whose vertical taps are now complete is produced and copied back.  Returns the number of lines written.
static int sws_scale_slice(B200SwsContext *c, const uint8_t *const srcSlice[], const int srcStride[],
                           int srcSliceY, int srcSliceH, uint8_t *const dst[], const int dstStride[])
{
    const SwsPlan &p = c->plan;
    // parameter checks of scale_internal (macro_height_src = 2 for yuv420p)
    if ((srcSliceY & 1) || ((srcSliceH & 1) && srcSliceY + srcSliceH != p.srcH) || srcSliceY + srcSliceH > p.srcH ||
        srcSliceY < 0 || srcSliceH < 0) {
        b200_set_error("Slice parameters %d, %d are invalid", srcSliceY, srcSliceH);
        return B200_EINVAL;
    }
    if (srcSliceH == 0) return 0;
    if (!c->slice_open && srcSliceY != 0) {
        b200_set_error("Slices start in the middle!");
        return B200_EINVAL;
    }
    B200Device *d = c->dev;
    B200_CUDA_OK(cudaSetDevice(d->ordinal));
    const PackedLayout L = packed_layout(p);
    cudaStream_t st = d->stream;
    if (!c->slice_buf) B200_CUDA_OK(cudaMalloc(&c->slice_buf, L.srcBytes + L.dstBytes));
    uint8_t *sb = (uint8_t *)c->slice_buf, *db = sb + L.srcBytes;
    if (srcSliceY == 0) { c->next_dst_y = 0; c->slice_open = true; }
    const int chrY = srcSliceY >> 1, chrH = -((-srcSliceH) >> 1);                       // AV_CEIL_RSHIFT
    B200_CUDA_OK(b200_h2d_rows(sb + L.yOff + (size_t)srcSliceY * L.yPitch, L.yPitch, srcSlice[0], srcStride[0], p.srcW, srcSliceH, st));
    const size_t cp1 = p.src_nv ? 2 * L.cPitch : L.cPitch;       // nv12 / nv21: plane 1 is twice as wide and holds both components
    B200_CUDA_OK(b200_h2d_rows(sb + L.uOff + (size_t)chrY * cp1, cp1, srcSlice[1], srcStride[1], p.src_nv ? 2 * p.chrSrcW : p.chrSrcW, chrH, st));
    if (!p.src_nv)
        B200_CUDA_OK(b200_h2d_rows(sb + L.vOff + (size_t)chrY * L.cPitch, L.cPitch, srcSlice[2], srcStride[2], p.chrSrcW, chrH, st));
    const uint8_t *sp[3] = { sb + L.yOff, sb + L.uOff, sb + L.vOff };
    const long long ss[3] = { (long long)L.yPitch, (long long)cp1, (long long)L.cPitch };
    const long long fs[3] = { 0, 0, 0 };
    int y0, y1;
    if (p.unscaled_lut) {                                   // convert_unscaled handles exactly the band it is given
        y0 = srcSliceY; y1 = srcSliceY + (srcSliceH & ~1);
    } else {
        y0 = c->next_dst_y;
        const int avail_l = srcSliceY + srcSliceH, avail_c = -((-(srcSliceY + srcSliceH)) >> 1);
        for (y1 = y0; y1 < p.dstH; y1++) {                  // "enough_lines", swscale.c:463-465
            const int firstLum = std::max(1 - p.vLum.size, p.vLum.pos[y1]);
            const int firstChr = std::max(1 - p.vChr.size, p.vChr.pos[y1]);
            const int lastLum = std::min(p.srcH, firstLum + p.vLum.size) - 1;
            const int lastChr = std::min(p.chrSrcH, firstChr + p.vChr.size) - 1;
            if (!(lastLum < avail_l && lastChr < avail_c)) break;
        }
        c->next_dst_y = y1;
    }
    const SwsRows R = { y0, y1 - y0, srcSliceY, srcSliceH, chrY, chrH };
    int ret = launch_batch(c, st, sp, ss, fs, db, (long long)L.dPitch, 0, 1, &R);
    if (ret < 0) return ret;
    if (y1 > y0 && sws_written_row_bytes(p))
        B200_CUDA_OK(b200_d2h_rows(dst[0] + (long long)y0 * dstStride[0], dstStride[0], db + (size_t)y0 * L.dPitch, L.dPitch,
                                   sws_written_row_bytes(p), y1 - y0, st));
    B200_CUDA_OK(cudaStreamSynchronize(st));
    if (srcSliceY + srcSliceH == p.srcH) c->slice_open = false;
    return p.unscaled_lut ? srcSliceH : y1 - y0;
}

B200_API int b200_sws_scale(B200SwsContext *c, const uint8_t *const srcSlice[], const int srcStride[],
                            int srcSliceY, int srcSliceH, uint8_t *const dst[], const int dstStride[])
{
    if (!c || !srcSlice || !srcStride || !dst || !dstStride) return B200_EINVAL;
    B200_LOCK_DEVICE(c->dev);      // contexts of one device share its stream and scratch (slice threads call N child contexts concurrently)
    const SwsPlan &p = c->plan;
    // Slice direction (scale_internal, libswscale/swscale.c:1096-1103): a sequence that starts with the band touching the bottom
    // of the picture runs bottom-up; the reference then flips the picture internally (:1141-1159: negated strides, pointers on the last
    // line of the band / of the destination, srcSliceY counted from the bottom) and so does this wrapper, band by band.
    if (!c->slice_open)
        c->slice_dir = (srcSliceY != 0 && srcSliceH != p.srcH && srcSliceY + srcSliceH == p.srcH && !p.src_rgb && !p.bgr24_yv12) ? -1 : 1;
    if (c->slice_dir == -1) {
        if ((p.srcH & 1) || (srcSliceH & 1) || (srcSliceY & 1) || srcSliceH <= 0 || srcSliceY < 0 || srcSliceY + srcSliceH > p.srcH ||
            (p.planar && (p.dstH & 1))) {
            b200_set_error("bottom-up slices: only even heights are implemented");
            return B200_ENOSYS;
        }
        const uint8_t *s2[4] = { srcSlice[0], srcSlice[1], p.src_nv ? nullptr : srcSlice[2], nullptr };
        int ss2[4] = { -srcStride[0], -srcStride[1], p.src_nv ? 0 : -srcStride[2], 0 };
        uint8_t *d2[4] = { dst[0], p.planar ? dst[1] : nullptr, p.planar && !p.dst_nv ? dst[2] : nullptr, nullptr };
        int ds2[4] = { -dstStride[0], p.planar ? -dstStride[1] : 0, p.planar && !p.dst_nv ? -dstStride[2] : 0, 0 };
        if (!s2[0] || !s2[1] || (!p.src_nv && !s2[2]) || !d2[0] || (p.planar && !d2[1]) || (p.planar && !p.dst_nv && !d2[2])) return B200_EINVAL;
        s2[0] += (long long)(srcSliceH - 1) * srcStride[0];
        s2[1] += (long long)((srcSliceH >> 1) - 1) * srcStride[1];
        if (s2[2]) s2[2] += (long long)((srcSliceH >> 1) - 1) * srcStride[2];
        d2[0] += (long long)(p.dstH - 1) * dstStride[0];
        if (d2[1]) d2[1] += (long long)((p.dstH >> 1) - 1) * dstStride[1];
        if (d2[2]) d2[2] += (long long)((p.dstH >> 1) - 1) * dstStride[2];
        const int yint = p.srcH - srcSliceY - srcSliceH;
        if (p.planar) return sws_scale_planar_host(c, s2, ss2, yint, srcSliceH, d2, ds2);
        return sws_scale_slice(c, s2, ss2, yint, srcSliceH, d2, ds2);
    }
    if (p.planar) return sws_scale_planar_host(c, srcSlice, srcStride, srcSliceY, srcSliceH, dst, dstStride);
    if (p.src_rgb && (srcSliceY != 0 || srcSliceH != p.srcH || c->slice_open)) {
        // packed RGB -> packed RGB, top-down slice sequence: bands accumulate in a device copy of the source, the picture is converted again
        // after each band and the lines whose vertical taps are complete (ff_swscale's "enough lines", swscale.c:463-465) are copied back
        if (srcSliceY + srcSliceH > p.srcH || srcSliceY < 0 || srcSliceH < 0) { b200_set_error("Slice parameters %d, %d are invalid", srcSliceY, srcSliceH); return B200_EINVAL; }
        if (srcSliceH == 0) return 0;
        if (!c->slice_open && srcSliceY != 0) { b200_set_error("Slices start in the middle!"); return B200_EINVAL; }
        if (!srcSlice[0] || !dst[0]) return B200_EINVAL;
        B200Device *dv = c->dev;
        B200_CUDA_OK(cudaSetDevice(dv->ordinal));
        const size_t sPitch = ((size_t)p.srcW * p.src_rgb + 255) & ~(size_t)255, dPitch = ((size_t)p.dstW * p.out.bpp + 255) & ~(size_t)255;
        if (p.rgb_shuffle) {                                      // convert_unscaled handles exactly the band it is given
            B200_LOCK_DEVICE(dv);
            uint8_t *scr3 = (uint8_t *)b200_scratch(dv, (sPitch + dPitch) * (size_t)srcSliceH);
            if (!scr3) return B200_ENOMEM;
            uint8_t *dd3 = scr3 + sPitch * (size_t)srcSliceH;
            cudaStream_t st3 = dv->stream;
            B200_CUDA_OK(b200_h2d_rows(scr3, sPitch, srcSlice[0], srcStride[0], (size_t)p.srcW * p.src_rgb, srcSliceH, st3));
            launch_rgb_shuffle(p, st3, scr3, (long long)sPitch, 0, dd3, (long long)dPitch, 0, srcSliceH, 1);
            B200_CUDA_OK(cudaGetLastError());
            B200_CUDA_OK(b200_d2h_rows(dst[0] + (long long)srcSliceY * dstStride[0], dstStride[0], dd3, dPitch, (size_t)p.dstW * p.out.bpp, srcSliceH, st3));
            B200_CUDA_OK(cudaStreamSynchronize(st3));
            c->slice_open = srcSliceY + srcSliceH < p.srcH;
            return srcSliceH;
        }
        cudaStream_t st2 = dv->stream;
        if (!c->slice_buf) {
            B200_CUDA_OK(cudaMalloc(&c->slice_buf, sPitch * p.srcH + dPitch * p.dstH));
            B200_CUDA_OK(cudaMemsetAsync(c->slice_buf, 0, sPitch * p.srcH + dPitch * p.dstH, st2));
        }
        uint8_t *sb = (uint8_t *)c->slice_buf, *db = sb + sPitch * p.srcH;
        if (srcSliceY == 0) { c->next_dst_y = 0; c->slice_open = true; }
        B200_CUDA_OK(b200_h2d_rows(sb + (size_t)srcSliceY * sPitch, sPitch, srcSlice[0], srcStride[0], (size_t)p.srcW * p.src_rgb, srcSliceH, st2));
        const int y0 = c->next_dst_y, avail = srcSliceY + srcSliceH;
        int y1;
        for (y1 = y0; y1 < p.dstH; y1++) {
            const int firstLum = std::max(1 - p.vLum.size, p.vLum.pos[y1]), firstChr = std::max(1 - p.vChr.size, p.vChr.pos[y1]);
            const int lastLum = std::min(p.srcH, firstLum + p.vLum.size) - 1, lastChr = std::min(p.chrSrcH, firstChr + p.vChr.size) - 1;
            if (!(lastLum < avail && lastChr < avail)) break;
        }
        c->next_dst_y = y1;
        if (y1 > y0) {
            const int r2 = launch_rgbsrc_packed(c, st2, sb, (long long)sPitch, 0, db, (long long)dPitch, 0, 1);
            if (r2 < 0) return r2;
            B200_CUDA_OK(b200_d2h_rows(dst[0] + (long long)y0 * dstStride[0], dstStride[0], db + (size_t)y0 * dPitch, dPitch, (size_t)p.dstW * p.out.bpp, y1 - y0, st2));
        }
        B200_CUDA_OK(cudaStreamSynchronize(st2));
        if (avail == p.srcH) c->slice_open = false;
        return y1 - y0;
    }
    if (p.src_rgb) {                                              // packed RGB -> packed RGB: a whole frame
        if (!srcSlice[0] || !dst[0]) return B200_EINVAL;
        if (srcStride[0] < 0 || dstStride[0] < 0) return B200_ENOSYS;
        B200Device *dv = c->dev;
        B200_CUDA_OK(cudaSetDevice(dv->ordinal));
        const size_t sPitch = ((size_t)p.srcW * p.src_rgb + 255) & ~(size_t)255, dPitch = ((size_t)p.dstW * p.out.bpp + 255) & ~(size_t)255;
        B200_LOCK_DEVICE(dv);      // scratch + stream are per device: one host-pointer call at a time (released on return)
        uint8_t *scr2 = (uint8_t *)b200_scratch(dv, sPitch * p.srcH + dPitch * p.dstH);
        if (!scr2) return B200_ENOMEM;
        cudaStream_t st2 = dv->stream;
        B200_CUDA_OK(cudaMemcpy2DAsync(scr2, sPitch, srcSlice[0], (size_t)srcStride[0], (size_t)p.srcW * p.src_rgb, p.srcH, cudaMemcpyHostToDevice, st2));
        uint8_t *dd2 = scr2 + sPitch * p.srcH;
        const int r2 = launch_rgbsrc_packed(c, st2, scr2, (long long)sPitch, 0, dd2, (long long)dPitch, 0, 1);
        if (r2 < 0) return r2;
        B200_CUDA_OK(cudaMemcpy2DAsync(dst[0], (size_t)dstStride[0], dd2, dPitch, (size_t)p.dstW * p.out.bpp, p.dstH, cudaMemcpyDeviceToHost, st2));
        B200_CUDA_OK(cudaStreamSynchronize(st2));
        return p.dstH;
    }
    if (srcSliceY != 0 || srcSliceH != p.srcH)
        return sws_scale_slice(c, srcSlice, srcStride, srcSliceY, srcSliceH, dst, dstStride);
    c->slice_open = false;
    B200Device *d = c->dev;
    B200_CUDA_OK(cudaSetDevice(d->ordinal));
    const PackedLayout L = packed_layout(p);
    uint8_t *scr = (uint8_t *)b200_scratch(d, L.srcBytes + L.dstBytes);
    if (!scr) return B200_ENOMEM;
    cudaStream_t st = d->stream;
    const int nsp = p.src_nv ? 2 : 3;                             // nv12 / nv21: plane 1 carries both chroma components
    const int wbytes[3] = { p.srcW, p.src_nv ? 2 * p.chrSrcW : p.chrSrcW, p.chrSrcW }, rows[3] = { p.srcH, p.chrSrcH, p.chrSrcH };
    const size_t pitch[3] = { L.yPitch, p.src_nv ? 2 * L.cPitch : L.cPitch, L.cPitch }, poff[3] = { L.yOff, L.uOff, L.vOff };
    const uint8_t *sp[3] = { nullptr, nullptr, nullptr }; long long ss[3] = { 0, 0, 0 };
    for (int pl = 0; pl < nsp; pl++) {
        const long long hs = srcStride[pl];
        const long long habs = hs < 0 ? -hs : hs;
        // negative stride (bottom-up, swscale.c:1141-1159): copy from the lowest address, walk upwards on the device
        const uint8_t *lo = hs < 0 ? srcSlice[pl] + (long long)(rows[pl] - 1) * hs : srcSlice[pl];
        B200_CUDA_OK(cudaMemcpy2DAsync(scr + poff[pl], pitch[pl], lo, (size_t)habs, wbytes[pl], rows[pl], cudaMemcpyHostToDevice, st));
        sp[pl] = hs < 0 ? scr + poff[pl] + (size_t)(rows[pl] - 1) * pitch[pl] : scr + poff[pl];
        ss[pl] = hs < 0 ? -(long long)pitch[pl] : (long long)pitch[pl];
    }
    const long long fs[3] = { 0, 0, 0 };
    uint8_t *dd = scr + L.srcBytes;
    int ret = launch_batch(c, st, sp, ss, fs, dd, (long long)L.dPitch, 0, 1);
    if (ret < 0) return ret;
    const long long dsl = dstStride[0];
    const long long dabs = dsl < 0 ? -dsl : dsl;
    const size_t wb = sws_written_row_bytes(p);
    if (!wb) {
        // a one-pixel-wide picture through the pair-wise converter: nothing is written
    } else if (dsl < 0) {
        // flip while copying back: row r of the device picture goes to dst[0] + r*dsl
        for (int r = 0; r < p.dstH; r++)
            B200_CUDA_OK(cudaMemcpyAsync(dst[0] + (long long)r * dsl, dd + (size_t)r * L.dPitch, wb, cudaMemcpyDeviceToHost, st));
    } else {
        B200_CUDA_OK(cudaMemcpy2DAsync(dst[0], (size_t)dabs, dd, L.dPitch, wb, p.dstH, cudaMemcpyDeviceToHost, st));
    }
    B200_CUDA_OK(cudaStreamSynchronize(st));
    return p.dstH;
}

B200_API int b200_sws_func(void *c, const uint8_t *const src[], const int srcStride[], int srcSliceY, int srcSliceH,
                           uint8_t *const dst[], const int dstStride[])
{
    return b200_sws_scale((B200SwsContext *)c, src, srcStride, srcSliceY, srcSliceH, dst, dstStride);
}
