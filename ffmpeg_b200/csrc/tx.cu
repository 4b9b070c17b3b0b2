// tx.cu — libavutil/tx float32 power-of-two FFT and MDCT on sm_90a: kernels + the C ABI (include/b200dsp.h, "tx").
//
// Reference semantics reproduced with the SAME float operation order, so results are bit-identical to the
// *_float_c codelets (checker: oracle/tx_oracle.c; build uses --fmad=false so no product/sum is contracted):
//   ff_tx_fft{2..131072}_ns, ff_tx_fft_sr_combine   libavutil/tx_template.c:562-722
//   ff_tx_fft (permute + codelet)                   libavutil/tx_template.c:763-778
//   ff_tx_mdct_fwd / ff_tx_mdct_inv                 libavutil/tx_template.c:1273-1342
//   tables: ff_tx_init_tab_N (:65-77), ff_tx_mdct_gen_exp (:2107-2134), ff_tx_gen_ptwo_revtab (tx.c:125-154)
//
// The reference's recursion  fft(S) = fft(S/2) | fft(S/4) | fft(S/4) ; combine(S)  is flattened into levels: all
// blocks of one size are independent, so a CTA keeps one transform in shared memory and sweeps S = 2, 4, ..., N with
// one barrier per level.  The hard-coded base cases are instances of the same rule (fft4 = fft2 + butterflies,
// fft8 = fft4 + 2 fft2 + combine, fft16 = fft8 + 2 fft4 + combine) except that for S <= 16 the j = 0 butterfly
// skips the multiplication by (1, 0); that distinction is kept.
// HBM traffic per transform is the algorithmic 8N in + 8N out (FFT) or 4*len in + 4*len out (iMDCT).
#include "common.h"
#include "tx_pfa.h"
#include "tx_double.h"
#include "tx_dct.h"
#include "tx_int32.h"
#include "tx_r16.h"
#include <vector>
#include <cmath>
#include <cstring>
#include <new>

namespace {

struct TxDev {                 // device-side plan
    int n;                     // complex FFT points
    int nlevels;               // levels S = 2^1 .. 2^nlevels
    const int *blk_off;        // block offsets, all levels concatenated
    int lvl_start[18], lvl_cnt[18];
    const float *tab;          // cosine tables, tab_off[k] = start of tab_{2^k}
    int tab_off[18];
    const int *leaf16; int n_leaf16;   // offsets of the size-16 blocks (done in registers)
    const int *leaf8;  int n_leaf8;    // offsets of size-8 blocks that are not part of a size-16 block
    const int *bfd;            // levels >= 5: padded index of the first element of every butterfly, all levels concatenated
    const float2 *tw2;         // levels >= 5: (tab_S[j], tab_S[S/4 - j]) pairs
    int bfd_start[18], tw2_start[18];
    const int *scatter;        // FFT: z[scatter[g]] = src[g]
    const int *imap;           // inverse MDCT: z[imap[m]] gets the pair (in[len-1-2m], in[2m])
    const int *sub_map;        // MDCT index map (doubled for the inverse)
    const float2 *exp;         // MDCT twiddles
    int len;                   // MDCT / RDFT length (2n)
    const float *rexp;         // RDFT: 8 factors, then tcos[len/4], tsin[len/4] (ff_tx_rdft_init, tx_template.c:1601-1653)
};

__device__ __forceinline__ void butterflies(float2 &a0, float2 &a1, float2 &a2, float2 &a3, float t1, float t2, float t5, float t6)
{
    const float r0 = a0.x, i0 = a0.y, r1 = a1.x, i1 = a1.y;
    const float t3 = t5 - t1; t5 = t5 + t1;
    a2.x = r0 - t5; a0.x = r0 + t5;
    a3.y = i1 - t3; a1.y = i1 + t3;
    const float t4 = t2 - t6; t6 = t2 + t6;
    a3.x = r1 - t4; a1.x = r1 + t4;
    a2.y = i0 - t6; a0.y = i0 + t6;
}

// shared-memory index with one pad element per 16 (kills the bank conflicts of the bit-reversal-like scatter)
__device__ __forceinline__ int PAD(int i) { return i + (i >> 4); }

__device__ __forceinline__ void fft2r(float2 &a, float2 &b)
{
    const float2 s0 = a, s1 = b;
    a = make_float2(s0.x + s1.x, s0.y + s1.y);
    b = make_float2(s0.x - s1.x, s0.y - s1.y);
}
__device__ __forceinline__ void bfly_nomul(float2 &a0, float2 &a1, float2 &a2, float2 &a3) { butterflies(a0, a1, a2, a3, a2.x, a2.y, a3.x, a3.y); }
__device__ __forceinline__ void bfly_mul(float2 &a0, float2 &a1, float2 &a2, float2 &a3, float wre, float wim)
{
    const float t1 = a2.x * wre - a2.y * (-wim);
    const float t2 = a2.x * (-wim) + a2.y * wre;
    const float t5 = a3.x * wre - a3.y * wim;
    const float t6 = a3.x * wim + a3.y * wre;
    butterflies(a0, a1, a2, a3, t1, t2, t5, t6);
}
// ff_tx_fft8_ns on v[0..7] (tx_template.c:660-679), c8 = tab_8[1]
__device__ __forceinline__ void leaf_fft8(float2 *v, float c8)
{
    fft2r(v[0], v[1]); fft2r(v[4], v[5]); fft2r(v[6], v[7]);
    bfly_nomul(v[0], v[1], v[2], v[3]);
    bfly_nomul(v[0], v[2], v[4], v[6]);
    bfly_mul(v[1], v[3], v[5], v[7], c8, c8);
}
// ff_tx_fft16_ns on v[0..15] (tx_template.c:681-704)
__device__ __forceinline__ void leaf_fft16(float2 *v, float c8, float c1, float c2, float c3)
{
    leaf_fft8(v, c8);
    fft2r(v[8], v[9]);   bfly_nomul(v[8], v[9], v[10], v[11]);
    fft2r(v[12], v[13]); bfly_nomul(v[12], v[13], v[14], v[15]);
    bfly_nomul(v[0], v[4], v[8], v[12]);
    bfly_mul(v[2], v[6], v[10], v[14], c2, c2);
    bfly_mul(v[1], v[5], v[9], v[13], c1, c3);
    bfly_mul(v[3], v[7], v[11], v[15], c3, c1);
}

// All levels on TB transforms held in z[k*zs + PAD(0..n)), k < TB.  A CTA works on TB transforms at once so that the
// per-butterfly table word and twiddle pair are fetched once for TB butterflies and every barrier covers TB times
// more work (the loads of the TB inputs are also all in flight together).
template <int TB>
__device__ void fft_levels(const TxDev &p, float2 *z, int zs)
{
    int first = 1;
    if (p.nlevels >= 5) {                                  // sizes 2..16 in registers, one thread per leaf block
        const float c8 = __ldg(p.tab + p.tab_off[3] + 1);
        const float *t16 = p.tab + p.tab_off[4];
        const float c1 = __ldg(t16 + 1), c2 = __ldg(t16 + 2), c3 = __ldg(t16 + 3);
        const int nleaf = p.n_leaf16 + p.n_leaf8;
        for (int bb = threadIdx.x; bb < nleaf * TB; bb += blockDim.x) {
            const int k = bb / nleaf, b = bb - k * nleaf;
            float2 *zk = z + k * zs;
            float2 v[16];
            if (b < p.n_leaf16) {
                const int o = __ldg(p.leaf16 + b);
#pragma unroll
                for (int i = 0; i < 16; i++) v[i] = zk[PAD(o) + i];           // o is a multiple of 16: one pad run
                leaf_fft16(v, c8, c1, c2, c3);
#pragma unroll
                for (int i = 0; i < 16; i++) zk[PAD(o) + i] = v[i];
            } else {
                const int o = __ldg(p.leaf8 + b - p.n_leaf16);                // multiple of 8
#pragma unroll
                for (int i = 0; i < 8; i++) v[i] = zk[PAD(o) + i];
                leaf_fft8(v, c8);
#pragma unroll
                for (int i = 0; i < 8; i++) zk[PAD(o) + i] = v[i];
            }
        }
        __syncthreads();
        first = 5;
    }
    for (int L = first; L <= p.nlevels; L++) {
        const int S = 1 << L;
        const int *off = p.blk_off + p.lvl_start[L];
        if (L >= 5) {
            // one table word per butterfly (padded index of a0) and one float2 per twiddle pair; the other three elements
            // sit at fixed padded distances: k*q + (k*q >> 4) for q >= 16, and 8 / 17 / 25 for q == 8
            const int lq = L - 2, q = 1 << lq;
            const int d1 = q == 8 ? 8 : q + (q >> 4), d2 = q == 8 ? 17 : 2 * q + (q >> 3), d3 = q == 8 ? 25 : 3 * q + ((3 * q) >> 4);
            const int *bd = p.bfd + p.bfd_start[L];
            const float2 *tw = p.tw2 + p.tw2_start[L];
            const int total = p.lvl_cnt[L] << lq;
            for (int b = threadIdx.x; b < total; b += blockDim.x) {
                const int i0 = __ldg(bd + b);
                const float2 w = __ldg(tw + (b & (q - 1)));
#pragma unroll
                for (int k = 0; k < TB; k++) {
                    float2 *zk = z + k * zs + i0;
                    float2 a0 = zk[0], a1 = zk[d1], a2 = zk[d2], a3 = zk[d3];
                    bfly_mul(a0, a1, a2, a3, w.x, w.y);
                    zk[0] = a0; zk[d1] = a1; zk[d2] = a2; zk[d3] = a3;
                }
            }
            __syncthreads();
            continue;
        }
        for (int k = 0; k < TB; k++) {
            float2 *zk = z + k * zs;
            if (L == 1) {
                for (int b = threadIdx.x; b < p.lvl_cnt[L]; b += blockDim.x) {
                    const int o = __ldg(off + b);
                    fft2r(zk[PAD(o)], zk[PAD(o + 1)]);
                }
            } else {
                const int lq = L - 2, q = 1 << lq;
                const float *tab = p.tab + p.tab_off[L];
                const int total = p.lvl_cnt[L] << lq;
                for (int b = threadIdx.x; b < total; b += blockDim.x) {
                    const int o = __ldg(off + (b >> lq)), j = b & (q - 1);
                    const int i0 = PAD(o + j), i1 = PAD(o + q + j), i2 = PAD(o + 2 * q + j), i3 = PAD(o + 3 * q + j);
                    float2 a0 = zk[i0], a1 = zk[i1], a2 = zk[i2], a3 = zk[i3];
                    if (S <= 16 && j == 0) bfly_nomul(a0, a1, a2, a3);
                    else bfly_mul(a0, a1, a2, a3, __ldg(tab + j), __ldg(tab + q - j));
                    zk[i0] = a0; zk[i1] = a1; zk[i2] = a2; zk[i3] = a3;
                }
            }
        }
        __syncthreads();
    }
}

// TB transforms per CTA; steps are in BYTES between consecutive transforms
template <int TB>
__global__ void __launch_bounds__(256)
tx_fft_kernel(TxDev p, float2 *out, const float2 *in, long long out_step, long long in_step, long long count)
{
    extern __shared__ float2 z[];
    const int zs = p.n + (p.n >> 4) + 1;
    const long long t0 = (long long)blockIdx.x * TB;
#pragma unroll
    for (int k = 0; k < TB; k++) {
        if (t0 + k >= count) break;
        const float2 *src = reinterpret_cast<const float2 *>(reinterpret_cast<const char *>(in) + (t0 + k) * in_step);
        for (int g = threadIdx.x; g < p.n; g += blockDim.x) z[k * zs + PAD(__ldg(p.scatter + g))] = src[g];
    }
    __syncthreads();
    fft_levels<TB>(p, z, zs);
#pragma unroll
    for (int k = 0; k < TB; k++) {
        if (t0 + k >= count) break;
        float2 *dst = reinterpret_cast<float2 *>(reinterpret_cast<char *>(out) + (t0 + k) * out_step);
        for (int i = threadIdx.x; i < p.n; i += blockDim.x) dst[i] = z[k * zs + PAD(i)];
    }
}

// ff_tx_rdft_r2c / ff_tx_rdft_c2r (DECL_RDFT, tx_template.c:1655-1724): the even/odd separation butterfly on the pair
// (data[i], data[len2 - i]), 1 <= i < len4, and the two special elements 0 and len4.
__device__ __forceinline__ void rdft_pair(const float *fact, float tc, float ts, float2 &a, float2 &b)
{
    const float t0re = fact[4] * (a.x + b.x), t0im = fact[5] * (a.y - b.y);
    const float t1re = fact[6] * (a.y + b.y), t1im = fact[7] * (a.x - b.x);
    const float t2re = t1re * tc - t1im * ts, t2im = t1re * ts + t1im * tc;
    a = make_float2(t0re + t2re, t2im - t0im);
    b = make_float2(t0re - t2re, t2im + t0im);
}
__device__ __forceinline__ void rdft_special(const float *fact, float2 &d0, float2 &dq)
{
    const float t0re = d0.x;
    d0.x = t0re + d0.y; d0.y = t0re - d0.y;
    d0.x = fact[0] * d0.x; d0.y = fact[1] * d0.y;
    dq.x = fact[2] * dq.x; dq.y = fact[3] * dq.y;
}

// r2c: len floats in, len/2 + 1 complex out
template <int TB>
__global__ void __launch_bounds__(256)
tx_rdft_r2c_kernel(TxDev p, float2 *out, const float2 *in, long long out_step, long long in_step, long long count)
{
    extern __shared__ float2 z[];
    const int zs = p.n + (p.n >> 4) + 1;
    const long long t0 = (long long)blockIdx.x * TB;
    const int len2 = p.n, len4 = p.n >> 1;
#pragma unroll
    for (int k = 0; k < TB; k++) {
        if (t0 + k >= count) break;
        const float2 *src = reinterpret_cast<const float2 *>(reinterpret_cast<const char *>(in) + (t0 + k) * in_step);
        for (int g = threadIdx.x; g < p.n; g += blockDim.x) z[k * zs + PAD(__ldg(p.scatter + g))] = src[g];
    }
    __syncthreads();
    fft_levels<TB>(p, z, zs);
    const float *fact = p.rexp, *tcos = fact + 8, *tsin = tcos + len4;
#pragma unroll
    for (int k = 0; k < TB; k++) {
        float2 *zk = z + k * zs;
        for (int i = threadIdx.x; i < max(len4, 1); i += blockDim.x) {
            if (i == 0) {
                float2 d0 = zk[PAD(0)], dq = zk[PAD(len4)];
                rdft_special(fact, d0, dq);
                if (len4 > 0) zk[PAD(len4)] = dq;
                zk[PAD(0)] = d0;
            } else {
                float2 a = zk[PAD(i)], b = zk[PAD(len2 - i)];
                rdft_pair(fact, __ldg(tcos + i), __ldg(tsin + i), a, b);
                zk[PAD(i)] = a; zk[PAD(len2 - i)] = b;
            }
        }
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < TB; k++) {
        if (t0 + k >= count) break;
        float2 *dst = reinterpret_cast<float2 *>(reinterpret_cast<char *>(out) + (t0 + k) * out_step);
        const float2 *zk = z + k * zs;
        for (int i = threadIdx.x; i <= len2; i += blockDim.x) {
            float2 v;
            if (i == 0) v = make_float2(zk[PAD(0)].x, 0.0f);
            else if (i == len2) v = make_float2(zk[PAD(0)].y, 0.0f);          // data[len2].re = data[0].im
            else v = zk[PAD(i)];
            dst[i] = v;
        }
    }
}

// c2r: len/2 + 1 complex in, len floats out.  The reference modifies its input in place before the inverse FFT; the
// modified values are written to `wb` when it is not NULL (the host av_tx_fn path hands them back to the caller).
template <int TB>
__global__ void __launch_bounds__(256)
tx_rdft_c2r_kernel(TxDev p, float2 *out, const float2 *in, float2 *wb, long long out_step, long long in_step, long long count)
{
    extern __shared__ float2 z[];
    const int zs = p.n + (p.n >> 4) + 1;
    const long long t0 = (long long)blockIdx.x * TB;
    const int len2 = p.n, len4 = p.n >> 1;
    const float *fact = p.rexp, *tcos = fact + 8, *tsin = tcos + len4;
#pragma unroll
    for (int k = 0; k < TB; k++) {
        if (t0 + k >= count) break;
        const float2 *src = reinterpret_cast<const float2 *>(reinterpret_cast<const char *>(in) + (t0 + k) * in_step);
        float2 *w = wb ? reinterpret_cast<float2 *>(reinterpret_cast<char *>(wb) + (t0 + k) * in_step) : nullptr;
        float2 *zk = z + k * zs;
        for (int i = threadIdx.x; i < max(len4, 1); i += blockDim.x) {
            if (i == 0) {
                float2 d0 = src[0], dq = src[len4];
                d0.y = src[len2].x;                                           // data[0].im = data[len2].re
                rdft_special(fact, d0, dq);
                zk[PAD(__ldg(p.scatter + 0))] = d0;
                if (len4 > 0) zk[PAD(__ldg(p.scatter + len4))] = dq;
                if (w) { w[0] = d0; if (len4 > 0) w[len4] = dq; }
            } else {
                float2 a = src[i], b = src[len2 - i];
                rdft_pair(fact, __ldg(tcos + i), __ldg(tsin + i), a, b);
                zk[PAD(__ldg(p.scatter + i))] = a; zk[PAD(__ldg(p.scatter + len2 - i))] = b;
                if (w) { w[i] = a; w[len2 - i] = b; }
            }
        }
    }
    __syncthreads();
    fft_levels<TB>(p, z, zs);
#pragma unroll
    for (int k = 0; k < TB; k++) {
        if (t0 + k >= count) break;
        float2 *dst = reinterpret_cast<float2 *>(reinterpret_cast<char *>(out) + (t0 + k) * out_step);
        for (int i = threadIdx.x; i < p.n; i += blockDim.x) dst[i] = z[k * zs + PAD(i)];
    }
}

// ff_tx_mdct_inv: len floats in (element k at in + k*stride floats), len floats out (contiguous)
template <int TB>
__global__ void __launch_bounds__(256)
tx_mdct_inv_kernel(TxDev p, float *out, const float *in, long long stride, long long out_step, long long in_step, long long count)
{
    extern __shared__ float2 z[];
    const int zs = p.n + (p.n >> 4) + 1;
    const long long t0 = (long long)blockIdx.x * TB;
    const int len2 = p.len >> 1, len4 = p.len >> 2;
    const float2 *e = p.exp + len2;                         // twiddles in natural order
#pragma unroll
    for (int k = 0; k < TB; k++) {
        if (t0 + k >= count) break;
        const float *src = reinterpret_cast<const float *>(reinterpret_cast<const char *>(in) + (t0 + k) * in_step);
        const float *in1 = src, *in2 = src + (long long)(len2 * 2 - 1) * stride;
        for (int m = threadIdx.x; m < len2; m += blockDim.x) {  // source order (coalesced reads), scattered into z
            const float are = in2[-(long long)(2 * m) * stride], aim = in1[(long long)(2 * m) * stride];
            const float2 w = __ldg(e + m);
            z[k * zs + PAD(__ldg(p.imap + m))] = make_float2(are * w.x - aim * w.y, are * w.y + aim * w.x);
        }
    }
    __syncthreads();
    fft_levels<TB>(p, z, zs);
#pragma unroll
    for (int k = 0; k < TB; k++) {
        float2 *zk = z + k * zs;
        for (int i = threadIdx.x; i < len4; i += blockDim.x) {
            const int i0 = len4 + i, i1 = len4 - i - 1;
            const float2 z1 = zk[PAD(i1)], z0 = zk[PAD(i0)], e1 = __ldg(e + i1), e0 = __ldg(e + i0);
            const float s1re = z1.y, s1im = z1.x, s0re = z0.y, s0im = z0.x;
            float2 o1, o0;
            o1.x = s1re * e1.y - s1im * e1.x;      // z[i1].re
            o0.y = s1re * e1.x + s1im * e1.y;      // z[i0].im
            o0.x = s0re * e0.y - s0im * e0.x;      // z[i0].re
            o1.y = s0re * e0.x + s0im * e0.y;      // z[i1].im
            zk[PAD(i1)] = o1; zk[PAD(i0)] = o0;
        }
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < TB; k++) {
        if (t0 + k >= count) break;
        float2 *dst = reinterpret_cast<float2 *>(reinterpret_cast<char *>(out) + (t0 + k) * out_step);
        for (int i = threadIdx.x; i < len2; i += blockDim.x) dst[i] = z[k * zs + PAD(i)];
    }
}

// ff_tx_mdct_fwd: 2*len floats in (contiguous), len floats out (element k at out + k*stride floats)
template <int TB>
__global__ void __launch_bounds__(256)
tx_mdct_fwd_kernel(TxDev p, float *out, const float *in, long long stride, long long out_step, long long in_step, long long count)
{
    extern __shared__ float2 z[];
    const int zs = p.n + (p.n >> 4) + 1;
    const long long t0 = (long long)blockIdx.x * TB;
    const int len2 = p.len >> 1, len4 = p.len >> 2, len3 = len2 * 3;
#pragma unroll
    for (int k = 0; k < TB; k++) {
        if (t0 + k >= count) break;
        const float *src = reinterpret_cast<const float *>(reinterpret_cast<const char *>(in) + (t0 + k) * in_step);
        for (int i = threadIdx.x; i < len2; i += blockDim.x) {
            const int kk = 2 * i, idx = __ldg(p.sub_map + i);
            float re, im;
            if (kk < len2) {
                re = -src[len2 + kk] + src[1 * len2 - 1 - kk];
                im = -src[len3 + kk] + -src[1 * len3 - 1 - kk];
            } else {
                re = -src[len2 + kk] + -src[5 * len2 - 1 - kk];
                im = src[-len2 + kk] + -src[1 * len3 - 1 - kk];
            }
            const float2 ee = __ldg(p.exp + i);
            z[k * zs + PAD(idx)] = make_float2(re * ee.y + im * ee.x, re * ee.x - im * ee.y); // (.re, .im) = (dim, dre) of the reference's CMUL
        }
    }
    __syncthreads();
    fft_levels<TB>(p, z, zs);
#pragma unroll
    for (int k = 0; k < TB; k++) {
        if (t0 + k >= count) break;
        float *dst = reinterpret_cast<float *>(reinterpret_cast<char *>(out) + (t0 + k) * out_step);
        const float2 *zk = z + k * zs;
        for (int i = threadIdx.x; i < len4; i += blockDim.x) {
            const int i0 = len4 + i, i1 = len4 - i - 1;
            const float2 s1 = zk[PAD(i1)], s0 = zk[PAD(i0)], e1 = __ldg(p.exp + i1), e0 = __ldg(p.exp + i0);
            dst[(2LL * i1 + 1) * stride] = s0.x * e0.y - s0.y * e0.x;
            dst[(2LL * i0) * stride]     = s0.x * e0.x + s0.y * e0.y;
            dst[(2LL * i0 + 1) * stride] = s1.x * e1.y - s1.y * e1.x;
            dst[(2LL * i1) * stride]     = s1.x * e1.x + s1.y * e1.y;
        }
    }
}

int sr_perm(int i, int len, int inv)       // split_radix_permutation, tx.c:125-134
{
    len >>= 1;
    if (len <= 1) return i & 1;
    if (!(i & len)) return sr_perm(i, len, inv) * 2;
    len >>= 1;
    return sr_perm(i, len, inv) * 4 + 1 - 2 * (!(i & len) ^ inv);
}

void collect_blocks(std::vector<std::vector<int>> &lv, int L, int off)   // block of size 2^L at `off`
{
    if (L < 1) return;
    lv[L].push_back(off);
    const int S = 1 << L;
    collect_blocks(lv, L - 1, off);
    if (L >= 2) {
        collect_blocks(lv, L - 2, off + S / 2);
        collect_blocks(lv, L - 2, off + 3 * S / 4);
    }
}

} // namespace

struct B200TXContext {
    B200Device *dev = nullptr;
    TxPfa *pfa = nullptr;            // compound 15 x M MDCT (tx_pfa.cu): everything below d is unused then
    TxDct *dct = nullptr;            // AV_TX_FLOAT_DCT (tx_dct.cu): stages around a child RDFT context
    TxI32 *i32 = nullptr;            // AV_TX_INT32_FFT / _MDCT (tx_int32.cu)
    TxDbl *dbl = nullptr;            // AV_TX_DOUBLE_FFT / _MDCT (tx_double.cu)
    TxR16 *r16 = nullptr;            // 512 ... 4096-point FFT / inverse MDCT: register-resident passes (tx_r16.cu), else the kernels below
    int type = 0, inv = 0, len = 0;
    bool full = false;               // AV_TX_FULL_IMDCT: ff_tx_mdct_inv_full around the inverse MDCT (tx_template.c:1372-1413)
    TxDev d{};
    void *blob = nullptr;
    size_t smem = 0;
    int tb = 1;
};

static int tx_build(B200TXContext *c, float scale)
{
    const int n = c->type == 0 ? c->len : c->len >> 1;
    int k = 0;
    while ((1 << k) < n) k++;
    TxDev &d = c->d;
    d.n = n; d.nlevels = k; d.len = c->len;
    std::vector<std::vector<int>> lv(18);
    collect_blocks(lv, k, 0);
    std::vector<int> leaf16 = lv[4], leaf8;
    for (int o : lv[3]) {                                            // size-8 blocks that are quarter blocks of a size-32 block
        bool inside16 = false;
        for (int o16 : lv[4]) if (o >= o16 && o < o16 + 16) { inside16 = true; break; }
        if (!inside16) leaf8.push_back(o);
    }
    std::vector<int> blk;
    for (int L = 0; L < 18; L++) {
        d.lvl_start[L] = (int)blk.size();
        d.lvl_cnt[L] = (int)lv[L].size();
        blk.insert(blk.end(), lv[L].begin(), lv[L].end());
    }
    std::vector<float> tab;
    for (int L = 0; L < 18; L++) {
        d.tab_off[L] = (int)tab.size();
        if (L >= 3 && L <= k) {                                      // ff_tx_init_tab_N, tx_template.c:65-77
            const int N = 1 << L;
            const double freq = 2 * M_PI / N;
            for (int i = 0; i < N / 4; i++) tab.push_back((float)cos(i * freq));
            tab.push_back(0.0f);
        } else if (L == 2) {                                         // never multiplied (S <= 16, j == 0 only) but keep indexing valid
            tab.push_back(1.0f); tab.push_back(0.0f);
        }
    }
    std::vector<int> gather(n), scatter(n), sub_map;
    const bool mdct_scatter = c->type == 1 && !c->inv;               // ff_tx_mdct_init: map_dir = !inv ? SCATTER : GATHER
    for (int i = 0; i < n; i++) {
        const int p = n == 1 ? 0 : (-sr_perm(i, n, c->inv)) & (n - 1);
        if (mdct_scatter) gather[p] = i; else gather[i] = p;
    }
    for (int i = 0; i < n; i++) scatter[gather[i]] = i;              // dst[i] = src[gather[i]]  <=>  dst[scatter[g]] = src[g]
    std::vector<float2> ex;
    if (c->type == 1) {                                              // ff_tx_mdct_gen_exp, tx_template.c:2107-2134
        const int len4 = c->len >> 1;
        const double sc = (double)scale;
        const double theta = (sc < 0 ? len4 : 0) + 1.0 / 8.0;
        const double amp = sqrt(fabs(sc));
        std::vector<float2> full(len4);
        for (int i = 0; i < len4; i++) {
            const double alpha = M_PI_2 * (i + theta) / len4;
            full[i] = make_float2((float)(cos(alpha) * amp), (float)(sin(alpha) * amp));
        }
        sub_map.resize(len4);
        if (c->inv) {
            ex.resize(2 * (size_t)len4);
            for (int i = 0; i < len4; i++) { ex[len4 + i] = full[i]; ex[i] = full[gather[i]]; sub_map[i] = gather[i] << 1; }
            c->r16 = tx_r16_create(1, n, gather.data(), full.data(), c->dev->sm_count);
        } else {
            ex = full;
            for (int i = 0; i < len4; i++) sub_map[i] = gather[i];
        }
    }
    if (c->type == 0) c->r16 = tx_r16_create(0, n, gather.data(), nullptr, c->dev->sm_count);
    auto al = [](size_t v) { return (v + 255) & ~(size_t)255; };
    size_t off = 0;
    const size_t o_blk = off; off += al(blk.size() * 4);
    const size_t o_tab = off; off += al(tab.size() * 4);
    const size_t o_sc = off;  off += al(scatter.size() * 4);
    const size_t o_sm = off;  off += al(sub_map.size() * 4 + 4);
    const size_t o_ex = off;  off += al(ex.size() * 8 + 8);
    std::vector<int> bfd;
    std::vector<float2> tw2;
    for (int L = 0; L < 18; L++) {
        d.bfd_start[L] = (int)bfd.size();
        d.tw2_start[L] = (int)tw2.size();
        if (L >= 5 && L <= k) {
            const int q = 1 << (L - 2);
            for (int o : lv[L])
                for (int j = 0; j < q; j++) bfd.push_back((o + j) + ((o + j) >> 4));
            const float *tb = &tab[d.tab_off[L]];
            for (int j = 0; j < q; j++) tw2.push_back(make_float2(tb[j], tb[q - j]));
        }
    }
    const size_t o_bfd = off; off += al(bfd.size() * 4 + 4);
    const size_t o_tw2 = off; off += al(tw2.size() * 8 + 8);
    std::vector<float> rexp;
    if (c->type == 6) {                                              // ff_tx_rdft_init, tx_template.c:1601-1653
        const int len = c->len, len4 = len >> 2, inv = c->inv;
        const double f = 2 * M_PI / len, m = inv ? 2 * (double)scale : (double)scale;
        rexp.push_back((float)((inv ? 0.5 : 1.0) * m));
        rexp.push_back((float)(inv ? 0.5 * m : 1.0 * m));
        rexp.push_back((float)(m));
        rexp.push_back((float)(-m));
        rexp.push_back((float)((0.5 - 0.0) * m));
        rexp.push_back((float)((0.0 - 0.5) * m));
        rexp.push_back((float)((0.5 - inv) * m));
        rexp.push_back((float)(-(0.5 - inv) * m));
        for (int i = 0; i < len4; i++) rexp.push_back((float)cos(i * f));
        for (int i = 0; i < len4; i++) rexp.push_back((float)cos(((len - i * 4) / 4.0) * f) * (inv ? 1 : -1));
    }
    const size_t o_rx = off; off += al(rexp.size() * 4 + 4);
    std::vector<int> imap(sub_map.size() + 1, 0);
    if (c->type == 1 && c->inv)
        for (size_t i = 0; i < sub_map.size(); i++) imap[sub_map[i] >> 1] = (int)i;
    const size_t o_im = off;  off += al(imap.size() * 4);
    const size_t o_l16 = off; off += al(leaf16.size() * 4 + 4);
    const size_t o_l8 = off;  off += al(leaf8.size() * 4 + 4);
    std::vector<uint8_t> host(off, 0);
    memcpy(&host[o_blk], blk.data(), blk.size() * 4);
    memcpy(&host[o_tab], tab.data(), tab.size() * 4);
    memcpy(&host[o_sc], scatter.data(), scatter.size() * 4);
    if (!sub_map.empty()) memcpy(&host[o_sm], sub_map.data(), sub_map.size() * 4);
    if (!ex.empty()) memcpy(&host[o_ex], ex.data(), ex.size() * 8);
    if (!bfd.empty()) memcpy(&host[o_bfd], bfd.data(), bfd.size() * 4);
    if (!tw2.empty()) memcpy(&host[o_tw2], tw2.data(), tw2.size() * 8);
    memcpy(&host[o_im], imap.data(), imap.size() * 4);
    if (!leaf16.empty()) memcpy(&host[o_l16], leaf16.data(), leaf16.size() * 4);
    if (!leaf8.empty()) memcpy(&host[o_l8], leaf8.data(), leaf8.size() * 4);
    if (!rexp.empty()) memcpy(&host[o_rx], rexp.data(), rexp.size() * 4);
    B200_CUDA_OK(cudaMalloc(&c->blob, off));
    B200_CUDA_OK(cudaMemcpy(c->blob, host.data(), off, cudaMemcpyHostToDevice));
    uint8_t *b = (uint8_t *)c->blob;
    d.blk_off = (const int *)(b + o_blk); d.tab = (const float *)(b + o_tab); d.scatter = (const int *)(b + o_sc);
    d.sub_map = (const int *)(b + o_sm); d.exp = (const float2 *)(b + o_ex);
    d.imap = (const int *)(b + o_im);
    d.rexp = (const float *)(b + o_rx);
    d.bfd = (const int *)(b + o_bfd); d.tw2 = (const float2 *)(b + o_tw2);
    d.leaf16 = (const int *)(b + o_l16); d.n_leaf16 = (int)leaf16.size();
    d.leaf8 = (const int *)(b + o_l8); d.n_leaf8 = (int)leaf8.size();
    c->tb = n <= 1024 ? 4 : n <= 2048 ? 2 : 1;                     // transforms per CTA (about 35 KB of shared memory up to n = 2048)
    c->smem = (size_t)c->tb * (n + (n >> 4) + 1) * sizeof(float2);
    if (c->smem > 48 * 1024) {
#define TX_SMEM(K) B200_CUDA_OK(cudaFuncSetAttribute(K, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)c->smem))
#define TX_SMEM_ALL(TB) do { TX_SMEM(tx_fft_kernel<TB>); TX_SMEM(tx_mdct_inv_kernel<TB>); TX_SMEM(tx_mdct_fwd_kernel<TB>); \
                             TX_SMEM(tx_rdft_r2c_kernel<TB>); TX_SMEM(tx_rdft_c2r_kernel<TB>); } while (0)
        if (c->tb == 4) TX_SMEM_ALL(4); else if (c->tb == 2) TX_SMEM_ALL(2); else TX_SMEM_ALL(1);
#undef TX_SMEM_ALL
#undef TX_SMEM
    }
    return 0;
}

// ff_tx_mdct_inv_full (tx_template.c:1386-1398): the inverse MDCT has put its n outputs at out[n/2 .. 3n/2); the first and the last
// quarter of the 2n outputs are mirrors of them (the first one negated).  One thread per mirrored pair.
__global__ void __launch_bounds__(256)
tx_imdct_full_mirror_kernel(float *out, long long out_step_floats, int n, long long count)
{
    const int n2 = n >> 1;
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= count * n2) return;
    float *d = out + (t / n2) * out_step_floats;
    const int k = (int)(t % n2);
    d[k] = -d[n - k - 1];
    d[2 * n - k - 1] = d[n + k];
}

static int tx_launch_half(B200TXContext *c, cudaStream_t st, void *out, const void *in, ptrdiff_t stride, int64_t count,
                          ptrdiff_t out_step, ptrdiff_t in_step, void *c2r_writeback);

static int tx_launch(B200TXContext *c, cudaStream_t st, void *out, const void *in, ptrdiff_t stride, int64_t count,
                     ptrdiff_t out_step, ptrdiff_t in_step, void *c2r_writeback = nullptr)
{
    if (!c->full) return tx_launch_half(c, st, out, in, stride, count, out_step, in_step, c2r_writeback);
    if (count <= 0) return 0;
    if (out_step & 3) return B200_EINVAL;
    const int ret = tx_launch_half(c, st, (float *)out + (c->len >> 1), in, stride, count, out_step, in_step, nullptr);
    if (ret < 0) return ret;
    const long long per = 0x7fffffffLL * 256 / (c->len >> 1);        // transforms per launch (grid.x limit)
    for (int64_t c0 = 0; c0 < count; c0 += per) {
        const long long cnt = count - c0 < per ? count - c0 : per;
        const long long threads = cnt * (c->len >> 1);
        tx_imdct_full_mirror_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, st>>>((float *)((char *)out + c0 * out_step), out_step / 4, c->len, cnt);
        B200_LAUNCHED();
    }
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

static int tx_launch_half(B200TXContext *c, cudaStream_t st, void *out, const void *in, ptrdiff_t stride, int64_t count,
                          ptrdiff_t out_step, ptrdiff_t in_step, void *c2r_writeback)
{
    if (count <= 0) return 0;
    if (c->pfa) return tx_pfa_launch(c->pfa, st, out, in, stride, count, out_step, in_step);
    if (c->dct) return tx_dct_launch(c->dct, st, out, in, count, out_step, in_step);
    if (c->i32) return tx_i32_launch(c->i32, st, out, in, stride, count, out_step, in_step);
    if (c->dbl) return tx_dbl_launch(c->dbl, st, out, in, stride, count, out_step, in_step);
    if (c->r16 && (c->type == 0 || stride == 4) && tx_r16_accepts(c->r16, out, in, out_step, in_step))
        return tx_r16_launch(c->r16, st, out, in, out_step, in_step, count);
    const int threads = c->d.n >= 1024 ? 256 : c->d.n >= 256 ? 128 : 64;     // threads per CTA grow with the transform
    const long long per = 0x7fffffffLL / 4 * c->tb;              // transforms per launch (grid.x limit)
    for (int64_t c0 = 0; c0 < count; c0 += per) {
        const long long cnt = count - c0 < per ? count - c0 : per;
        const unsigned nb = (unsigned)((cnt + c->tb - 1) / c->tb);
        char *o = (char *)out + c0 * out_step;
        const char *i = (const char *)in + c0 * in_step;
#define TX_LAUNCH(TB)                                                                                                          \
        do {                                                                                                                   \
            if (c->type == 0)   tx_fft_kernel<TB><<<nb, threads, c->smem, st>>>(c->d, (float2 *)o, (const float2 *)i, out_step, in_step, cnt); \
            else if (c->type == 6 && !c->inv) tx_rdft_r2c_kernel<TB><<<nb, threads, c->smem, st>>>(c->d, (float2 *)o, (const float2 *)i, out_step, in_step, cnt); \
            else if (c->type == 6) tx_rdft_c2r_kernel<TB><<<nb, threads, c->smem, st>>>(c->d, (float2 *)o, (const float2 *)i, (float2 *)(c2r_writeback ? (char *)c2r_writeback + c0 * in_step : nullptr), out_step, in_step, cnt); \
            else if (c->inv)    tx_mdct_inv_kernel<TB><<<nb, threads, c->smem, st>>>(c->d, (float *)o, (const float *)i, stride / 4, out_step, in_step, cnt); \
            else                tx_mdct_fwd_kernel<TB><<<nb, threads, c->smem, st>>>(c->d, (float *)o, (const float *)i, stride / 4, out_step, in_step, cnt); \
        } while (0)
        if (c->tb == 4) TX_LAUNCH(4); else if (c->tb == 2) TX_LAUNCH(2); else TX_LAUNCH(1);
#undef TX_LAUNCH
        B200_LAUNCHED();
    }
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}

// av_tx_fn shaped entry: HOST pointers, one transform
static void tx_host_fn(B200TXContext *c, void *out, void *in, ptrdiff_t stride)
{
    if (c->i32) { tx_i32_host_fn(c->i32, out, in, stride); return; }
    if (c->dbl) { tx_dbl_host_fn(c->dbl, out, in, stride); return; }
    const size_t n = c->d.n, len = c->len;
    size_t in_elems, out_elems;            // floats
    if (c->dct) { in_elems = out_elems = (size_t)tx_dct_points(c->dct); }     // DCT-II: len in / len out; DCT-III: 2*len in / 2*len out
    else if (c->type == 0) { in_elems = out_elems = 2 * (c->pfa ? len : n); }
    else if (c->type == 6) { in_elems = c->inv ? len + 2 : len; out_elems = c->inv ? len : len + 2; }
    else if (c->inv) { in_elems = len; out_elems = c->full ? 2 * len : len; }
    else { in_elems = 2 * len; out_elems = len; }
    if (c->full && stride != 4) B200HostCall::fail("av_tx_fn", "AV_TX_FULL_IMDCT takes stride == sizeof(float) (the reference mirrors with the input stride)");
    B200HostCall call("av_tx_fn", c->dev, (in_elems + out_elems) * 4 + 512);
    float *din = (float *)call.scratch, *dout = din + ((in_elems + 63) & ~(size_t)63);
    cudaStream_t st = call.stream;
    cudaError_t e;
    const bool strided_in = c->type == 1 && c->inv && stride != 4;
    const bool strided_out = c->type == 1 && !c->inv && stride != 4;
    const bool strided_cpx = c->type == 0 && c->pfa && stride != 8;  // ff_tx_fft_pfa stores out[i * stride] (tx_template.c:1078-1079)
    if (strided_in) e = cudaMemcpy2DAsync(din, 4, in, (size_t)stride, 4, in_elems, cudaMemcpyHostToDevice, st);
    else e = cudaMemcpyAsync(din, in, in_elems * 4, cudaMemcpyHostToDevice, st);
    call.check(e, "h2d");
    const bool clobbers = c->type == 6 && c->inv;                    // ff_tx_rdft_c2r rewrites its input (tx_template.c:1670-1696)
    call.launched(tx_launch(c, st, dout, din, c->type == 0 ? 8 : 4, 1, 0, 0, clobbers ? din : nullptr));
    if (clobbers) call.check(cudaMemcpyAsync(in, din, (in_elems - 2) * 4, cudaMemcpyDeviceToHost, st), "d2h input");
    if (strided_out) e = cudaMemcpy2DAsync(out, (size_t)stride, dout, 4, 4, out_elems, cudaMemcpyDeviceToHost, st);
    else if (strided_cpx) e = cudaMemcpy2DAsync(out, (size_t)stride, dout, 8, 8, out_elems / 2, cudaMemcpyDeviceToHost, st);
    else e = cudaMemcpyAsync(out, dout, out_elems * 4, cudaMemcpyDeviceToHost, st);
    call.check(e, "d2h");
    call.sync();
}

B200_API int b200_tx_init_device(B200Device *dev, B200TXContext **ctx, b200_tx_fn *tx, int type, int inv, int len,
                                 const void *scale, uint64_t flags)
{
    if (!ctx || !len) return B200_EINVAL;                            // av_tx_init, tx.c:903-940
    *ctx = nullptr;
    if (!dev) return B200_ENODEV;
    if (type != B200_TX_FLOAT_FFT && type != B200_TX_FLOAT_MDCT && type != B200_TX_FLOAT_RDFT && type != B200_TX_FLOAT_DCT &&
        type != B200_TX_INT32_FFT && type != B200_TX_INT32_MDCT && type != B200_TX_DOUBLE_FFT && type != B200_TX_DOUBLE_MDCT) return B200_ENOSYS;
    if (flags & ~(uint64_t)(B200_TX_INPLACE | B200_TX_UNALIGNED | B200_TX_FULL_IMDCT)) return B200_ENOSYS;    // REAL_TO_* not implemented
    // AV_TX_INPLACE: the complex FFT kernels stage a whole transform in shared memory before they store, so out == in is always
    // fine for them and gives the bits of the out-of-place call (as ff_tx_fft_inplace does, tx_template.c:780-812); other types refuse
    if ((flags & B200_TX_INPLACE) && !(type == B200_TX_FLOAT_FFT && len >= 2 && (!(len & (len - 1)) || tx_pfa_fft_length_ok(len)))) return B200_ENOSYS;
    const bool full = (flags & B200_TX_FULL_IMDCT) != 0;
    if (full && !(type == B200_TX_FLOAT_MDCT && inv)) return B200_ENOSYS;      // only the inverse MDCT has such a codelet (tx.c:762-771)
    if (type == B200_TX_DOUBLE_FFT || type == B200_TX_DOUBLE_MDCT) { // double precision (tx_double.cu); the scale of these types is a const double *
        if (flags & ~(uint64_t)B200_TX_UNALIGNED) return B200_ENOSYS;
        if (!tx_dbl_length_ok(type, len)) return B200_ENOSYS;
        double scdd = 1.0;
        if (type == B200_TX_DOUBLE_MDCT && scale) scdd = *(const double *)scale;
        B200TXContext *cd2 = new (std::nothrow) B200TXContext();
        if (!cd2) return B200_ENOMEM;
        cd2->dev = dev; cd2->type = type; cd2->inv = !!inv; cd2->len = len;
        if (cudaSetDevice(dev->ordinal) != cudaSuccess) { delete cd2; return B200_EEXTERNAL; }
        cd2->dbl = tx_dbl_create(dev, type, cd2->inv, len, scdd);
        if (!cd2->dbl) { delete cd2; return B200_EEXTERNAL; }
        *ctx = cd2;
        if (tx) *tx = tx_host_fn;
        return 0;
    }
    if (type == B200_TX_INT32_FFT || type == B200_TX_INT32_MDCT) {   // 32-bit fixed point (tx_int32.cu)
        if (!tx_i32_length_ok(type, len)) return B200_ENOSYS;
        float sci = 1.0f;
        if (type == B200_TX_INT32_MDCT && scale) sci = *(const float *)scale;
        B200TXContext *ci = new (std::nothrow) B200TXContext();
        if (!ci) return B200_ENOMEM;
        ci->dev = dev; ci->type = type; ci->inv = !!inv; ci->len = len;
        if (cudaSetDevice(dev->ordinal) != cudaSuccess) { delete ci; return B200_EEXTERNAL; }
        ci->i32 = tx_i32_create(dev, type, ci->inv, len, sci);
        if (!ci->i32) { delete ci; return B200_EEXTERNAL; }
        *ctx = ci;
        if (tx) *tx = tx_host_fn;
        return 0;
    }
    if (type == B200_TX_FLOAT_DCT) {                                 // DCT-II / DCT-III around a child real-DFT context (tx_dct.cu)
        if (!tx_dct_length_ok(!!inv, len)) return B200_ENOSYS;
        float scd = 1.0f;
        if (scale) scd = *(const float *)scale;
        B200TXContext *cd = new (std::nothrow) B200TXContext();
        if (!cd) return B200_ENOMEM;
        cd->dev = dev; cd->type = type; cd->inv = !!inv; cd->len = len;
        if (cudaSetDevice(dev->ordinal) != cudaSuccess) { delete cd; return B200_EEXTERNAL; }
        cd->dct = tx_dct_create(dev, cd->inv, len, scd);
        if (!cd->dct) { delete cd; return B200_EEXTERNAL; }
        *ctx = cd;
        if (tx) *tx = tx_host_fn;
        return 0;
    }
    if (type == B200_TX_FLOAT_FFT && tx_pfa_fft_length_ok(len)) {    // N x 2^k complex FFT: fft_pfa over fftN_ns (N = 15, 9, 7, 5, 3) and the split-radix transform
        B200TXContext *cp = new (std::nothrow) B200TXContext();
        if (!cp) return B200_ENOMEM;
        cp->dev = dev; cp->type = type; cp->inv = !!inv; cp->len = len; cp->full = false;
        if (cudaSetDevice(dev->ordinal) != cudaSuccess) { delete cp; return B200_EEXTERNAL; }
        cp->pfa = tx_pfa_create_fft(cp->inv, len);
        if (!cp->pfa) { delete cp; return B200_EEXTERNAL; }
        *ctx = cp;
        if (tx) *tx = tx_host_fn;
        return 0;
    }
    if (type == B200_TX_FLOAT_MDCT && tx_pfa_length_ok(len)) {       // 15 x 2^k: the compound MDCT av_tx_init() picks (Opus CELT sizes)
        float scp = 1.0f;
        if (scale) scp = *(const float *)scale;
        B200TXContext *cp = new (std::nothrow) B200TXContext();
        if (!cp) return B200_ENOMEM;
        cp->dev = dev; cp->type = type; cp->inv = !!inv; cp->len = len; cp->full = full;
        if (cudaSetDevice(dev->ordinal) != cudaSuccess) { delete cp; return B200_EEXTERNAL; }
        cp->pfa = tx_pfa_create(cp->inv, len, scp);
        if (!cp->pfa) { delete cp; return B200_EEXTERNAL; }
        *ctx = cp;
        if (tx) *tx = tx_host_fn;
        return 0;
    }
    if (len < 2 || (len & (len - 1))) return B200_ENOSYS;            // nested / naive decompositions (45 x 2^n, 25 x n, primes > 7 ...) are not implemented
    if (type == B200_TX_FLOAT_RDFT && len < 4) return B200_ENOSYS;   // ff_tx_rdft_*_def: min_len 4
    if (type == B200_TX_FLOAT_MDCT && len < 4) return B200_ENOSYS;   // len 2: the reference falls back to its naive MDCT (no 1-point FFT)
    const int n = type == 0 ? len : len >> 1;
    if (n < 1 || n > 16384) return B200_ENOSYS;                      // one transform must fit a CTA's shared memory
    float sc = 1.0f;                                                 // default_scale_f
    if (type != B200_TX_FLOAT_FFT && scale) sc = *(const float *)scale;
    B200TXContext *c = new (std::nothrow) B200TXContext();
    if (!c) return B200_ENOMEM;
    c->dev = dev; c->type = type; c->inv = !!inv; c->len = len; c->full = full;
    if (cudaSetDevice(dev->ordinal) != cudaSuccess) { delete c; return B200_EEXTERNAL; }
    int ret = tx_build(c, sc);
    if (ret < 0) { if (c->blob) cudaFree(c->blob); tx_r16_destroy(c->r16); delete c; return ret; }
    *ctx = c;
    if (tx) *tx = tx_host_fn;
    return 0;
}

B200_API int b200_tx_init(B200TXContext **ctx, b200_tx_fn *tx, int type, int inv, int len, const void *scale, uint64_t flags)
{
    return b200_tx_init_device(b200_default_device(), ctx, tx, type, inv, len, scale, flags);
}

B200_API void b200_tx_uninit(B200TXContext **ctx)
{
    if (!ctx || !*ctx) return;
    B200TXContext *c = *ctx;
    cudaSetDevice(c->dev->ordinal);
    cudaStreamSynchronize(c->dev->stream);
    if (c->blob) cudaFree(c->blob);
    tx_pfa_free(c->pfa);
    tx_dct_free(c->dct);
    tx_i32_free(c->i32);
    tx_dbl_free(c->dbl);
    tx_r16_destroy(c->r16);
    delete c;
    *ctx = nullptr;
}

// Power-of-two float transforms: the level-by-level kernels above move the complex side of a transform as 8-byte float2 words
// (FFT in and out, RDFT r2c in (sample pairs) and out, c2r in and out, inverse-MDCT out) and everything else as single floats.
// The register-resident route asks for more (tx_r16_accepts) but falls back to those kernels, so their rule is the one to meet.
// The compound, DCT, int32 and double routes check their own rules in their launch functions.
static int tx_check_align(const B200TXContext *c, const void *out, const void *in, ptrdiff_t out_step, ptrdiff_t in_step)
{
    if (c->pfa || c->dct || c->i32 || c->dbl) return 0;
    const uintptr_t ia = c->type == 1 ? 3 : 7, oa = c->type == 1 && !c->inv ? 3 : 7;
    if (((uintptr_t)in | (uintptr_t)in_step) & ia) {
        b200_set_error("b200_tx_batch_device: input pointer and in_step must be multiples of %d bytes for this transform", (int)ia + 1);
        return B200_EINVAL;
    }
    if (((uintptr_t)out | (uintptr_t)out_step) & oa) {
        b200_set_error("b200_tx_batch_device: output pointer and out_step must be multiples of %d bytes for this transform", (int)oa + 1);
        return B200_EINVAL;
    }
    return 0;
}

B200_API int b200_tx_batch_device(B200TXContext *c, void *out, const void *in, ptrdiff_t stride, int64_t count,
                                  ptrdiff_t out_step, ptrdiff_t in_step)
{
    if (!c || !out || !in || count < 0) return B200_EINVAL;
    if ((c->type == 1 || c->type == B200_TX_INT32_MDCT) && (stride & 3)) return B200_EINVAL;
    if (c->full && stride != 4) return B200_EINVAL;                  // the reference mirrors with the input stride: only sizeof(float) is meaningful
    if (tx_check_align(c, out, in, out_step, in_step) < 0) return B200_EINVAL;
    B200_CUDA_OK(cudaSetDevice(c->dev->ordinal));
    return tx_launch(c, c->dev->stream, out, in, (c->type == 1 || c->type == B200_TX_INT32_MDCT || c->type == B200_TX_DOUBLE_MDCT || (c->type == 0 && c->pfa)) ? stride : 8, count, out_step, in_step);
}

// HOST buffers (pinned for real overlap): the batch is cut into chunks that rotate over the device's three pipeline streams, each chunk
// = one linear H2D of its inputs, the transform kernels, one linear D2H of its outputs.
B200_API int b200_tx_batch_host(B200TXContext *c, void *out, const void *in, ptrdiff_t stride, int64_t count,
                                ptrdiff_t out_step, ptrdiff_t in_step)
{
    if (!c || !out || !in || count < 0 || out_step <= 0 || in_step <= 0) return B200_EINVAL;
    if ((c->type == 1 || c->type == B200_TX_INT32_MDCT) && (stride & 3)) return B200_EINVAL;
    if (c->full && stride != 4) return B200_EINVAL;
    if (count == 0) return 0;
    B200Device *d = c->dev;
    B200_CUDA_OK(cudaSetDevice(d->ordinal));
    const ptrdiff_t st_arg = (c->type == 1 || c->type == B200_TX_INT32_MDCT || c->type == B200_TX_DOUBLE_MDCT || (c->type == 0 && c->pfa)) ? stride : 8;
    const size_t istep = ((size_t)in_step + 15) & ~(size_t)15, ostep = ((size_t)out_step + 15) & ~(size_t)15;
    if (istep != (size_t)in_step || ostep != (size_t)out_step) { b200_set_error("b200_tx_batch_host: steps must be multiples of 16 bytes"); return B200_EINVAL; }
    int64_t chunk = ((int64_t)48 << 20) / (int64_t)(istep + ostep);
    if (chunk < 1) chunk = 1;
    if (chunk > count) chunk = count;
    const int K = B200Device::kPipe;
    B200_LOCK_DEVICE(d);
    uint8_t *scr = (uint8_t *)b200_scratch(d, (size_t)chunk * (istep + ostep) * K);
    if (!scr) return B200_ENOMEM;
    B200_CUDA_OK(cudaStreamSynchronize(d->stream));
    int slot = 0;
    for (int64_t i0 = 0; i0 < count; i0 += chunk, slot = (slot + 1) % K) {
        const int64_t n = count - i0 < chunk ? count - i0 : chunk;
        cudaStream_t st = d->pipe[slot];
        uint8_t *din = scr + (size_t)slot * chunk * (istep + ostep), *dout = din + (size_t)chunk * istep;
        B200_CUDA_OK(cudaMemcpyAsync(din, (const uint8_t *)in + (size_t)i0 * istep, (size_t)n * istep, cudaMemcpyHostToDevice, st));
        int ret = tx_launch(c, st, dout, din, st_arg, n, (ptrdiff_t)ostep, (ptrdiff_t)istep);
        if (ret < 0) return ret;
        B200_CUDA_OK(cudaMemcpyAsync((uint8_t *)out + (size_t)i0 * ostep, dout, (size_t)n * ostep, cudaMemcpyDeviceToHost, st));
    }
    for (int i = 0; i < K; i++) B200_CUDA_OK(cudaStreamSynchronize(d->pipe[i]));
    return 0;
}

