// tx_pfa.cu — libavutil/tx compound N x M float MDCT (N = 15, 5, 3) on sm_90a: what av_tx_init(AV_TX_FLOAT_MDCT, len = 2 * N * 2^k) resolves to
// (mdct_pfa_15xM_{inv,fwd} carry the largest factor, libavutil/tx.c:391-395), i.e. the Opus CELT transforms of 120 ... 960
// (libavcodec/opus/dec_celt.c:569, enc.c:690).
//
// Reference semantics reproduced bit for bit (checker: the compound part of oracle/tx_oracle.c), libavutil/tx_template.c:
//   :172-209 fft3, :211-250 fft5 / fft5_m1..m3, :252-339 fft7, :341-463 fft9, :465-476 fft15 (float branches), tables ff_tx_tab_53 / _7 / _9 :91-130
//   :1430-1469 ff_tx_mdct_pfa_init (compound map libavutil/tx.c:75-123, 3x5 input map embedded tx_priv.h:275-284, twiddles
//              ff_tx_mdct_gen_exp :2107-2134, scatter permutation of the M-point transform tx.c:136-154)
//   :1471-1511 ff_tx_mdct_pfa_15xM_inv, :1533-1579 ff_tx_mdct_pfa_15xM_fwd, M-point split-radix transforms :540-722
// Every product and sum is rounded on its own (library built with --fmad=false), in the reference's order.
//
// First version, correctness before speed: ONE THREAD PER TRANSFORM, the 15 x M work array in a global scratch line per
// thread; the tuned version will put one transform per warp / CTA in shared memory like tx.cu does for powers of two.
#include "tx_pfa.h"
#include <vector>
#include <cmath>
#include <cstring>

namespace {

// [device-code tx_pfa] (tests/cuda_emu runs this block on the CPU against the checker; comment markers only)
struct PfaDev {
    const int *in_map, *out_map, *sub_map;     // in_map holds doubled positions (tx_template.c:1460-1462)
    const float2 *exp;
    const float *tab53;                        // ff_tx_tab_53 [12], then ff_tx_tab_7 [6] and ff_tx_tab_9 [8]
    const float *tabs[12];                     // tabs[k]: cosine table of the 2^k-point transform (k = 3 ... 9)
    int m, log2m, len;
    int nfac;                                  // the odd factor: 15, 9, 7, 5 or 3
    const int *blk;                            // offsets of the split-radix blocks of an m-point transform, level after level
    int lvl_start[12], lvl_cnt[12];            // level L (block size 2^L): blk[lvl_start[L] .. + lvl_cnt[L])
    int ms;                                    // pitch of one m-point sub-transform in shared memory: m + m / 16 + 1
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

__device__ __forceinline__ void transform(float2 &a0, float2 &a1, float2 &a2, float2 &a3, float wre, float wim)
{
    const float t1 = a2.x * wre - a2.y * (-wim);
    const float t2 = a2.x * (-wim) + a2.y * wre;
    const float t5 = a3.x * wre - a3.y * wim;
    const float t6 = a3.x * wim + a3.y * wre;
    butterflies(a0, a1, a2, a3, t1, t2, t5, t6);
}

// The nfac power-of-two sub-transforms of a compound MDCT, all at once and level by level, on data held in shared memory:
// z[j * ms + PADI(k)] is sample k of sub-transform j.  The reference's recursion  fft(S) = fft(S/2) | fft(S/4) | fft(S/4) ; combine(S)
// (ff_tx_fft{N}_ns / ff_tx_fft_sr_combine, tx_template.c:562-722) is flattened: all blocks of one size are independent, so the CTA
// sweeps S = 2, 4, ..., m with one barrier per size, every thread taking butterflies of any block of any sub-transform.  The
// hard-coded sizes 4, 8, 16 are instances of the same rule except that their j = 0 butterfly skips the multiplication by (1, 0).
__device__ __forceinline__ int PADI(int i) { return i + (i >> 4); }
__device__ void pfa_sub_ffts(const PfaDev &P, float2 *z)
{
    const int N = P.nfac;
    for (int L = 1; L <= P.log2m; L++) {
        const int *off = P.blk + P.lvl_start[L];
        const int cnt = P.lvl_cnt[L];
        if (L == 1) {
            for (int it = threadIdx.x; it < N * cnt; it += blockDim.x) {
                const int j = it / cnt, o = off[it - j * cnt];
                float2 &a = z[j * P.ms + PADI(o)], &b = z[j * P.ms + PADI(o + 1)];
                const float2 s0 = a, s1 = b;
                a = make_float2(s0.x + s1.x, s0.y + s1.y);
                b = make_float2(s0.x - s1.x, s0.y - s1.y);
            }
        } else {
            const int lq = L - 2, q = 1 << lq, per = cnt << lq;
            const float *tab = P.tabs[L];
            for (int it = threadIdx.x; it < N * per; it += blockDim.x) {
                const int j = it / per, r = it - j * per, o = off[r >> lq], jj = r & (q - 1);
                float2 *zj = z + j * P.ms;
                const int i0 = PADI(o + jj), i1 = PADI(o + q + jj), i2 = PADI(o + 2 * q + jj), i3 = PADI(o + 3 * q + jj);
                float2 a0 = zj[i0], a1 = zj[i1], a2 = zj[i2], a3 = zj[i3];
                if (L <= 4 && jj == 0) butterflies(a0, a1, a2, a3, a2.x, a2.y, a3.x, a3.y);
                else transform(a0, a1, a2, a3, tab[jj], tab[q - jj]);
                zj[i0] = a0; zj[i1] = a1; zj[i2] = a2; zj[i3] = a3;
            }
        }
        __syncthreads();
    }
}

__device__ __forceinline__ void fft3(const float *tab, float2 *out, const float2 *in, int stride)
{
    float2 t0 = in[0], t1, t2;
    t1.x = in[1].y - in[2].y; t2.y = in[1].y + in[2].y;
    t1.y = in[1].x - in[2].x; t2.x = in[1].x + in[2].x;
    out[0 * stride].x = t0.x + t2.x;
    out[0 * stride].y = t0.y + t2.y;
    t1.x = tab[8] * t1.x; t1.y = tab[9] * t1.y; t2.x = tab[10] * t2.x; t2.y = tab[10] * t2.y;
    out[1 * stride].x = t0.x - t2.x + t1.x;
    out[1 * stride].y = t0.y - t2.y - t1.y;
    out[2 * stride].x = t0.x - t2.x - t1.x;
    out[2 * stride].y = t0.y - t2.y + t1.y;
}

template <int D0, int D1, int D2, int D3, int D4>
__device__ __forceinline__ void fft5(const float *tab, float2 *out, const float2 *in, int stride)
{
    const float2 dc = in[0];
    float2 z0[4], t[6];
    t[1].y = in[1].x - in[4].x; t[0].x = in[1].x + in[4].x;
    t[1].x = in[1].y - in[4].y; t[0].y = in[1].y + in[4].y;
    t[3].y = in[2].x - in[3].x; t[2].x = in[2].x + in[3].x;
    t[3].x = in[2].y - in[3].y; t[2].y = in[2].y + in[3].y;
    out[D0 * stride].x = dc.x + t[0].x + t[2].x;
    out[D0 * stride].y = dc.y + t[0].y + t[2].y;
    { const float a = tab[0] * t[2].x - tab[2] * t[0].x, b = tab[0] * t[0].x - tab[2] * t[2].x; t[4].x = a; t[0].x = b; }
    { const float a = tab[0] * t[2].y - tab[2] * t[0].y, b = tab[0] * t[0].y - tab[2] * t[2].y; t[4].y = a; t[0].y = b; }
    { const float a = tab[4] * t[3].x - tab[6] * t[1].x, b = tab[4] * t[1].x + tab[6] * t[3].x; t[5].x = a; t[1].x = b; }
    { const float a = tab[4] * t[3].y - tab[6] * t[1].y, b = tab[4] * t[1].y + tab[6] * t[3].y; t[5].y = a; t[1].y = b; }
    z0[0].x = t[0].x - t[1].x; z0[3].x = t[0].x + t[1].x;
    z0[0].y = t[0].y - t[1].y; z0[3].y = t[0].y + t[1].y;
    z0[2].x = t[4].x - t[5].x; z0[1].x = t[4].x + t[5].x;
    z0[2].y = t[4].y - t[5].y; z0[1].y = t[4].y + t[5].y;
    out[D1 * stride].x = dc.x + z0[3].x; out[D1 * stride].y = dc.y + z0[0].y;
    out[D2 * stride].x = dc.x + z0[2].x; out[D2 * stride].y = dc.y + z0[1].y;
    out[D3 * stride].x = dc.x + z0[1].x; out[D3 * stride].y = dc.y + z0[2].y;
    out[D4 * stride].x = dc.x + z0[0].x; out[D4 * stride].y = dc.y + z0[3].y;
}

// fft7 (tx_template.c:252-339, float branch).  S[k] / D[k]: sum / difference of in[k + 1] and in[6 - k]; T = ff_tx_tab_7 as three
// (re, im) pairs.  The products and sums keep the reference's left-to-right order (the library is built without contraction).
__device__ __forceinline__ void fft7(const float *T, float2 *out, const float2 *in, int stride)
{
    const float c0 = T[0], s0 = T[1], c1 = T[2], s1 = T[3], c2 = T[4], s2 = T[5];
    const float2 dc = in[0];
    float2 S[3], D[3], z[3], u[3];
#pragma unroll
    for (int k = 0; k < 3; k++) {
        S[k].x = in[k + 1].x + in[6 - k].x; D[k].x = in[k + 1].x - in[6 - k].x;
        S[k].y = in[k + 1].y + in[6 - k].y; D[k].y = in[k + 1].y - in[6 - k].y;
    }
    out[0].x = dc.x + S[0].x + S[1].x + S[2].x;
    out[0].y = dc.y + S[0].y + S[1].y + S[2].y;
    z[0].x = c0 * S[0].x - c2 * S[2].x - c1 * S[1].x;
    z[1].x = c0 * S[2].x - c1 * S[0].x - c2 * S[1].x;
    z[2].x = c0 * S[1].x - c2 * S[0].x - c1 * S[2].x;
    z[0].y = c0 * S[0].y - c1 * S[1].y - c2 * S[2].y;
    z[1].y = c0 * S[2].y - c1 * S[0].y - c2 * S[1].y;
    z[2].y = c0 * S[1].y - c2 * S[0].y - c1 * S[2].y;
    u[0].x = s2 * D[0].y + s1 * D[2].y - s0 * D[1].y;
    u[1].x = s0 * D[2].y + s2 * D[1].y - s1 * D[0].y;
    u[2].x = s2 * D[2].y + s1 * D[1].y + s0 * D[0].y;
    u[0].y = s0 * D[0].x + s1 * D[1].x + s2 * D[2].x;
    u[1].y = s2 * D[1].x + s0 * D[2].x - s1 * D[0].x;
    u[2].y = s2 * D[0].x + s1 * D[2].x - s0 * D[1].x;
    out[1 * stride].x = dc.x + (z[0].x + u[2].x); out[1 * stride].y = dc.y + (z[0].y - u[0].y);
    out[2 * stride].x = dc.x + (z[1].x - u[1].x); out[2 * stride].y = dc.y + (z[1].y + u[1].y);
    out[3 * stride].x = dc.x + (z[2].x + u[0].x); out[3 * stride].y = dc.y + (z[2].y - u[2].y);
    out[4 * stride].x = dc.x + (z[2].x - u[0].x); out[4 * stride].y = dc.y + (z[2].y + u[2].y);
    out[5 * stride].x = dc.x + (z[1].x + u[1].x); out[5 * stride].y = dc.y + (z[1].y - u[1].y);
    out[6 * stride].x = dc.x + (z[0].x - u[2].x); out[6 * stride].y = dc.y + (z[0].y + u[0].y);
}

// fft9 (tx_template.c:341-463, float branch).  S[k] / D[k]: sum / difference of in[k + 1] and in[8 - k]; T = ff_tx_tab_9 as four pairs.
__device__ __forceinline__ void fft9(const float *T, float2 *out, const float2 *in, int stride)
{
    const float2 dc = in[0];
    float2 S[4], D[4], w[4], x[5], y[5], z0, z1;
#pragma unroll
    for (int k = 0; k < 4; k++) {
        S[k].x = in[k + 1].x + in[8 - k].x; D[k].x = in[k + 1].x - in[8 - k].x;
        S[k].y = in[k + 1].y + in[8 - k].y; D[k].y = in[k + 1].y - in[8 - k].y;
    }
    w[0].x = S[0].x - S[3].x; w[0].y = S[0].y - S[3].y;
    w[1].x = S[1].x - S[3].x; w[1].y = S[1].y - S[3].y;
    w[2].x = D[0].x - D[3].x; w[2].y = D[0].y - D[3].y;
    w[3].x = D[1].x + D[3].x; w[3].y = D[1].y + D[3].y;
    z0.x = dc.x + S[2].x; z0.y = dc.y + S[2].y;
    z1.x = S[0].x + S[1].x + S[3].x; z1.y = S[0].y + S[1].y + S[3].y;
    out[0].x = z0.x + z1.x; out[0].y = z0.y + z1.y;
    y[3].x = T[1] * (D[0].x - D[1].x + D[3].x);
    y[3].y = T[1] * (D[0].y - D[1].y + D[3].y);
    x[3].x = z0.x + T[0] * z1.x; x[3].y = z0.y + T[0] * z1.y;
    z0.x = dc.x + T[0] * S[2].x; z0.y = dc.y + T[0] * S[2].y;
    x[1].x = T[2] * w[0].x + T[5] * w[1].x; x[1].y = T[2] * w[0].y + T[5] * w[1].y;
    x[2].x = T[5] * w[0].x - T[6] * w[1].x; x[2].y = T[5] * w[0].y - T[6] * w[1].y;
    y[1].x = T[3] * w[2].x + T[4] * w[3].x; y[1].y = T[3] * w[2].y + T[4] * w[3].y;
    y[2].x = T[4] * w[2].x - T[7] * w[3].x; y[2].y = T[4] * w[2].y - T[7] * w[3].y;
    y[0].x = T[1] * D[2].x; y[0].y = T[1] * D[2].y;
    x[4].x = x[1].x + x[2].x; x[4].y = x[1].y + x[2].y;
    y[4].x = y[1].x - y[2].x; y[4].y = y[1].y - y[2].y;
    x[1].x = z0.x + x[1].x; x[1].y = z0.y + x[1].y;
    y[1].x = y[0].x + y[1].x; y[1].y = y[0].y + y[1].y;
    x[2].x = z0.x + x[2].x; x[2].y = z0.y + x[2].y;
    y[2].x = y[2].x - y[0].x; y[2].y = y[2].y - y[0].y;
    x[4].x = z0.x - x[4].x; x[4].y = z0.y - x[4].y;
    y[4].x = y[0].x - y[4].x; y[4].y = y[0].y - y[4].y;
#pragma unroll
    for (int k = 1; k <= 4; k++) {
        out[k * stride].x = x[k].x + y[k].y; out[k * stride].y = x[k].y - y[k].x;
        out[(9 - k) * stride].x = x[k].x - y[k].y; out[(9 - k) * stride].y = x[k].y + y[k].x;
    }
}

__device__ __forceinline__ void fft15(const float *tab, float2 *out, const float2 *in, int stride);
// the N-point transform DECL_COMP_IMDCT / DECL_COMP_MDCT instantiate for N = 3, 5, 7, 9, 15
__device__ __forceinline__ void fftN(int n, const float *tab, float2 *out, const float2 *in, int stride)
{
    if (n == 3) fft3(tab, out, in, stride);
    else if (n == 5) fft5<0, 1, 2, 3, 4>(tab, out, in, stride);
    else if (n == 7) fft7(tab + 12, out, in, stride);
    else if (n == 9) fft9(tab + 18, out, in, stride);
    else fft15(tab, out, in, stride);
}
__device__ __forceinline__ void fft15(const float *tab, float2 *out, const float2 *in, int stride)
{
    float2 tmp[15];
#pragma unroll
    for (int i = 0; i < 5; i++) fft3(tab, tmp + i, in + i * 3, 5);
    fft5<0, 6, 12, 3, 9>(tab, out, tmp + 0, stride);
    fft5<10, 1, 7, 13, 4>(tab, out, tmp + 5, stride);
    fft5<5, 11, 2, 8, 14>(tab, out, tmp + 10, stride);
}

// ff_tx_mdct_pfa_{15,9,7,5,3}xM_inv (tx_template.c:1430-1508): one CTA per transform.  Pre-rotation and the m small odd-size
// transforms (one per thread, straight into the shared-memory layout of the sub-transforms), the nfac m-point transforms
// cooperatively, then the post-rotation.  in: len floats with a stride (in floats), out: len floats.
constexpr int PFA_THREADS = 128;
__global__ void __launch_bounds__(PFA_THREADS)
tx_mdct_pfa_inv_kernel(const PfaDev P, float *out, const float *in, long long stride, long long out_step, long long in_step, long long count)
{
    extern __shared__ float2 pfa_z[];
    const int len4 = P.len >> 2, len2 = P.len >> 1, m = P.m, N = P.nfac;
    for (long long tr = blockIdx.x; tr < count; tr += gridDim.x) {
        float2 *z = reinterpret_cast<float2 *>(reinterpret_cast<char *>(out) + tr * out_step);
        const float *src = reinterpret_cast<const float *>(reinterpret_cast<const char *>(in) + tr * in_step);
        const float *in1 = src, *in2 = src + ((N * m * 2) - 1) * stride;
        for (int b = threadIdx.x; b < m; b += blockDim.x) {
            const float2 *e = P.exp + b * N;
            const int *in_map = P.in_map + b * N;
            float2 f15[15];
#pragma unroll
            for (int j = 0; j < 15; j++) {
                if (j < N) {
                    const int k = in_map[j];
                    const float are = in2[-k * stride], aim = in1[k * stride];
                    f15[j].x = are * e[j].x - aim * e[j].y;
                    f15[j].y = are * e[j].y + aim * e[j].x;
                }
            }
            fftN(N, P.tab53, pfa_z + PADI(P.sub_map[b]), f15, P.ms);
        }
        __syncthreads();
        pfa_sub_ffts(P, pfa_z);
        const float2 *e = P.exp + len2;
        for (int i = threadIdx.x; i < len4; i += blockDim.x) {
            const int i0 = len4 + i, i1 = len4 - i - 1, s0 = P.out_map[i0], s1 = P.out_map[i1];
            const float2 t1 = pfa_z[(s1 >> P.log2m) * P.ms + PADI(s1 & (m - 1))], t0 = pfa_z[(s0 >> P.log2m) * P.ms + PADI(s0 & (m - 1))];
            const float2 src1 = make_float2(t1.y, t1.x), src0 = make_float2(t0.y, t0.x);
            float2 o1, o0;
            o1.x = src1.x * e[i1].y - src1.y * e[i1].x;
            o0.y = src1.x * e[i1].x + src1.y * e[i1].y;
            o0.x = src0.x * e[i0].y - src0.y * e[i0].x;
            o1.y = src0.x * e[i0].x + src0.y * e[i0].y;
            z[i1] = o1; z[i0] = o0;
        }
        __syncthreads();                                   // the next transform reuses the buffer
    }
}

// ff_tx_mdct_pfa_{15,9,7,5,3}xM_fwd (tx_template.c:1510-1599): in: 2*len floats, out: len floats with a stride (in floats)
__global__ void __launch_bounds__(PFA_THREADS)
tx_mdct_pfa_fwd_kernel(const PfaDev P, float *out, const float *in, long long stride, long long out_step, long long in_step, long long count)
{
    extern __shared__ float2 pfa_z[];
    const int m = P.m, N = P.nfac, len4 = N * m, len3 = len4 * 3, len8 = P.len >> 2;
    const float2 *e = P.exp;
    for (long long tr = blockIdx.x; tr < count; tr += gridDim.x) {
        float *dst = reinterpret_cast<float *>(reinterpret_cast<char *>(out) + tr * out_step);
        const float *src = reinterpret_cast<const float *>(reinterpret_cast<const char *>(in) + tr * in_step);
        for (int b = threadIdx.x; b < m; b += blockDim.x) {
            float2 f15[15];
#pragma unroll
            for (int j = 0; j < 15; j++) {
                if (j < N) {
                    const int k = P.in_map[b * N + j];
                    float re, im;
                    if (k < len4) { re = -src[len4 + k] + src[1 * len4 - 1 - k]; im = -src[len3 + k] + -src[1 * len3 - 1 - k]; }
                    else          { re = -src[len4 + k] + -src[5 * len4 - 1 - k]; im = src[-len4 + k] + -src[1 * len3 - 1 - k]; }
                    f15[j].y = re * e[k >> 1].x - im * e[k >> 1].y;
                    f15[j].x = re * e[k >> 1].y + im * e[k >> 1].x;
                }
            }
            fftN(N, P.tab53, pfa_z + PADI(P.sub_map[b]), f15, P.ms);
        }
        __syncthreads();
        pfa_sub_ffts(P, pfa_z);
        for (int i = threadIdx.x; i < len8; i += blockDim.x) {
            const int i0 = len8 + i, i1 = len8 - i - 1, s0 = P.out_map[i0], s1 = P.out_map[i1];
            const float2 src1 = pfa_z[(s1 >> P.log2m) * P.ms + PADI(s1 & (m - 1))], src0 = pfa_z[(s0 >> P.log2m) * P.ms + PADI(s0 & (m - 1))];
            dst[(2 * i1 + 1) * stride] = src0.x * e[i0].y - src0.y * e[i0].x;
            dst[2 * i0 * stride]       = src0.x * e[i0].x + src0.y * e[i0].y;
            dst[(2 * i0 + 1) * stride] = src1.x * e[i1].y - src1.y * e[i1].x;
            dst[2 * i1 * stride]       = src1.x * e[i1].x + src1.y * e[i1].y;
        }
        __syncthreads();
    }
}
// ff_tx_fft_pfa (tx_template.c:1059-1080) for fftN_ns x 2^k: what av_tx_init(AV_TX_FLOAT_FFT, len = N * 2^k) resolves to (checkasm
// lengths 120 / 960 / 1920, tests/checkasm/av_tx.c:38-40).  One CTA per transform: the gathered N-point transforms (one per
// thread), the N power-of-two transforms cooperatively, the CRT-ordered output.  in: len complex; out: len complex with a stride
// (in complex).  Everything is read before anything is stored: out == in is fine.
__global__ void __launch_bounds__(PFA_THREADS)
tx_fft_pfa_kernel(const PfaDev P, float2 *out, const float2 *in, long long stride, long long out_step, long long in_step, long long count)
{
    extern __shared__ float2 pfa_z[];
    const int m = P.m, N = P.nfac, l = P.len;
    for (long long tr = blockIdx.x; tr < count; tr += gridDim.x) {
        float2 *dst = reinterpret_cast<float2 *>(reinterpret_cast<char *>(out) + tr * out_step);
        const float2 *src = reinterpret_cast<const float2 *>(reinterpret_cast<const char *>(in) + tr * in_step);
        for (int b = threadIdx.x; b < m; b += blockDim.x) {
            const int *in_map = P.in_map + b * N;
            float2 f15[15];
#pragma unroll
            for (int j = 0; j < 15; j++)
                if (j < N) f15[j] = src[in_map[j]];
            fftN(N, P.tab53, pfa_z + PADI(P.sub_map[b]), f15, P.ms);
        }
        __syncthreads();
        pfa_sub_ffts(P, pfa_z);
        for (int i = threadIdx.x; i < l; i += blockDim.x) {
            const int s = P.out_map[i];
            dst[i * stride] = pfa_z[(s >> P.log2m) * P.ms + PADI(s & (m - 1))];
        }
        __syncthreads();
    }
}
// [/device-code tx_pfa]

int sr_perm(int i, int len, int inv)                               // split_radix_permutation, libavutil/tx.c:125-134
{
    len >>= 1;
    if (len <= 1) return i & 1;
    if (!(i & len)) return sr_perm(i, len, inv) * 2;
    len >>= 1;
    return sr_perm(i, len, inv) * 4 + 1 - 2 * (!(i & len) ^ inv);
}
int mulinv(int n, int m)                                           // libavutil/tx.c:34-42
{
    n = n % m;
    for (int x = 1; x < m; x++) if (((n * x) % m) == 1) return x;
    return 0;
}

} // namespace

struct TxPfa {
    int inv = 0, len = 0, m = 0;
    bool fft = false;                  // compound complex FFT instead of the compound MDCT
    PfaDev d{};
    void *blob = nullptr;
    size_t smem = 0;
    int grid_cap = 0;
};

// the host tables of one transform (also used by the CPU test tier through b200_tx_pfa_tables)
struct PfaHost {
    std::vector<int> in_map, out_map, sub_map;
    std::vector<float> exp;            // interleaved re, im: inverse = 2 * l2 entries (pre-shuffled, then natural), forward = l2
    float tab53[26];                   // ff_tx_tab_53 [12], ff_tx_tab_7 [6], ff_tx_tab_9 [8]
    std::vector<float> cosk[12];
    int m = 0, log2m = 0, nfac = 0;
    std::vector<int> blk;              // split-radix block offsets of an m-point transform, level after level
    int lvl_start[12] = { 0 }, lvl_cnt[12] = { 0 };
};

static void pfa_collect_blocks(std::vector<std::vector<int>> &lv, int L, int off)   // block of size 2^L at `off` and everything below it
{
    if (L < 1) return;
    lv[L].push_back(off);
    const int S = 1 << L;
    pfa_collect_blocks(lv, L - 1, off);
    if (L >= 2) {
        pfa_collect_blocks(lv, L - 2, off + S / 2);
        pfa_collect_blocks(lv, L - 2, off + 3 * S / 4);
    }
}

// the odd factor av_tx_init() ends up with for this MDCT length: the largest of 15, 9, 7, 5, 3 that leaves a power of two (tx.c:391-395); 0 = none
static int pfa_factor(int len)
{
    if (len < 12 || (len & 1)) return 0;
    static const int factors[5] = { 15, 9, 7, 5, 3 };
    for (int n : factors) {
        const int l2 = len >> 1, m = l2 / n;
        if (l2 % n == 0 && m >= 2 && m <= 512 && !(m & (m - 1))) return n;
    }
    return 0;
}
bool tx_pfa_length_ok(int len) { return pfa_factor(len) != 0; }
// compound complex FFT: odd part 15, 9, 7, 5 or 3 times a power of two 2 ... 512 (the tree fft_pfa -> fftN_ns + fft2^k_ns the reference builds)
static int pfa_fft_factor(int len)
{
    if (len < 6) return 0;
    int m = 1;
    while (!(len & m)) m <<= 1;
    const int n = len / m;
    if (m < 2 || m > 512) return 0;
    return (n == 3 || n == 5 || n == 7 || n == 9 || n == 15) ? n : 0;
}
bool tx_pfa_fft_length_ok(int len) { return pfa_fft_factor(len) != 0; }

static void pfa_host_tables(PfaHost &H, int inv, int len, float scale, bool fft = false)
{
    const int n = fft ? pfa_fft_factor(len) : pfa_factor(len), l2 = fft ? len : len >> 1, m = l2 / n;
    H.nfac = n;
    H.m = m; H.log2m = 0;
    while ((1 << H.log2m) < m) H.log2m++;
    {
        std::vector<std::vector<int>> lv(12);
        pfa_collect_blocks(lv, H.log2m, 0);
        H.blk.clear();
        for (int L = 0; L < 12; L++) {
            H.lvl_start[L] = (int)H.blk.size(); H.lvl_cnt[L] = (int)lv[L].size();
            H.blk.insert(H.blk.end(), lv[L].begin(), lv[L].end());
        }
    }
    H.in_map.assign(l2, 0); H.out_map.assign(l2, 0); H.sub_map.assign(m, 0);
    const int m_inv = mulinv(m, n), n_inv = mulinv(n, m);
    for (int j = 0; j < m; j++)                                     // ff_tx_gen_compound_mapping, gather direction (tx.c:104-110)
        for (int i = 0; i < n; i++) {
            H.in_map[j * n + i] = (i * m + j * n) % l2;
            H.out_map[(i * m * m_inv + j * n * n_inv) % l2] = i * m + j;
        }
    if (fft) {
        // ff_tx_fft_pfa_init (tx_template.c:948-1057): the compound map is generated for the forward direction; the direction comes
        // from the map of the first sub-transform (ff_tx_fft_factor_init :478-494: 3 x 5 map for 15 points, ff_tx_gen_pfa_input_map
        // tx.c:44-71, else ff_tx_gen_default_map tx.c:525-542; the inverse reverses all but the DC), flattened into it (:1040-1046)
        int sub[15];
        if (n == 15) {
            for (int b = 0; b < 5; b++)
                for (int a = 0; a < 3; a++) {
                    if (inv) sub[(b * 3 + a * 5) % 15] = b * 3 + a;
                    else     sub[b * 3 + a] = (b * 3 + a * 5) % 15;
                }
            if (inv) for (int w = 1; w <= 7; w++) std::swap(sub[w], sub[15 - w]);
        } else {
            sub[0] = 0;
            for (int i = 1; i < n; i++) sub[i] = inv ? n - i : i;
        }
        for (int k = 0; k < l2; k += n) {
            int mt[15];
            memcpy(mt, &H.in_map[k], sizeof(int) * n);
            for (int i = 0; i < n; i++) H.in_map[k + i] = mt[sub[i]];
        }
        H.exp.clear();
    } else {
        if (inv)
            for (int i = 0; i < m; i++) {
                int *in = &H.in_map[i * n + 1];
                for (int j = 0; j < ((n - 1) >> 1); j++) std::swap(in[j], in[n - j - 2]);
            }
        for (int k = 0; n == 15 && k < l2; k += 15) {                   // TX_EMBED_INPUT_PFA_MAP(map, len, 3, 5): the 15-point transform is 3 x 5
            int mt[15];
            memcpy(mt, &H.in_map[k], sizeof(mt));
            for (int b = 0; b < 5; b++) for (int a = 0; a < 3; a++) H.in_map[k + b * 3 + a] = mt[(b * 3 + a * 5) % 15];
        }
        const double theta = (scale < 0 ? l2 : 0) + 1.0 / 8.0, sc = sqrt(fabs((double)scale));      // ff_tx_mdct_gen_exp
        std::vector<float> full(2 * (size_t)l2);
        for (int i = 0; i < l2; i++) {
            const double alpha = M_PI_2 * (i + theta) / l2;
            full[2 * i] = (float)(cos(alpha) * sc);
            full[2 * i + 1] = (float)(sin(alpha) * sc);
        }
        if (inv) {
            H.exp.assign(4 * (size_t)l2, 0.f);
            memcpy(&H.exp[2 * (size_t)l2], full.data(), sizeof(float) * 2 * l2);
            for (int i = 0; i < l2; i++) { H.exp[2 * i] = full[2 * H.in_map[i]]; H.exp[2 * i + 1] = full[2 * H.in_map[i] + 1]; }
        } else
            H.exp = full;
        for (int i = 0; i < l2; i++) H.in_map[i] <<= 1;
    }
    for (int i = 0; i < m; i++) H.sub_map[(-sr_perm(i, m, inv)) & (m - 1)] = i;
    const double c5 = cos(2 * M_PI / 5), c10 = cos(2 * M_PI / 10), s5 = sin(2 * M_PI / 5), s10 = sin(2 * M_PI / 10);
    H.tab53[0] = H.tab53[1] = (float)c5; H.tab53[2] = H.tab53[3] = (float)c10;
    H.tab53[4] = H.tab53[5] = (float)s5; H.tab53[6] = H.tab53[7] = (float)s10;
    H.tab53[8] = H.tab53[9] = (float)cos(2 * M_PI / 12); H.tab53[10] = (float)cos(2 * M_PI / 6); H.tab53[11] = (float)cos(8 * M_PI / 6);
    float *t7 = H.tab53 + 12, *t9 = H.tab53 + 18;                   // ff_tx_init_tab_7 / _9 (tx_template.c:110-130)
    t7[0] = (float)cos(2 * M_PI / 7); t7[1] = (float)sin(2 * M_PI / 7); t7[2] = (float)sin(2 * M_PI / 28);
    t7[3] = (float)cos(2 * M_PI / 28); t7[4] = (float)cos(2 * M_PI / 14); t7[5] = (float)sin(2 * M_PI / 14);
    t9[0] = (float)cos(2 * M_PI / 3); t9[1] = (float)sin(2 * M_PI / 3); t9[2] = (float)cos(2 * M_PI / 9); t9[3] = (float)sin(2 * M_PI / 9);
    t9[4] = (float)cos(2 * M_PI / 36); t9[5] = (float)sin(2 * M_PI / 36); t9[6] = t9[2] + t9[5]; t9[7] = t9[3] - t9[4];
    for (int k = 3; k <= H.log2m; k++) {                            // ff_tx_init_tab_N (tx_template.c:65-77)
        const int nn = 1 << k;
        H.cosk[k].assign(nn / 4 + 1, 0.f);
        const double freq = 2 * M_PI / nn;
        for (int i = 0; i < nn / 4; i++) H.cosk[k][i] = (float)cos(i * freq);
    }
}

// host-only: the tables of a transform, flattened, for the CPU test tier: [in_map l2][out_map l2][sub_map m] as int32, then
// floats: exp, tab53[12] + tab7[6] + tab9[8], cosine tables k = 3 .. log2m.  Returns the number of 32-bit words (or what it would need if cap is short).
B200_API int b200_tx_pfa_tables(int inv, int len, float scale, int32_t *words, int cap, int32_t *layout8)
{
    if (!tx_pfa_length_ok(len)) return B200_ENOSYS;
    PfaHost H;
    pfa_host_tables(H, inv, len, scale);
    std::vector<int32_t> w;
    auto addi = [&](const std::vector<int> &v) { for (int x : v) w.push_back(x); };
    auto addf = [&](const float *f, size_t n) { for (size_t i = 0; i < n; i++) { int32_t b; memcpy(&b, f + i, 4); w.push_back(b); } };
    int32_t lay[8] = { 0 };
    lay[0] = (int32_t)w.size(); addi(H.in_map);
    lay[1] = (int32_t)w.size(); addi(H.out_map);
    lay[2] = (int32_t)w.size(); addi(H.sub_map);
    lay[3] = (int32_t)w.size(); addf(H.exp.data(), H.exp.size());
    lay[4] = (int32_t)w.size(); addf(H.tab53, 26);
    lay[5] = (int32_t)w.size();
    for (int k = 3; k <= H.log2m; k++) addf(H.cosk[k].data(), H.cosk[k].size());
    lay[6] = H.m; lay[7] = H.log2m | (H.nfac << 8);
    for (int L = 0; L < 12; L++) w.push_back(H.lvl_start[L]);      // after the cosine tables: 12 level starts, 12 level counts, the offsets
    for (int L = 0; L < 12; L++) w.push_back(H.lvl_cnt[L]);
    addi(H.blk);
    if (layout8) memcpy(layout8, lay, sizeof(lay));
    if (words && cap >= (int)w.size()) memcpy(words, w.data(), w.size() * 4);
    return (int)w.size();
}

static TxPfa *pfa_create(bool fft, int inv, int len, float scale)
{
    if (!(fft ? tx_pfa_fft_length_ok(len) : tx_pfa_length_ok(len))) return nullptr;
    PfaHost H;
    pfa_host_tables(H, inv, len, scale, fft);
    const int l2 = fft ? len : len >> 1, m = H.m;
    auto al = [](size_t v) { return (v + 255) & ~(size_t)255; };
    size_t off = 0;
    const size_t o_in = off;  off += al(sizeof(int) * l2);
    const size_t o_out = off; off += al(sizeof(int) * l2);
    const size_t o_sub = off; off += al(sizeof(int) * m);
    const size_t o_exp = off; off += al(sizeof(float) * H.exp.size());
    const size_t o_53 = off;  off += al(sizeof(float) * 26);
    size_t o_cos[12] = { 0 };
    for (int k = 3; k <= H.log2m; k++) { o_cos[k] = off; off += al(sizeof(float) * H.cosk[k].size()); }
    const size_t o_blk = off; off += al(sizeof(int) * H.blk.size() + 4);
    std::vector<uint8_t> host(off, 0);
    memcpy(&host[o_blk], H.blk.data(), sizeof(int) * H.blk.size());
    memcpy(&host[o_in], H.in_map.data(), sizeof(int) * l2);
    memcpy(&host[o_out], H.out_map.data(), sizeof(int) * l2);
    memcpy(&host[o_sub], H.sub_map.data(), sizeof(int) * m);
    if (!H.exp.empty()) memcpy(&host[o_exp], H.exp.data(), sizeof(float) * H.exp.size());
    memcpy(&host[o_53], H.tab53, sizeof(float) * 26);
    for (int k = 3; k <= H.log2m; k++) memcpy(&host[o_cos[k]], H.cosk[k].data(), sizeof(float) * H.cosk[k].size());
    TxPfa *p = new (std::nothrow) TxPfa();
    if (!p) return nullptr;
    p->inv = inv; p->len = len; p->m = m; p->fft = fft;
    if (cudaMalloc(&p->blob, off) != cudaSuccess || cudaMemcpy(p->blob, host.data(), off, cudaMemcpyHostToDevice) != cudaSuccess) {
        b200_set_error("tx_pfa_create: device tables");
        if (p->blob) cudaFree(p->blob);
        delete p;
        return nullptr;
    }
    uint8_t *b = (uint8_t *)p->blob;
    PfaDev &d = p->d;
    d.in_map = (const int *)(b + o_in); d.out_map = (const int *)(b + o_out); d.sub_map = (const int *)(b + o_sub);
    d.exp = (const float2 *)(b + o_exp); d.tab53 = (const float *)(b + o_53);
    for (int k = 0; k < 12; k++) d.tabs[k] = k >= 3 && k <= H.log2m ? (const float *)(b + o_cos[k]) : nullptr;
    d.m = m; d.log2m = H.log2m; d.len = len; d.nfac = H.nfac;
    d.blk = (const int *)(b + o_blk);
    for (int L = 0; L < 12; L++) { d.lvl_start[L] = H.lvl_start[L]; d.lvl_cnt[L] = H.lvl_cnt[L]; }
    d.ms = m + (m >> 4) + 1;
    p->smem = (size_t)H.nfac * d.ms * sizeof(float2);
    if (p->smem > 48 * 1024 &&
        (cudaFuncSetAttribute(tx_mdct_pfa_inv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p->smem) != cudaSuccess ||
         cudaFuncSetAttribute(tx_mdct_pfa_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p->smem) != cudaSuccess ||
         cudaFuncSetAttribute(tx_fft_pfa_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p->smem) != cudaSuccess)) {
        b200_set_error("tx_pfa_create: %zu bytes of shared memory per transform", p->smem);
        cudaFree(p->blob);
        delete p;
        return nullptr;
    }
    int dev = 0, sms = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    p->grid_cap = (sms > 0 ? sms : 132) * 8;
    return p;
}

TxPfa *tx_pfa_create(int inv, int len, float scale) { return pfa_create(false, inv, len, scale); }
TxPfa *tx_pfa_create_fft(int inv, int len) { return pfa_create(true, inv, len, 1.0f); }

void tx_pfa_free(TxPfa *p)
{
    if (!p) return;
    if (p->blob) cudaFree(p->blob);
    delete p;
}

int tx_pfa_launch(TxPfa *p, cudaStream_t st, void *out, const void *in, ptrdiff_t stride, int64_t count, ptrdiff_t out_step, ptrdiff_t in_step)
{
    if (count <= 0) return 0;
    if (p->fft) {                                          // complex in, complex out with a stride in bytes
        if (((reinterpret_cast<uintptr_t>(out) | (uintptr_t)out_step | reinterpret_cast<uintptr_t>(in) | (uintptr_t)in_step | (uintptr_t)stride) & 7) || stride <= 0) {
            b200_set_error("b200_tx_batch_device: compound FFT pointers, steps and stride must be multiples of 8 bytes");
            return B200_EINVAL;
        }
        const unsigned nbf = (unsigned)(count < p->grid_cap ? count : p->grid_cap);
        tx_fft_pfa_kernel<<<nbf, PFA_THREADS, p->smem, st>>>(p->d, (float2 *)out, (const float2 *)in, (long long)(stride / 8), out_step, in_step, count);
        B200_LAUNCHED();
        B200_CUDA_OK(cudaGetLastError());
        return 0;
    }
    // the inverse writes its outputs as complex pairs (8-byte words); everything else moves single floats
    if (((reinterpret_cast<uintptr_t>(out) | (uintptr_t)out_step) & (p->inv ? 7 : 3)) || ((reinterpret_cast<uintptr_t>(in) | (uintptr_t)in_step) & 3)) {
        b200_set_error("b200_tx_batch_device: compound MDCT input must be 4-byte aligned, output %d-byte aligned (pointers and steps)", p->inv ? 8 : 4);
        return B200_EINVAL;
    }
    // one CTA per transform, CTAs stride over the batch
    const unsigned nb = (unsigned)(count < p->grid_cap ? count : p->grid_cap);
    if (p->inv) tx_mdct_pfa_inv_kernel<<<nb, PFA_THREADS, p->smem, st>>>(p->d, (float *)out, (const float *)in, (long long)(stride / 4), out_step, in_step, count);
    else        tx_mdct_pfa_fwd_kernel<<<nb, PFA_THREADS, p->smem, st>>>(p->d, (float *)out, (const float *)in, (long long)(stride / 4), out_step, in_step, count);
    B200_LAUNCHED();
    B200_CUDA_OK(cudaGetLastError());
    return 0;
}
