// hevcidct_dev.cuh — the HEVC residual arithmetic (hevc/dsp_template.c:46-309) shared by the transform batch (hevcidct.cu) and the
// picture intra reconstruction (hevcintra.cu): the 32-point matrix, the partial butterflies, the 4x4 DST, the col_limit masks and the
// per-line work of the two passes.  The semantics are those listed at the top of hevcidct.cu.
#pragma once
#include "common.h"

namespace {

enum { K_IDCT = B200_HEVC_TU_IDCT, K_DC = B200_HEVC_TU_IDCT_DC, K_DST4 = B200_HEVC_TU_DST4, K_SKIP = B200_HEVC_TU_SKIP,
       K_BYPASS = B200_HEVC_TU_BYPASS };

// The 32-point HEVC transform matrix (H.265 8.6.4.2): row k, column n is c(k (2n + 1) mod 128) with c(m) the scaled cos(pi m / 64)
// of the standard's coefficient list, by the cosine's symmetries; row 0 is 64.
struct Mat32 { int8_t v[32][32]; };
constexpr int cosv(int m)
{
    constexpr int c[33] = { 64, 90, 90, 90, 89, 88, 87, 85, 83, 82, 80, 78, 75, 73, 70, 67, 64, 61, 57, 54, 50, 46, 43, 38, 36, 31, 25, 22,
                            18, 13, 9, 4, 0 };
    return m <= 32 ? c[m] : m <= 64 ? -c[64 - m] : m <= 96 ? -c[m - 64] : c[128 - m];
}
constexpr Mat32 make_t32()
{
    Mat32 t{};
    for (int k = 0; k < 32; k++)
        for (int n = 0; n < 32; n++) t.v[k][n] = (int8_t)(k ? cosv((k * (2 * n + 1)) & 127) : 64);
    return t;
}
__constant__ Mat32 c_t32 = make_t32();

// partial butterfly of N points, inputs x[k S], k < N (the reference's TR_4 .. TR_32 with every input taken)
template <int N, int S>
__device__ __forceinline__ void idct1d(const int *x, int *y)
{
    if constexpr (N == 4) {
        const int e0 = 64 * x[0] + 64 * x[2 * S], e1 = 64 * x[0] - 64 * x[2 * S];
        const int o0 = 83 * x[S] + 36 * x[3 * S], o1 = 36 * x[S] - 83 * x[3 * S];
        y[0] = e0 + o0;
        y[1] = e1 + o1;
        y[2] = e1 - o1;
        y[3] = e0 - o0;
    } else {
        int e[N / 2];
        idct1d<N / 2, 2 * S>(x, e);
#pragma unroll
        for (int i = 0; i < N / 2; i++) {
            int o = 0;
#pragma unroll
            for (int j = 1; j < N; j += 2) o += c_t32.v[j * (32 / N)][i] * x[j * S];
            y[i] = e[i] + o;
            y[N - 1 - i] = e[i] - o;
        }
    }
}

// the DST of transform_4x4_luma (TR_4x4_LUMA)
__device__ __forceinline__ void dst4(const int *s, int *d)
{
    const int c0 = s[0] + s[2], c1 = s[2] + s[3], c2 = s[0] - s[3], c3 = 74 * s[1];
    d[2] = 74 * (s[0] - s[2] + s[3]);
    d[0] = 29 * c0 + 55 * c1 + c3;
    d[1] = 55 * c2 - 29 * c1 + c3;
    d[3] = 55 * c0 + 29 * c2 - c3;
}

__device__ __forceinline__ int clip16(int v) { return v < -32768 ? -32768 : v > 32767 ? 32767 : v; }

// input j of an N-point butterfly that the reference sums with end E (odd j < E; j = 2 mod 4 at 32 points by j / 2 < E / 2)
template <int N>
__device__ __forceinline__ bool kept(int j, int E)
{
    if (N == 4 || (j & 1) == 0 && (N != 32 || (j & 3) == 0)) return true;
    return (j & 1) ? j < E : (j >> 1) < (E >> 1);
}

// first-pass limit of column c: limit2 as the reference's loop leaves it (int arithmetic wrapping like the compiled reference's)
template <int N>
__device__ __forceinline__ int col_end(int col_limit, int c)
{
    const int l0 = (int)((unsigned)col_limit + 4u);
    int l = l0 < N ? l0 : N;
    for (int i = 4; i < c; i += 4)
        if (l < N) l = (int)((unsigned)l - 4u);
    return l;
}

// pass 1 of one op, column c: the coefficients A (N x N, row-major) to the pass-1 array B (rows of N + 2).  Op: anything with the
// members col_limit and flags (B200_HEVC_TU_*) of B200HevcTuOp
template <int N, typename Op>
__device__ __forceinline__ void pass1_col(const Op &op, int kind, int c, const int16_t *A, int16_t *B, int depth)
{
    if (kind == K_DC) return;
    int x[N], y[N];
#pragma unroll
    for (int j = 0; j < N; j++) x[j] = A[j * N + c];
    if (kind == K_IDCT || kind == K_DST4) {
        if (kind == K_DST4) {
            dst4(x, y);
        } else {
            const int E = col_end<N>(op.col_limit, c);
#pragma unroll
            for (int j = 0; j < N; j++) x[j] = kept<N>(j, E) ? x[j] : 0;
            idct1d<N, 1>(x, y);
        }
#pragma unroll
        for (int j = 0; j < N; j++) B[j * (N + 2) + c] = (int16_t)clip16((y[j] + 64) >> 7);
        return;
    }
    if (kind == K_SKIP) {
        if (N == 4 && (op.flags & B200_HEVC_TU_ROTATE)) {
#pragma unroll
            for (int j = 0; j < N; j++) x[j] = A[15 - (j * N + c)];
        }
        const int s = 15 - depth - (N == 4 ? 2 : N == 8 ? 3 : N == 16 ? 4 : 5);
        if (s > 0) {
#pragma unroll
            for (int j = 0; j < N; j++) x[j] = (int16_t)((x[j] + (1 << (s - 1))) >> s);
        } else if (s < 0) {
#pragma unroll
            for (int j = 0; j < N; j++) x[j] = (int16_t)(uint16_t)((unsigned)(uint16_t)x[j] << -s);
        }
    }
    if ((op.flags & (B200_HEVC_TU_RDPCM | B200_HEVC_TU_RDPCM_VER)) == (B200_HEVC_TU_RDPCM | B200_HEVC_TU_RDPCM_VER)) {
#pragma unroll
        for (int j = 1; j < N; j++) x[j] = (int16_t)(x[j] + x[j - 1]);
    }
#pragma unroll
    for (int j = 0; j < N; j++) B[j * (N + 2) + c] = (int16_t)x[j];
}

// pass 2 of one op, row r: the residual y[0 .. N - 1] of the row, from B (or from A[0] for the DC kind)
template <int N, typename Op>
__device__ __forceinline__ void pass2_row(const Op &op, int kind, int r, const int16_t *A, const int16_t *B, int depth, int *y)
{
    int x[N];
    if (kind == K_DC) {
        const int v = (((A[0] + 1) >> 1) + (1 << (13 - depth))) >> (14 - depth);
#pragma unroll
        for (int j = 0; j < N; j++) y[j] = v;
    } else {
#pragma unroll
        for (int j = 0; j < N; j++) x[j] = B[r * (N + 2) + j];
        const int sh = 20 - depth, add = 1 << (sh - 1);
        if (kind == K_IDCT || kind == K_DST4) {
            if (kind == K_DST4) {
                dst4(x, y);
            } else {
                const int E = op.col_limit < N ? op.col_limit : N;
#pragma unroll
                for (int j = 0; j < N; j++) x[j] = kept<N>(j, E) ? x[j] : 0;
                idct1d<N, 1>(x, y);
            }
#pragma unroll
            for (int j = 0; j < N; j++) y[j] = clip16((y[j] + add) >> sh);
        } else {
            if ((op.flags & (B200_HEVC_TU_RDPCM | B200_HEVC_TU_RDPCM_VER)) == B200_HEVC_TU_RDPCM) {
#pragma unroll
                for (int j = 1; j < N; j++) x[j] = (int16_t)(x[j] + x[j - 1]);
            }
#pragma unroll
            for (int j = 0; j < N; j++) y[j] = x[j];
        }
    }
}

// one destination word of 4 samples: load, add, clip, store
template <typename P>
__device__ __forceinline__ void add4(P *d, const int *r, int maxv)
{
    if constexpr (sizeof(P) == 1) {
        const unsigned w = *reinterpret_cast<const unsigned *>(d);
        unsigned o = 0;
#pragma unroll
        for (int k = 0; k < 4; k++) o |= (unsigned)min(max((int)((w >> (8 * k)) & 0xFF) + r[k], 0), maxv) << (8 * k);
        *reinterpret_cast<unsigned *>(d) = o;
    } else {
        const uint2 w = *reinterpret_cast<const uint2 *>(d);
        const int s0 = w.x & 0xFFFF, s1 = w.x >> 16, s2 = w.y & 0xFFFF, s3 = w.y >> 16;
        uint2 o;
        o.x = (unsigned)min(max(s0 + r[0], 0), maxv) | (unsigned)min(max(s1 + r[1], 0), maxv) << 16;
        o.y = (unsigned)min(max(s2 + r[2], 0), maxv) | (unsigned)min(max(s3 + r[3], 0), maxv) << 16;
        *reinterpret_cast<uint2 *>(d) = o;
    }
}

} // namespace
