/*
 * hevcidct_oracle.c — TEST INFRASTRUCTURE ONLY.  CPU restatement of the HEVC residual members of HEVCDSPContext
 * (libavcodec/hevc/dsp.h:47-125: add_residual[4], dequant, transform_rdpcm, transform_4x4_luma, idct[4], idct_dc[4]: 15 functions per depth) as
 * ff_hevc_dsp_init installs them for depth 8, 9, 10 and 12 (hevc/dsp.c:198-215), and the batch semantics of
 * b200_hevc_transform_add_batch_device (include/b200dsp.h).
 *
 * Follows (behaviour, not text) hevc/dsp_template.c:46-309, written as matrix products rather than butterflies:
 *   idct    each pass y[n] = sum over the kept inputs k of T32[k 32 / N][n] x[k], then clip16((y + add) >> shift), shift 7 then
 *           20 - depth; column c of pass 1 keeps odd k < L(c) (L(0) = min(col_limit + 4, N), minus 4 after columns 4, 8, ... while
 *           below N), every row of pass 2 odd k < min(col_limit, N); at N = 32 also k = 2 (mod 4) by k / 2 < end / 2; N = 4 keeps all
 *   idct_dc (((c0 + 1) >> 1) + 2^(13 - depth)) >> (14 - depth) everywhere
 *   dst4    the 4x4 DST matrix of H.265 8.6.4.2 with the idct's shifts
 *   dequant s = 15 - depth - log2: (c + 2^(s - 1)) >> s; s == 0 nothing; s < 0 (uint16) c << -s stored to int16
 *   rdpcm   running int16 sums along rows (mode 0) or down columns
 *   add     clip(dst + res)
 * T32 is the standard's 32-point matrix: T32[k][n] = c((k (2n + 1)) mod 128) from the scaled cosines c(0..32), row 0 all 64.
 */
#include <string.h>
#include "oracle.h"
#include "../include/b200dsp.h"

static int t32(int k, int n)
{
    static const int c[33] = { 64, 90, 90, 90, 89, 88, 87, 85, 83, 82, 80, 78, 75, 73, 70, 67, 64, 61, 57, 54, 50, 46, 43, 38, 36, 31, 25, 22,
                               18, 13, 9, 4, 0 };
    if (k == 0) return 64;
    const int m = (k * (2 * n + 1)) & 127;
    return m <= 32 ? c[m] : m <= 64 ? -c[64 - m] : m <= 96 ? -c[m - 64] : c[128 - m];
}
static int clip16(int v) { return v < -32768 ? -32768 : v > 32767 ? 32767 : v; }

/* does the reference's N-point butterfly with end `e` sum input k? */
static int kept(int N, int k, int e)
{
    if (N == 4 || k % 4 == 0 || (k % 2 == 0 && N != 32)) return 1;
    if (k % 2) return k < e;
    return k / 2 < (e >= 0 ? e / 2 : -1);
}

static void idct(int depth, int N, int16_t *c, int col_limit)
{
    int16_t t[32 * 32];
    long long l = (long long)col_limit + 4;                     /* the reference's int arithmetic, wrapping */
    l = (int)(unsigned)l;
    int lim2 = l < N ? (int)l : N;
    for (int col = 0; col < N; col++) {
        for (int n = 0; n < N; n++) {
            int s = 0;
            for (int k = 0; k < N; k++)
                if (kept(N, k, lim2)) s += t32(k * (32 / N), n) * c[k * N + col];
            t[n * N + col] = (int16_t)clip16((s + 64) >> 7);
        }
        if (lim2 < N && col % 4 == 0 && col) lim2 = (int)((unsigned)lim2 - 4u);
    }
    const int lim = col_limit < N ? col_limit : N, sh = 20 - depth;
    for (int r = 0; r < N; r++)
        for (int n = 0; n < N; n++) {
            int s = 0;
            for (int k = 0; k < N; k++)
                if (kept(N, k, lim)) s += t32(k * (32 / N), n) * t[r * N + k];
            c[r * N + n] = (int16_t)clip16((s + (1 << (sh - 1))) >> sh);
        }
}

/* DST-VII 4x4 of H.265 8.6.4.2: rows (29 55 74 84) (74 74 0 -74) (84 -29 -74 55) (55 -84 74 -29) */
static const int DST[4][4] = { { 29, 55, 74, 84 }, { 74, 74, 0, -74 }, { 84, -29, -74, 55 }, { 55, -84, 74, -29 } };

static void dst4(int depth, int16_t *c)
{
    int16_t t[16];
    for (int col = 0; col < 4; col++)
        for (int n = 0; n < 4; n++) {
            int s = 0;
            for (int k = 0; k < 4; k++) s += DST[k][n] * c[k * 4 + col];
            t[n * 4 + col] = (int16_t)clip16((s + 64) >> 7);
        }
    const int sh = 20 - depth;
    for (int r = 0; r < 4; r++)
        for (int n = 0; n < 4; n++) {
            int s = 0;
            for (int k = 0; k < 4; k++) s += DST[k][n] * t[r * 4 + k];
            c[r * 4 + n] = (int16_t)clip16((s + (1 << (sh - 1))) >> sh);
        }
}

static void dequant(int depth, int log2, int16_t *c)
{
    const int N = 1 << log2, s = 15 - depth - log2;
    for (int i = 0; i < N * N; i++) {
        if (s > 0) c[i] = (int16_t)((c[i] + (1 << (s - 1))) >> s);
        else if (s < 0) c[i] = (int16_t)(uint16_t)((unsigned)(uint16_t)c[i] << -s);
    }
}

static void rdpcm(int log2, int16_t *c, int mode)
{
    const int N = 1 << log2;
    for (int a = 0; a < N; a++)
        for (int b = 1; b < N; b++) {
            int16_t *p = mode ? &c[b * N + a] : &c[a * N + b];
            *p = (int16_t)(*p + (mode ? c[(b - 1) * N + a] : c[a * N + b - 1]));
        }
}

/* fn: 0 idct[log2 - 2](c, arg), 1 idct_dc[log2 - 2], 2 transform_4x4_luma, 3 dequant(c, log2), 4 transform_rdpcm(c, log2, arg);
 * -1 for arguments outside what the reference's functions take */
int orc_hevc_tx(int depth, int fn, int log2, int16_t *c, int arg)
{
    if (log2 < 2 || log2 > 5 || (fn == 2 && log2 != 2) || fn < 0 || fn > 4) return -1;
    const int N = 1 << log2;
    switch (fn) {
    case 0: idct(depth, N, c, arg); break;
    case 1: {
        const int v = (((c[0] + 1) >> 1) + (1 << (13 - depth))) >> (14 - depth);
        for (int i = 0; i < N * N; i++) c[i] = (int16_t)v;
        break;
    }
    case 2: dst4(depth, c); break;
    case 3: dequant(depth, log2, c); break;
    case 4: rdpcm(log2, c, arg); break;
    }
    return 0;
}

/* add_residual[log2 - 2] */
int orc_hevc_add_residual(int depth, int log2, uint8_t *dst, const int16_t *res, ptrdiff_t stride)
{
    const int N = 1 << log2, maxv = (1 << depth) - 1;
    if (log2 < 2 || log2 > 5) return -1;
    for (int y = 0; y < N; y++)
        for (int x = 0; x < N; x++) {
            uint8_t *row = dst + y * stride;
            const int v = (depth > 8 ? ((uint16_t *)row)[x] : row[x]) + res[y * N + x];
            const int o = v < 0 ? 0 : v > maxv ? maxv : v;
            if (depth > 8) ((uint16_t *)row)[x] = (uint16_t)o;
            else row[x] = (uint8_t)o;
        }
    return 0;
}

/* b200_hevc_transform_add_batch_device on host memory (coef is not written); returns the number of ops that wrote their block */
int64_t orc_hevc_tu_batch(int depth, int64_t nops, const B200HevcTuOp *ops, const int16_t *coef, uint8_t *dst, ptrdiff_t dst_stride)
{
    const int bps = depth > 8 ? 2 : 1;
    int16_t c[32 * 32];
    int64_t done = 0;
    for (int64_t i = 0; i < nops; i++) {
        const B200HevcTuOp *op = &ops[i];
        const int log2 = op->log2_size, N = 1 << (log2 & 7), k = op->kind, f = op->flags;
        if (log2 < 2 || log2 > 5 || k > B200_HEVC_TU_BYPASS || (k == B200_HEVC_TU_DST4 && log2 != 2) || (op->coef_off & 7) ||
            (op->dst_off % (4 * bps)))
            continue;
        memcpy(c, coef + op->coef_off, (size_t)N * N * sizeof(int16_t));
        if (k == B200_HEVC_TU_IDCT) orc_hevc_tx(depth, 0, log2, c, op->col_limit);
        else if (k == B200_HEVC_TU_IDCT_DC) orc_hevc_tx(depth, 1, log2, c, 0);
        else if (k == B200_HEVC_TU_DST4) orc_hevc_tx(depth, 2, log2, c, 0);
        else {
            if (k == B200_HEVC_TU_SKIP) {
                if ((f & B200_HEVC_TU_ROTATE) && log2 == 2)
                    for (int j = 0; j < 8; j++) { const int16_t t = c[j]; c[j] = c[15 - j]; c[15 - j] = t; }
                orc_hevc_tx(depth, 3, log2, c, 0);
            }
            if (f & B200_HEVC_TU_RDPCM) orc_hevc_tx(depth, 4, log2, c, !!(f & B200_HEVC_TU_RDPCM_VER));
        }
        orc_hevc_add_residual(depth, log2, dst + op->dst_off, c, dst_stride);
        done++;
    }
    return done;
}
