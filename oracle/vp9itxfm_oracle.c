/* vp9itxfm_oracle.c — TEST INFRASTRUCTURE ONLY.  The checker of ffmpeg_b200/csrc/vp9itxfm.cu: VP9's itxfm_add members
 * (libavcodec/vp9dsp_template.c:1155-1778) restated on the host for 8, 10 and 12 bit samples, and the batch entry's semantics.
 *
 * Written in a different form from the kernel so that each checks the other: every value is an int64_t, and the 8-bit storage class's
 * 32-bit wrapping is applied explicitly (fix(): the value modulo 2^32 read as int32) at every stored stage value and before every
 * rounding shift, where the kernel computes in native uint32_t; the first stages of the 16- and 32-point transforms are driven by
 * tables of (input, input, cos, sin) rotations; the sum / difference stages are loops over index pairs.  Truncation to the storage
 * type (int16 at 8 bit, int32 above) is written out at the pass boundaries. */
#include <stdint.h>
#include <stddef.h>
#include <string.h>
#include "vp9itxfm_oracle.h"

typedef int64_t I;

/* wrap = 1: 8-bit storage class (32-bit arithmetic), 0: 10 / 12 bit (exact int64) */
static I fix(int wrap, I v) { return wrap ? (I)(int32_t)(uint32_t)(uint64_t)v : v; }
static I rnd(int wrap, I v) { return fix(wrap, v + 8192) >> 14; }
static I store(int depth, I v) { return depth == 8 ? (I)(int16_t)(uint16_t)(uint64_t)v : (I)(int32_t)(uint32_t)(uint64_t)v; }

/* p = rnd(x c - y s), q = rnd(x s + y c) */
static void rotate(int w, I x, I y, int c, int s, I *p, I *q)
{
    *p = rnd(w, fix(w, x * c) - fix(w, y * s));
    *q = rnd(w, fix(w, x * s) + fix(w, y * c));
}

/* ---------------------------------------------------------------- inverse DCT, n = 4, 8, 16, 32: even half recursively, odd part */
static void dct(int w, int n, const I *x, I *y);

static void dct_odd8(int w, const I *od, I *o)                      /* od[k] = input 2k + 1 */
{
    I a4, a5, a6, a7;
    rotate(w, od[0], od[3], 3196, 16069, &a4, &a7);
    rotate(w, od[2], od[1], 13623, 9102, &a5, &a6);
    const I s4 = fix(w, a4 + a5), d5 = fix(w, a4 - a5), d6 = fix(w, a7 - a6), s7 = fix(w, a7 + a6);
    o[0] = s7;
    o[1] = rnd(w, fix(w, (d6 + d5) * 11585));
    o[2] = rnd(w, fix(w, (d6 - d5) * 11585));
    o[3] = s4;
}

/* first-stage rotations of the 16- and 32-point odd parts: outputs (lo, hi) = rotate(input i, input j, c, s) */
struct rot1 { int i, j, c, s, lo, hi; };
static const struct rot1 k16[4] = {                                  /* inputs and outputs numbered as in the 16-point transform */
    { 1, 15, 1606, 16305, 8, 15 }, { 9, 7, 12665, 10394, 9, 14 }, { 5, 11, 7723, 14449, 10, 13 }, { 13, 3, 15679, 4756, 11, 12 } };
static const struct rot1 k32[8] = {
    { 1, 31, 804, 16364, 16, 31 }, { 17, 15, 12140, 11003, 17, 30 }, { 9, 23, 7005, 14811, 18, 29 }, { 25, 7, 15426, 5520, 19, 28 },
    { 5, 27, 3981, 15893, 20, 27 }, { 21, 11, 14053, 8423, 21, 26 }, { 13, 19, 9760, 13160, 22, 25 }, { 29, 3, 16207, 2404, 23, 24 } };

/* sum / difference of groups of four: t[k] = a + b, t[k + 1] = a - b, t[k + 2] = d - c, t[k + 3] = d + c for (a, b, c, d) = s[k..k+3] */
static void sumdiff4(int w, const I *s, I *t, int from, int to)
{
    for (int k = from; k < to; k += 4) {
        t[k] = fix(w, s[k] + s[k + 1]);
        t[k + 1] = fix(w, s[k] - s[k + 1]);
        t[k + 2] = fix(w, s[k + 3] - s[k + 2]);
        t[k + 3] = fix(w, s[k + 3] + s[k + 2]);
    }
}

/* rotation whose first output is rounded as computed and whose second is rounded negated */
static void rotate_neg(int w, I x, I y, int c, int s, I *p, I *nq)
{
    *p = rnd(w, fix(w, x * c) - fix(w, y * s));
    *nq = rnd(w, -fix(w, x * s + y * c));
}

static void dct_odd16(int w, const I *x, I *o)                       /* x = the 16 inputs */
{
    I s[16], t[16];
    for (int r = 0; r < 4; r++) rotate(w, x[k16[r].i], x[k16[r].j], k16[r].c, k16[r].s, &s[k16[r].lo], &s[k16[r].hi]);
    /* pairs (8, 9), (11, 10), (12, 13), (15, 14) */
    sumdiff4(w, s, t, 8, 16);
    I u9, u14, u13, u10;
    rotate(w, t[14], t[9], 6270, 15137, &u9, &u14);
    rotate_neg(w, t[13], t[10], 6270, 15137, &u13, &u10);
    const I v8 = fix(w, t[8] + t[11]), v11 = fix(w, t[8] - t[11]), v12 = fix(w, t[15] - t[12]), v15 = fix(w, t[15] + t[12]);
    const I v9 = fix(w, u9 + u10), v10 = fix(w, u9 - u10), v13 = fix(w, u14 - u13), v14 = fix(w, u14 + u13);
    o[0] = v15;
    o[1] = v14;
    o[2] = rnd(w, fix(w, (v13 + v10) * 11585));
    o[3] = rnd(w, fix(w, (v12 + v11) * 11585));
    o[4] = rnd(w, fix(w, (v12 - v11) * 11585));
    o[5] = rnd(w, fix(w, (v13 - v10) * 11585));
    o[6] = v9;
    o[7] = v8;
}

static void dct_odd32(int w, const I *x, I *o)                       /* x = the 32 inputs */
{
    I s[32], t[32], u[32], v[32], z[32];
    for (int r = 0; r < 8; r++) rotate(w, x[k32[r].i], x[k32[r].j], k32[r].c, k32[r].s, &s[k32[r].lo], &s[k32[r].hi]);
    sumdiff4(w, s, t, 16, 32);
    for (int k = 16; k < 32; k++) u[k] = t[k];
    rotate(w, t[30], t[17], 3196, 16069, &u[17], &u[30]);
    rotate_neg(w, t[29], t[18], 3196, 16069, &u[29], &u[18]);
    rotate(w, t[26], t[21], 13623, 9102, &u[21], &u[26]);
    rotate_neg(w, t[25], t[22], 13623, 9102, &u[25], &u[22]);
    /* groups of eight: (a, b, c, d, e, f, g, h) = u[k..k+7] -> a + d, b + c, b - c, a - d, h - e, g - f, g + f, h + e */
    for (int k = 16; k < 32; k += 8) {
        v[k]     = fix(w, u[k] + u[k + 3]);
        v[k + 1] = fix(w, u[k + 1] + u[k + 2]);
        v[k + 2] = fix(w, u[k + 1] - u[k + 2]);
        v[k + 3] = fix(w, u[k] - u[k + 3]);
        v[k + 4] = fix(w, u[k + 7] - u[k + 4]);
        v[k + 5] = fix(w, u[k + 6] - u[k + 5]);
        v[k + 6] = fix(w, u[k + 6] + u[k + 5]);
        v[k + 7] = fix(w, u[k + 7] + u[k + 4]);
    }
    for (int k = 16; k < 32; k++) z[k] = v[k];
    rotate(w, v[29], v[18], 6270, 15137, &z[18], &z[29]);
    rotate(w, v[28], v[19], 6270, 15137, &z[19], &z[28]);
    rotate_neg(w, v[27], v[20], 6270, 15137, &z[27], &z[20]);
    rotate_neg(w, v[26], v[21], 6270, 15137, &z[26], &z[21]);
    /* the 16 + 16 butterfly of the two halves: f[16 + k] for k < 4 sums, 4..7 differences, mirrored above 24 */
    I f[32];
    for (int k = 0; k < 4; k++) {
        f[16 + k] = fix(w, z[16 + k] + z[23 - k]);
        f[23 - k] = fix(w, z[16 + k] - z[23 - k]);
        f[31 - k] = fix(w, z[31 - k] + z[24 + k]);
        f[24 + k] = fix(w, z[31 - k] - z[24 + k]);
    }
    for (int k = 0; k < 4; k++) {
        o[k] = f[31 - k];
        o[15 - k] = f[16 + k];
        o[4 + k] = rnd(w, fix(w, (f[27 - k] + f[20 + k]) * 11585));
        o[11 - k] = rnd(w, fix(w, (f[27 - k] - f[20 + k]) * 11585));
    }
}

static void dct(int w, int n, const I *x, I *y)
{
    if (n == 4) {
        const I e0 = rnd(w, fix(w, (x[0] + x[2]) * 11585)), e1 = rnd(w, fix(w, (x[0] - x[2]) * 11585));
        I o0, o1;
        rotate(w, x[1], x[3], 6270, 15137, &o0, &o1);
        y[0] = fix(w, e0 + o1);
        y[1] = fix(w, e1 + o0);
        y[2] = fix(w, e1 - o0);
        y[3] = fix(w, e0 - o1);
        return;
    }
    I ev[16], e[16], od[16], o[16];
    for (int k = 0; k < n / 2; k++) ev[k] = x[2 * k], od[k] = x[2 * k + 1];
    dct(w, n / 2, ev, e);
    if (n == 8) dct_odd8(w, od, o);
    else if (n == 16) dct_odd16(w, x, o);
    else dct_odd32(w, x, o);
    for (int i = 0; i < n / 2; i++) {
        y[i] = fix(w, e[i] + o[i]);
        y[n - 1 - i] = fix(w, e[i] - o[i]);
    }
}

/* ---------------------------------------------------------------- inverse ADST, n = 4, 8, 16 */
/* the ADST's input rotation, unrounded: p = x c + y s, q = x s - y c */
static void arot(int w, I x, I y, int c, int s, I *p, I *q)
{
    *p = fix(w, x * c + y * s);
    *q = fix(w, x * s - y * c);
}

static void adst(int w, int n, const I *x, I *y)
{
    if (n == 4) {
        const I s0 = fix(w, 5283 * x[0] + 15212 * x[2] + 9929 * x[3]), s1 = fix(w, 9929 * x[0] - 5283 * x[2] - 15212 * x[3]);
        const I s2 = fix(w, 13377 * fix(w, x[0] - x[2] + x[3])), s3 = fix(w, 13377 * x[1]);
        y[0] = rnd(w, s0 + s3);
        y[1] = rnd(w, s1 + s3);
        y[2] = rnd(w, s2);
        y[3] = rnd(w, s0 + s1 - s3);
        return;
    }
    /* stage 1: rotation k pairs input n - 1 - 2k with input 2k, by the cospi of (2k + 1) / (4n) turns, folded onto the first quadrant */
    static const int c8[4][2] = { { 16305, 1606 }, { 14449, 7723 }, { 10394, 12665 }, { 4756, 15679 } };
    static const int c16[8][2] = { { 16364, 804 }, { 15893, 3981 }, { 14811, 7005 }, { 13160, 9760 }, { 11003, 12140 }, { 8423, 14053 },
                                   { 5520, 15426 }, { 2404, 16207 } };
    const int h = n / 2;
    I p[16], q[16];
    for (int k = 0; k < h; k++) {
        const int *c = n == 8 ? c8[k] : c16[k];
        arot(w, x[n - 1 - 2 * k], x[2 * k], c[0], c[1], &p[2 * k], &p[2 * k + 1]);
    }
    for (int k = 0; k < h; k++) {
        q[k] = rnd(w, p[k] + p[k + h]);
        q[k + h] = rnd(w, p[k] - p[k + h]);
    }
    I r[16];
    if (n == 16) {                                                   /* the 16-point transform's extra stage on the upper half */
        I u[16];
        arot(w, q[8], q[9], 16069, 3196, &u[8], &u[9]);
        arot(w, q[10], q[11], 9102, 13623, &u[10], &u[11]);
        arot(w, q[13], q[12], 3196, 16069, &u[13], &u[12]);
        arot(w, q[15], q[14], 13623, 9102, &u[15], &u[14]);
        for (int k = 0; k < 4; k++) {
            r[k] = fix(w, q[k] + q[k + 4]);
            r[k + 4] = fix(w, q[k] - q[k + 4]);
            r[k + 8] = rnd(w, u[k + 8] + u[k + 12]);
            r[k + 12] = rnd(w, u[k + 8] - u[k + 12]);
        }
    } else {
        for (int k = 0; k < 8; k++) r[k] = q[k];
    }
    /* the last stages, applied to each group of eight: r[g..g+7] -> outputs through the map below */
    const int groups = n / 8;
    I o[16];
    for (int g = 0; g < groups; g++) {
        const I *a = r + 8 * g;
        I w4, w5, w6, w7;
        arot(w, a[4], a[5], 15137, 6270, &w4, &w5);
        arot(w, a[7], a[6], 6270, 15137, &w7, &w6);
        I *b = o + 8 * g;
        b[0] = fix(w, a[0] + a[2]);                                   /* pre-sign outputs of the group, in order: */
        b[1] = fix(w, a[1] + a[3]);                                   /*  0: a0 + a2, 1: a1 + a3, 2: rnd(w4 + w6), 3: rnd(w5 + w7) */
        b[2] = rnd(w, w4 + w6);
        b[3] = rnd(w, w5 + w7);
        const I d2 = fix(w, a[0] - a[2]), d3 = fix(w, a[1] - a[3]), d6 = rnd(w, w4 - w6), d7 = rnd(w, w5 - w7);
        b[4] = fix(w, d2 + d3);                                       /*  4: d2 + d3 (then x 11585), 5: d2 - d3, 6: d6 + d7, 7: d6 - d7 */
        b[5] = fix(w, d2 - d3);
        b[6] = fix(w, d6 + d7);
        b[7] = fix(w, d6 - d7);
    }
    if (n == 8) {
        y[0] = o[0];
        y[7] = fix(w, -o[1]);
        y[1] = fix(w, -o[2]);
        y[6] = o[3];
        y[3] = fix(w, -rnd(w, fix(w, o[4] * 11585)));
        y[4] = rnd(w, fix(w, o[5] * 11585));
        y[2] = rnd(w, fix(w, o[6] * 11585));
        y[5] = fix(w, -rnd(w, fix(w, o[7] * 11585)));
        return;
    }
    /* 16 points: group 0 (r[0..7]) and group 1 (r[8..15]) */
    y[0] = o[0];
    y[15] = fix(w, -o[1]);
    y[3] = fix(w, -o[2]);
    y[12] = o[3];
    y[7] = rnd(w, fix(w, -o[4] * 11585));
    y[8] = rnd(w, fix(w, o[5] * 11585));
    y[4] = rnd(w, fix(w, o[6] * 11585));
    y[11] = rnd(w, fix(w, -o[7] * 11585));
    y[1] = fix(w, -o[8]);
    y[14] = o[9];
    y[2] = o[10];
    y[13] = fix(w, -o[11]);
    y[6] = rnd(w, fix(w, o[12] * 11585));
    y[9] = rnd(w, fix(w, -o[13] * 11585));
    y[5] = rnd(w, fix(w, -o[14] * 11585));
    y[10] = rnd(w, fix(w, o[15] * 11585));
}

/* ---------------------------------------------------------------- Walsh-Hadamard, 32-bit ints at every depth */
static void wht(const I *x, I *y, int first)
{
    const int sh = first ? 2 : 0;
    const I a = (int32_t)x[0] >> sh, c = (int32_t)x[1] >> sh, d = (int32_t)x[2] >> sh, b = (int32_t)x[3] >> sh;
    const I s = fix(1, a + c), t = fix(1, d - b), m = fix(1, s - t) >> 1;
    const I y1 = fix(1, m - b), y2 = fix(1, m - c);
    y[0] = fix(1, s - y1);
    y[1] = y1;
    y[2] = y2;
    y[3] = fix(1, t + y2);
}

enum { DCT, ADST, WHT };

static void tx1(int depth, int kind, int n, int first, const I *x, I *y)
{
    const int w = depth == 8;
    I t[32];
    if (kind == WHT) wht(x, t, first);
    else if (kind == ADST) adst(w, n, x, t);
    else dct(w, n, x, t);
    for (int k = 0; k < n; k++) y[k] = store(depth, t[k]);
}

static int clip(int v, int maxv) { return v < 0 ? 0 : v > maxv ? maxv : v; }

static I get(int depth, const void *b, int64_t i) { return depth == 8 ? ((const int16_t *)b)[i] : ((const int32_t *)b)[i]; }

/* dst += residual of the block read from `coef`; returns 1 for the DC-only path */
static int itxfm(int depth, int tx, int type, uint8_t *dst, ptrdiff_t stride, const void *coef, int eob)
{
    const int n = tx == 4 ? 4 : 4 << tx, maxv = (1 << depth) - 1;
    const int bits = tx == 4 ? 0 : tx == 0 ? 4 : tx == 1 ? 5 : 6;
    const int dconly = eob == 1 && (tx == 3 || (tx < 3 && type == 0));
    int res[32][32];                                                 /* [row][column] */
    if (dconly) {
        const int64_t c0 = get(depth, coef, 0);
        const int64_t t1 = depth == 8 ? (int64_t)(((int32_t)c0 * 11585 + 8192) >> 14) : (c0 * 11585 + 8192) >> 14;
        const int t = (int32_t)(uint32_t)(uint64_t)((t1 * 11585 + 8192) >> 14);
        const int v = (int32_t)((uint32_t)t + (1u << (bits - 1))) >> bits;
        for (int j = 0; j < n; j++)
            for (int i = 0; i < n; i++) res[j][i] = v;
    } else {
        const int ka = tx == 4 ? WHT : tx == 3 ? DCT : (type == 1 || type == 3) ? ADST : DCT;
        const int kb = tx == 4 ? WHT : tx == 3 ? DCT : (type == 2 || type == 3) ? ADST : DCT;
        I tmp[32][32], col[32], out[32];
        for (int i = 0; i < n; i++) {                                /* pass 1: column i of the block -> row i of tmp */
            for (int k = 0; k < n; k++) col[k] = get(depth, coef, i + (int64_t)k * n);
            tx1(depth, ka, n, 1, col, tmp[i]);
        }
        for (int i = 0; i < n; i++) {                                /* pass 2: column i of tmp -> column i of dst */
            for (int k = 0; k < n; k++) col[k] = tmp[k][i];
            tx1(depth, kb, n, 0, col, out);
            for (int j = 0; j < n; j++)
                res[j][i] = bits ? (int32_t)((uint32_t)(int32_t)out[j] + (1u << (bits - 1))) >> bits : (int32_t)out[j];
        }
    }
    for (int j = 0; j < n; j++)
        for (int i = 0; i < n; i++) {
            if (depth == 8) {
                uint8_t *p = dst + j * stride + i;
                *p = (uint8_t)clip((int32_t)((uint32_t)*p + (uint32_t)res[j][i]), maxv);
            } else {
                uint16_t *p = (uint16_t *)(dst + j * stride) + i;
                *p = (uint16_t)clip((int32_t)((uint32_t)*p + (uint32_t)res[j][i]), maxv);
            }
        }
    return dconly;
}

int orc_vp9_itxfm(int depth, int tx, int type, uint8_t *dst, ptrdiff_t stride, void *block, int eob)
{
    if ((depth != 8 && depth != 10 && depth != 12) || tx < 0 || tx > 4 || type < 0 || type > 3) return -1;
    const int n = tx == 4 ? 4 : 4 << tx, cs = depth == 8 ? 2 : 4;
    const int dconly = itxfm(depth, tx, type, dst, stride, block, eob);
    memset(block, 0, dconly ? (size_t)cs : (size_t)n * n * cs);
    return 0;
}

int64_t orc_vp9_itxfm_batch(int depth, int64_t nops, const B200Vp9TxOp *ops, const void *coef, uint8_t *dst, ptrdiff_t dst_stride)
{
    if (depth != 8 && depth != 10 && depth != 12) return -1;
    const int bps = depth == 8 ? 1 : 2, cs = depth == 8 ? 2 : 4;
    int64_t done = 0;
    for (int64_t i = 0; i < nops; i++) {
        const B200Vp9TxOp *op = &ops[i];
        if (op->tx > 4 || op->type > 3 || (op->coef_off & 15) || (op->dst_off % (4 * bps))) continue;
        itxfm(depth, op->tx, op->type, dst + op->dst_off, dst_stride, (const uint8_t *)coef + op->coef_off * cs, op->eob);
        done++;
    }
    return done;
}
