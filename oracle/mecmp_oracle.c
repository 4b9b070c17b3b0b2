/*
 * mecmp_oracle.c — TEST INFRASTRUCTURE ONLY.  CPU restatement of libavcodec's me_cmp SAD/SSE and of the exhaustive
 * search that drives it.
 *
 * Follows (behaviour, not text):
 *   pix_abs16_c / pix_abs8_c ........ libavcodec/me_cmp.c:117-143, 272-290     sum |a-b| over w x h, one stride for both
 *   pix_abs{16,8}_{x2,y2,xy2}_c ..... libavcodec/me_cmp.c:145-385             blk2 interpolated: avg2 = (a+b+1)>>1,
 *                                                                             avg4 = (a+b+c+d+2)>>2 (:114-115)
 *   sse16_c / sse8_c / sse4_c ....... libavcodec/me_cmp.c:37-103               sum (a-b)^2
 *   vsad / vsad_intra, vsse / vsse_intra  libavcodec/me_cmp.c:843-931          vertical gradient of the difference (or of the block itself)
 *   nsse16_c / nsse8_c .............. libavcodec/me_cmp.c:387-437             SSE + weight * |difference of the two blocks' 2x2 gradient energy|
 *   pix_median_abs16_c / 8_c ........ libavcodec/me_cmp.c:145-183, 292-330    residual of the difference after median (left, top, gradient) prediction
 *   hadamard8_intra8x8_c / 16 ....... libavcodec/me_cmp.c:564-612, 944        SATD of the block itself minus |DC|
 *   sum_abs_dctelem_c ............... libavcodec/me_cmp.c:105-112             sum |block[i]|, i < 64
 *   dct_sad8x8_c / dct_max8x8_c ..... libavcodec/me_cmp.c:614-622, 678-693     forward DCT of blk1 - blk2 (pixblockdsp.c:40-59), then sum / max of |coef|
 *   ff_jpeg_fdct_islow_8 ............ libavcodec/jfdctint_template.c:173-340   FDCTDSPContext.fdct for FF_DCT_AUTO (fdctdsp.c:27-45): LL&M, 13-bit
 *                                                                             constants, PASS1_BITS 4, products modulo 2^32, stores truncated to int16
 *   ff_fdct_ifast ................... libavcodec/jfdctfst.c:140-284            FF_DCT_FASTINT: AA&N, 8-bit constants, (x * c) >> 8 without rounding
 *   dct264_sad8x8_c ................. libavcodec/me_cmp.c:624-675              H.264 8x8 integer transform, rows stored as int16, columns summed
 *   16 wide entries ................. libavcodec/me_cmp.c:933-959              WRAPPER8_16_SQ: two blocks, four when h == 16 (the scores add up)
 *   table layout .................... libavcodec/me_cmp.c:961-1027             sad[0]=16 wide, sad[1]=8; sse[0..2]=16,8,4;
 *                                                                             pix_abs[0=16,1=8][0 full,1 x2,2 y2,3 xy2]
 *   ff_me_cmp_sad, ff_me_search_esa . libavfilter/motion_estimation.c:60-97   cost(0 mv) first, return at once if it is 0,
 *                                                                             raster scan, strict '<' keeps the first minimum
 *   frame driver .................... libavfilter/vf_mestimate.c:85-127       mv initialised to the block's own position,
 *                                                                             window clipped to [0, (b_w-1)<<log2] etc.
 */
#include "oracle.h"
#include <stdlib.h>

static int sad_wh(const uint8_t *a, const uint8_t *b, ptrdiff_t stride, int w, int h, int mode)
{
    int s = 0;
    for (int y = 0; y < h; y++, a += stride, b += stride)
        for (int x = 0; x < w; x++) {
            int p;
            switch (mode) {
            case 0:  p = b[x]; break;
            case 1:  p = (b[x] + b[x + 1] + 1) >> 1; break;
            case 2:  p = (b[x] + b[x + stride] + 1) >> 1; break;
            default: p = (b[x] + b[x + 1] + b[x + stride] + b[x + stride + 1] + 2) >> 2; break;
            }
            s += abs(a[x] - p);
        }
    return s;
}

static int sse_wh(const uint8_t *a, const uint8_t *b, ptrdiff_t stride, int w, int h)
{
    int s = 0;
    for (int y = 0; y < h; y++, a += stride, b += stride)
        for (int x = 0; x < w; x++) {
            int d = a[x] - b[x];
            s += d * d;
        }
    return s;
}

/* hadamard8_diff8x8_c (me_cmp.c:514-562): sum of the absolute values of the 8x8 Hadamard transform of src - dst; the result is
 * the same whatever order the butterflies run in (exact integers).  The 16-wide entry is the WRAPPER8_16_SQ of it (:933-950):
 * two 8x8 blocks side by side, two more below them when h == 16; the 8-wide entry ignores h. */
static int satd8x8(const uint8_t *dst, const uint8_t *src, ptrdiff_t stride)
{
    int t[64], sum = 0;
    for (int i = 0; i < 8; i++)
        for (int j = 0; j < 8; j++) t[8 * i + j] = src[stride * i + j] - dst[stride * i + j];
    for (int pass = 0; pass < 2; pass++) {                         /* rows, then columns */
        const int es = pass ? 8 : 1, ls = pass ? 1 : 8;
        for (int l = 0; l < 8; l++)
            for (int span = 1; span < 8; span <<= 1)
                for (int a = 0; a < 8; a++)
                    if (!(a & span)) {
                        const int x = t[l * ls + a * es], y = t[l * ls + (a + span) * es];
                        t[l * ls + a * es] = x + y; t[l * ls + (a + span) * es] = x - y;
                    }
    }
    for (int i = 0; i < 64; i++) sum += abs(t[i]);
    return sum;
}

static int mid3(int a, int b, int c)            /* mid_pred (libavutil/common.h / mathops.h): median of three */
{
    if (a > b) { if (c > b) { b = c > a ? a : c; } }
    else       { if (b > c) { b = c > a ? c : a; } }
    return b;
}

/* vsad / vsse (intra = the block itself): rows 1 .. h-1 against the row above */
static int vgrad_wh(const uint8_t *s1, const uint8_t *s2, ptrdiff_t stride, int w, int h, int intra, int sq)
{
    int score = 0;
    for (int y = 1; y < h; y++, s1 += stride, s2 += stride)
        for (int x = 0; x < w; x++) {
            const int d = intra ? s1[x] - s1[x + stride] : s1[x] - s2[x] - s1[x + stride] + s2[x + stride];
            score += sq ? d * d : abs(d);
        }
    return score;
}

static int nsse_wh(const uint8_t *s1, const uint8_t *s2, ptrdiff_t stride, int w, int h, int weight)
{
    int score1 = 0, score2 = 0;
    for (int y = 0; y < h; y++, s1 += stride, s2 += stride) {
        for (int x = 0; x < w; x++) score1 += (s1[x] - s2[x]) * (s1[x] - s2[x]);
        if (y + 1 < h)
            for (int x = 0; x < w - 1; x++)
                score2 += abs(s1[x] - s1[x + stride] - s1[x + 1] + s1[x + stride + 1]) -
                          abs(s2[x] - s2[x + stride] - s2[x + 1] + s2[x + stride + 1]);
    }
    return score1 + abs(score2) * weight;
}

static int median_sad_wh(const uint8_t *p1, const uint8_t *p2, ptrdiff_t stride, int w, int h)
{
    int s = 0;
#define V(x) (p1[x] - p2[x])
    s += abs(V(0));
    for (int j = 1; j < w; j++) s += abs(V(j) - V(j - 1));
    p1 += stride; p2 += stride;
    for (int i = 1; i < h; i++, p1 += stride, p2 += stride) {
        s += abs(V(0) - V(-stride));
        for (int j = 1; j < w; j++)
            s += abs(V(j) - mid3(V(j - stride), V(j - 1), V(j - stride) + V(j - 1) - V(j - stride - 1)));
    }
#undef V
    return s;
}

/* hadamard8_intra8x8_c: the transform of the block itself; the DC term (sum of all 64 samples) is left out */
static int satd8x8_intra(const uint8_t *src, ptrdiff_t stride)
{
    int t[64], sum = 0;
    for (int i = 0; i < 8; i++)
        for (int j = 0; j < 8; j++) t[8 * i + j] = src[stride * i + j];
    for (int pass = 0; pass < 2; pass++) {
        const int es = pass ? 8 : 1, ls = pass ? 1 : 8;
        for (int l = 0; l < 8; l++)
            for (int span = 1; span < 8; span <<= 1)
                for (int a = 0; a < 8; a++)
                    if (!(a & span)) {
                        const int x = t[l * ls + a * es], y = t[l * ls + (a + span) * es];
                        t[l * ls + a * es] = x + y; t[l * ls + (a + span) * es] = x - y;
                    }
    }
    for (int i = 0; i < 64; i++) sum += abs(t[i]);
    return sum - abs(t[0]);
}

/* ---- transform-domain comparisons: dct_sad (fn 8), dct_max (fn 9), dct264_sad (fn 10) ---- */
static int g_dct_algo = 0;                      /* AVCodecContext.dct_algo: 0 FF_DCT_AUTO (islow), 1 FF_DCT_FASTINT (ifast) */
void orc_me_cmp_set_dct_algo(int algo) { g_dct_algo = algo; }

static int16_t descale16(uint32_t x, int n) { return (int16_t)(((int32_t)x + (1 << (n - 1))) >> n); }

/* one 1-D pass of the "slow" integer DCT over eight samples at p[0], p[st], ...; second = the column pass */
static void islow_pass_bits(int16_t *p, int st, int second, int p1, int outs);
static void islow_pass(int16_t *p, int st, int second) { islow_pass_bits(p, st, second, 4, 4); }
/* p1 = PASS1_BITS, outs = OUT_SHIFT: 4 / 4 for 8-bit samples, 1 / 2 for 10-bit (jfdctint_template.c:84-92) */
static void islow_pass_bits(int16_t *p, int st, int second, int p1, int outs)
{
    const int x0 = p[0], x1 = p[st], x2 = p[2 * st], x3 = p[3 * st], x4 = p[4 * st], x5 = p[5 * st], x6 = p[6 * st], x7 = p[7 * st];
    const int s0 = x0 + x7, s1 = x1 + x6, s2 = x2 + x5, s3 = x3 + x4;
    const int d0 = x0 - x7, d1 = x1 - x6, d2 = x2 - x5, d3 = x3 - x4;
    const int e0 = s0 + s3, e3 = s0 - s3, e1 = s1 + s2, e2 = s1 - s2;
    const int sh = second ? 13 + outs : 13 - p1, rnd = 1 << (outs - 1);
    if (second) { p[0] = (int16_t)((e0 + e1 + rnd) >> outs); p[4 * st] = (int16_t)((e0 - e1 + rnd) >> outs); }
    else        { p[0] = (int16_t)((e0 + e1) * (1 << p1)); p[4 * st] = (int16_t)((e0 - e1) * (1 << p1)); }
    const uint32_t r = (uint32_t)(e2 + e3) * 4433u;
    p[2 * st] = descale16(r + (uint32_t)e3 * 6270u, sh);
    p[6 * st] = descale16(r - (uint32_t)e2 * 15137u, sh);
    uint32_t z1 = (uint32_t)(d3 + d0), z2 = (uint32_t)(d2 + d1), z3 = (uint32_t)(d3 + d1), z4 = (uint32_t)(d2 + d0);
    const uint32_t z5 = (z3 + z4) * 9633u;
    const uint32_t t4 = (uint32_t)d3 * 2446u, t5 = (uint32_t)d2 * 16819u, t6 = (uint32_t)d1 * 25172u, t7 = (uint32_t)d0 * 12299u;
    z1 *= (uint32_t)-7373; z2 *= (uint32_t)-20995; z3 = z3 * (uint32_t)-16069 + z5; z4 = z4 * (uint32_t)-3196 + z5;
    p[7 * st] = descale16(t4 + z1 + z3, sh);
    p[5 * st] = descale16(t5 + z2 + z4, sh);
    p[3 * st] = descale16(t6 + z2 + z3, sh);
    p[1 * st] = descale16(t7 + z1 + z4, sh);
}

static int ifast_mul(int v, int c) { return (int16_t)((v * c) >> 8); }
static void ifast_pass(int16_t *p, int st)
{
    const int x0 = p[0], x1 = p[st], x2 = p[2 * st], x3 = p[3 * st], x4 = p[4 * st], x5 = p[5 * st], x6 = p[6 * st], x7 = p[7 * st];
    const int s0 = x0 + x7, s1 = x1 + x6, s2 = x2 + x5, s3 = x3 + x4;
    const int d0 = x0 - x7, d1 = x1 - x6, d2 = x2 - x5, d3 = x3 - x4;
    const int e0 = s0 + s3, e3 = s0 - s3, e1 = s1 + s2, e2 = s1 - s2;
    p[0] = (int16_t)(e0 + e1); p[4 * st] = (int16_t)(e0 - e1);
    const int r = ifast_mul(e2 + e3, 181);
    p[2 * st] = (int16_t)(e3 + r); p[6 * st] = (int16_t)(e3 - r);
    const int a = d3 + d2, b = d2 + d1, c = d1 + d0;
    const int z5 = ifast_mul(a - c, 98), z2 = ifast_mul(a, 139) + z5, z4 = ifast_mul(c, 334) + z5, z3 = ifast_mul(b, 181);
    const int z11 = d0 + z3, z13 = d0 - z3;
    p[5 * st] = (int16_t)(z13 + z2); p[3 * st] = (int16_t)(z13 - z2); p[1 * st] = (int16_t)(z11 + z4); p[7 * st] = (int16_t)(z11 - z4);
}

/* column pass of the 2-4-8 DCT (ff_fdct248_islow, jfdctint_template.c:347-412; ff_fdct_ifast248, jfdctfst.c:286-343): the even part of the
 * 1-D DCT on the sums of line pairs (rows 0 4 2 6) and on their differences (rows 1 5 3 7) */
static void col248(int16_t *p, int fast, int outs)
{
    const int x[8] = { p[0], p[8], p[16], p[24], p[32], p[40], p[48], p[56] };
    for (int half = 0; half < 2; half++) {
        int a[4];
        for (int k = 0; k < 4; k++) a[k] = half ? x[2 * k] - x[2 * k + 1] : x[2 * k] + x[2 * k + 1];
        const int t10 = a[0] + a[3], t11 = a[1] + a[2], t12 = a[1] - a[2], t13 = a[0] - a[3];
        int16_t *o = p + 8 * half;
        if (fast) {
            o[0] = (int16_t)(t10 + t11); o[32] = (int16_t)(t10 - t11);
            const int z = ifast_mul(t12 + t13, 181);
            o[16] = (int16_t)(t13 + z); o[48] = (int16_t)(t13 - z);
        } else {
            const int rnd = 1 << (outs - 1);
            o[0] = (int16_t)((t10 + t11 + rnd) >> outs); o[32] = (int16_t)((t10 - t11 + rnd) >> outs);
            const uint32_t z = (uint32_t)(t12 + t13) * 4433u;
            o[16] = descale16(z + (uint32_t)t13 * 6270u, 13 + outs);
            o[48] = descale16(z - (uint32_t)t12 * 15137u, 13 + outs);
        }
    }
}

/* FDCTDSPContext.fdct / .fdct248 (fdctdsp.c:27-45): kind 0 islow 8-bit, 1 ifast, 2 islow 10-bit */
void orc_fdct(int kind, int is248, int16_t *block)
{
    const int p1 = kind == 2 ? 1 : 4, outs = kind == 2 ? 2 : 4;
    for (int i = 0; i < 8; i++) { if (kind == 1) ifast_pass(block + 8 * i, 1); else islow_pass_bits(block + 8 * i, 1, 0, p1, outs); }
    for (int j = 0; j < 8; j++) {
        if (is248) col248(block + j, kind == 1, outs);
        else if (kind == 1) ifast_pass(block + j, 8);
        else islow_pass_bits(block + j, 8, 1, p1, outs);
    }
}

/* the H.264 8x8 forward transform's 1-D step: in[] -> out[] */
static void dct264_1d(const int *in, int *out)
{
    const int s07 = in[0] + in[7], s16 = in[1] + in[6], s25 = in[2] + in[5], s34 = in[3] + in[4];
    const int d07 = in[0] - in[7], d16 = in[1] - in[6], d25 = in[2] - in[5], d34 = in[3] - in[4];
    const int a0 = s07 + s34, a1 = s16 + s25, a2 = s07 - s34, a3 = s16 - s25;
    const int a4 = d16 + d25 + (d07 + (d07 >> 1)), a5 = d07 - d34 - (d25 + (d25 >> 1));
    const int a6 = d07 + d34 - (d16 + (d16 >> 1)), a7 = d16 - d25 + (d34 + (d34 >> 1));
    out[0] = a0 + a1; out[1] = a4 + (a7 >> 2); out[2] = a2 + (a3 >> 1); out[3] = a5 + (a6 >> 2);
    out[4] = a0 - a1; out[5] = a6 - (a5 >> 2); out[6] = (a2 >> 1) - a3; out[7] = (a4 >> 2) - a7;
}

static int dct_cmp8x8(int fn, const uint8_t *s1, const uint8_t *s2, ptrdiff_t stride)
{
    int16_t t[64];
    for (int i = 0; i < 8; i++)
        for (int j = 0; j < 8; j++) t[8 * i + j] = (int16_t)(s1[i * stride + j] - s2[i * stride + j]);
    int sum = 0;
    if (fn == 10) {
        for (int i = 0; i < 8; i++) {
            int in[8], out[8];
            for (int j = 0; j < 8; j++) in[j] = t[8 * i + j];
            dct264_1d(in, out);
            for (int j = 0; j < 8; j++) t[8 * i + j] = (int16_t)out[j];
        }
        for (int j = 0; j < 8; j++) {
            int in[8], out[8];
            for (int i = 0; i < 8; i++) in[i] = t[8 * i + j];
            dct264_1d(in, out);
            for (int i = 0; i < 8; i++) sum += abs(out[i]);
        }
        return sum;
    }
    for (int i = 0; i < 8; i++) { if (g_dct_algo == 1) ifast_pass(t + 8 * i, 1); else islow_pass(t + 8 * i, 1, 0); }
    for (int j = 0; j < 8; j++) { if (g_dct_algo == 1) ifast_pass(t + j, 8); else islow_pass(t + j, 8, 1); }
    for (int i = 0; i < 64; i++) { const int v = abs(t[i]); if (fn == 8) sum += v; else if (v > sum) sum = v; }
    return sum;
}

int orc_sum_abs_dctelem(const int16_t *block)
{
    int sum = 0;
    for (int i = 0; i < 64; i++) sum += abs(block[i]);
    return sum;
}

/* nsse's weight: avctx->nsse_weight of the encoder context, 8 for a NULL context (me_cmp.c:407-410) */
static int g_nsse_weight = 8;
void orc_me_cmp_set_nsse_weight(int weight) { g_nsse_weight = weight; }

int orc_me_cmp(int fn, int idx, const uint8_t *blk1, const uint8_t *blk2, ptrdiff_t stride, int h)
{
    if (fn >= 8 && fn <= 10) {                                     /* dct_sad / dct_max / dct264_sad: [0] 16 wide, [1] 8x8 */
        if (idx != 0 && idx != 1) return -1;
        int s = dct_cmp8x8(fn, blk1, blk2, stride);
        if (idx == 1) return s;
        s += dct_cmp8x8(fn, blk1 + 8, blk2 + 8, stride);
        if (h == 16) s += dct_cmp8x8(fn, blk1 + 8 * stride, blk2 + 8 * stride, stride) + dct_cmp8x8(fn, blk1 + 8 * stride + 8, blk2 + 8 * stride + 8, stride);
        return s;
    }
    if (fn == 3 && (idx == 4 || idx == 5)) {                       /* hadamard8_diff[4] = intra16, [5] = intra8x8 */
        if (idx == 5) return satd8x8_intra(blk1, stride);
        int s = satd8x8_intra(blk1, stride) + satd8x8_intra(blk1 + 8, stride);
        if (h == 16) s += satd8x8_intra(blk1 + 8 * stride, stride) + satd8x8_intra(blk1 + 8 * stride + 8, stride);
        return s;
    }
    if (fn == 4 || fn == 5) {                                      /* vsad / vsse: [0] 16, [1] 8, [4] intra16, [5] intra8 */
        if (idx != 0 && idx != 1 && idx != 4 && idx != 5) return -1;
        return vgrad_wh(blk1, blk2, stride, idx & 1 ? 8 : 16, h, idx >= 4, fn == 5);
    }
    if (fn == 6) return idx == 0 || idx == 1 ? nsse_wh(blk1, blk2, stride, 16 >> idx, h, g_nsse_weight) : -1;
    if (fn == 7) return idx == 0 || idx == 1 ? median_sad_wh(blk1, blk2, stride, 16 >> idx, h) : -1;
    if (fn == 3) {
        if (idx == 1) return satd8x8(blk1, blk2, stride);
        if (idx != 0) return -1;
        int s = satd8x8(blk1, blk2, stride) + satd8x8(blk1 + 8, blk2 + 8, stride);
        if (h == 16) s += satd8x8(blk1 + 8 * stride, blk2 + 8 * stride, stride) + satd8x8(blk1 + 8 * stride + 8, blk2 + 8 * stride + 8, stride);
        return s;
    }
    if (fn == 0) return idx == 0 ? sad_wh(blk1, blk2, stride, 16, h, 0) : idx == 1 ? sad_wh(blk1, blk2, stride, 8, h, 0) : -1;
    if (fn == 1) return idx <= 2 ? sse_wh(blk1, blk2, stride, 16 >> idx, h) : -1;
    if (fn == 2) return idx < 8 ? sad_wh(blk1, blk2, stride, idx < 4 ? 16 : 8, h, idx & 3) : -1;
    return -1;
}

/* out[i] = orc_me_cmp(fn, idx, f1 + off1[i], f2 + off2[i], stride, h): one call for a whole batch */
void orc_me_cmp_batch(int fn, int idx, const uint8_t *f1, const uint8_t *f2, ptrdiff_t stride, int h,
                      const int64_t *off1, const int64_t *off2, int64_t n, int32_t *out)
{
    for (int64_t i = 0; i < n; i++) out[i] = orc_me_cmp(fn, idx, f1 + off1[i], f2 + off2[i], stride, h);
}

void orc_esa_frame(const uint8_t *cur, const uint8_t *ref, int linesize, int width, int height,
                   int mb_size, int search_param, int mb_row0, int mb_row1, int32_t *out_mv, uint64_t *out_cost)
{
    int log2_mb = 0;
    while ((1 << log2_mb) < mb_size) log2_mb++;
    const int b_w = width >> log2_mb, b_h = height >> log2_mb;
    const int gx_max = (b_w - 1) << log2_mb, gy_max = (b_h - 1) << log2_mb;
    if (mb_row1 > b_h) mb_row1 = b_h;
    for (int by = mb_row0; by < mb_row1; by++)
        for (int bx = 0; bx < b_w; bx++) {
            const int x_mb = bx << log2_mb, y_mb = by << log2_mb;
            const uint8_t *c = cur + (ptrdiff_t)y_mb * linesize + x_mb;
            int best_x = x_mb, best_y = y_mb;
            uint64_t best = 0;
            for (int j = 0; j < mb_size; j++)
                for (int i = 0; i < mb_size; i++)
                    best += abs(ref[(ptrdiff_t)(y_mb + j) * linesize + x_mb + i] - c[(ptrdiff_t)j * linesize + i]);
            if (best) {
                const int x0 = x_mb - search_param > 0 ? x_mb - search_param : 0;
                const int y0 = y_mb - search_param > 0 ? y_mb - search_param : 0;
                const int x1 = x_mb + search_param < gx_max ? x_mb + search_param : gx_max;
                const int y1 = y_mb + search_param < gy_max ? y_mb + search_param : gy_max;
                for (int y = y0; y <= y1; y++)
                    for (int x = x0; x <= x1; x++) {
                        uint64_t cost = 0;
                        const uint8_t *r = ref + (ptrdiff_t)y * linesize + x;
                        for (int j = 0; j < mb_size; j++)
                            for (int i = 0; i < mb_size; i++)
                                cost += abs(r[(ptrdiff_t)j * linesize + i] - c[(ptrdiff_t)j * linesize + i]);
                        if (cost < best) { best = cost; best_x = x; best_y = y; }
                    }
            }
            out_mv[2 * (by * b_w + bx)] = best_x;
            out_mv[2 * (by * b_w + bx) + 1] = best_y;
            out_cost[by * b_w + bx] = best;
        }
}

/* av_pixelutils_get_sad_fn(bits, bits, ...) (libavutil/pixelutils.c:43-111): square blocks of 1 << bits pixels, one stride per block */
int orc_pixelutils_sad(int bits, const uint8_t *src1, ptrdiff_t stride1, const uint8_t *src2, ptrdiff_t stride2)
{
    if (bits < 1 || bits > 5) return -1;
    const int size = 1 << bits;
    int sum = 0;
    for (int y = 0; y < size; y++)
        for (int x = 0; x < size; x++) {
            const int d = src1[y * stride1 + x] - src2[y * stride2 + x];
            sum += d < 0 ? -d : d;
        }
    return sum;
}
