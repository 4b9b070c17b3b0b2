/* vc1dsp_oracle.c — TEST INFRASTRUCTURE ONLY: the checker of ffmpeg_b200/csrc/vc1mc.cu and vc1idct.cu, restated from
 * libavcodec/vc1dsp.c (the mspel, chroma and transform members), hpeldsp.c / h264chroma.c (the members the decoder takes for hpel luma
 * and rounded chroma), vc1_mc.c (the progressive sequence of ff_vc1_mc_1mv, ff_vc1_mc_4mv_luma, ff_vc1_mc_4mv_chroma and
 * ff_vc1_interp_mc: edge test, emulated_edge_mc window, range reduction, IC LUT, member call) and vc1_block.c:1124-1240 (the transform
 * dispatch of vc1_decode_p_block).  Each function follows the reference's own order of operations, block by block, on host memory. */
#include <string.h>
#include "vc1dsp_oracle.h"

static uint8_t clip8(int v) { return v < 0 ? 0 : v > 255 ? 255 : (uint8_t)v; }
static int clampi(int v, int lo, int hi) { return v < lo ? lo : v > hi ? hi : v; }

/* ---------------------------------------------------------------- mspel (vc1dsp.c:541-778) */
static const int TAPS[4][4] = { { 0, 0, 0, 0 }, { -4, 53, 18, -3 }, { -1, 9, 9, -1 }, { -3, 18, 53, -4 } };
static const int SHIFT[4] = { 0, 5, 1, 5 };

static int taps8(const uint8_t *s, ptrdiff_t step, int mode)
{
    return TAPS[mode][0] * s[-step] + TAPS[mode][1] * s[0] + TAPS[mode][2] * s[step] + TAPS[mode][3] * s[2 * step];
}

static void store(uint8_t *d, int v, int avg) { *d = avg ? (uint8_t)((*d + clip8(v) + 1) >> 1) : clip8(v); }

static void mspel_block(int avg, int n, uint8_t *dst, ptrdiff_t dstride, const uint8_t *src, ptrdiff_t sstride, int hm, int vm, int rnd)
{
    if (hm && vm) {
        const int shift = (SHIFT[hm] + SHIFT[vm]) >> 1, r = (1 << (shift - 1)) + rnd - 1;
        int16_t tmp[16][19];                                   /* column i of tmp is source column i - 1 */
        for (int j = 0; j < n; j++)
            for (int i = 0; i < n + 3; i++) tmp[j][i] = (int16_t)((taps8(src + j * sstride + i - 1, sstride, vm) + r) >> shift);
        for (int j = 0; j < n; j++)
            for (int i = 0; i < n; i++) {
                const int16_t *t = &tmp[j][i];
                store(dst + j * dstride + i, (TAPS[hm][0] * t[0] + TAPS[hm][1] * t[1] + TAPS[hm][2] * t[2] + TAPS[hm][3] * t[3] + 64 - rnd) >> 7, avg);
            }
        return;
    }
    for (int j = 0; j < n; j++)
        for (int i = 0; i < n; i++) {
            const uint8_t *s = src + j * sstride + i;
            int v;
            if (vm) v = (taps8(s, sstride, vm) + (vm == 2 ? 8 : 32) - (1 - rnd)) >> (vm == 2 ? 4 : 6);
            else if (hm) v = (taps8(s, 1, hm) + (hm == 2 ? 8 : 32) - rnd) >> (hm == 2 ? 4 : 6);
            else v = s[0];                                      /* [size][0]: put_ / avg_pixels{16x16,8x8}_c */
            store(dst + j * dstride + i, v, avg);
        }
}

int orc_vc1_mspel(int avg, int size, int dxy, uint8_t *dst, const uint8_t *src, ptrdiff_t stride, int rnd)
{
    if (size < 0 || size > 1 || dxy < 0 || dxy > 15) return -1;
    mspel_block(avg, size ? 8 : 16, dst, stride, src, stride, dxy & 3, dxy >> 2, rnd);
    return 0;
}

/* ---------------------------------------------------------------- hpel (hpeldsp.c) and chroma (h264chroma_template.c, vc1dsp.c:780-877) */
static void hpel_block(int avg, int n, uint8_t *dst, ptrdiff_t dstride, const uint8_t *src, ptrdiff_t sstride, int dxy, int no_rnd)
{
    for (int j = 0; j < n; j++)
        for (int i = 0; i < n; i++) {
            const uint8_t *s = src + j * sstride + i;
            int v = s[0];
            if (dxy == 1) v = (s[0] + s[1] + 1 - no_rnd) >> 1;
            else if (dxy == 2) v = (s[0] + s[sstride] + 1 - no_rnd) >> 1;
            else if (dxy == 3) v = (s[0] + s[1] + s[sstride] + s[sstride + 1] + 2 - no_rnd) >> 2;
            store(dst + j * dstride + i, v, avg);
        }
}

static void chroma_block(int avg, int w, int h, uint8_t *dst, ptrdiff_t dstride, const uint8_t *src, ptrdiff_t sstride, int x, int y, int bias)
{
    const int A = (8 - x) * (8 - y), B = x * (8 - y), C = (8 - x) * y, D = x * y;
    for (int j = 0; j < h; j++)
        for (int i = 0; i < w; i++) {
            const uint8_t *s = src + j * sstride + i;
            store(dst + j * dstride + i, (A * s[0] + B * s[1] + C * s[sstride] + D * s[sstride + 1] + bias) >> 6, avg);
        }
}

int orc_vc1_chroma(int avg, int idx, uint8_t *dst, const uint8_t *src, ptrdiff_t stride, int h, int x, int y)
{
    if (idx < 0 || idx > 1 || x < 0 || x > 7 || y < 0 || y > 7 || h < 0) return -1;
    chroma_block(avg, idx ? 4 : 8, h, dst, stride, src, stride, x, y, 28);
    return 0;
}

/* ---------------------------------------------------------------- transforms (vc1dsp.c:240-537) */
/* 8-point: out[k] for k = 0..7 of in[0..7] with bias b, shift sh, + r on the last four outputs */
static void tx8(const int *in, int b, int sh, int r, int *out)
{
    const int e0 = 12 * (in[0] + in[4]) + b, e1 = 12 * (in[0] - in[4]) + b, e2 = 16 * in[2] + 6 * in[6], e3 = 6 * in[2] - 16 * in[6];
    const int ev[4] = { e0 + e2, e1 + e3, e1 - e3, e0 - e2 };
    const int od[4] = { 16 * in[1] + 15 * in[3] + 9 * in[5] + 4 * in[7], 15 * in[1] - 4 * in[3] - 16 * in[5] - 9 * in[7],
                        9 * in[1] - 16 * in[3] + 4 * in[5] + 15 * in[7], 4 * in[1] - 9 * in[3] + 15 * in[5] - 16 * in[7] };
    for (int k = 0; k < 4; k++) {
        out[k] = (ev[k] + od[k]) >> sh;
        out[7 - k] = (ev[k] - od[k] + r) >> sh;
    }
}

static void tx4(const int *in, int b, int sh, int *out)
{
    const int e0 = 17 * (in[0] + in[2]) + b, e1 = 17 * (in[0] - in[2]) + b, o0 = 22 * in[1] + 10 * in[3], o1 = 22 * in[3] - 10 * in[1];
    out[0] = (e0 + o0) >> sh;
    out[1] = (e1 - o1) >> sh;
    out[2] = (e1 + o1) >> sh;
    out[3] = (e0 - o0) >> sh;
}

int orc_vc1_itx(int tt, int dc, uint8_t *dest, ptrdiff_t stride, int16_t *block)
{
    if (tt < 0 || tt > 3) return -1;
    const int w = tt == B200_VC1_TT_8X8 || tt == B200_VC1_TT_8X4 ? 8 : 4, h = tt == B200_VC1_TT_8X8 || tt == B200_VC1_TT_4X8 ? 8 : 4;
    if (dc) {
        int d = block[0];
        if (w == 8) d = (3 * d + 1) >> 1;
        else d = (17 * d + 4) >> 3;
        if (h == 8) d = w == 8 ? (3 * d + 16) >> 5 : (12 * d + 64) >> 7;
        else d = (17 * d + 64) >> 7;
        for (int j = 0; j < h; j++)
            for (int i = 0; i < w; i++) dest[j * stride + i] = clip8(dest[j * stride + i] + d);
        return 0;
    }
    int in[8], out[8];
    if (tt == B200_VC1_TT_8X8) {                                 /* columns into temp[col][k], then temp's columns into block rows */
        int16_t temp[8][8];
        for (int c = 0; c < 8; c++) {
            for (int k = 0; k < 8; k++) in[k] = block[8 * k + c];
            tx8(in, 4, 3, 0, out);
            for (int k = 0; k < 8; k++) temp[c][k] = (int16_t)out[k];
        }
        for (int i = 0; i < 8; i++) {
            for (int k = 0; k < 8; k++) in[k] = temp[k][i];
            tx8(in, 64, 7, 1, out);
            for (int k = 0; k < 8; k++) block[8 * k + i] = (int16_t)out[k];
        }
        return 0;
    }
    for (int j = 0; j < h; j++) {                                /* rows, written back into block */
        for (int k = 0; k < w; k++) in[k] = block[8 * j + k];
        if (w == 8) tx8(in, 4, 3, 0, out);
        else tx4(in, 4, 3, out);
        for (int k = 0; k < w; k++) block[8 * j + k] = (int16_t)out[k];
    }
    for (int i = 0; i < w; i++) {                                /* columns, added to dest */
        for (int k = 0; k < h; k++) in[k] = block[8 * k + i];
        if (h == 8) tx8(in, 64, 7, 1, out);
        else tx4(in, 64, 7, out);
        for (int k = 0; k < h; k++) dest[k * stride + i] = clip8(dest[k * stride + i] + out[k]);
    }
    return 0;
}

/* ---------------------------------------------------------------- the decoder's progressive MC sequence */
enum { EMU_PITCH = 32 };

/* the window of k x k samples from (x0, y0) of a w x h plane, edge-replicated, then range reduction and the LUT pair (vc1_mc.c:35-104) */
static void window(uint8_t *buf, const uint8_t *plane, ptrdiff_t ls, int k, int x0, int y0, int w, int h, int rr, const uint8_t (*lut)[256])
{
    for (int r = 0; r < k; r++)
        for (int c = 0; c < k; c++) buf[r * EMU_PITCH + c] = plane[clampi(y0 + r, 0, h - 1) * ls + clampi(x0 + c, 0, w - 1)];
    if (rr)
        for (int r = 0; r < k; r++)
            for (int c = 0; c < k; c++) buf[r * EMU_PITCH + c] = (uint8_t)(((buf[r * EMU_PITCH + c] - 128) >> 1) + 128);
    if (lut) {
        const uint8_t *lut1 = lut[(0 + y0) & 1], *lut2 = lut[(1 + y0) & 1];
        for (int r = 0; r < k; r++)
            for (int c = 0; c < k; c++) buf[r * EMU_PITCH + c] = (r & 1 ? lut2 : lut1)[buf[r * EMU_PITCH + c]];
    }
}

static int op_valid(const B200Vc1McOp *op, int nrefs, int mbw, int mbh)
{
    const int nsrc = op->flags & B200_VC1_MC_AVG ? 2 : 1;
    if (op->kind > B200_VC1_MC_CHROMA8 || (nsrc == 2 && op->kind != B200_VC1_MC_1MV)) return 0;
    for (int s = 0; s < nsrc; s++) {
        const B200Vc1McSrc *S = &op->src[s];
        if (S->ref >= nrefs || S->mx > 3 || S->my > 3 || S->uvmx > 3 || S->uvmy > 3) return 0;
    }
    const int n = op->kind == B200_VC1_MC_1MV ? 16 : 8, sc = op->kind == B200_VC1_MC_CHROMA8 ? 8 : 16;
    return op->dst_x >= 0 && op->dst_y >= 0 && op->dst_x % 8 == 0 && op->dst_y % 8 == 0 && op->dst_x + n <= sc * mbw && op->dst_y + n <= sc * mbh;
}

int64_t orc_vc1_mc_frame(int nrefs, const B200Vc1McRef *refs, uint8_t *const dst[3], ptrdiff_t ls_y, ptrdiff_t ls_uv, int mb_width,
                         int mb_height, int H, int V, int64_t nops, const B200Vc1McOp *ops)
{
    if (nops < 0 || nrefs < 1 || nrefs > 2 || mb_width < 1 || mb_height < 1 || mb_width > 2047 || mb_height > 2047 || H < 1 || V < 1 ||
        H > 32767 || V > 32767)
        return -1;
    for (int r = 0; r < nrefs; r++)
        if (refs[r].interlaced) return -1;
    int64_t wrote = 0;
    uint8_t ybuf[19 * EMU_PITCH], ubuf[9 * EMU_PITCH], vbuf[9 * EMU_PITCH];
    for (int64_t i = 0; i < nops; i++) {
        const B200Vc1McOp *op = &ops[i];
        if (!op_valid(op, nrefs, mb_width, mb_height)) continue;
        const int ms = !!(op->flags & B200_VC1_MC_MSPEL), rnd = !!(op->flags & B200_VC1_MC_RND);
        const int nsrc = op->flags & B200_VC1_MC_AVG ? 2 : 1;
        for (int s = 0; s < nsrc; s++) {
            const B200Vc1McSrc *S = &op->src[s];
            const B200Vc1McRef *R = &refs[S->ref];
            const int avg = s == 1;
            int emu;
            if (op->kind == B200_VC1_MC_1MV && s == 0)               /* ff_vc1_mc_1mv */
                emu = R->rangeredfrm || R->use_ic || H < 22 || V < 22 || (unsigned)(S->x - ms) > (unsigned)(H - S->mx - 16 - ms * 3) ||
                      (unsigned)(S->y - 1) > (unsigned)(V - S->my - 16 - 3);
            else if (op->kind == B200_VC1_MC_1MV)                    /* ff_vc1_interp_mc */
                emu = R->rangeredfrm || H < 22 || V < 22 || R->use_ic || (unsigned)(S->x - 1) > (unsigned)(H - S->mx - 16 - 3) ||
                      (unsigned)(S->y - 1) > (unsigned)(V - S->my - 16 - 3);
            else if (op->kind == B200_VC1_MC_LUMA8)                  /* ff_vc1_mc_4mv_luma */
                emu = R->rangeredfrm || R->use_ic || H < 13 || V < 23 || (unsigned)(S->x - ms) > (unsigned)(H - S->mx - 8 - ms * 2) ||
                      (unsigned)(S->y - ms) > (unsigned)(V - S->my - (8 + ms * 2));
            else                                                     /* ff_vc1_mc_4mv_chroma */
                emu = R->rangeredfrm || R->use_ic || H < 18 || V < 18 || (unsigned)S->uvx > (unsigned)((H >> 1) - 9) ||
                      (unsigned)S->uvy > (unsigned)((V >> 1) - 9);
            if (op->kind != B200_VC1_MC_CHROMA8) {
                const int n = op->kind == B200_VC1_MC_1MV ? 16 : 8;
                const uint8_t *src = R->y + S->y * R->ls_y + S->x;
                ptrdiff_t sls = R->ls_y;
                if (emu) {
                    window(ybuf, R->y, R->ls_y, n + 1 + 2 * ms, S->x - ms, S->y - ms, H, V, R->rangeredfrm, R->use_ic ? R->luty : NULL);
                    src = ybuf + ms * (1 + EMU_PITCH);
                    sls = EMU_PITCH;
                }
                uint8_t *d = dst[0] + op->dst_y * ls_y + op->dst_x;
                if (ms) mspel_block(avg, n, d, ls_y, src, sls, S->mx, S->my, rnd);
                else hpel_block(avg, n, d, ls_y, src, sls, (S->my & 2) | ((S->mx & 2) >> 1), rnd);
            }
            if (op->kind != B200_VC1_MC_LUMA8) {
                const uint8_t *su = R->u + S->uvy * R->ls_uv + S->uvx, *sv = R->v + S->uvy * R->ls_uv + S->uvx;
                ptrdiff_t sls = R->ls_uv;
                if (emu) {
                    window(ubuf, R->u, R->ls_uv, 9, S->uvx, S->uvy, H >> 1, V >> 1, R->rangeredfrm, R->use_ic ? R->lutuv : NULL);
                    window(vbuf, R->v, R->ls_uv, 9, S->uvx, S->uvy, H >> 1, V >> 1, R->rangeredfrm, R->use_ic ? R->lutuv : NULL);
                    su = ubuf;
                    sv = vbuf;
                    sls = EMU_PITCH;
                }
                const int cx = op->kind == B200_VC1_MC_CHROMA8 ? op->dst_x : op->dst_x / 2, cy = op->kind == B200_VC1_MC_CHROMA8 ? op->dst_y : op->dst_y / 2;
                const int bias = rnd ? 28 : 32;                         /* put_no_rnd_vc1_chroma / put_h264_chroma */
                chroma_block(avg, 8, 8, dst[1] + cy * ls_uv + cx, ls_uv, su, sls, S->uvmx << 1, S->uvmy << 1, bias);
                chroma_block(avg, 8, 8, dst[2] + cy * ls_uv + cx, ls_uv, sv, sls, S->uvmx << 1, S->uvmy << 1, bias);
            }
        }
        wrote++;
    }
    return wrote;
}

/* ---------------------------------------------------------------- vc1_decode_p_block's transform calls */
int64_t orc_vc1_residual_frame(uint8_t *const dst[3], ptrdiff_t ls_y, ptrdiff_t ls_uv, int mb_width, int mb_height, const int16_t *coef,
                               int64_t nops, const B200Vc1ResidualOp *ops)
{
    if (nops < 0 || mb_width < 1 || mb_height < 1 || mb_width > 2047 || mb_height > 2047) return -1;
    int64_t wrote = 0;
    for (int64_t i = 0; i < nops; i++) {
        const B200Vc1ResidualOp *op = &ops[i];
        const int sc = op->plane ? 8 : 16;
        if (op->plane > 2 || op->ttblk > 3 || op->coef_off < 0 || op->coef_off % 8 || op->x < 0 || op->y < 0 || op->x % 8 || op->y % 8 ||
            op->x + 8 > sc * mb_width || op->y + 8 > sc * mb_height)
            continue;
        int16_t block[64];
        memcpy(block, coef + op->coef_off, sizeof(block));
        const ptrdiff_t ls = op->plane ? ls_uv : ls_y;
        uint8_t *d = dst[op->plane] + op->y * ls + op->x;
        const int pat = op->subblkpat;
        switch (op->ttblk) {
        case B200_VC1_TT_8X8:
            if (op->dc & 1) {
                orc_vc1_itx(B200_VC1_TT_8X8, 1, d, ls, block);
            } else {
                orc_vc1_itx(B200_VC1_TT_8X8, 0, NULL, 0, block);
                for (int j = 0; j < 8; j++)                            /* add_pixels_clamped */
                    for (int k = 0; k < 8; k++) d[j * ls + k] = clip8(d[j * ls + k] + block[8 * j + k]);
            }
            break;
        case B200_VC1_TT_4X4:
            for (int j = 0; j < 4; j++)
                if (!(pat & (1 << (3 - j))))
                    orc_vc1_itx(B200_VC1_TT_4X4, (op->dc >> j) & 1, d + (j & 1) * 4 + (j & 2) * 2 * ls, ls, block + (j & 1) * 4 + (j & 2) * 16);
            break;
        case B200_VC1_TT_8X4:
            for (int j = 0; j < 2; j++)
                if (!(pat & (1 << (1 - j)))) orc_vc1_itx(B200_VC1_TT_8X4, (op->dc >> j) & 1, d + j * 4 * ls, ls, block + j * 32);
            break;
        case B200_VC1_TT_4X8:
            for (int j = 0; j < 2; j++)
                if (!(pat & (1 << (1 - j)))) orc_vc1_itx(B200_VC1_TT_4X8, (op->dc >> j) & 1, d + j * 4, ls, block + j * 4);
            break;
        }
        wrote++;
    }
    return wrote;
}
