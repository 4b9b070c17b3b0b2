/*
 * hevcmc_oracle.c — TEST INFRASTRUCTURE ONLY.  CPU restatement of HEVC motion compensation: the 40 distinct functions per depth behind
 * the put_hevc_{q,e}pel, _uni, _uni_w, _bi, _bi_w tables of HEVCDSPContext (libavcodec/hevc/dsp.h:47-125) as ff_hevc_dsp_init installs
 * them for depth 8, 9, 10 and 12 (hevc/dsp.c:140-196), and the batch semantics of b200_hevc_mc_batch_device (include/b200dsp.h).
 *
 * Follows (behaviour, not text) libavcodec/h26x/h2656_inter_template.c and hevc/dsp_template.c:368-809:
 *   v(x, y)  pixels  S << (14 - depth)
 *            h / v   (8 taps at -3..+4, qpel; 4 taps at -1..+2, epel) >> (depth - 8)
 *            hv      the horizontal sums >> (depth - 8) kept as int16 for rows -B .. height + A - 1, then the vertical sum >> 6
 *   plain    dst16 = (int16) v                                  (the int16 dst at the 64-element MAX_PB_SIZE stride)
 *   uni      clip((v + 2^(13 - depth)) >> (14 - depth))
 *   uni_w    clip(((v wx + 2^(s - 1)) >> s) + ox 2^(depth - 8)),   s = denom + 14 - depth
 *   bi       clip((v + src2 + 2^(14 - depth)) >> (15 - depth))
 *   bi_w     clip((v wx1 + src2 wx0 + (ox 2^(depth - 8) + 1) 2^l) >> (l + 1)),   l = denom + 14 - depth
 * The filter rows are H.265's luma / chroma interpolation coefficients; phase 0 is the reference's all-zero dummy row, which a
 * member whose table position filters in that direction uses when it is called with phase 0.
 * Batch op: the decoder's sequence (hevcdec.c:1722-2040): UNI / UNI_W = the _uni[_w] member on reference 0; BI / BI_W = the plain
 * member into an int16 tmp on reference 0, then the _bi[_w] member on reference 1 with that tmp; the member of table position
 * [!!my][!!mx]; source samples through coordinates clamped to the picture (what emulated_edge_mc's windows give).
 */
#include <string.h>
#include "oracle.h"
#include "../include/b200dsp.h"

static const int8_t QF[4][8] = { { 0 }, { -1, 4, -10, 58, 17, -5, 1, 0 }, { -1, 4, -11, 40, 40, -11, 4, -1 }, { 0, 1, -5, 17, 58, -10, 4, -1 } };
static const int8_t EF[8][4] = { { 0 }, { -2, 58, 10, -2 }, { -4, 54, 16, -2 }, { -6, 46, 28, -4 }, { -4, 36, 36, -4 }, { -4, 28, 46, -6 },
                                 { -2, 16, 54, -4 }, { -2, 10, 58, -2 } };

static int sample(const uint8_t *src, ptrdiff_t stride, int hbd, int x, int y)
{
    const uint8_t *row = src + y * stride;
    return hbd ? ((const uint16_t *)row)[x] : row[x];
}
static int clipd(int v, int depth) { return v < 0 ? 0 : v > (1 << depth) - 1 ? (1 << depth) - 1 : v; }

/* form: 0 plain, 1 uni, 2 uni_w, 3 bi, 4 bi_w; (vdir, hdir) = the table position [!!my][!!mx]; strides in bytes; -1 for arguments
 * outside what the reference's functions take (width / height 1..64, phases inside the filter table) */
int orc_hevc_mc(int depth, int epel, int form, int vdir, int hdir, void *dst, ptrdiff_t dststride, const void *src_, ptrdiff_t srcstride,
                const int16_t *src2, int height, int denom, int wx0, int wx1, int ox, int mx, int my, int width)
{
    const uint8_t *src = src_;
    const int T = epel ? 4 : 8, B = epel ? 1 : 3, hbd = depth > 8, sh8 = depth - 8;
    if (width < 1 || width > 64 || height < 1 || height > 64 || mx < 0 || my < 0 || mx > (epel ? 7 : 3) || my > (epel ? 7 : 3)) return -1;
    const int8_t *hf = epel ? EF[mx] : QF[mx], *vf = epel ? EF[my] : QF[my];
    static int16_t tmp[(64 + 7) * 64];
    if (hdir && vdir) {
        for (int y = -B; y < height + T - 1 - B; y++)
            for (int x = 0; x < width; x++) {
                int s = 0;
                for (int k = 0; k < T; k++) s += hf[k] * sample(src, srcstride, hbd, x - B + k, y);
                tmp[(y + B) * 64 + x] = (int16_t)(s >> sh8);
            }
    }
    for (int y = 0; y < height; y++)
        for (int x = 0; x < width; x++) {
            int v = 0;
            if (hdir && vdir) {
                for (int k = 0; k < T; k++) v += vf[k] * tmp[(y + k) * 64 + x];
                v >>= 6;
            } else if (hdir) {
                for (int k = 0; k < T; k++) v += hf[k] * sample(src, srcstride, hbd, x - B + k, y);
                v >>= sh8;
            } else if (vdir) {
                for (int k = 0; k < T; k++) v += vf[k] * sample(src, srcstride, hbd, x, y - B + k);
                v >>= sh8;
            } else {
                v = sample(src, srcstride, hbd, x, y) << (14 - depth);
            }
            if (form == 0) {
                ((int16_t *)dst)[y * 64 + x] = (int16_t)v;
                continue;
            }
            int out;
            const int s2 = form >= 3 ? src2[y * 64 + x] : 0;
            if (form == 1) out = (v + (1 << (13 - depth))) >> (14 - depth);
            else if (form == 2) {
                const int s = denom + 14 - depth;
                out = ((v * wx0 + (1 << (s - 1))) >> s) + ox * (1 << sh8);
            } else if (form == 3) out = (v + s2 + (1 << (14 - depth))) >> (15 - depth);
            else {
                const int l = denom + 14 - depth;
                out = (v * wx1 + s2 * wx0 + (ox * (1 << sh8) + 1) * (1 << l)) >> (l + 1);
            }
            uint8_t *row = (uint8_t *)dst + y * dststride;
            if (hbd) ((uint16_t *)row)[x] = (uint16_t)clipd(out, depth);
            else row[x] = (uint8_t)clipd(out, depth);
        }
    return 0;
}

/* b200_hevc_mc_batch_device on host memory; returns the number of ops that wrote their block */
int64_t orc_hevc_mc_batch(int depth, int epel, int64_t nops, const B200HevcMcOp *ops, uint8_t *dst, ptrdiff_t dst_stride, const uint8_t *ref,
                          ptrdiff_t ref_stride, int pic_w, int pic_h)
{
    const int T = epel ? 4 : 8, B = epel ? 1 : 3, bps = depth > 8 ? 2 : 1, maxp = epel ? 7 : 3;
    static uint8_t win[2][(64 + 7) * (64 + 7) * 2];
    static int16_t tmp[64 * 64];
    int64_t done = 0;
    for (int64_t i = 0; i < nops; i++) {
        const B200HevcMcOp *op = &ops[i];
        const int bi = op->kind == B200_HEVC_MC_BI || op->kind == B200_HEVC_MC_BI_W, nref = bi ? 2 : 1;
        int ok = op->kind <= 3 && op->w >= 1 && op->w <= 64 && op->h >= 1 && op->h <= 64 && op->denom <= 7;
        for (int r = 0; r < nref; r++) ok = ok && op->mx[r] <= maxp && op->my[r] <= maxp && !(op->ref_off[r] % bps);
        if (!ok || op->dst_off % bps) continue;
        const int wp = (op->w + T - 1) * bps;                              /* window: the block and B / T - 1 - B samples around it */
        for (int r = 0; r < nref; r++)
            for (int y = 0; y < op->h + T - 1; y++)
                for (int x = 0; x < op->w + T - 1; x++) {
                    long long yy = (long long)op->y[r] - B + y, xx = (long long)op->x[r] - B + x;
                    yy = yy < 0 ? 0 : yy >= pic_h ? pic_h - 1 : yy;
                    xx = xx < 0 ? 0 : xx >= pic_w ? pic_w - 1 : xx;
                    memcpy(win[r] + y * wp + x * bps, ref + op->ref_off[r] + yy * ref_stride + xx * bps, bps);
                }
        uint8_t *d = dst + op->dst_off;
        const int kind = op->kind;
        if (!bi) {
            orc_hevc_mc(depth, epel, 1 + kind, !!op->my[0], !!op->mx[0], d, dst_stride, win[0] + B * wp + B * bps, wp, NULL, op->h, op->denom,
                        op->wx0, 0, op->ox, op->mx[0], op->my[0], op->w);
        } else {
            orc_hevc_mc(depth, epel, 0, !!op->my[0], !!op->mx[0], tmp, 0, win[0] + B * wp + B * bps, wp, NULL, op->h, 0, 0, 0, 0, op->mx[0],
                        op->my[0], op->w);
            orc_hevc_mc(depth, epel, kind == B200_HEVC_MC_BI ? 3 : 4, !!op->my[1], !!op->mx[1], d, dst_stride, win[1] + B * wp + B * bps, wp, tmp,
                        op->h, op->denom, op->wx0, op->wx1, op->ox, op->mx[1], op->my[1], op->w);
        }
        done++;
    }
    return done;
}
