/* hevcpred_oracle.c — TEST INFRASTRUCTURE ONLY: a plain-C restatement of HEVC intra prediction (libavcodec/hevc/pred_template.c),
 * the checker for ffmpeg_b200/csrc/hevcpred.cu.  Written from the reference's behaviour, sequentially and with int edge arrays:
 *   orc_hevc_pred_planar / _dc / _angular   the three prediction members (stride in samples, as intra_pred passes it);
 *   orc_hevc_filter_3tap / _strong          the two reference-sample filters, with the reference's writes;
 *   orc_hevc_intra_plane                    one call of b200_hevc_intra_pred_batch_device: each B200HevcIntraOp in turn runs
 *                                           intra_pred's flow on the plane (neighbour fetch, constrained-intra PU checks and
 *                                           substitution, the availability if-chain, the filter decision and filter, prediction).
 * Unlike the kernel, the substitution of unavailable samples follows the reference's if-chain step by step, so the kernel's closed
 * form is checked against an independent statement of it.  Checked bit for bit against the compiled reference by
 * tests/test_hevc_pred.py. */
#include <stdint.h>
#include <stddef.h>
#include <string.h>

#include "../include/b200dsp.h"

#define API __attribute__((visibility("default")))

static int rd(const uint8_t *p, int depth, ptrdiff_t i) { return depth == 8 ? p[i] : ((const uint16_t *)p)[i]; }
static void wr(uint8_t *p, int depth, ptrdiff_t i, int v)
{
    if (depth == 8) p[i] = (uint8_t)v;
    else ((uint16_t *)p)[i] = (uint16_t)v;
}
static int clipv(int v, int maxv) { return v < 0 ? 0 : v > maxv ? maxv : v; }
static int iabs(int v) { return v < 0 ? -v : v; }

static const int angle_tab[33] = { 32, 26, 21, 17, 13, 9, 5, 2, 0, -2, -5, -9, -13, -17, -21, -26, -32,
                                   -26, -21, -17, -13, -9, -5, -2, 0, 2, 5, 9, 13, 17, 21, 26, 32 };
static const int inv_angle_tab[15] = { -4096, -1638, -910, -630, -482, -390, -315, -256, -315, -390, -482, -630, -910, -1638, -4096 };

/* the three predictions on int edge arrays (index -1 = corner), into an int block of size x size */
static void predict(int *blk, const int *top, const int *left, int log2, int mode, int luma, int depth)
{
    const int n = 1 << log2, maxv = (1 << depth) - 1;
    if (mode == 0) {                                             /* planar: both linear interpolations, averaged */
        for (int y = 0; y < n; y++)
            for (int x = 0; x < n; x++)
                blk[y * n + x] = ((n - 1 - x) * left[y] + (x + 1) * top[n] + (n - 1 - y) * top[x] + (y + 1) * left[n] + n) >> (log2 + 1);
        return;
    }
    if (mode == 1) {                                             /* DC, with the luma edge smoothing below 32x32 */
        int sum = n;
        for (int i = 0; i < n; i++) sum += top[i] + left[i];
        const int dc = sum >> (log2 + 1);
        for (int i = 0; i < n * n; i++) blk[i] = dc;
        if (luma && n < 32) {
            blk[0] = (left[0] + 2 * dc + top[0] + 2) >> 2;
            for (int x = 1; x < n; x++) blk[x] = (top[x] + 3 * dc + 2) >> 2;
            for (int y = 1; y < n; y++) blk[y * n] = (left[y] + 3 * dc + 2) >> 2;
        }
        return;
    }
    /* angular: project along the main array (top for the vertical modes 18..34, left for 2..17); for negative angles whose
     * projection leaves the main array, extend it backwards with samples of the side array at the inverse angle */
    const int vertical = mode >= 18, angle = angle_tab[mode - 2];
    const int *mainp = vertical ? top : left, *side = vertical ? left : top;
    int ext[3 * 32 + 8];
    int *e = ext + n;                                            /* e[k] = reference sample k - 1 of the main direction */
    for (int k = 0; k <= 2 * n; k++) e[k] = mainp[k - 1];
    const int last = (n * angle) >> 5;
    if (angle < 0 && last < -1)
        for (int k = last; k <= -1; k++) e[k] = side[-1 + ((k * inv_angle_tab[mode - 11] + 128) >> 8)];
    for (int j = 0; j < n; j++) {                                /* j across the main direction (row for vertical modes) */
        const int pos = (j + 1) * angle, idx = pos >> 5, fact = pos & 31;
        for (int i = 0; i < n; i++) {
            const int a = e[i + idx + 1], b = e[i + idx + 2];
            const int v = fact ? ((32 - fact) * a + fact * b + 16) >> 5 : a;
            if (vertical) blk[j * n + i] = v;
            else blk[i * n + j] = v;
        }
    }
    if (luma && n < 32) {                                        /* the pure vertical / horizontal modes' edge correction */
        if (mode == 26)
            for (int y = 0; y < n; y++) blk[y * n] = clipv(top[0] + ((left[y] - left[-1]) >> 1), maxv);
        if (mode == 10)
            for (int x = 0; x < n; x++) blk[x] = clipv(left[0] + ((top[x] - top[-1]) >> 1), maxv);
    }
}

static void load_edges(int *t, int *l, const uint8_t *top, const uint8_t *left, int depth, int from, int to)
{
    for (int i = from; i < to; i++) { t[i] = rd(top, depth, i); l[i] = rd(left, depth, i); }
}

static void store_block(uint8_t *dst, ptrdiff_t stride, const int *blk, int n, int depth)
{
    for (int y = 0; y < n; y++)
        for (int x = 0; x < n; x++) wr(dst, depth, y * stride + x, blk[y * n + x]);
}

API void orc_hevc_pred_planar(int depth, int log2, uint8_t *dst, const uint8_t *top, const uint8_t *left, ptrdiff_t stride)
{
    int ta[130] = { 0 }, la[130] = { 0 }, blk[32 * 32];
    load_edges(ta + 1, la + 1, top, left, depth, 0, (1 << log2) + 1);
    predict(blk, ta + 1, la + 1, log2, 0, 0, depth);
    store_block(dst, stride, blk, 1 << log2, depth);
}

API void orc_hevc_pred_dc(int depth, uint8_t *dst, const uint8_t *top, const uint8_t *left, ptrdiff_t stride, int log2, int c_idx)
{
    int ta[130] = { 0 }, la[130] = { 0 }, blk[32 * 32];
    if (log2 < 2 || log2 > 5) return;
    load_edges(ta + 1, la + 1, top, left, depth, 0, 1 << log2);
    predict(blk, ta + 1, la + 1, log2, 1, c_idx == 0, depth);
    store_block(dst, stride, blk, 1 << log2, depth);
}

API void orc_hevc_pred_angular(int depth, int log2, uint8_t *dst, const uint8_t *top, const uint8_t *left, ptrdiff_t stride, int c_idx,
                               int mode)
{
    int ta[130] = { 0 }, la[130] = { 0 }, blk[32 * 32];
    if (mode < 2 || mode > 34) return;
    load_edges(ta + 1, la + 1, top, left, depth, -1, 2 << log2);
    predict(blk, ta + 1, la + 1, log2, mode, c_idx == 0, depth);
    store_block(dst, stride, blk, 1 << log2, depth);
}

/* [1 2 1] / 4 along each array, the last sample kept, the corner from left[0], the corner and top[0] */
static void filt3(int *fl, int *ft, const int *l, const int *t, int n)
{
    fl[n - 1] = l[n - 1];
    ft[n - 1] = t[n - 1];
    for (int i = 0; i < n - 1; i++) {
        fl[i] = (l[i - 1] + 2 * l[i] + l[i + 1] + 2) >> 2;
        ft[i] = (t[i - 1] + 2 * t[i] + t[i + 1] + 2) >> 2;
    }
    fl[-1] = ft[-1] = (l[0] + 2 * l[-1] + t[0] + 2) >> 2;
}

/* bilinear between the corner and sample 63 of each array; the top into ft, the left in place */
static void filt_strong(int *ft, int *l, const int *t)
{
    ft[-1] = t[-1];
    ft[63] = t[63];
    const int l0 = l[-1], l63 = l[63];
    for (int i = 0; i < 63; i++) {
        ft[i] = ((63 - i) * t[-1] + (i + 1) * t[63] + 32) >> 6;
        l[i] = ((63 - i) * l0 + (i + 1) * l63 + 32) >> 6;
    }
}

API void orc_hevc_filter_3tap(int depth, uint8_t *fl, uint8_t *ft, const uint8_t *left, const uint8_t *top, int size)
{
    int ta[130] = { 0 }, la[130] = { 0 }, fla[130], fta[130];
    const int n = 2 * size;
    load_edges(ta + 1, la + 1, top, left, depth, -1, n);
    filt3(fla + 1, fta + 1, la + 1, ta + 1, n);
    for (int i = -1; i < n; i++) { wr(fl, depth, i, fla[1 + i]); wr(ft, depth, i, fta[1 + i]); }
}

API void orc_hevc_filter_strong(int depth, uint8_t *ft, uint8_t *left, const uint8_t *top)
{
    int ta[130] = { 0 }, la[130] = { 0 }, fta[130];
    load_edges(ta + 1, la + 1, top, left, depth, -1, 64);
    filt_strong(fta + 1, la + 1, ta + 1);
    for (int i = -1; i < 64; i++) wr(ft, depth, i, fta[1 + i]);
    for (int i = 0; i < 63; i++) wr(left, depth, i, la[1 + i]);
}

/* ---- one batch call */
typedef struct Pic {
    uint8_t *pix;
    ptrdiff_t stride;                                            /* samples */
    int depth, W, H, hs, vs, pw, ph;
    const uint8_t *map;
    ptrdiff_t mstride;
    int log2_pu, mpw, mph;
} Pic;

/* intra / inter of the luma min PU (px, py); outside the map: not intra */
static int pu_intra(const Pic *p, int px, int py)
{
    return px >= 0 && py >= 0 && px < p->mpw && py < p->mph && p->map[py * p->mstride + px] != 0;
}
/* intra_pred's IS_INTRA(x, y): x, y in component samples relative to the block at luma (x0, y0) */
static int nb_intra(const Pic *p, int x0, int y0, int x, int y)
{
    return pu_intra(p, (x0 + x * (1 << p->hs)) >> p->log2_pu, (y0 + y * (1 << p->vs)) >> p->log2_pu);
}

static void fill(int *a, int v, int len)                         /* the reference's 4-sample EXTEND */
{
    for (int i = 0; i < len; i += 4) a[i] = a[i + 1] = a[i + 2] = a[i + 3] = v;
}

static void one_op(const Pic *p, const B200HevcIntraOp *op)
{
    const int log2 = op->log2_size, mode = op->mode, f = op->flags;
    if (log2 < 2 || log2 > 5 || mode > 34) return;
    const int n = 1 << log2, x = op->x, y = op->y;
    int bl = !!(f & B200_HEVC_INTRA_CAND_BL), l = !!(f & B200_HEVC_INTRA_CAND_L), ul = !!(f & B200_HEVC_INTRA_CAND_UL);
    int u = !!(f & B200_HEVC_INTRA_CAND_U), ur = !!(f & B200_HEVC_INTRA_CAND_UR);
    if (x < 0 || y < 0 || x + n > p->pw || y + n > p->ph || (x < 1 && (bl || l || ul)) || (y < 1 && (ul || u || ur))) return;
    const int luma = !!(f & B200_HEVC_INTRA_LUMA), depth = p->depth;
    const int x0 = x << p->hs, y0 = y << p->vs, nh = n << p->hs, nv = n << p->vs;
    const int bls = ((y0 + 2 * nv < p->H ? y0 + 2 * nv : p->H) - (y0 + nv)) >> p->vs;
    const int trs = ((x0 + 2 * nh < p->W ? x0 + 2 * nh : p->W) - (x0 + nh)) >> p->hs;
    const ptrdiff_t base = (ptrdiff_t)y * p->stride + x;
#define PIX(xx, yy) rd(p->pix, depth, base + (ptrdiff_t)(yy) * p->stride + (xx))
    int la[8 + 2 * 64 + 16], ta[8 + 2 * 64 + 16], fla[2 * 64 + 1], fta[2 * 64 + 1];
    int *left = la + 4, *top = ta + 4;                           /* index -1 .. 2 * 64 + 10 */
    memset(la, 0, sizeof(la));
    memset(ta, 0, sizeof(ta));

    if (p->map) {                                                /* constrained intra: drop candidates whose PUs are all inter */
        const int lp = p->log2_pu;
        int pv = nv >> lp, ph = nh >> lp;
        const int edge_x = (x0 & ((1 << lp) - 1)) == 0, edge_y = (y0 & ((1 << lp) - 1)) == 0;
        if (ph == 0) ph = 1;
        if (bl && edge_x) {
            const int py = (y0 + nv) >> lp, cnt = pv < p->mph - py ? pv : p->mph - py;
            bl = 0;
            for (int i = 0; i < cnt; i += 2) bl |= pu_intra(p, (x0 - 1) >> lp, py + i);
        }
        if (l && edge_x) {
            const int py = y0 >> lp, cnt = pv < p->mph - py ? pv : p->mph - py;
            l = 0;
            for (int i = 0; i < cnt; i += 2) l |= pu_intra(p, (x0 - 1) >> lp, py + i);
        }
        if (ul) ul = pu_intra(p, (x0 - 1) >> lp, (y0 - 1) >> lp);
        if (u && edge_y) {
            const int px = x0 >> lp, cnt = ph < p->mpw - px ? ph : p->mpw - px;
            u = 0;
            for (int i = 0; i < cnt; i += 2) u |= pu_intra(p, px + i, (y0 - 1) >> lp);
        }
        if (ur && edge_y) {
            const int px = (x0 + nh) >> lp, cnt = ph < p->mpw - px ? ph : p->mpw - px;
            ur = 0;
            for (int i = 0; i < cnt; i += 2) ur |= pu_intra(p, px + i, (y0 - 1) >> lp);
        }
        const int byte128 = depth == 8 ? 128 : 0x8080;           /* memset(.., 128, ..) on the sample arrays */
        for (int i = 0; i < 128; i++) left[i] = top[i] = byte128;
        top[-1] = 128;
    }
    /* the available neighbours, the bottom-left / top-right runs clipped to the picture and extended with their last sample */
    if (ul) left[-1] = top[-1] = PIX(-1, -1);
    if (u) for (int i = 0; i < n; i++) top[i] = PIX(i, -1);
    if (ur) for (int i = 0; i < n; i++) top[n + i] = i < trs ? PIX(n + i, -1) : PIX(n + trs - 1, -1);
    if (l) for (int i = 0; i < n; i++) left[i] = PIX(-1, i);
    if (bl) for (int i = 0; i < n; i++) left[n + i] = i < bls ? PIX(-1, n + i) : PIX(-1, n + bls - 1);

    if (p->map && (bl || l || ul || u || ur)) {                  /* constrained intra substitution (pred_template.c:234-295) */
        int mx = x0 + ((2 * n) << p->hs) < p->W ? 2 * n : (p->W - x0) >> p->hs;
        int my = y0 + ((2 * n) << p->vs) < p->H ? 2 * n : (p->H - y0) >> p->vs;
        if (!ur) mx = x0 + (n << p->hs) < p->W ? n : (p->W - x0) >> p->hs;
        if (!bl) my = y0 + (n << p->vs) < p->H ? n : (p->H - y0) >> p->vs;
        int j;
        if (bl || l || ul) {
            j = n + (bl ? bls : 0) - 1;
            while (j > -1 && !nb_intra(p, x0, y0, -1, j)) j--;
            if (!nb_intra(p, x0, y0, -1, j)) {                   /* no intra sample on the left: take the first intra one on top */
                j = 0;
                while (j < mx && !nb_intra(p, x0, y0, j, -1)) j++;
                for (int i = j; i >= 0; i--)
                    if (!nb_intra(p, x0, y0, i - 1, -1)) top[i - 1] = top[i];
                left[-1] = top[-1];
            }
        } else {
            j = 0;
            while (j < mx && !nb_intra(p, x0, y0, j, -1)) j++;
            if (j > 0) {
                for (int i = j; i > 0; i--)
                    if (!nb_intra(p, x0, y0, i - 1, -1)) top[i - 1] = top[i];
                top[-1] = top[0];
            }
        }
        left[-1] = top[-1];
        if (bl || l) {
            int carry = left[-1];
            for (int i = 0; i < my; i += 4) {
                if (nb_intra(p, x0, y0, -1, i)) carry = left[i + 3];
                else fill(left + i, carry, 4);
            }
        }
        if (!l) fill(left, left[-1], n);
        if (!bl) fill(left + n, left[n - 1], n);
        if (x0 == 0) {
            fill(left, 0, my);
        } else {
            int carry = left[my - 1];
            for (int i = my - 1; i >= 0; i -= 4) {
                if (nb_intra(p, x0, y0, -1, i - 3)) carry = left[i - 3];
                else fill(left + i - 3, carry, 4);
            }
            if (y0 != 0 && !nb_intra(p, x0, y0, -1, -1)) left[-1] = left[0];
        }
        top[-1] = left[-1];
        if (y0 != 0) {
            int carry = left[-1];
            for (int i = 0; i < mx; i += 4) {
                if (nb_intra(p, x0, y0, i, -1)) carry = top[i + 3];
                else fill(top + i, carry, 4);
            }
        }
    }
    /* unavailable samples, the reference's if-chain (pred_template.c:296-332) */
    if (!bl) {
        if (l) {
            fill(left + n, left[n - 1], n);
        } else if (ul) {
            fill(left, left[-1], 2 * n);
            l = 1;
        } else if (u) {
            left[-1] = top[0];
            fill(left, left[-1], 2 * n);
            ul = l = 1;
        } else if (ur) {
            fill(top, top[n], n);
            left[-1] = top[n];
            fill(left, left[-1], 2 * n);
            u = ul = l = 1;
        } else {
            left[-1] = 1 << (depth - 1);
            fill(top, left[-1], 2 * n);
            fill(left, left[-1], 2 * n);
        }
    }
    if (!l) fill(left, left[n], n);
    if (!ul) left[-1] = left[0];
    if (!u) fill(top, left[-1], n);
    if (!ur) fill(top + n, top[n - 1], n);
    top[-1] = left[-1];

    const int *pt = top, *pl = left;
    if ((f & B200_HEVC_INTRA_SMOOTH) && mode != 1 && n != 4) {
        const int dist = iabs(mode - 26) < iabs(mode - 10) ? iabs(mode - 26) : iabs(mode - 10);
        const int limit = log2 == 3 ? 7 : log2 == 4 ? 1 : 0;
        if (dist > limit) {
            const int thr = 1 << (depth - 5);
            if ((f & B200_HEVC_INTRA_STRONG) && luma && log2 == 5 && iabs(top[-1] + top[63] - 2 * top[31]) < thr &&
                iabs(left[-1] + left[63] - 2 * left[31]) < thr) {
                filt_strong(fta + 1, left, top);
                pt = fta + 1;
            } else {
                filt3(fla + 1, fta + 1, left, top, 2 * n);
                pt = fta + 1;
                pl = fla + 1;
            }
        }
    }
    int blk[32 * 32];
    predict(blk, pt, pl, log2, mode, luma, depth);
    for (int yy = 0; yy < n; yy++)
        for (int xx = 0; xx < n; xx++) wr(p->pix, depth, base + (ptrdiff_t)yy * p->stride + xx, blk[yy * n + xx]);
#undef PIX
}

/* the ops of one b200_hevc_intra_pred_batch_device call, one after the other (the same result as the batch for independent ops);
 * stride and map_stride in bytes; returns 0, -1 for arguments the entry refuses */
API int orc_hevc_intra_plane(int depth, uint8_t *pix, ptrdiff_t stride, int width, int height, int hshift, int vshift, int64_t nops,
                             const B200HevcIntraOp *ops, const uint8_t *map, ptrdiff_t map_stride, int log2_min_pu)
{
    if ((depth != 8 && depth != 9 && depth != 10 && depth != 12) || nops < 0 || width < 1 || height < 1 || hshift < 0 || hshift > 1 ||
        vshift < 0 || vshift > 1)
        return -1;
    const int bps = depth > 8 ? 2 : 1;
    Pic p = { pix, stride / bps, depth, width, height, hshift, vshift, width >> hshift, height >> vshift, map, map_stride,
              map ? log2_min_pu : 2, 0, 0 };
    p.mpw = width >> p.log2_pu;
    p.mph = height >> p.log2_pu;
    for (int64_t k = 0; k < nops; k++) one_op(&p, &ops[k]);
    return 0;
}
