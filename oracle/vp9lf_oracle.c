/* vp9lf_oracle.c — TEST INFRASTRUCTURE ONLY.  The checker of ffmpeg_b200/csrc/vp9lf.cu: VP9's loop-filter members
 * (libavcodec/vp9dsp_template.c:1780-1967) and the frame driver ff_vp9_loopfilter_sb (vp9lpf.c:27-203) restated on the host for 8, 10
 * and 12 bit samples.
 *
 * Written in a different form from the kernel so that each checks the other: the dispatch follows the driver's loops over pairs of
 * 8-line halves and emits edge descriptors (position, direction, width, level) for a superblock's plane first, which are then applied
 * one after the other; the 16- and 8-wide smoothing filters are running sums over a window whose ends repeat the outermost samples,
 * where the kernel sums each output's taps afresh. */
#include <stdint.h>
#include <stddef.h>
#include <stdlib.h>
#include <string.h>
#include "vp9lf_oracle.h"

typedef struct {
    uint8_t *base;
    ptrdiff_t ls;
    int bps;
} Plane;

static int get(const Plane *p, int x, int y)
{
    const uint8_t *q = p->base + (ptrdiff_t)y * p->ls + (ptrdiff_t)x * p->bps;
    return p->bps == 1 ? q[0] : ((const uint16_t *)q)[0];
}
static void put(const Plane *p, int x, int y, int v)
{
    uint8_t *q = p->base + (ptrdiff_t)y * p->ls + (ptrdiff_t)x * p->bps;
    if (p->bps == 1) q[0] = (uint8_t)v;
    else ((uint16_t *)q)[0] = (uint16_t)v;
}
static int iabs(int v) { return v < 0 ? -v : v; }
static int clampi(int v, int lo, int hi) { return v < lo ? lo : v > hi ? hi : v; }

/* x[0..15] = p7..p0 q0..q7 of one line; returns the filtered line in y (y = x where nothing changes) */
static void filter_line(int depth, int wd, int E, int I, int H, const int *x, int *y)
{
    const int s = depth - 8, F = 1 << s, top = (1 << (depth - 1)) - 1, pmax = (1 << depth) - 1;
    memcpy(y, x, 16 * sizeof(int));
    E <<= s, I <<= s, H <<= s;
    const int *p = x + 8;                                    /* p[-4..3] = p3..q3 */
    for (int k = -4; k < 3; k++)
        if (k != -1 && iabs(p[k + 1] - p[k]) > I) return;
    if (2 * iabs(p[-1] - p[0]) + (iabs(p[-2] - p[1]) >> 1) > E) return;
    int in = wd >= 8, out = wd >= 16;
    for (int k = 1; k <= 3 && in; k++) in = iabs(p[-1 - k] - p[-1]) <= F && iabs(p[k] - p[0]) <= F;
    for (int k = 4; k <= 7 && out; k++) out = iabs(p[-1 - k] - p[-1]) <= F && iabs(p[k] - p[0]) <= F;
    if (in && out) {                                         /* 15 taps from p7..q7, the ends repeated, the centre once more */
        int sum = 0;
        for (int d = -7; d <= 7; d++) sum += x[clampi(1 + d, 0, 15)];
        for (int j = 1; j <= 14; j++) {
            y[j] = (sum + x[j] + 8) >> 4;
            sum += x[clampi(j + 8, 0, 15)] - x[clampi(j - 7, 0, 15)];
        }
    } else if (in) {                                         /* 7 taps from p3..q3 */
        int sum = 0;
        for (int d = -3; d <= 3; d++) sum += x[clampi(5 + d, 4, 11)];
        for (int j = 5; j <= 10; j++) {
            y[j] = (sum + x[j] + 4) >> 3;
            sum += x[clampi(j + 4, 4, 11)] - x[clampi(j - 3, 4, 11)];
        }
    } else {
        const int hev = iabs(p[-2] - p[-1]) > H || iabs(p[1] - p[0]) > H;
        int f = clampi(3 * (p[0] - p[-1]) + (hev ? clampi(p[-2] - p[1], -top - 1, top) : 0), -top - 1, top);
        const int f1 = (f + 4 > top ? top : f + 4) >> 3, f2 = (f + 3 > top ? top : f + 3) >> 3;
        y[7] = clampi(p[-1] + f2, 0, pmax);
        y[8] = clampi(p[0] - f1, 0, pmax);
        if (!hev) {
            y[6] = clampi(p[-2] + ((f1 + 1) >> 1), 0, pmax);
            y[9] = clampi(p[1] - ((f1 + 1) >> 1), 0, pmax);
        }
    }
}

/* 8 lines of one edge: line l's q0 at (x + l, y) for dir 1 (row edge), (x, y + l) for dir 0 (column edge) */
static void filter_edge(int depth, const Plane *pl, int dir, int x, int y, int wd, int E, int I, int H)
{
    const int reach = wd >= 16 ? 8 : 4, wr = wd >= 16 ? 7 : wd >= 8 ? 3 : 2;
    for (int l = 0; l < 8; l++) {
        int a[16] = { 0 }, b[16];
        for (int k = -reach; k < reach; k++) a[8 + k] = dir ? get(pl, x + l, y + k) : get(pl, x + k, y + l);
        filter_line(depth, wd, E, I, H, a, b);
        for (int k = -wr; k < wr; k++) {
            if (dir) put(pl, x + l, y + k, b[8 + k]);
            else put(pl, x + k, y + l, b[8 + k]);
        }
    }
}

int orc_vp9_lf_member(int depth, int m, uint8_t *dst, ptrdiff_t stride, int E, int I, int H)
{
    if ((depth != 8 && depth != 10 && depth != 12) || m < 0 || m > 15) return -1;
    const int bps = depth > 8 ? 2 : 1, dir = m & 1;
    Plane pl = { dst, stride, bps };
    int wd[2], e[2] = { E, E }, i[2] = { I, I }, h[2] = { H, H };
    if (m < 6) wd[0] = 4 << (m >> 1), wd[1] = 0;
    else if (m < 8) wd[0] = wd[1] = 16;
    else {
        wd[0] = 4 << ((m - 8) >> 2), wd[1] = 4 << (((m - 8) >> 1) & 1);
        e[0] = E & 0xff, i[0] = I & 0xff, h[0] = H & 0xff;
        e[1] = E >> 8, i[1] = I >> 8, h[1] = H >> 8;
    }
    for (int k = 0; k < 2; k++)
        if (wd[k]) filter_edge(depth, &pl, dir, dir ? 8 * k : 0, dir ? 0 : 8 * k, wd[k], e[k], i[k], h[k]);
    return 0;
}

/* ---------------------------------------------------------------- frame */
typedef struct { int x, y, dir, wd, L; } EdgeDesc;          /* 8 lines; (x, y) = q0 of the first line in plane coordinates */

typedef struct {
    EdgeDesc e[1024];
    int n;
} EdgeList;

static void emit(EdgeList *el, int x, int y, int dir, int wd, int L)
{
    EdgeDesc d = { x, y, dir, wd, L & 63 };
    el->e[el->n++] = d;
}

/* filter_plane_cols (vp9lpf.c:27-100) for the superblock whose plane origin is (x0, y0) */
static void cols_edges(EdgeList *el, int first_col, int ss_h, int ss_v, const uint8_t *lvl, const uint8_t (*mask)[4], int x0, int y0)
{
    for (int y = 0; y < 8; y += 2 << ss_v) {
        const uint8_t *h1 = mask[y], *h2 = mask[y + 1 + ss_v];
        const unsigned hm1 = h1[0] | h1[1] | h1[2], hm2 = h2[1] | h2[2], all = hm1 | hm2 | h1[3] | h2[3];
        const int py = y0 + (y >> ss_v) * 8, l1 = y * 8, l2 = (y + (1 << ss_v)) * 8;
        int lc = 0;
        for (int bit = 0; bit < 8 && (all >> bit); bit++) {
            const unsigned x = 1u << bit;
            const int px = x0 + bit * (8 >> ss_h);
            if (!first_col || bit > 0) {
                if (hm1 & x) {
                    if (h1[0] & x) {
                        emit(el, px, py, 0, 16, lvl[l1 + lc]);
                        if (h2[0] & x) emit(el, px, py + 8, 0, 16, lvl[l1 + lc]);
                    } else {
                        emit(el, px, py, 0, (h1[1] & x) ? 8 : 4, lvl[l1 + lc]);
                        if (hm2 & x) emit(el, px, py + 8, 0, (h2[1] & x) ? 8 : 4, lvl[l2 + lc]);
                    }
                } else if (hm2 & x) {
                    emit(el, px, py + 8, 0, (h2[1] & x) ? 8 : 4, lvl[l2 + lc]);
                }
            }
            if (ss_h) {
                if (bit & 1) lc += 2;
            } else {
                if (h1[3] & x) emit(el, px + 4, py, 0, 4, lvl[l1 + lc]);
                if (h2[3] & x) emit(el, px + 4, py + 8, 0, 4, lvl[l2 + lc]);
                lc++;
            }
        }
    }
}

/* filter_plane_rows (vp9lpf.c:102-177) */
static void rows_edges(EdgeList *el, int first_row, int ss_h, int ss_v, const uint8_t *lvl, const uint8_t (*mask)[4], int x0, int y0)
{
    for (int y = 0; y < 8; y++) {
        const uint8_t *v = mask[y];
        const unsigned vm = v[0] | v[1] | v[2];
        const int py = y0 + y * (8 >> ss_v), lr = (ss_v ? y & ~1 : y) * 8;
        for (int bit = 0, k = 0; bit < 8 && (vm >> bit); bit += 2 << ss_h, k++) {
            const unsigned a = 1u << bit, b = 1u << (bit + 1 + ss_h);
            const int px = x0 + 16 * k, La = lvl[lr + bit], Lb = lvl[lr + bit + 1 + ss_h];
            if (!first_row || y) {
                if (vm & a) {
                    if (v[0] & a) {
                        emit(el, px, py, 1, 16, La);
                        if (v[0] & b) emit(el, px + 8, py, 1, 16, La);
                    } else {
                        emit(el, px, py, 1, (v[1] & a) ? 8 : 4, La);
                        if (vm & b) emit(el, px + 8, py, 1, (v[1] & b) ? 8 : 4, Lb);
                    }
                } else if (vm & b) {
                    emit(el, px + 8, py, 1, (v[1] & b) ? 8 : 4, Lb);
                }
            }
            if (!ss_v) {
                if (v[3] & a) emit(el, px, py + 4, 1, 4, La);
                if (v[3] & b) emit(el, px + 8, py + 4, 1, 4, Lb);
            }
        }
    }
}

typedef struct {
    int depth, ss_h, ss_v, cols, rows;
    Plane pl[3];
    const B200Vp9Filter *lflvl;
    int64_t lstride;
    const uint8_t *lim, *mblim;
} Frame;

/* the record of superblock (r, c) with the mask bits the entry ignores cleared */
static void record(const Frame *f, int r, int c, B200Vp9Filter *out)
{
    *out = f->lflvl[(int64_t)r * f->lstride + c];
    const int nc = f->cols - 8 * c, nr = f->rows - 8 * r;
    const unsigned keep = nc >= 8 ? 0xFF : (1u << nc) - 1;
    for (int ch = 0; ch < 2; ch++)
        for (int d = 0; d < 2; d++)
            for (int y = 0; y < 8; y++)
                for (int w = 0; w < 4; w++) out->mask[ch][d][y][w] &= y < nr ? keep : 0;
    /* chroma 16-wide edges at bit 7 / row 7 of a subsampled direction (mask_edges sets them only at 0 and 4) */
    for (int y = 0; y < 8; y++)
        if (f->ss_h) out->mask[1][0][y][0] &= 0x7F;
    if (f->ss_v) out->mask[1][1][7][0] = 0;
}

/* pass bit 0: column edges, bit 1: row edges, of every plane of superblock (r, c) */
static void run_sb(const Frame *f, int r, int c, int pass)
{
    B200Vp9Filter rec;
    record(f, r, c, &rec);
    static EdgeList el;
    for (int p = 0; p < 3; p++) {
        const int sh = p ? f->ss_h : 0, sv = p ? f->ss_v : 0, mi = p ? (f->ss_h | f->ss_v) : 0;
        const int x0 = c * (64 >> sh), y0 = r * (64 >> sv);
        for (int d = 0; d < 2; d++) {
            if (!(pass >> d & 1)) continue;
            el.n = 0;
            if (d == 0) cols_edges(&el, c == 0, sh, sv, rec.level, (const uint8_t (*)[4])rec.mask[mi][0], x0, y0);
            else rows_edges(&el, r == 0, sh, sv, rec.level, (const uint8_t (*)[4])rec.mask[mi][1], x0, y0);
            for (int i = 0; i < el.n; i++) {
                const EdgeDesc *e = &el.e[i];
                filter_edge(f->depth, &f->pl[p], e->dir, e->x, e->y, e->wd, f->mblim[e->L], f->lim[e->L], e->L >> 4);
            }
        }
    }
}

int orc_vp9_lf_frame(int depth, int ss_h, int ss_v, int width, int height, uint8_t *const planes[3], ptrdiff_t ls_y, ptrdiff_t ls_uv,
                     const B200Vp9Filter *lflvl, int64_t lflvl_stride, const uint8_t lim_lut[64], const uint8_t mblim_lut[64], int order)
{
    if ((depth != 8 && depth != 10 && depth != 12) || (ss_h & ~1) || (ss_v & ~1) || width < 1 || height < 1 || order < -1) return -1;
    const int bps = depth > 8 ? 2 : 1;
    Frame f = { depth, ss_h, ss_v, (width + 7) >> 3, (height + 7) >> 3,
                { { planes[0], ls_y, bps }, { planes[1], ls_uv, bps }, { planes[2], ls_uv, bps } }, lflvl, lflvl_stride, lim_lut, mblim_lut };
    const int sbc = (f.cols + 7) >> 3, sbr = (f.rows + 7) >> 3;
    if (lflvl_stride < sbc) return -1;
    if (order == -1) {
        for (int pass = 1; pass <= 2; pass++)
            for (int r = 0; r < sbr; r++)
                for (int c = 0; c < sbc; c++) run_sb(&f, r, c, pass);
    } else if (order == 0) {
        for (int r = 0; r < sbr; r++)
            for (int c = 0; c < sbc; c++) run_sb(&f, r, c, 3);
    } else {
        for (int s = 0; s < sbc + order * (sbr - 1); s++)
            for (int r = sbr - 1; r >= 0; r--)               /* lower rows first: what a wait that is too short lets happen */
                if (s - order * r >= 0 && s - order * r < sbc) run_sb(&f, r, s - order * r, 3);
    }
    return 0;
}
