/* vp8lf_oracle.c — TEST INFRASTRUCTURE ONLY.  The checker of ffmpeg_b200/csrc/vp8lf.cu: the VP8 / VP7 loop-filter members
 * (libavcodec/vp8dsp.c:263-457) and the decoder's per-macroblock sequence filter_mb / filter_mb_simple (vp8.c:2181-2299) run over a
 * frame in raster order, restated on the host.
 *
 * Written in a different form from the kernel so that each checks the other: a macroblock first emits edge descriptors (plane,
 * direction, position, kind, limits) in three groups (column edges filtered before the row edges, the row edges, VP7's late inner column
 * edges), which are then applied one after the other in the order asked for; the line filter indexes p[-4..3] around q0 and takes the
 * MB-edge taps from a table; hev_thresh counts the thresholds a level has reached.  The orders other than raster are the wrong ones a
 * frame entry could fall into (a slope-1 wavefront, a frame-wide order, VP8's edge order for VP7), for the tests that show that the
 * fixture frames tell them apart. */
#include <stdint.h>
#include <stddef.h>
#include <stdlib.h>
#include <string.h>
#include "vp8lf_oracle.h"

enum { K_MBEDGE, K_INNER, K_SIMPLE };

static int clampi(int v, int lo, int hi) { return v < lo ? lo : v > hi ? hi : v; }
static int ad(int a, int b) { return a > b ? a - b : b - a; }

/* p[-4..3] = p3..q3 of one line, filtered in place (the simple kind touches only p[-2..1]) */
static void filter_line(int vp7, int kind, int E, int I, int H, int *p)
{
    const int edge = vp7 ? ad(p[-1], p[0]) : 2 * ad(p[-1], p[0]) + (ad(p[-2], p[1]) >> 1);
    if (edge > E) return;
    if (kind != K_SIMPLE)
        for (int k = -4; k < 3; k++)
            if (k != -1 && ad(p[k], p[k + 1]) > I) return;
    const int hev = kind == K_SIMPLE || ad(p[-2], p[-1]) > H || ad(p[1], p[0]) > H;
    if (!hev && kind == K_MBEDGE) {
        static const int taps[3] = { 27, 18, 9 };            /* p0 / q0, p1 / q1, p2 / q2 */
        const int w = clampi(clampi(p[-2] - p[1], -128, 127) + 3 * (p[0] - p[-1]), -128, 127);
        for (int k = 0; k < 3; k++) {
            const int d = (taps[k] * w + 63) >> 7;
            p[-1 - k] = clampi(p[-1 - k] + d, 0, 255);
            p[k] = clampi(p[k] - d, 0, 255);
        }
        return;
    }
    const int a = clampi(3 * (p[0] - p[-1]) + (hev ? clampi(p[-2] - p[1], -128, 127) : 0), -128, 127);
    const int f1 = (a + 4 > 127 ? 127 : a + 4) >> 3;
    const int f2 = vp7 ? ((a & 7) == 4 ? f1 - 1 : f1) : (a + 3 > 127 ? 127 : a + 3) >> 3;
    const int p1 = p[-2], q1 = p[1];
    p[-1] = clampi(p[-1] + f2, 0, 255);
    p[0] = clampi(p[0] - f1, 0, 255);
    if (!hev) {
        p[-2] = clampi(p1 + ((f1 + 1) >> 1), 0, 255);
        p[1] = clampi(q1 - ((f1 + 1) >> 1), 0, 255);
    }
}

typedef struct { uint8_t *base; ptrdiff_t ls; } Plane;

/* n lines of the edge whose q0 of line 0 is at (x, y): dir 0 the edge left of column x (line l is row y + l), dir 1 the edge above row y
 * (line l is column x + l) */
static void filter_edge(const Plane *pl, int vp7, int dir, int x, int y, int n, int kind, int E, int I, int H)
{
    const int reach = kind == K_SIMPLE ? 2 : 4;
    for (int l = 0; l < n; l++) {
        int v[8] = { 0 };
        const ptrdiff_t step = dir ? pl->ls : 1;
        uint8_t *q0 = pl->base + (ptrdiff_t)(dir ? y : y + l) * pl->ls + (dir ? x + l : x);
        for (int k = -reach; k < reach; k++) v[4 + k] = q0[k * step];
        filter_line(vp7, kind, E, I, H, v + 4);
        for (int k = -reach; k < reach; k++) q0[k * step] = (uint8_t)v[4 + k];
    }
}

int orc_vp8_lf_member(int is_vp7, int m, uint8_t *dst, uint8_t *dstv, ptrdiff_t stride, int E, int I, int H)
{
    if ((is_vp7 != 0 && is_vp7 != 1) || m < 0 || m > 9) return -1;
    const int dir = !(m & 1), kind = m >= 8 ? K_SIMPLE : m >= 4 ? K_INNER : K_MBEDGE, uv = m < 8 && (m & 2);
    Plane a = { dst, stride }, b = { dstv, stride };
    filter_edge(&a, is_vp7, dir, 0, 0, uv ? 8 : 16, kind, E, I, H);
    if (uv) filter_edge(&b, is_vp7, dir, 0, 0, 8, kind, E, I, H);
    return 0;
}

/* ---------------------------------------------------------------- frame */
typedef struct { int p, dir, x, y, n, kind, E, I, H; } EdgeDesc;
typedef struct { EdgeDesc e[3][24]; int n[3]; } MbEdges;    /* groups: 0 column edges first, 1 row edges, 2 VP7's late inner columns */

static void emit(MbEdges *m, int g, int p, int dir, int x, int y, int kind, int E, int I, int H)
{
    EdgeDesc d = { p, dir, x, y, p ? 8 : 16, kind, E, I, H };
    m->e[g][m->n[g]++] = d;
}

/* hev_thresh_lut[keyframe][level] (vp8.c:2191-2202): the number of thresholds 15, 20 (inter frames only), 40 the level has reached */
static int hev_threshold(int keyframe, int level)
{
    static const int th[2][3] = { { 15, 20, 40 }, { 15, 40, 1 << 20 } };
    int n = 0;
    for (int k = 0; k < 3; k++) n += level >= th[keyframe][k];
    return n;
}

static void mb_edges(int vp7, int simple, int keyframe, int mb_x, int mb_y, const uint8_t *rec, MbEdges *m)
{
    memset(m->n, 0, sizeof(m->n));
    const int L = rec[0], il = rec[1], inner = rec[2] != 0;
    if (L == 0 || L > 63) return;
    const int H = hev_threshold(keyframe, L);
    if (simple) {                                            /* filter_mb_simple: luma, the VP8 limits for both codecs */
        const int b = 2 * L + il, mb = b + 4, x = 16 * mb_x, y = 16 * mb_y;
        if (mb_x) emit(m, 0, 0, 0, x, y, K_SIMPLE, mb, 0, 0);
        for (int k = 4; inner && k < 16; k += 4) emit(m, 0, 0, 0, x + k, y, K_SIMPLE, b, 0, 0);
        if (mb_y) emit(m, 1, 0, 1, x, y, K_SIMPLE, mb, 0, 0);
        for (int k = 4; inner && k < 16; k += 4) emit(m, 1, 0, 1, x, y + k, K_SIMPLE, b, 0, 0);
        return;
    }
    const int by = vp7 ? L : 2 * L + il, buv = vp7 ? 2 * L : by, mb = vp7 ? L + 2 : by + 4;
    for (int p = 0; p < 3; p++) {
        const int s = p ? 8 : 16, x = s * mb_x, y = s * mb_y, b = p ? buv : by;
        if (mb_x) emit(m, 0, p, 0, x, y, K_MBEDGE, mb, il, H);
        for (int k = 4; inner && k < s; k += 4) emit(m, vp7 ? 2 : 0, p, 0, x + k, y, K_INNER, b, il, H);
        if (mb_y) emit(m, 1, p, 1, x, y, K_MBEDGE, mb, il, H);
        for (int k = 4; inner && k < s; k += 4) emit(m, 1, p, 1, x, y + k, K_INNER, b, il, H);
    }
}

static void run_groups(const Plane *pl, int vp7, const MbEdges *m, const int *groups, int ng)
{
    for (int i = 0; i < ng; i++)
        for (int j = 0; j < m->n[groups[i]]; j++) {
            const EdgeDesc *d = &m->e[groups[i]][j];
            filter_edge(&pl[d->p], vp7, d->dir, d->x, d->y, d->n, d->kind, d->E, d->I, d->H);
        }
}

int orc_vp8_lf_frame(int is_vp7, int simple, int keyframe, int mb_width, int mb_height, uint8_t *const planes[3], ptrdiff_t ls_y,
                     ptrdiff_t ls_uv, const B200Vp8FilterStrength *f, int64_t f_stride, int order)
{
    if ((is_vp7 | simple | keyframe) & ~1 || mb_width < 1 || mb_height < 1 || f_stride < mb_width || order < -2) return -1;
    const Plane pl[3] = { { planes[0], ls_y }, { planes[1], ls_uv }, { planes[2], ls_uv } };
    const uint8_t *recs = (const uint8_t *)f;
    MbEdges m;
    static const int all[3] = { 0, 1, 2 }, cols[2] = { 0, 2 }, rows[1] = { 1 }, vp8_order[3] = { 0, 2, 1 };
#define REC(r, c) (recs + 3 * ((int64_t)(r) * f_stride + (c)))
    if (order == -1) {
        for (int pass = 0; pass < 2; pass++)
            for (int r = 0; r < mb_height; r++)
                for (int c = 0; c < mb_width; c++) {
                    mb_edges(is_vp7, simple, keyframe, c, r, REC(r, c), &m);
                    if (pass == 0) run_groups(pl, is_vp7, &m, cols, 2);
                    else run_groups(pl, is_vp7, &m, rows, 1);
                }
        return 0;
    }
    const int k = order > 0 ? order : 0;
    const int steps = k ? mb_width + k * (mb_height - 1) : mb_width * mb_height;
    for (int s = 0; s < steps; s++)
        for (int r = mb_height - 1; r >= 0; r--) {
            const int c = k ? s - k * r : (s / mb_width == r ? s % mb_width : -1);
            if (c < 0 || c >= mb_width) continue;
            mb_edges(is_vp7, simple, keyframe, c, r, REC(r, c), &m);
            run_groups(pl, is_vp7, &m, order == -2 ? vp8_order : all, 3);
        }
#undef REC
    return 0;
}
