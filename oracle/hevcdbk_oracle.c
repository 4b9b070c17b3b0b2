/*
 * hevcdbk_oracle.c — TEST INFRASTRUCTURE ONLY.  CPU restatement of the HEVC deblocking members of HEVCDSPContext
 * (libavcodec/hevc/dsp.h:47-125: hevc_{h,v}_loop_filter_{luma,chroma} and the identical _c twins) as ff_hevc_dsp_init installs them
 * for depth 8, 9, 10 and 12 (hevc/dsp.c:237-244), and the picture-level semantics of b200_hevc_deblock_plane_device
 * (include/b200dsp.h): every vertical segment of the plane, then every horizontal one.
 *
 * Follows (behaviour, not text) hevc/dsp_template.c:834-928 and h26x/h2656_deblock_template.c, written per 4-line segment: the
 * segment's samples are addressed as s(i, k), line i = 0..3 along the edge, k = -4..3 across it (k < 0 the P side), so one routine
 * serves both edge directions and both the member and the plane forms.  It also counts which branch each segment (and weak-filter
 * line) takes, so tests can show that an input reaches every branch:
 *   cnt[0] luma, tc > 0, skipped by d >= beta      cnt[1] luma strong
 *   cnt[2] / cnt[3] luma weak with nd_p 1 / 2       cnt[4] / cnt[5] luma weak with nd_q 1 / 2
 *   cnt[6] luma weak lines skipped by |delta0| >= 10 tc
 *   cnt[7] segments with tc <= 0 (luma or chroma)   cnt[8] chroma segments filtered
 */
#include <stdint.h>
#include <stddef.h>
#include <stdlib.h>
#include "../include/b200dsp.h"

typedef struct {
    uint8_t *base;        /* sample (line 0, k = 0) */
    ptrdiff_t along;      /* bytes from line i to line i + 1 */
    ptrdiff_t across;     /* bytes from k to k + 1 */
    int bps;
} Seg;

static int rd(const Seg *s, int i, int k)
{
    const uint8_t *p = s->base + i * s->along + k * s->across;
    return s->bps == 1 ? *p : *(const uint16_t *)p;
}
static void wr(const Seg *s, int i, int k, int v)
{
    uint8_t *p = s->base + i * s->along + k * s->across;
    if (s->bps == 1) *p = (uint8_t)v;
    else *(uint16_t *)p = (uint16_t)v;
}
static int clip(int v, int lo, int hi) { return v < lo ? lo : v > hi ? hi : v; }

/* second difference on one side of line i: side -1 = P (p2 - 2 p1 + p0), +1 = Q */
static int d2(const Seg *s, int i, int side)
{
    return side < 0 ? abs(rd(s, i, -3) - 2 * rd(s, i, -2) + rd(s, i, -1)) : abs(rd(s, i, 2) - 2 * rd(s, i, 1) + rd(s, i, 0));
}

static void luma_seg(const Seg *s, int depth, int beta8, int tc8, int no_p, int no_q, int64_t *cnt)
{
    const int maxv = (1 << depth) - 1;
    const int beta = beta8 * (1 << (depth - 8)), tc = tc8 * (1 << (depth - 8));
    if (tc <= 0) { cnt[7]++; return; }
    const int dp = d2(s, 0, -1) + d2(s, 3, -1), dq = d2(s, 0, 1) + d2(s, 3, 1);
    if (dp + dq >= beta) { cnt[0]++; return; }
    int strong = 1;
    for (int i = 0; i <= 3; i += 3) {
        const int d = d2(s, i, -1) + d2(s, i, 1);
        strong &= abs(rd(s, i, -4) - rd(s, i, -1)) + abs(rd(s, i, 3) - rd(s, i, 0)) < beta / 8 &&
                  abs(rd(s, i, -1) - rd(s, i, 0)) < (5 * tc + 1) / 2 && 2 * d < beta / 4;
    }
    if (strong) {
        cnt[1]++;
        const int lim = 2 * tc;
        for (int i = 0; i < 4; i++) {
            int a[8];                                          /* a[k + 4] = sample k */
            for (int k = -4; k < 4; k++) a[k + 4] = rd(s, i, k);
            for (int side = 0; side < 2; side++) {
                if (side == 0 ? no_p : no_q) continue;
                int v0, v1, v2, v3, w0, w1;                      /* own side at distance 0..3 from the edge, the other side 0..1 */
                if (side == 0) { v0 = a[3]; v1 = a[2]; v2 = a[1]; v3 = a[0]; w0 = a[4]; w1 = a[5]; }
                else           { v0 = a[4]; v1 = a[5]; v2 = a[6]; v3 = a[7]; w0 = a[3]; w1 = a[2]; }
                const int n0 = (v2 + 2 * v1 + 2 * v0 + 2 * w0 + w1 + 4) >> 3;
                const int n1 = (v2 + v1 + v0 + w0 + 2) >> 2;
                const int n2 = (2 * v3 + 3 * v2 + v1 + v0 + w0 + 4) >> 3;
                const int sg = side == 0 ? -1 : 1, o = side == 0 ? -1 : 0;
                wr(s, i, o, v0 + clip(n0 - v0, -lim, lim));
                wr(s, i, o + sg, v1 + clip(n1 - v1, -lim, lim));
                wr(s, i, o + 2 * sg, v2 + clip(n2 - v2, -lim, lim));
            }
        }
        return;
    }
    const int thr = (beta + beta / 2) / 8;
    const int ndp = dp < thr ? 2 : 1, ndq = dq < thr ? 2 : 1;
    cnt[ndp == 2 ? 3 : 2]++;
    cnt[ndq == 2 ? 5 : 4]++;
    for (int i = 0; i < 4; i++) {
        const int p2 = rd(s, i, -3), p1 = rd(s, i, -2), p0 = rd(s, i, -1), q0 = rd(s, i, 0), q1 = rd(s, i, 1), q2 = rd(s, i, 2);
        int delta = (9 * (q0 - p0) - 3 * (q1 - p1) + 8) >> 4;
        if (abs(delta) >= 10 * tc) { cnt[6]++; continue; }
        delta = clip(delta, -tc, tc);
        if (!no_p) {
            wr(s, i, -1, clip(p0 + delta, 0, maxv));
            if (ndp == 2) wr(s, i, -2, clip(p1 + clip((((p2 + p0 + 1) >> 1) - p1 + delta) >> 1, -(tc >> 1), tc >> 1), 0, maxv));
        }
        if (!no_q) {
            wr(s, i, 0, clip(q0 - delta, 0, maxv));
            if (ndq == 2) wr(s, i, 1, clip(q1 + clip((((q2 + q0 + 1) >> 1) - q1 - delta) >> 1, -(tc >> 1), tc >> 1), 0, maxv));
        }
    }
}

static void chroma_seg(const Seg *s, int depth, int tc8, int no_p, int no_q, int64_t *cnt)
{
    const int maxv = (1 << depth) - 1, tc = tc8 * (1 << (depth - 8));
    if (tc <= 0) { cnt[7]++; return; }
    cnt[8]++;
    for (int i = 0; i < 4; i++) {
        const int p1 = rd(s, i, -2), p0 = rd(s, i, -1), q0 = rd(s, i, 0), q1 = rd(s, i, 1);
        const int delta = clip((4 * (q0 - p0) + p1 - q1 + 4) >> 3, -tc, tc);
        if (!no_p) wr(s, i, -1, clip(p0 + delta, 0, maxv));
        if (!no_q) wr(s, i, 0, clip(q0 - delta, 0, maxv));
    }
}

/* one member call: horiz 0 = hevc_v_loop_filter_*, 1 = hevc_h_loop_filter_*; beta ignored for chroma; cnt may be NULL */
void orc_hevc_dbk_member(int depth, int chroma, int horiz, uint8_t *pix, ptrdiff_t stride, int beta, const int32_t *tc, const uint8_t *no_p,
                         const uint8_t *no_q, int64_t *cnt)
{
    int64_t dummy[9] = { 0 };
    const int bps = depth > 8 ? 2 : 1;
    if (!cnt) cnt = dummy;
    for (int j = 0; j < 2; j++) {
        Seg s;
        s.bps = bps;
        s.along = horiz ? bps : stride;
        s.across = horiz ? stride : bps;
        s.base = pix + 4 * j * s.along;
        if (chroma) chroma_seg(&s, depth, tc[j], no_p[j], no_q[j], cnt);
        else luma_seg(&s, depth, beta, tc[j], no_p[j], no_q[j], cnt);
    }
}

/* the plane entry's semantics: every vertical segment, then every horizontal one; returns 0, cnt[9] branch counts (may be NULL) */
int orc_hevc_dbk_plane(int depth, int chroma, uint8_t *pix, ptrdiff_t stride, int width, int height, const B200HevcDbkSeg *vseg, int64_t vstride,
                       const B200HevcDbkSeg *hseg, int64_t hstride, int64_t *cnt)
{
    int64_t dummy[9] = { 0 };
    const int bps = depth > 8 ? 2 : 1;
    if (!cnt) cnt = dummy;
    for (int pass = 0; pass < 2; pass++)
        for (int y = pass ? 8 : 0; y < height; y += pass ? 8 : 4)
            for (int x = pass ? 0 : 8; x < width; x += pass ? 4 : 8) {
                const B200HevcDbkSeg *g = pass ? &hseg[(int64_t)(y / 8) * hstride + x / 4] : &vseg[(int64_t)(y / 4) * vstride + x / 8];
                Seg s;
                s.bps = bps;
                s.base = pix + (ptrdiff_t)y * stride + (ptrdiff_t)x * bps;
                s.along = pass ? bps : stride;
                s.across = pass ? stride : bps;
                const int np = !!(g->flags & B200_HEVC_DBK_NO_P), nq = !!(g->flags & B200_HEVC_DBK_NO_Q);
                if (chroma) chroma_seg(&s, depth, g->tc, np, nq, cnt);
                else luma_seg(&s, depth, g->beta, g->tc, np, nq, cnt);
            }
    return 0;
}
