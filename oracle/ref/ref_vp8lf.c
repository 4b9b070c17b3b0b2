/* TEST INFRASTRUCTURE — the reference's VP8 / VP7 loop filter (the ten loop-filter functions of libavcodec/vp8dsp.c, compiled unmodified
 * where it lies by oracle/ref/vp8lf.mk into oracle/_ref/libffref_vp8lf.so) exposed through a flat C ABI: one
 * loop-filter member of ff_vp8dsp_init / ff_vp7dsp_init per call, and the decoder's per-macroblock sequence over a frame in raster order:
 * filter_mb / filter_mb_simple (vp8.c:2181-2299, static there) restated around the reference members, with the limits and the edge
 * order they use, and the 70 pointers of both contexts.  Plus the compile-time proof that
 * B200Vp8FilterStrength has VP8FilterStrength's layout.  tests/vp8lflib.py loads it. */
#include <stdint.h>
#include <stddef.h>
#include <string.h>

#include "config.h"
#include "libavcodec/vp8dsp.h"
#include "libavcodec/vp8.h"
#include "../../include/b200dsp.h"

#define API __attribute__((visibility("default")))

_Static_assert(sizeof(VP8FilterStrength) == sizeof(B200Vp8FilterStrength), "B200Vp8FilterStrength size");
_Static_assert(offsetof(VP8FilterStrength, filter_level) == offsetof(B200Vp8FilterStrength, filter_level), "filter_level");
_Static_assert(offsetof(VP8FilterStrength, inner_limit) == offsetof(B200Vp8FilterStrength, inner_limit), "inner_limit");
_Static_assert(offsetof(VP8FilterStrength, inner_filter) == offsetof(B200Vp8FilterStrength, inner_filter), "inner_filter");

API const char ffref_vp8lf_layout_check[] = "b200dsp.h B200Vp8FilterStrength matches VP8FilterStrength";

static VP8DSPContext *lf_ctx(int is_vp7)
{
    static VP8DSPContext c[2];
    static int ok[2];
    if (is_vp7 != 0 && is_vp7 != 1) return NULL;
    if (!ok[is_vp7]) {
        memset(&c[is_vp7], 0, sizeof(c[is_vp7]));
        ff_vp78dsp_init(&c[is_vp7]);
        if (is_vp7) ff_vp7dsp_init(&c[is_vp7]);
        else ff_vp8dsp_init(&c[is_vp7]);
        ok[is_vp7] = 1;
    }
    return &c[is_vp7];
}

/* the 70 pointers of the context after ff_vp78dsp_init and ff_vp8dsp_init / ff_vp7dsp_init, in member order */
API int ffref_vp8lf_pointers(int is_vp7, void **out)
{
    VP8DSPContext *c = lf_ctx(is_vp7);
    if (!c) return -1;
    memcpy(out, c, sizeof(*c));
    return 0;
}

/* member m in member order: 0 v16y, 1 h16y, 2 v8uv, 3 h8uv, 4 v16y_inner, 5 h16y_inner, 6 v8uv_inner, 7 h8uv_inner, 8 v_simple,
 * 9 h_simple (dstv for 8uv only; E is flim for the simple members) */
API int ffref_vp8_lf_member(int is_vp7, int m, uint8_t *dst, uint8_t *dstv, ptrdiff_t stride, int E, int I, int H)
{
    VP8DSPContext *c = lf_ctx(is_vp7);
    if (!c || m < 0 || m > 9) return -1;
    switch (m) {
    case 0: c->vp8_v_loop_filter16y(dst, stride, E, I, H); break;
    case 1: c->vp8_h_loop_filter16y(dst, stride, E, I, H); break;
    case 2: c->vp8_v_loop_filter8uv(dst, dstv, stride, E, I, H); break;
    case 3: c->vp8_h_loop_filter8uv(dst, dstv, stride, E, I, H); break;
    case 4: c->vp8_v_loop_filter16y_inner(dst, stride, E, I, H); break;
    case 5: c->vp8_h_loop_filter16y_inner(dst, stride, E, I, H); break;
    case 6: c->vp8_v_loop_filter8uv_inner(dst, dstv, stride, E, I, H); break;
    case 7: c->vp8_h_loop_filter8uv_inner(dst, dstv, stride, E, I, H); break;
    case 8: c->vp8_v_loop_filter_simple(dst, stride, E); break;
    default: c->vp8_h_loop_filter_simple(dst, stride, E); break;
    }
    return 0;
}

/* hev_thresh_lut[keyframe][level] of filter_mb (vp8.c:2191-2202), level 0..63 */
static int hev_thresh(int keyframe, int level)
{
    if (level >= 40) return keyframe ? 2 : 3;
    if (level >= 20) return keyframe ? 1 : 2;
    return level >= 15;
}

/* filter_mb's inner column edges (H_LOOP_FILTER_16Y_INNER, vp8.c:2226-2241) */
static void h_inner(const VP8DSPContext *d, uint8_t *const dst[3], int bedge_lim_y, int bedge_lim_uv, int inner_limit, int hev,
                    ptrdiff_t linesize, ptrdiff_t uvlinesize)
{
    for (int k = 4; k < 16; k += 4) d->vp8_h_loop_filter16y_inner(dst[0] + k, linesize, bedge_lim_y, inner_limit, hev);
    d->vp8_h_loop_filter8uv_inner(dst[1] + 4, dst[2] + 4, uvlinesize, bedge_lim_uv, inner_limit, hev);
}

/* filter_mb (vp8.c:2181-2266) */
static void filter_mb(const VP8DSPContext *d, uint8_t *const dst[3], const VP8FilterStrength *f, int mb_x, int mb_y, int is_vp7,
                      int keyframe, ptrdiff_t linesize, ptrdiff_t uvlinesize)
{
    const int filter_level = f->filter_level, inner_limit = f->inner_limit, inner_filter = f->inner_filter;
    int mbedge_lim, bedge_lim_y, bedge_lim_uv;
    if (!filter_level) return;
    if (is_vp7) {
        bedge_lim_y = filter_level;
        bedge_lim_uv = filter_level * 2;
        mbedge_lim = filter_level + 2;
    } else {
        bedge_lim_y = bedge_lim_uv = filter_level * 2 + inner_limit;
        mbedge_lim = bedge_lim_y + 4;
    }
    const int hev = hev_thresh(keyframe, filter_level);
    if (mb_x) {
        d->vp8_h_loop_filter16y(dst[0], linesize, mbedge_lim, inner_limit, hev);
        d->vp8_h_loop_filter8uv(dst[1], dst[2], uvlinesize, mbedge_lim, inner_limit, hev);
    }
    if (!is_vp7 && inner_filter) h_inner(d, dst, bedge_lim_y, bedge_lim_uv, inner_limit, hev, linesize, uvlinesize);
    if (mb_y) {
        d->vp8_v_loop_filter16y(dst[0], linesize, mbedge_lim, inner_limit, hev);
        d->vp8_v_loop_filter8uv(dst[1], dst[2], uvlinesize, mbedge_lim, inner_limit, hev);
    }
    if (inner_filter) {
        for (int k = 4; k < 16; k += 4) d->vp8_v_loop_filter16y_inner(dst[0] + k * linesize, linesize, bedge_lim_y, inner_limit, hev);
        d->vp8_v_loop_filter8uv_inner(dst[1] + 4 * uvlinesize, dst[2] + 4 * uvlinesize, uvlinesize, bedge_lim_uv, inner_limit, hev);
    }
    if (is_vp7 && inner_filter) h_inner(d, dst, bedge_lim_y, bedge_lim_uv, inner_limit, hev, linesize, uvlinesize);
}

/* filter_mb_simple (vp8.c:2268-2299) */
static void filter_mb_simple(const VP8DSPContext *d, uint8_t *dst, const VP8FilterStrength *f, int mb_x, int mb_y, ptrdiff_t linesize)
{
    const int filter_level = f->filter_level, inner_limit = f->inner_limit, inner_filter = f->inner_filter;
    if (!filter_level) return;
    const int bedge_lim = 2 * filter_level + inner_limit, mbedge_lim = bedge_lim + 4;
    if (mb_x) d->vp8_h_loop_filter_simple(dst, linesize, mbedge_lim);
    if (inner_filter)
        for (int k = 4; k < 16; k += 4) d->vp8_h_loop_filter_simple(dst + k, linesize, bedge_lim);
    if (mb_y) d->vp8_v_loop_filter_simple(dst, linesize, mbedge_lim);
    if (inner_filter)
        for (int k = 4; k < 16; k += 4) d->vp8_v_loop_filter_simple(dst + k * linesize, linesize, bedge_lim);
}

/* filter_mb_row (vp8.c:2523-2574) over every row in order, HOST planes; MBs with filter_level > 63 are skipped (the decoder never
 * produces them; the reference would read past hev_thresh_lut) */
API int ffref_vp8_lf_frame(int is_vp7, int simple, int keyframe, int mb_width, int mb_height, uint8_t *const planes[3], ptrdiff_t ls_y,
                           ptrdiff_t ls_uv, const B200Vp8FilterStrength *f, int64_t f_stride)
{
    const VP8DSPContext *d = lf_ctx(is_vp7);
    if (!d || (simple & ~1) || (keyframe & ~1) || mb_width < 1 || mb_height < 1 || f_stride < mb_width) return -1;
    for (int mb_y = 0; mb_y < mb_height; mb_y++)
        for (int mb_x = 0; mb_x < mb_width; mb_x++) {
            const VP8FilterStrength *s = (const VP8FilterStrength *)(f + (int64_t)mb_y * f_stride + mb_x);
            if (s->filter_level > 63) continue;
            uint8_t *const dst[3] = { planes[0] + (ptrdiff_t)16 * mb_y * ls_y + 16 * mb_x, planes[1] + (ptrdiff_t)8 * mb_y * ls_uv + 8 * mb_x,
                                      planes[2] + (ptrdiff_t)8 * mb_y * ls_uv + 8 * mb_x };
            if (simple) {
                filter_mb_simple(d, dst[0], s, mb_x, mb_y, ls_y);
                continue;
            }
            filter_mb(d, dst, s, mb_x, mb_y, is_vp7, keyframe, ls_y, ls_uv);
        }
    return 0;
}
