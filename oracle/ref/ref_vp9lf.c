/* TEST INFRASTRUCTURE — the reference's VP9 loop filter (libavcodec/vp9lpf.c with the loop-filter functions of vp9dsp.c,
 * vp9dsp_8bpp.c, vp9dsp_10bpp.c, vp9dsp_12bpp.c, compiled unmodified where they lie by oracle/ref/vp9lf.mk into
 * oracle/_ref/libffref_vp9lf.so) exposed through a flat C ABI: one loop-filter member of ff_vp9dsp_init(.., bpp, 1) per call, and
 * ff_vp9_loopfilter_sb over a frame's superblocks on a hand-set VP9Context (the fields vp9lpf.c reads: dsp, filter_lut, bytesperpixel,
 * ss_h, ss_v and the current frame's data / linesize), in raster order or in a wavefront order.  tests/vp9lflib.py loads it. */
#include <stdint.h>
#include <stddef.h>
#include <string.h>

#include "config.h"
#include "libavutil/frame.h"
#include "libavcodec/avcodec.h"
#include "libavcodec/vp9dec.h"
#include "../../include/b200dsp.h"

#define API __attribute__((visibility("default")))

_Static_assert(sizeof(VP9Filter) == sizeof(B200Vp9Filter), "B200Vp9Filter size");
_Static_assert(offsetof(VP9Filter, level) == offsetof(B200Vp9Filter, level), "B200Vp9Filter level");
_Static_assert(offsetof(VP9Filter, mask) == offsetof(B200Vp9Filter, mask), "B200Vp9Filter mask");
_Static_assert(sizeof(((VP9Filter *)0)->mask) == sizeof(((B200Vp9Filter *)0)->mask), "B200Vp9Filter mask size");

static VP9Context ctx;
static AVFrame frame;
static AVCodecContext avctx;

static int setup(int depth, int ss_h, int ss_v)
{
    if (depth != 8 && depth != 10 && depth != 12) return -1;
    memset(&ctx, 0, sizeof(ctx));
    ff_vp9dsp_init(&ctx.dsp, depth, 1);
    ctx.bytesperpixel = depth > 8 ? 2 : 1;
    ctx.ss_h = ss_h;
    ctx.ss_v = ss_v;
    ctx.s.frames[CUR_FRAME].tf.f = &frame;
    avctx.priv_data = &ctx;
    return 0;
}

/* member m: 0..5 loop_filter_8[m >> 1][m & 1], 6..7 loop_filter_16[m & 1], 8..15 loop_filter_mix2[(m - 8) >> 2][((m - 8) >> 1) & 1][m & 1] */
API int ffref_vp9_lf_member(int depth, int m, uint8_t *dst, ptrdiff_t stride, int E, int I, int H)
{
    if (setup(depth, 0, 0) || m < 0 || m > 15) return -1;
    if (m < 6) ctx.dsp.loop_filter_8[m >> 1][m & 1](dst, stride, E, I, H);
    else if (m < 8) ctx.dsp.loop_filter_16[m & 1](dst, stride, E, I, H);
    else ctx.dsp.loop_filter_mix2[(m - 8) >> 2][((m - 8) >> 1) & 1][m & 1](dst, stride, E, I, H);
    return 0;
}

/* 1 if the 16 loop-filter pointers are distinct */
API int ffref_vp9_lf_distinct(int depth)
{
    void *p[16];
    if (setup(depth, 0, 0)) return -1;
    memcpy(p, ctx.dsp.loop_filter_8, 6 * sizeof(void *));
    memcpy(p + 6, ctx.dsp.loop_filter_16, 2 * sizeof(void *));
    memcpy(p + 8, ctx.dsp.loop_filter_mix2, 8 * sizeof(void *));
    for (int a = 0; a < 16; a++)
        for (int b = 0; b < a; b++)
            if (p[a] == p[b]) return 0;
    return 1;
}

/* ff_vp9_loopfilter_sb for every superblock (HOST planes): k = 0 raster order, k >= 1 the wavefront in which superblock (r, c) runs at
 * step c + k r (lower rows first within a step: the order a wait that is too short would allow) */
API int ffref_vp9_lf_frame(int depth, int ss_h, int ss_v, int width, int height, uint8_t *const planes[3], ptrdiff_t ls_y, ptrdiff_t ls_uv,
                           const B200Vp9Filter *lflvl, int64_t lstride, const uint8_t lim[64], const uint8_t mblim[64], int k)
{
    if (setup(depth, ss_h, ss_v) || k < 0) return -1;
    const int bps = ctx.bytesperpixel, cols = (width + 7) >> 3, rows = (height + 7) >> 3;
    const int sb_cols = (cols + 7) >> 3, sb_rows = (rows + 7) >> 3;
    memcpy(ctx.filter_lut.lim_lut, lim, 64);
    memcpy(ctx.filter_lut.mblim_lut, mblim, 64);
    for (int p = 0; p < 3; p++) frame.data[p] = planes[p];
    frame.linesize[0] = (int)ls_y;
    frame.linesize[1] = frame.linesize[2] = (int)ls_uv;
    const int steps = k ? sb_cols + k * (sb_rows - 1) : sb_rows * sb_cols;
    for (int s = 0; s < steps; s++)
        for (int r = sb_rows - 1; r >= 0; r--) {
            const int c = k ? s - k * r : (s / sb_cols == r ? s % sb_cols : -1);
            if (c < 0 || c >= sb_cols) continue;
            VP9Filter *f = (VP9Filter *)(lflvl + (int64_t)r * lstride + c);
            ff_vp9_loopfilter_sb(&avctx, f, r * 8, c * 8, (ptrdiff_t)r * 64 * ls_y + (ptrdiff_t)c * 64 * bps,
                                 (ptrdiff_t)r * (64 >> ss_v) * ls_uv + (ptrdiff_t)c * (64 >> ss_h) * bps);
        }
    return 0;
}
