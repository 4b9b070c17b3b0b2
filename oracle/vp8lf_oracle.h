/* vp8lf_oracle.h — TEST INFRASTRUCTURE ONLY.  Declarations of the VP8 / VP7 loop-filter checker (vp8lf_oracle.c, part of liboracle.so). */
#ifndef VP8LF_ORACLE_H
#define VP8LF_ORACLE_H
#include <stdint.h>
#include <stddef.h>
#include "../include/b200dsp.h"
#ifdef __cplusplus
extern "C" {
#endif

/* loop-filter member m of VP8DSPContext (VP8 or VP7), in member order: 0 v16y, 1 h16y, 2 v8uv, 3 h8uv, 4 v16y_inner, 5 h16y_inner,
 * 6 v8uv_inner, 7 h8uv_inner, 8 v_simple, 9 h_simple (HOST pointers; dstv only for 8uv; E is flim for the simple members, I and H
 * unused there); -1 for is_vp7 or m outside the table */
int orc_vp8_lf_member(int is_vp7, int m, uint8_t *dst, uint8_t *dstv, ptrdiff_t stride, int E, int I, int H);
/* b200_vp8_loopfilter_frame_device (include/b200dsp.h) on HOST planes.  order 0: macroblocks in raster order (the entry's result);
 * k >= 1: MB (r, c) at wavefront step c + k r, lower rows first within a step; -1: every MB's column edges, then every MB's row edges
 * (a frame-wide order); -2: per MB in raster order with VP8's edge order for VP7 too (the inner column edges before the row edges).
 * -1 for invalid arguments. */
int orc_vp8_lf_frame(int is_vp7, int simple, int keyframe, int mb_width, int mb_height, uint8_t *const planes[3], ptrdiff_t ls_y,
                     ptrdiff_t ls_uv, const B200Vp8FilterStrength *f, int64_t f_stride, int order);

#ifdef __cplusplus
}
#endif
#endif
