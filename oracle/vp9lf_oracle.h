/* vp9lf_oracle.h — TEST INFRASTRUCTURE ONLY.  Declarations of the VP9 loop-filter checker (vp9lf_oracle.c, part of liboracle.so). */
#ifndef VP9LF_ORACLE_H
#define VP9LF_ORACLE_H
#include <stdint.h>
#include <stddef.h>
#include "../include/b200dsp.h"
#ifdef __cplusplus
extern "C" {
#endif

/* member m of VP9DSPContext at depth 8, 10, 12 (HOST pointers, stride in bytes): 0..5 loop_filter_8[m >> 1][m & 1], 6..7
 * loop_filter_16[m & 1], 8..15 loop_filter_mix2[(m - 8) >> 2][((m - 8) >> 1) & 1][m & 1]; -1 for a depth or m outside the table */
int orc_vp9_lf_member(int depth, int m, uint8_t *dst, ptrdiff_t stride, int E, int I, int H);
/* b200_vp9_loopfilter_frame_device (include/b200dsp.h) on HOST planes.  order 0: superblocks in raster order (the entry's result);
 * k >= 1: superblock (r, c) at wavefront step c + k r, lower rows first within a step; -1: every superblock's column edges, then every superblock's row edges (the
 * frame-wide order of HEVC deblocking).  -1 for invalid arguments. */
int orc_vp9_lf_frame(int depth, int ss_h, int ss_v, int width, int height, uint8_t *const planes[3], ptrdiff_t ls_y, ptrdiff_t ls_uv,
                     const B200Vp9Filter *lflvl, int64_t lflvl_stride, const uint8_t lim_lut[64], const uint8_t mblim_lut[64], int order);

#ifdef __cplusplus
}
#endif
#endif
