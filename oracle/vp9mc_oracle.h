/* vp9mc_oracle.h — TEST INFRASTRUCTURE ONLY.  Declarations of the VP9 motion-compensation checker (vp9mc_oracle.c, part of liboracle.so). */
#ifndef VP9MC_ORACLE_H
#define VP9MC_ORACLE_H
#include <stdint.h>
#include <stddef.h>
#include "../include/b200dsp.h"
#ifdef __cplusplus
extern "C" {
#endif

/* VP9DSPContext.mc[size of w][bank][avg][hdir][vdir] / .smc[size of w][bank][avg] at depth 8, 10, 12; bank in FilterMode order
 * (smooth, regular, sharp, bilinear); strides in bytes; -1 for arguments outside the reference's contract */
int orc_vp9_mc(int depth, int bank, int avg, int hdir, int vdir, void *dst, ptrdiff_t dst_stride, const void *src, ptrdiff_t src_stride,
               int w, int h, int mx, int my);
int orc_vp9_smc(int depth, int bank, int avg, void *dst, ptrdiff_t dst_stride, const void *src, ptrdiff_t src_stride, int w, int h, int mx,
                int my, int dx, int dy);
/* the three 8-tap banks, [3][16][8] */
const int16_t *orc_vp9_subpel_filters(void);
/* b200_vp9_mc_batch_device (include/b200dsp.h) on host memory; returns the number of ops that wrote their block */
int64_t orc_vp9_mc_batch(int depth, int nrefs, const B200Vp9McRef *refs, int64_t nops, const B200Vp9McOp *ops, uint8_t *dst,
                         ptrdiff_t dst_stride);

#ifdef __cplusplus
}
#endif
#endif
