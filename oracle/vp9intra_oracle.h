/* vp9intra_oracle.h — TEST INFRASTRUCTURE ONLY.  Declarations of the VP9 intra-prediction checker (vp9intra_oracle.c, part of
 * liboracle.so). */
#ifndef VP9INTRA_ORACLE_H
#define VP9INTRA_ORACLE_H
#include <stdint.h>
#include <stddef.h>
#include "../include/b200dsp.h"
#ifdef __cplusplus
extern "C" {
#endif

/* VP9DSPContext.intra_pred[tx][mode] at depth 8, 10, 12 (HOST pointers, stride in bytes, left / top as the reference takes them);
 * -1 for a depth, tx or mode outside the table */
int orc_vp9_intra_pred(int depth, int tx, int mode, uint8_t *dst, ptrdiff_t stride, const uint8_t *left, const uint8_t *top);
/* b200_vp9_intra_recon_frame_device (include/b200dsp.h) on HOST planes, coef read only.  order 0: the ops one after the other (the
 * entry's result); 1: no dependencies, every op reads the planes as they were before the call.  Returns the number of ops that wrote
 * samples, or -1 for invalid arguments. */
int64_t orc_vp9_intra_frame(int depth, int ss_h, int ss_v, int width, int height, uint8_t *const planes[3], ptrdiff_t ls_y, ptrdiff_t ls_uv,
                            int64_t nops, const B200Vp9IntraOp *ops, const void *coef, int order);

#ifdef __cplusplus
}
#endif
#endif
