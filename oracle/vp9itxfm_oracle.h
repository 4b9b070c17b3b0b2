/* vp9itxfm_oracle.h — TEST INFRASTRUCTURE ONLY.  Declarations of the VP9 inverse-transform checker (vp9itxfm_oracle.c, part of
 * liboracle.so). */
#ifndef VP9ITXFM_ORACLE_H
#define VP9ITXFM_ORACLE_H
#include <stdint.h>
#include <stddef.h>
#include "../include/b200dsp.h"
#ifdef __cplusplus
extern "C" {
#endif

/* VP9DSPContext.itxfm_add[tx][type] at depth 8, 10, 12: block = sz * sz int16 (8 bit) / int32 (10 / 12 bit) coefficients, left as the
 * reference leaves them; stride in bytes; -1 for a depth, tx or type outside the table */
int orc_vp9_itxfm(int depth, int tx, int type, uint8_t *dst, ptrdiff_t stride, void *block, int eob);
/* b200_vp9_itxfm_add_batch_device (include/b200dsp.h) on host memory, coef read only; returns the number of ops that wrote their block */
int64_t orc_vp9_itxfm_batch(int depth, int64_t nops, const B200Vp9TxOp *ops, const void *coef, uint8_t *dst, ptrdiff_t dst_stride);

#ifdef __cplusplus
}
#endif
#endif
