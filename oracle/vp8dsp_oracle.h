/* vp8dsp_oracle.h — TEST INFRASTRUCTURE ONLY.  Declarations of the VP8 / VP7 motion-compensation and residual checker (vp8dsp_oracle.c,
 * part of liboracle.so). */
#ifndef VP8DSP_ORACLE_H
#define VP8DSP_ORACLE_H
#include <stdint.h>
#include <stddef.h>
#include "../include/b200dsp.h"
#ifdef __cplusplus
extern "C" {
#endif

/* put_vp8_epel_pixels_tab[size of w][v][h] (bilinear = 0) / put_vp8_bilinear_pixels_tab[size of w][v][h] (bilinear = 1); v, h 0..2;
 * -1 for a NULL table position or arguments outside the reference's contract (h 1..2w, filtered phases 1..7 epel / 0..7 bilinear) */
int orc_vp8_mc(int bilinear, int w, int v, int h_idx, uint8_t *dst, ptrdiff_t dst_stride, const uint8_t *src, ptrdiff_t src_stride, int h,
               int mx, int my);
/* subpel_filters[7][6] as the reference stores it (unsigned magnitudes) */
const uint8_t *orc_vp8_subpel_filters(void);
/* vp8_luma_dc_wht (dc_only = 0) / vp8_luma_dc_wht_dc (dc_only = 1) */
void orc_vp8_wht(int is_vp7, int dc_only, int16_t *block, int16_t *dc);
/* which 0 vp8_idct_add, 1 vp8_idct_dc_add, 2 vp8_idct_dc_add4y, 3 vp8_idct_dc_add4uv */
void orc_vp8_idct(int is_vp7, int which, uint8_t *dst, int16_t *block, ptrdiff_t stride);
/* b200_vp8_mc_frame_device / b200_vp8_residual_frame_device on host memory (refs' planes host addresses); return the number of ops that
 * wrote their block */
int64_t orc_vp8_mc_frame(int bilinear, int mb_width, int mb_height, int nrefs, const B200Vp8McRef *refs, int64_t nops, const B200Vp8McOp *ops,
                         uint8_t *const dst[3], ptrdiff_t ls_y, ptrdiff_t ls_uv);
int64_t orc_vp8_residual_frame(int is_vp7, int64_t nops, const B200Vp8ResidualOp *ops, const int16_t *coef, uint8_t *const dst[3],
                               ptrdiff_t ls_y, ptrdiff_t ls_uv);

#ifdef __cplusplus
}
#endif
#endif
