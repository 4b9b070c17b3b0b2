/* vc1dsp_oracle.h — TEST INFRASTRUCTURE ONLY.  Declarations of the VC-1 motion-compensation and inverse-transform checker
 * (vc1dsp_oracle.c, part of liboracle.so). */
#ifndef VC1DSP_ORACLE_H
#define VC1DSP_ORACLE_H
#include <stdint.h>
#include <stddef.h>
#include "../include/b200dsp.h"
#ifdef __cplusplus
extern "C" {
#endif

/* put_ (avg = 0) / avg_vc1_mspel_pixels_tab[size][dxy] (size 0: 16x16, 1: 8x8); -1 outside the table */
int orc_vc1_mspel(int avg, int size, int dxy, uint8_t *dst, const uint8_t *src, ptrdiff_t stride, int rnd);
/* put_ / avg_no_rnd_vc1_chroma_pixels_tab[idx] (0: 8 wide, 1: 4 wide); -1 outside the table or for x, y outside 0..7, h < 0 */
int orc_vc1_chroma(int avg, int idx, uint8_t *dst, const uint8_t *src, ptrdiff_t stride, int h, int x, int y);
/* vc1_inv_trans_<tt> (dc = 0) / vc1_inv_trans_<tt>_dc (dc = 1), tt a B200_VC1_TT_*; vc1_inv_trans_8x8 ignores dest; -1 for bad tt */
int orc_vc1_itx(int tt, int dc, uint8_t *dest, ptrdiff_t stride, int16_t *block);
/* b200_vc1_mc_frame_device / b200_vc1_residual_frame_device on host memory (refs' planes host addresses); return the number of ops that
 * wrote, or -1 where the entry refuses the call */
int64_t orc_vc1_mc_frame(int nrefs, const B200Vc1McRef *refs, uint8_t *const dst[3], ptrdiff_t ls_y, ptrdiff_t ls_uv, int mb_width,
                         int mb_height, int h_edge_pos, int v_edge_pos, int64_t nops, const B200Vc1McOp *ops);
int64_t orc_vc1_residual_frame(uint8_t *const dst[3], ptrdiff_t ls_y, ptrdiff_t ls_uv, int mb_width, int mb_height, const int16_t *coef,
                               int64_t nops, const B200Vc1ResidualOp *ops);

#ifdef __cplusplus
}
#endif
#endif
