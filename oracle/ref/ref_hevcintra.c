/* TEST INFRASTRUCTURE — the reference's HEVC intra reconstruction of a whole picture (built by oracle/ref/Makefile into
 * oracle/_ref/libffref_hevcintra.so; tests/hevcintralib.py loads it): all three components TU by TU in decode order, each TU through the
 * reference's own intra_pred[] (libavcodec/hevc/pred.c, compiled unmodified where it lies) over minimal decoder contexts, then its
 * residual through ffref_hevc_tu_batch (ref_hevcidct.c: the decoder's member sequence of hevc/cabac.c:1550-1592 and add_residual). */
#include <stdint.h>
#include <stddef.h>
#include <stdlib.h>
#include <string.h>

#include "config.h"
#include "libavcodec/hevc/hevcdec.h"
#include "libavcodec/hevc/pred.h"
#include "../../include/b200dsp.h"

#define API __attribute__((visibility("default")))

int64_t ffref_hevc_tu_batch(int depth, int64_t nops, const B200HevcTuOp *ops, const int16_t *coef, uint8_t *dst, ptrdiff_t dst_stride);

/* One TU as the decoder calls intra_pred for it: luma position of the call, log2 size of the block, component, mode, the five
 * na.cand_* values; then the residual (kind B200_HEVC_TU_NONE: none) */
typedef struct RefReconTu {
    int32_t x0, y0, log2_size, c_idx, mode, na;
    int64_t coef_off;
    int32_t kind, flags, col_limit, pad;
} RefReconTu;

API int ffref_hevc_intra_picture(int depth, int chroma_format_idc, int W, int H, int log2_ctb, int log2_min_tb, int log2_min_pu,
                                 uint8_t *const planes[3], int ls_y, int ls_uv, int ntu, const RefReconTu *tus, const int16_t *coef,
                                 const uint8_t *intra_map, int smoothing_disabled, int strong_enabled)
{
    static HEVCPredContext hpcs[13];
    static int ok[13];
    if (depth != 8 && depth != 9 && depth != 10 && depth != 12) return -1;
    if (!ok[depth]) { ff_hevc_pred_init(&hpcs[depth], depth); ok[depth] = 1; }
    HEVCPredContext *hpc = &hpcs[depth];
    HEVCSPS *sps = calloc(1, sizeof(*sps));
    HEVCPPS *pps = calloc(1, sizeof(*pps));
    HEVCContext *s = calloc(1, sizeof(*s));
    HEVCLocalContext *lc = calloc(1, sizeof(*lc));
    HEVCFrame *frame = calloc(1, sizeof(*frame));
    AVFrame *f = calloc(1, sizeof(*f));
    const int mpw = W >> log2_min_pu, mph = H >> log2_min_pu;

    sps->width = W; sps->height = H;
    sps->log2_ctb_size = log2_ctb; sps->log2_min_tb_size = log2_min_tb; sps->log2_min_pu_size = log2_min_pu;
    sps->min_pu_width = mpw; sps->min_pu_height = mph;
    sps->tb_mask = (1 << (log2_ctb - log2_min_tb)) - 1;
    sps->chroma_format_idc = chroma_format_idc;
    sps->hshift[1] = sps->hshift[2] = chroma_format_idc == 1 || chroma_format_idc == 2;
    sps->vshift[1] = sps->vshift[2] = chroma_format_idc == 1;
    sps->bit_depth = depth; sps->pixel_shift = depth > 8;
    sps->intra_smoothing_disabled = !!smoothing_disabled;
    sps->strong_intra_smoothing_enabled = !!strong_enabled;

    /* min_tb_addr_zs as hevc/ps.c builds it: the z-scan address inside a CTB, -1 in the row and column before it */
    const int tw = sps->tb_mask + 2, log2_diff = log2_ctb - log2_min_tb;
    int *zs_tab = malloc(sizeof(int) * tw * tw);
    for (int i = 0; i < tw; i++) zs_tab[i] = zs_tab[i * tw] = -1;
    pps->min_tb_addr_zs = zs_tab + tw + 1;
    for (int y = 0; y < tw - 1; y++)
        for (int x = 0; x < tw - 1; x++) {
            int v = 0;
            for (int i = 0; i < log2_diff; i++) {
                const int m = 1 << i;
                v += (m & x ? m * m : 0) + (m & y ? 2 * m * m : 0);
            }
            pps->min_tb_addr_zs[y * tw + x] = v;
        }
    pps->sps = sps;
    pps->constrained_intra_pred_flag = intra_map != NULL;

    MvField *mvf = calloc((size_t)(mph + 2) * mpw + 2, sizeof(MvField));
    for (size_t i = 0; i < (size_t)(mph + 2) * mpw + 2; i++) mvf[i].pred_flag = PF_L0;
    if (intra_map)
        for (int i = 0; i < mpw * mph; i++) mvf[1 + mpw + i].pred_flag = intra_map[i] ? PF_INTRA : PF_L0;
    frame->tab_mvf = mvf + 1 + mpw;
    for (int c = 0; c < 3; c++) { f->data[c] = planes[c]; f->linesize[c] = c ? ls_uv : ls_y; }
    frame->f = f;
    s->cur_frame = frame;
    s->hpc = *hpc;
    lc->parent = s;

    for (int k = 0; k < ntu; k++) {
        const RefReconTu *t = &tus[k];
        const int c = t->c_idx, hs = c ? sps->hshift[1] : 0, vs = c ? sps->vshift[1] : 0, ls = c ? ls_uv : ls_y;
        lc->na.cand_bottom_left = t->na & 1;
        lc->na.cand_left = !!(t->na & 2);
        lc->na.cand_up_left = !!(t->na & 4);
        lc->na.cand_up = !!(t->na & 8);
        lc->na.cand_up_right = !!(t->na & 16);
        lc->tu.intra_pred_mode = lc->tu.intra_pred_mode_c = t->mode;
        hpc->intra_pred[t->log2_size - 2](lc, pps, t->x0, t->y0, c);
        if (t->kind == B200_HEVC_TU_NONE) continue;
        B200HevcTuOp op;
        memset(&op, 0, sizeof(op));
        op.dst_off = (int64_t)(t->y0 >> vs) * ls + (int64_t)((t->x0 >> hs) << sps->pixel_shift);
        op.coef_off = t->coef_off; op.log2_size = t->log2_size; op.kind = t->kind; op.flags = t->flags; op.col_limit = t->col_limit;
        ffref_hevc_tu_batch(depth, 1, &op, coef, planes[c], ls);
    }
    free(mvf); free(zs_tab);
    free(f); free(frame); free(lc); free(s); free(pps); free(sps);
    return 0;
}
