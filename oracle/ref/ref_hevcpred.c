/* TEST INFRASTRUCTURE — the reference's HEVC intra prediction exposed through a flat C ABI (built by oracle/ref/hevcpred.mk into
 * oracle/_ref/libffref_hevcpred.so; tests/hevcpredlib.py loads it):
 *  - the members of HEVCPredContext (libavcodec/hevc/pred.c, compiled unmodified where it lies), called through the context
 *    ff_hevc_pred_init fills;
 *  - whole planes through the reference's own intra_pred[]: TU by TU in decode order over minimal HEVCContext / HEVCFrame / AVFrame /
 *    HEVCLocalContext / HEVCSPS / HEVCPPS (na, tu.intra_pred_mode / _c, min_tb_addr_zs, tab_mvf[].pred_flag, the shifts, sizes and
 *    smoothing flags), each TU followed by a residual added through the reference's add_residual (libavcodec/hevc/dsp.c).
 * Plus the compile-time proof that B200HEVCPredContext (include/b200dsp.h) has HEVCPredContext's layout. */
#include <stdint.h>
#include <stddef.h>
#include <stdlib.h>
#include <string.h>

#include "config.h"
#include "libavcodec/hevc/hevcdec.h"
#include "libavcodec/hevc/dsp.h"
#include "libavcodec/hevc/pred.h"
#include "../../include/b200dsp.h"

#define API __attribute__((visibility("default")))

#define SAME_OFF(A, B, m)  _Static_assert(offsetof(A, m) == offsetof(B, m), "offset of " #m " in " #A " / " #B)
#define SAME_SIZE(A, B, m) _Static_assert(sizeof(((A *)0)->m) == sizeof(((B *)0)->m), "size of " #m " in " #A " / " #B)
#define SAME(A, B, m)      SAME_OFF(A, B, m); SAME_SIZE(A, B, m)

_Static_assert(sizeof(HEVCPredContext) == sizeof(B200HEVCPredContext), "size of HEVCPredContext / B200HEVCPredContext");
SAME(HEVCPredContext, B200HEVCPredContext, intra_pred);
SAME(HEVCPredContext, B200HEVCPredContext, pred_planar);
SAME(HEVCPredContext, B200HEVCPredContext, pred_dc);
SAME(HEVCPredContext, B200HEVCPredContext, pred_angular);
SAME(HEVCPredContext, B200HEVCPredContext, ref_filter_3tap);
SAME(HEVCPredContext, B200HEVCPredContext, ref_filter_strong);
API const char ffref_hevcpred_layout_check[] = "B200HEVCPredContext == HEVCPredContext";

static HEVCPredContext *ref_hpc(int depth)
{
    static HEVCPredContext c[13];
    static int ok[13];
    if (depth != 8 && depth != 9 && depth != 10 && depth != 12) return NULL;
    if (!ok[depth]) { ff_hevc_pred_init(&c[depth], depth); ok[depth] = 1; }
    return &c[depth];
}

static HEVCDSPContext *ref_dsp(int depth)
{
    static HEVCDSPContext c[13];
    static int ok[13];
    if (!ok[depth]) { ff_hevc_dsp_init(&c[depth], depth); ok[depth] = 1; }
    return &c[depth];
}

/* which: 0 planar, 1 DC, 2 angular */
API int ffref_hevc_pred(int depth, int which, int log2_size, uint8_t *dst, const uint8_t *top, const uint8_t *left, ptrdiff_t stride,
                        int c_idx, int mode)
{
    HEVCPredContext *c = ref_hpc(depth);
    if (!c || log2_size < 2 || log2_size > 5) return -1;
    if (which == 0) c->pred_planar[log2_size - 2](dst, top, left, stride);
    else if (which == 1) c->pred_dc(dst, top, left, stride, log2_size, c_idx);
    else c->pred_angular[log2_size - 2](dst, top, left, stride, c_idx, mode);
    return 0;
}

API int ffref_hevc_filter_3tap(int depth, int idx, uint8_t *fl, uint8_t *ft, const uint8_t *left, const uint8_t *top, int size)
{
    HEVCPredContext *c = ref_hpc(depth);
    if (!c || idx < 0 || idx > 2) return -1;
    c->ref_filter_3tap[idx](fl, ft, left, top, size);
    return 0;
}

API int ffref_hevc_filter_strong(int depth, uint8_t *ft, uint8_t *left, const uint8_t *top)
{
    HEVCPredContext *c = ref_hpc(depth);
    if (!c) return -1;
    c->ref_filter_strong(ft, left, top);
    return 0;
}

/* One TU as the caller records it: luma position, log2 size of the block predicted, component, mode, the five na.cand_* values */
typedef struct RefTu { int32_t x0, y0, log2_size, c_idx, mode, na; } RefTu;

/* One component plane predicted and reconstructed TU by TU in decode order.  plane / linesize: the component's samples (edited in
 * place); W x H the luma picture; log2_ctb / log2_min_tb / log2_min_pu the SPS sizes; intra_map: NULL or one byte per luma min PU
 * (non-zero = PF_INTRA), which also switches constrained_intra_pred_flag on.  tab_mvf gets one guard row above and below the picture
 * whose entries are inter: for a block on the top row intra_pred reads the row above the picture (see INTEGRATION.md).  res: per TU
 * its (1 << log2_size)^2 int16 residual, added by add_residual after the prediction. */
API int ffref_hevc_intra_plane(int depth, int chroma_format_idc, int W, int H, int log2_ctb, int log2_min_tb, int log2_min_pu,
                               uint8_t *plane, int linesize, int c_idx, int ntu, const RefTu *tus, const int16_t *res,
                               const uint8_t *intra_map, int smoothing_disabled, int strong_enabled)
{
    HEVCPredContext *hpc = ref_hpc(depth);
    if (!hpc) return -1;
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
    f->data[c_idx] = plane; f->linesize[c_idx] = linesize;
    frame->f = f;
    s->cur_frame = frame;
    s->hpc = *hpc;
    lc->parent = s;

    HEVCDSPContext *dsp = ref_dsp(depth);
    const int hs = sps->hshift[c_idx], vs = sps->vshift[c_idx];
    for (int k = 0; k < ntu; k++) {
        const RefTu *t = &tus[k];
        lc->na.cand_bottom_left = t->na & 1;
        lc->na.cand_left = !!(t->na & 2);
        lc->na.cand_up_left = !!(t->na & 4);
        lc->na.cand_up = !!(t->na & 8);
        lc->na.cand_up_right = !!(t->na & 16);
        lc->tu.intra_pred_mode = lc->tu.intra_pred_mode_c = t->mode;
        hpc->intra_pred[t->log2_size - 2](lc, pps, t->x0, t->y0, c_idx);
        uint8_t *dst = plane + (ptrdiff_t)(t->y0 >> vs) * linesize + ((t->x0 >> hs) << sps->pixel_shift);
        dsp->add_residual[t->log2_size - 2](dst, (int16_t *)res, linesize);
        res += 1 << (2 * t->log2_size);
    }
    free(mvf); free(zs_tab);
    free(f); free(frame); free(lc); free(s); free(pps); free(sps);
    return 0;
}
