/* CHECKER — HEVC intra reconstruction of a whole picture (b200_hevc_intra_recon_picture_device), restated op by op in decode order:
 * each op's intra_pred through the prediction checker (orc_hevc_intra_plane, one op at a time), then its residual through the
 * residual checker's per-op sequence (orc_hevc_tu_batch, one op).  order 1 ("no dependencies") gives every op the planes as they were
 * before the call, so that a test can show a picture whose result depends on the decode order. */
#include <stdint.h>
#include <stddef.h>
#include <stdlib.h>
#include <string.h>

#include "../include/b200dsp.h"

#define API __attribute__((visibility("default")))

int orc_hevc_intra_plane(int depth, uint8_t *pix, ptrdiff_t stride, int width, int height, int hshift, int vshift, int64_t nops,
                         const B200HevcIntraOp *ops, const uint8_t *map, ptrdiff_t map_stride, int log2_min_pu);
int64_t orc_hevc_tu_batch(int depth, int64_t nops, const B200HevcTuOp *ops, const int16_t *coef, uint8_t *dst, ptrdiff_t dst_stride);

/* the entry's op guard: what the batch entries refuse, the plane index and 4-aligned positions */
static int op_ok(const B200HevcIntraReconOp *op, int np, int pw, int ph)
{
    const int f = op->flags, size = 1 << (op->log2_size & 7);
    if (op->plane >= np || (op->x & 3) || (op->y & 3) || op->log2_size < 2 || op->log2_size > 5 || op->mode > 34) return 0;
    if (op->x < 0 || op->y < 0 || op->x > pw - size || op->y > ph - size) return 0;
    if (op->x < 1 && (f & (B200_HEVC_INTRA_CAND_BL | B200_HEVC_INTRA_CAND_L | B200_HEVC_INTRA_CAND_UL))) return 0;
    if (op->y < 1 && (f & (B200_HEVC_INTRA_CAND_UL | B200_HEVC_INTRA_CAND_U | B200_HEVC_INTRA_CAND_UR))) return 0;
    if (op->tu_kind == B200_HEVC_TU_NONE) return 1;
    return op->tu_kind <= B200_HEVC_TU_BYPASS && (op->tu_kind != B200_HEVC_TU_DST4 || op->log2_size == 2) && op->coef_off >= 0 &&
           !(op->coef_off & 7);
}

static void one(int depth, uint8_t *pix, ptrdiff_t ls, int W, int H, int hs, int vs, const B200HevcIntraReconOp *op, const int16_t *coef,
                const uint8_t *map, ptrdiff_t map_stride, int log2_min_pu)
{
    B200HevcIntraOp p;
    memset(&p, 0, sizeof(p));
    p.x = op->x; p.y = op->y; p.log2_size = op->log2_size; p.mode = op->mode; p.flags = op->flags;
    orc_hevc_intra_plane(depth, pix, ls, W, H, hs, vs, 1, &p, map, map_stride, log2_min_pu);
    if (op->tu_kind == B200_HEVC_TU_NONE) return;
    B200HevcTuOp t;
    memset(&t, 0, sizeof(t));
    t.dst_off = (int64_t)op->y * ls + (int64_t)op->x * (depth > 8 ? 2 : 1);
    t.coef_off = op->coef_off; t.log2_size = op->log2_size; t.kind = op->tu_kind; t.flags = op->tu_flags; t.col_limit = op->col_limit;
    orc_hevc_tu_batch(depth, 1, &t, coef, pix, ls);
}

/* planes / line sizes as the entry takes them; order 0: decode order, 1: every op reads the planes as they were before the call */
API int orc_hevc_intra_picture(int depth, int chroma_format_idc, int W, int H, uint8_t *const planes[3], ptrdiff_t ls_y, ptrdiff_t ls_uv,
                               int64_t nops, const B200HevcIntraReconOp *ops, const int16_t *coef, const uint8_t *map, ptrdiff_t map_stride,
                               int log2_min_pu, int order)
{
    const int np = chroma_format_idc ? 3 : 1, bps = depth > 8 ? 2 : 1;
    const int chs = chroma_format_idc == 1 || chroma_format_idc == 2, cvs = chroma_format_idc == 1;
    uint8_t *work[3] = { NULL, NULL, NULL };
    if (order) {                                                     /* copies of the planes as they are before the call */
        for (int p = 0; p < np; p++) {
            const ptrdiff_t ls = p ? ls_uv : ls_y;
            const int ph = p ? H >> cvs : H;
            work[p] = malloc((size_t)ls * ph);
            memcpy(work[p], planes[p], (size_t)ls * ph);
        }
    }
    uint8_t blk[32 * 32 * 2];
    for (int64_t k = 0; k < nops; k++) {
        const B200HevcIntraReconOp *op = &ops[k];
        const int p = op->plane < 3 ? op->plane : 0;
        const int hs = p ? chs : 0, vs = p ? cvs : 0;
        const ptrdiff_t ls = p ? ls_uv : ls_y;
        if (!op_ok(op, np, W >> hs, H >> vs)) continue;
        if (!order) {
            one(depth, planes[p], ls, W, H, hs, vs, op, coef, map, map_stride, log2_min_pu);
            continue;
        }
        const int n = 1 << op->log2_size;                            /* on the copy, then the block moved over and the copy restored */
        const size_t row = (size_t)n * bps, o = (size_t)op->y * ls + (size_t)op->x * bps;
        for (int y = 0; y < n; y++) memcpy(blk + y * row, work[p] + o + y * ls, row);
        one(depth, work[p], ls, W, H, hs, vs, op, coef, map, map_stride, log2_min_pu);
        for (int y = 0; y < n; y++) {
            memcpy(planes[p] + o + y * ls, work[p] + o + y * ls, row);
            memcpy(work[p] + o + y * ls, blk + y * row, row);
        }
    }
    for (int p = 0; p < 3; p++) free(work[p]);
    return 0;
}
