/* TEST INFRASTRUCTURE — the reference's HEVC sample adaptive offset exposed through a flat C ABI (built by oracle/ref/hevcsao.mk into
 * oracle/_ref/libffref_hevcsao.so; tests/hevcsaolib.py loads it):
 *  - the SAO members of HEVCDSPContext (libavcodec/hevc/dsp.c, compiled unmodified where it lies), called through the context
 *    ff_hevc_dsp_init fills, one call at a time or, for sao_edge_restore, swept over every class, border and edge-flag combination
 *    with the results folded into one digest;
 *  - whole pictures through the decoder's own loop filter (libavcodec/hevc/filter.c, compiled unmodified where it lies):
 *    ff_hevc_hls_filters / ff_hevc_hls_filter driven CTB by CTB in tile-scan order over minimal HEVCContext / HEVCLayerContext /
 *    HEVCSPS / HEVCPPS, every boundary strength zero (so deblocking_filter_CTB changes nothing), with the per-CTB SAOParams, slice
 *    addresses, filter_slice_edges, tile maps and is_pcm the caller describes.  The saved-sample buffers, the SAO_APPLIED
 *    bookkeeping, the unfilterable-edge flags and restore_tqb_pixels are then the decoder's.
 * Plus the compile-time proof that B200SAOParams (include/b200dsp.h) has SAOParams' layout.  The three symbols filter.c links
 * against outside what is compiled here are stubbed below; none of them is reached with the settings used. */
#include <stdint.h>
#include <stddef.h>
#include <stdlib.h>
#include <string.h>

#include "config.h"
#include "libavcodec/hevc/hevcdec.h"
#include "libavcodec/hevc/dsp.h"
#include "../../include/b200dsp.h"

#define API __attribute__((visibility("default")))

#define SAME_OFF(A, B, m)  _Static_assert(offsetof(A, m) == offsetof(B, m), "offset of " #m " in " #A " / " #B)
#define SAME_SIZE(A, B, m) _Static_assert(sizeof(((A *)0)->m) == sizeof(((B *)0)->m), "size of " #m " in " #A " / " #B)
#define SAME(A, B, m)      SAME_OFF(A, B, m); SAME_SIZE(A, B, m)

/* SAOParams, libavcodec/hevc/dsp.h:34-45 */
_Static_assert(sizeof(SAOParams) == sizeof(B200SAOParams), "size of SAOParams / B200SAOParams");
SAME(SAOParams, B200SAOParams, offset_abs);
SAME(SAOParams, B200SAOParams, offset_sign);
SAME(SAOParams, B200SAOParams, band_position);
SAME(SAOParams, B200SAOParams, eo_class);
SAME(SAOParams, B200SAOParams, offset_val);
SAME(SAOParams, B200SAOParams, type_idx);

/* stubs for the symbols filter.c references: ff_hevc_get_ref_list is only called from ff_hevc_deblocking_boundary_strengths and
 * ff_progress_frame_report only with frame threading, neither of which runs here */
const RefPicList *ff_hevc_get_ref_list(const HEVCFrame *frame, int x0, int y0) { abort(); }
void ff_progress_frame_report(ProgressFrame *f, int progress) { abort(); }

static HEVCDSPContext *ref_hevcdsp(int depth)
{
    static HEVCDSPContext c[13];
    static int ok[13];
    if (depth != 8 && depth != 9 && depth != 10 && depth != 12) return NULL;
    if (!ok[depth]) { ff_hevc_dsp_init(&c[depth], depth); ok[depth] = 1; }
    return &c[depth];
}

API int ffref_hevc_sao_band(int depth, int idx, uint8_t *dst, const uint8_t *src, ptrdiff_t stride_dst, ptrdiff_t stride_src,
                            const int16_t *off, int left_class, int w, int h)
{
    HEVCDSPContext *c = ref_hevcdsp(depth);
    if (!c || idx < 0 || idx > 4) return -1;
    c->sao_band_filter[idx](dst, src, stride_dst, stride_src, off, left_class, w, h);
    return 0;
}

/* src at the members' implicit stride of 192 bytes */
API int ffref_hevc_sao_edge(int depth, int idx, uint8_t *dst, const uint8_t *src, ptrdiff_t stride_dst, const int16_t *off, int eo, int w, int h)
{
    HEVCDSPContext *c = ref_hevcdsp(depth);
    if (!c || idx < 0 || idx > 4) return -1;
    c->sao_edge_filter[idx](dst, src, stride_dst, off, eo, w, h);
    return 0;
}

typedef void (*restore_fn)(uint8_t *, const uint8_t *, ptrdiff_t, ptrdiff_t, const SAOParams *, const int *, int, int, int,
                           const uint8_t *, const uint8_t *, const uint8_t *);

API int ffref_hevc_sao_restore(int depth, int which, uint8_t *dst, const uint8_t *src, ptrdiff_t stride_dst, ptrdiff_t stride_src,
                               const void *sao, const int *borders, int w, int h, int c_idx, const uint8_t *vert_edge,
                               const uint8_t *horiz_edge, const uint8_t *diag_edge)
{
    HEVCDSPContext *c = ref_hevcdsp(depth);
    if (!c || which < 0 || which > 1) return -1;
    c->sao_edge_restore[which](dst, src, stride_dst, stride_src, (const SAOParams *)sao, borders, w, h, c_idx, vert_edge, horiz_edge,
                               diag_edge);
    return 0;
}

/* the reference member's address, for the checker's sweep (orc_hevc_sao_restore_sweep), which runs the same loop over it */
API void *ffref_hevc_sao_restore_fn(int depth, int which)
{
    HEVCDSPContext *c = ref_hevcdsp(depth);
    return c && (which == 0 || which == 1) ? (void *)c->sao_edge_restore[which] : NULL;
}

/* One picture through the decoder's loop filter.  planes[c] / linesize[c]: the deblocked component planes, filtered in place
 * (luma W x H, chroma (W >> hshift) x (H >> vshift) for chroma_format_idc 1 / 2 / 3; 0 = luma only).  Per CTB in raster order:
 * sao[] (type_idx, band_position, eo_class, offset_val are read), slice_addr[], lf_across_slices[].  Tiles: ncols / nrows tiles with
 * boundaries col_bd[0..ncols] / row_bd[0..nrows] in CTBs (tiles_enabled when either is above 1).  is_pcm: one byte per luma min PU,
 * (W >> log2_min_pu) per row, read by restore_tqb_pixels when pcm_or_bypass (pcm_enabled and pcm_loop_filter_disabled set). */
API int ffref_hevc_sao_picture(int depth, int chroma_format_idc, int W, int H, int log2_ctb, uint8_t **planes, const int *linesize,
                               const void *sao_in, const int32_t *slice_addr, const uint8_t *lf_across_slices, int ncols, const int *col_bd,
                               int nrows, const int *row_bd, int lf_across_tiles, const uint8_t *is_pcm, int log2_min_pu, int pcm_or_bypass)
{
    HEVCDSPContext *dsp = ref_hevcdsp(depth);
    if (!dsp || log2_ctb < 4 || log2_ctb > 6 || chroma_format_idc < 0 || chroma_format_idc > 3) return -1;
    HEVCSPS *sps = calloc(1, sizeof(*sps));
    HEVCPPS *pps = calloc(1, sizeof(*pps));
    HEVCLayerContext *l = calloc(1, sizeof(*l));
    HEVCContext *s = calloc(1, sizeof(*s));
    HEVCLocalContext *lc = calloc(1, sizeof(*lc));
    AVCodecContext *avctx = calloc(1, sizeof(*avctx));
    HEVCFrame *frame = calloc(1, sizeof(*frame));
    AVFrame *f = calloc(1, sizeof(*f));
    const int ctb = 1 << log2_ctb, cw = (W + ctb - 1) >> log2_ctb, ch = (H + ctb - 1) >> log2_ctb, n = cw * ch;
    const int ncomp = chroma_format_idc ? 3 : 1;

    sps->width = W; sps->height = H;
    sps->log2_ctb_size = log2_ctb; sps->ctb_width = cw; sps->ctb_height = ch; sps->ctb_size = n;
    sps->log2_min_pu_size = log2_min_pu; sps->min_pu_width = W >> log2_min_pu; sps->min_pu_height = H >> log2_min_pu;
    sps->chroma_format_idc = chroma_format_idc;
    sps->hshift[1] = sps->hshift[2] = chroma_format_idc == 1 || chroma_format_idc == 2;
    sps->vshift[1] = sps->vshift[2] = chroma_format_idc == 1;
    sps->bit_depth = depth; sps->pixel_shift = depth > 8;
    sps->sao_enabled = 1;
    sps->pcm_enabled = sps->pcm_loop_filter_disabled = !!pcm_or_bypass;

    pps->sps = sps;
    pps->tiles_enabled_flag = ncols > 1 || nrows > 1;
    pps->loop_filter_across_tiles_enabled_flag = !!lf_across_tiles;
    pps->ctb_addr_rs_to_ts = calloc(n, sizeof(int));
    pps->ctb_addr_ts_to_rs = calloc(n, sizeof(int));
    pps->tile_id = calloc(n, sizeof(int));
    int ts = 0;
    for (int tr = 0; tr < nrows; tr++)                       /* tile scan: tiles in raster order, CTBs in raster order inside */
        for (int tc = 0; tc < ncols; tc++)
            for (int y = row_bd[tr]; y < row_bd[tr + 1]; y++)
                for (int x = col_bd[tc]; x < col_bd[tc + 1]; x++) {
                    pps->ctb_addr_rs_to_ts[y * cw + x] = ts;
                    pps->ctb_addr_ts_to_rs[ts] = y * cw + x;
                    pps->tile_id[ts] = tr * ncols + tc;
                    ts++;
                }

    l->sao = calloc(n, sizeof(SAOParams));
    memcpy(l->sao, sao_in, n * sizeof(SAOParams));
    l->deblock = calloc(n, sizeof(DBParams));
    l->filter_slice_edges = calloc(n, 1);
    memcpy(l->filter_slice_edges, lf_across_slices, n);
    l->tab_slice_address = calloc(n, sizeof(int32_t));
    memcpy(l->tab_slice_address, slice_addr, n * sizeof(int32_t));
    l->is_pcm = calloc((size_t)(sps->min_pu_width + 1) * (sps->min_pu_height + 1), 1);
    memcpy(l->is_pcm, is_pcm, (size_t)sps->min_pu_width * sps->min_pu_height);
    l->bs_width = (W >> 2) + 1; l->bs_height = (H >> 2) + 1;
    l->horizontal_bs = calloc(l->bs_width, l->bs_height);   /* bs 0 everywhere: deblocking_filter_CTB makes no member call */
    l->vertical_bs = calloc(l->bs_width, l->bs_height);
    for (int c = 0; c < ncomp; c++) {
        const int w = W >> sps->hshift[c], h = H >> sps->vshift[c];
        l->sao_pixel_buffer_h[c] = calloc((size_t)(w * 2 * ch) << sps->pixel_shift, 1);
        l->sao_pixel_buffer_v[c] = calloc((size_t)(h * 2 * cw) << sps->pixel_shift, 1);
    }

    for (int c = 0; c < ncomp; c++) { f->data[c] = planes[c]; f->linesize[c] = linesize[c]; }
    frame->f = f;
    s->avctx = avctx;                                        /* skip_loop_filter AVDISCARD_DEFAULT, no frame threading */
    s->cur_frame = frame;
    s->hevcdsp = *dsp;
    lc->parent = s;

    int x = 0, y = 0;
    for (ts = 0; ts < n; ts++) {                             /* hls_decode_entry's calls, hevc/hevcdec.c:2771-2805 */
        const int rs = pps->ctb_addr_ts_to_rs[ts];
        x = (rs % cw) << log2_ctb;
        y = (rs / cw) << log2_ctb;
        ff_hevc_hls_filters(lc, l, pps, x, y, ctb);
    }
    if (x + ctb >= W && y + ctb >= H)
        ff_hevc_hls_filter(lc, l, pps, x, y, ctb);

    for (int c = 0; c < ncomp; c++) { free(l->sao_pixel_buffer_h[c]); free(l->sao_pixel_buffer_v[c]); }
    free(l->horizontal_bs); free(l->vertical_bs); free(l->is_pcm); free(l->tab_slice_address); free(l->filter_slice_edges);
    free(l->deblock); free(l->sao);
    free(pps->ctb_addr_rs_to_ts); free(pps->ctb_addr_ts_to_rs); free(pps->tile_id);
    free(f); free(frame); free(avctx); free(lc); free(s); free(l); free(pps); free(sps);
    return 0;
}
