/* TEST INFRASTRUCTURE — the reference's HEVC deblocking members (libavcodec/hevc/dsp.c, compiled unmodified where it lies by
 * oracle/ref/Makefile into oracle/_ref/libffref_hevcdbk.so) exposed through a flat C ABI, called through the HEVCDSPContext that
 * ff_hevc_dsp_init fills: one member per call, and a whole plane driven in the decoder's own order (hevc/filter.c:501-676, restated
 * in plane sample coordinates): CTBs in raster order; in each, per 8-row band, the band's vertical edges, then its horizontal edge
 * lagged 8 samples to the left (the last 8 columns of a CTB wait for the next CTB's first vertical edge).  tests/hevcdbklib.py loads it. */
#include <stdint.h>
#include <stddef.h>

#include "config.h"
#include "libavcodec/hevc/dsp.h"
#include "../../include/b200dsp.h"

#define API __attribute__((visibility("default")))

static HEVCDSPContext *ref_hevcdsp(int depth)
{
    static HEVCDSPContext c[13];
    static int ok[13];
    if (depth != 8 && depth != 9 && depth != 10 && depth != 12) return NULL;
    if (!ok[depth]) { ff_hevc_dsp_init(&c[depth], depth); ok[depth] = 1; }
    return &c[depth];
}

/* fn: 0 hevc_h_loop_filter_luma, 1 _v_luma, 2 _h_chroma, 3 _v_chroma, 4..7 the same four _c members */
API int ffref_hevc_dbk_member(int depth, int fn, uint8_t *pix, ptrdiff_t stride, int beta, const int32_t *tc, const uint8_t *no_p,
                              const uint8_t *no_q)
{
    HEVCDSPContext *h = ref_hevcdsp(depth);
    if (!h) return -1;
    switch (fn) {
    case 0: h->hevc_h_loop_filter_luma(pix, stride, beta, tc, no_p, no_q); return 0;
    case 1: h->hevc_v_loop_filter_luma(pix, stride, beta, tc, no_p, no_q); return 0;
    case 2: h->hevc_h_loop_filter_chroma(pix, stride, tc, no_p, no_q); return 0;
    case 3: h->hevc_v_loop_filter_chroma(pix, stride, tc, no_p, no_q); return 0;
    case 4: h->hevc_h_loop_filter_luma_c(pix, stride, beta, tc, no_p, no_q); return 0;
    case 5: h->hevc_v_loop_filter_luma_c(pix, stride, beta, tc, no_p, no_q); return 0;
    case 6: h->hevc_h_loop_filter_chroma_c(pix, stride, tc, no_p, no_q); return 0;
    case 7: h->hevc_v_loop_filter_chroma_c(pix, stride, tc, no_p, no_q); return 0;
    }
    return -1;
}

/* the member call for the 8-sample edge whose first segment is `a` and second `b` (b NULL past the plane: tc 0, as the decoder's
 * boundary strength is 0 there); two calls, one per segment, when the segments' beta differ (the member takes one beta) */
static void edge(HEVCDSPContext *h, int chroma, int horiz, uint8_t *pix, ptrdiff_t stride, const B200HevcDbkSeg *a, const B200HevcDbkSeg *b)
{
    const B200HevcDbkSeg zero = { 0, 0, 0, 0 };
    if (!b) b = &zero;
    const int split = !chroma && a->beta != b->beta && a->tc && b->tc;
    for (int k = 0; k < (split ? 2 : 1); k++) {
        const int32_t tc[2] = { split && k == 1 ? 0 : a->tc, split && k == 0 ? 0 : b->tc };
        const uint8_t no_p[2] = { !!(a->flags & B200_HEVC_DBK_NO_P), !!(b->flags & B200_HEVC_DBK_NO_P) };
        const uint8_t no_q[2] = { !!(a->flags & B200_HEVC_DBK_NO_Q), !!(b->flags & B200_HEVC_DBK_NO_Q) };
        const int beta = k == 1 || !a->tc ? b->beta : a->beta;
        if (chroma) (horiz ? h->hevc_h_loop_filter_chroma : h->hevc_v_loop_filter_chroma)(pix, stride, tc, no_p, no_q);
        else (horiz ? h->hevc_h_loop_filter_luma : h->hevc_v_loop_filter_luma)(pix, stride, beta, tc, no_p, no_q);
    }
}

/* the plane through the members in CTB order, CTBs of (1 << log2_w) x (1 << log2_h) plane samples (the luma CTB size shifted by the
 * chroma subsampling); the buffer must hold 4 more rows / columns past the plane where height / width is 4 (mod 8), which the
 * members read for the segment beyond the plane */
API int ffref_hevc_dbk_plane_ctb(int depth, int chroma, uint8_t *pix, ptrdiff_t stride, int width, int height, const B200HevcDbkSeg *vseg,
                                 int64_t vstride, const B200HevcDbkSeg *hseg, int64_t hstride, int log2_w, int log2_h)
{
    HEVCDSPContext *h = ref_hevcdsp(depth);
    const int bps = depth > 8 ? 2 : 1, cw = 1 << log2_w, ch = 1 << log2_h;
    if (!h || log2_w < 3 || log2_h < 3) return -1;
    for (int y0 = 0; y0 < height; y0 += ch)
        for (int x0 = 0; x0 < width; x0 += cw) {
            const int x_end = x0 + cw < width ? x0 + cw : width, y_end = y0 + ch < height ? y0 + ch : height;
            const int x_end2 = x_end == width ? x_end : x_end - 8;
            for (int y = y0; y < y_end; y += 8) {
                for (int x = x0 ? x0 : 8; x < x_end; x += 8)                                  /* filter.c:551, 615 */
                    edge(h, chroma, 0, pix + (ptrdiff_t)y * stride + x * bps, stride, &vseg[(int64_t)(y / 4) * vstride + x / 8],
                         y + 4 < height ? &vseg[(int64_t)(y / 4 + 1) * vstride + x / 8] : NULL);
                if (!y) continue;
                for (int x = x0 ? x0 - 8 : 0; x < x_end2; x += 8)                             /* filter.c:580, 649 */
                    edge(h, chroma, 1, pix + (ptrdiff_t)y * stride + x * bps, stride, &hseg[(int64_t)(y / 8) * hstride + x / 4],
                         x + 4 < width ? &hseg[(int64_t)(y / 8) * hstride + x / 4 + 1] : NULL);
            }
        }
    return 0;
}
