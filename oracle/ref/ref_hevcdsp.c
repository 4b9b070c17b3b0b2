/* TEST INFRASTRUCTURE — the reference's HEVC DSP (libavcodec/hevc/dsp.c, compiled unmodified where it lies by oracle/ref/Makefile
 * into oracle/_ref/libffref_hevcdsp.so, next to libffref.so which it links against for emulated_edge_mc) exposed through a flat C
 * ABI: one table member per call, and the decoder's per-prediction-unit sequence (hevcdec.c:1722-2040: the emulated_edge_mc window
 * where the block's window leaves the picture, then the member calls) for a batch of B200HevcMcOp.  Plus the compile-time proof that
 * include/b200dsp.h's B200HEVCDSPContext can be copied member for member into HEVCDSPContext (same size, member offsets and
 * function-pointer types).  tests/hevcmclib.py loads it and reads the marker below. */
#include <stdint.h>
#include <stddef.h>
#include <string.h>

#include "config.h"
#include "libavcodec/hevc/dsp.h"
#include "../../include/b200dsp.h"

#define API __attribute__((visibility("default")))

#define SAME_OFF(A, B, m)  _Static_assert(offsetof(A, m) == offsetof(B, m), "offset of " #m " in " #A " / " #B)
#define SAME_TYPE(A, B, m) _Static_assert(__builtin_types_compatible_p(__typeof__(((A *)0)->m), __typeof__(((B *)0)->m)), "type of " #m " in " #A " / " #B)
#define SAME(A, B, m)      SAME_OFF(A, B, m); SAME_TYPE(A, B, m)

/* HEVCDSPContext, libavcodec/hevc/dsp.h:47-125 */
_Static_assert(sizeof(HEVCDSPContext) == sizeof(B200HEVCDSPContext), "size of HEVCDSPContext / B200HEVCDSPContext");
SAME(HEVCDSPContext, B200HEVCDSPContext, put_pcm);
SAME(HEVCDSPContext, B200HEVCDSPContext, add_residual);
SAME(HEVCDSPContext, B200HEVCDSPContext, dequant);
SAME(HEVCDSPContext, B200HEVCDSPContext, transform_rdpcm);
SAME(HEVCDSPContext, B200HEVCDSPContext, transform_4x4_luma);
SAME(HEVCDSPContext, B200HEVCDSPContext, idct);
SAME(HEVCDSPContext, B200HEVCDSPContext, idct_dc);
SAME(HEVCDSPContext, B200HEVCDSPContext, sao_band_filter);
SAME(HEVCDSPContext, B200HEVCDSPContext, sao_edge_filter);
SAME(HEVCDSPContext, B200HEVCDSPContext, sao_edge_restore);
SAME(HEVCDSPContext, B200HEVCDSPContext, put_hevc_qpel);
SAME(HEVCDSPContext, B200HEVCDSPContext, put_hevc_qpel_uni);
SAME(HEVCDSPContext, B200HEVCDSPContext, put_hevc_qpel_uni_w);
SAME(HEVCDSPContext, B200HEVCDSPContext, put_hevc_qpel_bi);
SAME(HEVCDSPContext, B200HEVCDSPContext, put_hevc_qpel_bi_w);
SAME(HEVCDSPContext, B200HEVCDSPContext, put_hevc_epel);
SAME(HEVCDSPContext, B200HEVCDSPContext, put_hevc_epel_uni);
SAME(HEVCDSPContext, B200HEVCDSPContext, put_hevc_epel_uni_w);
SAME(HEVCDSPContext, B200HEVCDSPContext, put_hevc_epel_bi);
SAME(HEVCDSPContext, B200HEVCDSPContext, put_hevc_epel_bi_w);
SAME(HEVCDSPContext, B200HEVCDSPContext, hevc_h_loop_filter_luma);
SAME(HEVCDSPContext, B200HEVCDSPContext, hevc_v_loop_filter_luma);
SAME(HEVCDSPContext, B200HEVCDSPContext, hevc_h_loop_filter_chroma);
SAME(HEVCDSPContext, B200HEVCDSPContext, hevc_v_loop_filter_chroma);
SAME(HEVCDSPContext, B200HEVCDSPContext, hevc_h_loop_filter_luma_c);
SAME(HEVCDSPContext, B200HEVCDSPContext, hevc_v_loop_filter_luma_c);
SAME(HEVCDSPContext, B200HEVCDSPContext, hevc_h_loop_filter_chroma_c);
SAME(HEVCDSPContext, B200HEVCDSPContext, hevc_v_loop_filter_chroma_c);
_Static_assert(MAX_PB_SIZE == 64, "MAX_PB_SIZE");

API const char ffref_hevcdsp_layout_check[] = "b200dsp.h B200HEVCDSPContext matches HEVCDSPContext";

/* libffref.so (oracle/ref/ref_shim.c): VideoDSPContext.emulated_edge_mc for 8-bit and for 16-bit samples */
void ffref_emulated_edge_mc(uint8_t *buf, const uint8_t *src, ptrdiff_t buf_linesize, ptrdiff_t src_linesize, int block_w, int block_h,
                            int src_x, int src_y, int w, int h);
void ffref_emulated_edge_mc_hbd(uint8_t *buf, const uint8_t *src, ptrdiff_t buf_linesize, ptrdiff_t src_linesize, int block_w, int block_h,
                                int src_x, int src_y, int w, int h);

static HEVCDSPContext *ref_hevcdsp(int depth)
{
    static HEVCDSPContext c[13];
    static int ok[13];
    if (depth != 8 && depth != 9 && depth != 10 && depth != 12) return NULL;
    if (!ok[depth]) { ff_hevc_dsp_init(&c[depth], depth); ok[depth] = 1; }
    return &c[depth];
}

/* hevcdec.c:62 */
static int pel_idx(int w)
{
    static const int8_t t[65] = { [2] = 0, [4] = 1, [6] = 2, [8] = 3, [12] = 4, [16] = 5, [24] = 6, [32] = 7, [48] = 8, [64] = 9 };
    return w >= 0 && w <= 64 ? t[w] : 0;
}

/* one member of ff_hevc_dsp_init(depth): form 0 put_hevc_?pel, 1 _uni, 2 _uni_w, 3 _bi, 4 _bi_w at [idx of width][vdir][hdir] */
API int ffref_hevc_mc(int depth, int epel, int form, int vdir, int hdir, void *dst, ptrdiff_t dststride, const void *src, ptrdiff_t srcstride,
                      const int16_t *src2, int height, int denom, int wx0, int wx1, int ox, int mx, int my, int width)
{
    HEVCDSPContext *c = ref_hevcdsp(depth);
    const int i = pel_idx(width), v = !!vdir, h = !!hdir;
    if (!c) return -1;
    switch (form) {
    case 0: (epel ? c->put_hevc_epel : c->put_hevc_qpel)[i][v][h](dst, src, srcstride, height, mx, my, width); return 0;
    case 1: (epel ? c->put_hevc_epel_uni : c->put_hevc_qpel_uni)[i][v][h](dst, dststride, src, srcstride, height, mx, my, width); return 0;
    case 2: (epel ? c->put_hevc_epel_uni_w : c->put_hevc_qpel_uni_w)[i][v][h](dst, dststride, src, srcstride, height, denom, wx0, ox, mx, my, width);
            return 0;
    case 3: (epel ? c->put_hevc_epel_bi : c->put_hevc_qpel_bi)[i][v][h](dst, dststride, src, srcstride, src2, height, mx, my, width); return 0;
    case 4: (epel ? c->put_hevc_epel_bi_w : c->put_hevc_qpel_bi_w)[i][v][h](dst, dststride, src, srcstride, src2, height, denom, wx0, wx1, ox,
                                                                            mx, my, width);
            return 0;
    }
    return -1;
}

/* one reference's source pointer as luma_mc_* / chroma_mc_* compute it: the picture itself where the block's filter window lies inside
 * (by the decoder's own test), else an emulated_edge_mc window in buf */
static const uint8_t *mc_src(int depth, int epel, const uint8_t *pic, ptrdiff_t stride, int x, int y, int w, int h, int pic_w, int pic_h,
                             uint8_t *buf, ptrdiff_t *srcstride)
{
    const int before = epel ? 1 : 3, after = epel ? 2 : 4, extra = epel ? 3 : 7, bps = depth > 8 ? 2 : 1;
    const ptrdiff_t emu_stride = 80 * bps;                                  /* EDGE_EMU_BUFFER_STRIDE << pixel_shift */
    const uint8_t *src = pic + (ptrdiff_t)y * stride + (ptrdiff_t)x * bps;
    *srcstride = stride;
    if (x < before || y < after || x >= pic_w - w - after || y >= pic_h - h - after) {
        const ptrdiff_t off = before * stride + before * bps;
        (bps == 2 ? ffref_emulated_edge_mc_hbd : ffref_emulated_edge_mc)(buf, src - off, emu_stride, stride, w + extra, h + extra, x - before,
                                                                         y - before, pic_w, pic_h);
        src = buf + before * emu_stride + before * bps;
        *srcstride = emu_stride;
    }
    return src;
}

/* the decoder's sequence for each op of a batch (the same op guard as the product); returns the number of ops that wrote their block */
API int64_t ffref_hevc_mc_batch(int depth, int epel, int64_t nops, const B200HevcMcOp *ops, uint8_t *dst, ptrdiff_t dst_stride,
                                const uint8_t *ref, ptrdiff_t ref_stride, int pic_w, int pic_h)
{
    static uint8_t buf[2][80 * 2 * (64 + 7)];
    static int16_t tmp[64 * 64];                                            /* lc->tmp */
    const int bps = depth > 8 ? 2 : 1, maxp = epel ? 7 : 3;
    int64_t done = 0;
    if (!ref_hevcdsp(depth)) return -1;
    for (int64_t i = 0; i < nops; i++) {
        const B200HevcMcOp *op = &ops[i];
        const int bi = op->kind == B200_HEVC_MC_BI || op->kind == B200_HEVC_MC_BI_W, nref = bi ? 2 : 1;
        int ok = op->kind <= 3 && op->w >= 1 && op->w <= 64 && op->h >= 1 && op->h <= 64 && op->denom <= 7 && !(op->dst_off % bps);
        for (int r = 0; r < nref; r++) ok = ok && op->mx[r] <= maxp && op->my[r] <= maxp && !(op->ref_off[r] % bps);
        if (!ok) continue;
        const uint8_t *src[2];
        ptrdiff_t ss[2];
        for (int r = 0; r < nref; r++)
            src[r] = mc_src(depth, epel, ref + op->ref_off[r], ref_stride, op->x[r], op->y[r], op->w, op->h, pic_w, pic_h, buf[r], &ss[r]);
        uint8_t *d = dst + op->dst_off;
        if (!bi) {
            ffref_hevc_mc(depth, epel, 1 + op->kind, op->my[0], op->mx[0], d, dst_stride, src[0], ss[0], NULL, op->h, op->denom, op->wx0, 0,
                          op->ox, op->mx[0], op->my[0], op->w);
        } else {
            ffref_hevc_mc(depth, epel, 0, op->my[0], op->mx[0], tmp, 0, src[0], ss[0], NULL, op->h, 0, 0, 0, 0, op->mx[0], op->my[0], op->w);
            ffref_hevc_mc(depth, epel, op->kind == B200_HEVC_MC_BI ? 3 : 4, op->my[1], op->mx[1], d, dst_stride, src[1], ss[1], tmp, op->h,
                          op->denom, op->wx0, op->wx1, op->ox, op->mx[1], op->my[1], op->w);
        }
        done++;
    }
    return done;
}
