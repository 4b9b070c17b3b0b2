/* TEST INFRASTRUCTURE — the reference's VP9 DSP (libavcodec/vp9dsp.c, vp9dsp_8bpp.c, vp9dsp_10bpp.c, vp9dsp_12bpp.c, compiled
 * unmodified where they lie by oracle/ref/vp9dsp.mk into oracle/_ref/libffref_vp9dsp.so, next to libffref.so which it links against
 * for emulated_edge_mc) exposed through a flat C ABI: one mc / smc table member per call, the address of ff_vp9_subpel_filters, and
 * the decoder's per-block sequence (vp9recon.c:299-551: the emulated_edge_mc window where the decoder's own test says the block's
 * window leaves the picture, then the member call; vp9_mc_template.c: put from the first reference, avg from the second) for a batch
 * of B200Vp9McOp.  Plus the compile-time proof that include/b200dsp.h's B200VP9DSPContext can be copied member for member into
 * VP9DSPContext (same size, member offsets and function-pointer types).  tests/vp9mclib.py loads it and reads the marker below. */
#include <stdint.h>
#include <stddef.h>
#include <string.h>

#include "config.h"
#include "libavcodec/vp9dsp.h"
#include "../../include/b200dsp.h"

#define API __attribute__((visibility("default")))

#define SAME_OFF(A, B, m)  _Static_assert(offsetof(A, m) == offsetof(B, m), "offset of " #m " in " #A " / " #B)
#define SAME_TYPE(A, B, m) _Static_assert(__builtin_types_compatible_p(__typeof__(((A *)0)->m), __typeof__(((B *)0)->m)), "type of " #m " in " #A " / " #B)
#define SAME(A, B, m)      SAME_OFF(A, B, m); SAME_TYPE(A, B, m)

/* VP9DSPContext, libavcodec/vp9dsp.h:40-122 */
_Static_assert(sizeof(VP9DSPContext) == sizeof(B200VP9DSPContext), "size of VP9DSPContext / B200VP9DSPContext");
SAME(VP9DSPContext, B200VP9DSPContext, intra_pred);
SAME(VP9DSPContext, B200VP9DSPContext, itxfm_add);
SAME(VP9DSPContext, B200VP9DSPContext, loop_filter_8);
SAME(VP9DSPContext, B200VP9DSPContext, loop_filter_16);
SAME(VP9DSPContext, B200VP9DSPContext, loop_filter_mix2);
SAME(VP9DSPContext, B200VP9DSPContext, mc);
SAME(VP9DSPContext, B200VP9DSPContext, smc);
_Static_assert(FILTER_8TAP_SMOOTH == 0 && FILTER_8TAP_REGULAR == 1 && FILTER_8TAP_SHARP == 2 && FILTER_BILINEAR == 3, "FilterMode order");

API const char ffref_vp9dsp_layout_check[] = "b200dsp.h B200VP9DSPContext matches VP9DSPContext";

/* libffref.so (oracle/ref/ref_shim.c): VideoDSPContext.emulated_edge_mc for 8-bit and for 16-bit samples */
void ffref_emulated_edge_mc(uint8_t *buf, const uint8_t *src, ptrdiff_t buf_linesize, ptrdiff_t src_linesize, int block_w, int block_h,
                            int src_x, int src_y, int w, int h);
void ffref_emulated_edge_mc_hbd(uint8_t *buf, const uint8_t *src, ptrdiff_t buf_linesize, ptrdiff_t src_linesize, int block_w, int block_h,
                                int src_x, int src_y, int w, int h);

static VP9DSPContext *ref_vp9dsp(int depth)
{
    static VP9DSPContext c[13];
    static int ok[13];
    if (depth != 8 && depth != 10 && depth != 12) return NULL;
    if (!ok[depth]) { ff_vp9dsp_init(&c[depth], depth, 1); ok[depth] = 1; }
    return &c[depth];
}

/* table index of a block width: 64, 32, 16, 8, 4 -> 0..4; -1 for any other */
static int size_idx(int w)
{
    for (int i = 0; i < 5; i++)
        if (w == 64 >> i) return i;
    return -1;
}

API const int16_t *ffref_vp9_subpel_filters(void) { return &ff_vp9_subpel_filters[0][0][0]; }

/* mc[size of w][bank][avg][hdir][vdir] of ff_vp9dsp_init(depth) */
API int ffref_vp9_mc(int depth, int bank, int avg, int hdir, int vdir, void *dst, ptrdiff_t dst_stride, const void *src, ptrdiff_t src_stride,
                     int w, int h, int mx, int my)
{
    VP9DSPContext *c = ref_vp9dsp(depth);
    const int i = size_idx(w);
    if (!c || i < 0 || bank < 0 || bank > 3) return -1;
    c->mc[i][bank][!!avg][!!hdir][!!vdir](dst, dst_stride, src, src_stride, h, mx, my);
    return 0;
}

/* smc[size of w][bank][avg] */
API int ffref_vp9_smc(int depth, int bank, int avg, void *dst, ptrdiff_t dst_stride, const void *src, ptrdiff_t src_stride, int w, int h, int mx,
                      int my, int dx, int dy)
{
    VP9DSPContext *c = ref_vp9dsp(depth);
    const int i = size_idx(w);
    if (!c || i < 0 || bank < 0 || bank > 3) return -1;
    c->smc[i][bank][!!avg](dst, dst_stride, src, src_stride, h, mx, my, dx, dy);
    return 0;
}

/* 1 if the four full-pel entries of every size and put / avg are one function (vp9dsp_template.c:2308-2322) */
API int ffref_vp9_fpel_shared(int depth)
{
    VP9DSPContext *c = ref_vp9dsp(depth);
    if (!c) return -1;
    for (int i = 0; i < 5; i++)
        for (int a = 0; a < 2; a++)
            for (int f = 1; f < 4; f++)
                if (c->mc[i][f][a][0][0] != c->mc[i][0][a][0][0]) return 0;
    return 1;
}

/* one slot of one op as mc_luma_unscaled / mc_chroma_unscaled (vp9recon.c:325-336, :368-388) and mc_luma_scaled / mc_chroma_scaled
 * (:450-469, :520-549) run it, from the point where x, y, mx, my are known */
static void mc_slot(VP9DSPContext *c, int depth, const B200Vp9McRef *f, const B200Vp9McOp *op, int r, uint8_t *dst, ptrdiff_t dst_stride,
                    uint8_t *edge_emu_buffer)
{
    const int bytesperpixel = depth > 8 ? 2 : 1, bw = op->w, bh = op->h, w = f->w, h = f->h, i = size_idx(bw);
    const int x = op->x[r], y = op->y[r], mx = op->mx[r], my = op->my[r];
    const uint8_t *ref = f->data + (ptrdiff_t)y * f->stride + (ptrdiff_t)x * bytesperpixel;
    ptrdiff_t ref_stride = f->stride;
    void (*emu)(uint8_t *, const uint8_t *, ptrdiff_t, ptrdiff_t, int, int, int, int, int, int) =
        bytesperpixel == 2 ? ffref_emulated_edge_mc_hbd : ffref_emulated_edge_mc;
    if (f->dx == 16 && f->dy == 16) {
        if (x < !!mx * 3 || y < !!my * 3 || x + !!mx * 4 > w - bw || y + !!my * 5 > h - bh) {
            emu(edge_emu_buffer, ref - !!my * 3 * ref_stride - !!mx * 3 * bytesperpixel, 160, ref_stride, bw + !!mx * 7, bh + !!my * 7,
                x - !!mx * 3, y - !!my * 3, w, h);
            ref = edge_emu_buffer + !!my * 3 * 160 + !!mx * 3 * bytesperpixel;
            ref_stride = 160;
        }
        c->mc[i][op->filter][r][!!mx][!!my](dst, dst_stride, ref, ref_stride, bh, mx, my);
    } else {
        const int refbw_m1 = ((bw - 1) * f->dx + mx) >> 4, refbh_m1 = ((bh - 1) * f->dy + my) >> 4;
        if (x < 3 || y < 3 || x + 4 >= w - refbw_m1 || y + 5 >= h - refbh_m1) {
            emu(edge_emu_buffer, ref - 3 * ref_stride - 3 * bytesperpixel, 288, ref_stride, refbw_m1 + 8, refbh_m1 + 8, x - 3, y - 3, w, h);
            ref = edge_emu_buffer + 3 * 288 + 3 * bytesperpixel;
            ref_stride = 288;
        }
        c->smc[i][op->filter][r](dst, dst_stride, ref, ref_stride, bh, mx, my, f->dx, f->dy);
    }
}

/* the decoder's sequence for each op of a batch (the same op guard as the product; refs[].data are host addresses); returns the number
 * of ops that wrote their block */
API int64_t ffref_vp9_mc_batch(int depth, int nrefs, const B200Vp9McRef *refs, int64_t nops, const B200Vp9McOp *ops, uint8_t *dst,
                               ptrdiff_t dst_stride)
{
    static uint8_t edge_emu_buffer[135 * 288];                             /* td->edge_emu_buffer, vp9dec.h */
    VP9DSPContext *c = ref_vp9dsp(depth);
    const int bps = depth > 8 ? 2 : 1;
    int64_t done = 0;
    if (!c) return -1;
    for (int64_t i = 0; i < nops; i++) {
        const B200Vp9McOp *op = &ops[i];
        const int nslot = op->kind == B200_VP9_MC_COMPOUND ? 2 : 1;
        int ok = op->kind <= 1 && op->filter <= 3 && size_idx(op->w) >= 0 && op->h >= 1 && op->h <= 64 && !(op->dst_off % bps);
        for (int r = 0; r < nslot; r++) ok = ok && op->ref[r] < nrefs && op->mx[r] <= 15 && op->my[r] <= 15;
        if (!ok) continue;
        for (int r = 0; r < nslot; r++) mc_slot(c, depth, &refs[op->ref[r]], op, r, dst + op->dst_off, dst_stride, edge_emu_buffer);
        done++;
    }
    return done;
}
