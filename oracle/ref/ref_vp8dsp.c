/* TEST INFRASTRUCTURE — the reference's VP8 / VP7 DSP (libavcodec/vp8dsp.c, compiled unmodified where it lies by oracle/ref/vp8dsp.mk
 * with CONFIG_VP7_DECODER and CONFIG_VP8_DECODER on, into oracle/_ref/libffref_vp8dsp.so, next to libffref.so which it links against
 * for emulated_edge_mc) exposed through a flat C ABI: one member per call of either context (ff_vp78dsp_init plus ff_vp8dsp_init or
 * ff_vp7dsp_init), the pointers of both contexts, and the decoder's two sequences for the frame entries of include/b200dsp.h:
 * vp8_mc_luma / vp8_mc_chroma (vp8.c:1831-1929) from the point where the source position and phase are known — the edge test, an
 * emulated_edge_mc window of EDGE_EMU_LINESIZE, the member call — and, per macroblock, the luma DC WHT of decode_mb_coeffs
 * (vp8.c:1517-1524) followed by idct_mb's calls (vp8.c:2085-2146) on a copy of the coefficients.  Plus the compile-time proof that
 * B200VP8DSPContext can be copied member for member into VP8DSPContext.  tests/vp8dsplib.py loads it and reads the marker below. */
#include <stdint.h>
#include <stddef.h>
#include <string.h>

#include "config.h"
#include "libavutil/intreadwrite.h"
#include "libavutil/mem_internal.h"
#include "libavcodec/vp8dsp.h"
#include "../../include/b200dsp.h"

#define API __attribute__((visibility("default")))

#define SAME_OFF(A, B, m)  _Static_assert(offsetof(A, m) == offsetof(B, m), "offset of " #m " in " #A " / " #B)
#define SAME_TYPE(A, B, m) _Static_assert(__builtin_types_compatible_p(__typeof__(((A *)0)->m), __typeof__(((B *)0)->m)), "type of " #m " in " #A " / " #B)
#define SAME(A, B, m)      SAME_OFF(A, B, m); SAME_TYPE(A, B, m)

/* VP8DSPContext, libavcodec/vp8dsp.h:37-82 */
_Static_assert(sizeof(VP8DSPContext) == sizeof(B200VP8DSPContext) && sizeof(VP8DSPContext) == 70 * sizeof(void *), "size of VP8DSPContext");
SAME(VP8DSPContext, B200VP8DSPContext, vp8_luma_dc_wht);
SAME(VP8DSPContext, B200VP8DSPContext, vp8_luma_dc_wht_dc);
SAME(VP8DSPContext, B200VP8DSPContext, vp8_idct_add);
SAME(VP8DSPContext, B200VP8DSPContext, vp8_idct_dc_add);
SAME(VP8DSPContext, B200VP8DSPContext, vp8_idct_dc_add4y);
SAME(VP8DSPContext, B200VP8DSPContext, vp8_idct_dc_add4uv);
SAME(VP8DSPContext, B200VP8DSPContext, vp8_v_loop_filter16y);
SAME(VP8DSPContext, B200VP8DSPContext, vp8_h_loop_filter16y);
SAME(VP8DSPContext, B200VP8DSPContext, vp8_v_loop_filter8uv);
SAME(VP8DSPContext, B200VP8DSPContext, vp8_h_loop_filter8uv);
SAME(VP8DSPContext, B200VP8DSPContext, vp8_v_loop_filter16y_inner);
SAME(VP8DSPContext, B200VP8DSPContext, vp8_h_loop_filter16y_inner);
SAME(VP8DSPContext, B200VP8DSPContext, vp8_v_loop_filter8uv_inner);
SAME(VP8DSPContext, B200VP8DSPContext, vp8_h_loop_filter8uv_inner);
SAME(VP8DSPContext, B200VP8DSPContext, vp8_v_loop_filter_simple);
SAME(VP8DSPContext, B200VP8DSPContext, vp8_h_loop_filter_simple);
SAME(VP8DSPContext, B200VP8DSPContext, put_vp8_epel_pixels_tab);
SAME(VP8DSPContext, B200VP8DSPContext, put_vp8_bilinear_pixels_tab);

API const char ffref_vp8dsp_layout_check[] = "b200dsp.h B200VP8DSPContext matches VP8DSPContext";

/* libffref.so (oracle/ref/ref_shim.c): VideoDSPContext.emulated_edge_mc for 8-bit samples */
void ffref_emulated_edge_mc(uint8_t *buf, const uint8_t *src, ptrdiff_t buf_linesize, ptrdiff_t src_linesize, int block_w, int block_h,
                            int src_x, int src_y, int w, int h);

static VP8DSPContext *ref_vp8dsp(int is_vp7)
{
    static VP8DSPContext c[2];
    static int ok[2];
    if (is_vp7 != 0 && is_vp7 != 1) return NULL;
    if (!ok[is_vp7]) {
        memset(&c[is_vp7], 0, sizeof(c[is_vp7]));
        ff_vp78dsp_init(&c[is_vp7]);
        if (is_vp7) ff_vp7dsp_init(&c[is_vp7]);
        else ff_vp8dsp_init(&c[is_vp7]);
        ok[is_vp7] = 1;
    }
    return &c[is_vp7];
}

/* the 70 pointers of the context, in member order */
API int ffref_vp8_pointers(int is_vp7, void **out)
{
    VP8DSPContext *c = ref_vp8dsp(is_vp7);
    if (!c) return -1;
    memcpy(out, c, sizeof(*c));
    return 0;
}

static int size_idx(int w) { return w == 16 ? 0 : w == 8 ? 1 : w == 4 ? 2 : -1; }

/* put_vp8_epel_pixels_tab / put_vp8_bilinear_pixels_tab[size of w][v][h]; -1 for a NULL position */
API int ffref_vp8_mc(int bilinear, int w, int v, int hi, uint8_t *dst, ptrdiff_t dst_stride, const uint8_t *src, ptrdiff_t src_stride, int h,
                     int mx, int my)
{
    VP8DSPContext *c = ref_vp8dsp(0);
    const int i = size_idx(w);
    if (i < 0 || v < 0 || v > 2 || hi < 0 || hi > 2) return -1;
    vp8_mc_func f = bilinear ? c->put_vp8_bilinear_pixels_tab[i][v][hi] : c->put_vp8_epel_pixels_tab[i][v][hi];
    if (!f) return -1;
    f(dst, dst_stride, src, src_stride, h, mx, my);
    return 0;
}

API void ffref_vp8_wht(int is_vp7, int dc_only, int16_t *block, int16_t *dc)
{
    VP8DSPContext *c = ref_vp8dsp(is_vp7);
    (dc_only ? c->vp8_luma_dc_wht_dc : c->vp8_luma_dc_wht)((int16_t (*)[4][16])block, dc);
}

/* which 0 idct_add, 1 idct_dc_add, 2 idct_dc_add4y, 3 idct_dc_add4uv */
API void ffref_vp8_idct(int is_vp7, int which, uint8_t *dst, int16_t *block, ptrdiff_t stride)
{
    VP8DSPContext *c = ref_vp8dsp(is_vp7);
    switch (which) {
    case 0: c->vp8_idct_add(dst, block, stride); break;
    case 1: c->vp8_idct_dc_add(dst, block, stride); break;
    case 2: c->vp8_idct_dc_add4y(dst, (int16_t (*)[16])block, stride); break;
    case 3: c->vp8_idct_dc_add4uv(dst, (int16_t (*)[16])block, stride); break;
    }
}

static const uint8_t subpel_idx[3][8] = {                  /* vp8.c:1809-1814 */
    { 0, 1, 2, 1, 2, 1, 2, 1 },
    { 0, 3, 5, 3, 5, 3, 5, 3 },
    { 0, 2, 3, 2, 3, 2, 3, 2 },
};
#define EDGE_EMU_LINESIZE 32

/* the decoder's sequence for each op of a frame (the same op guard as the product; refs' planes are host addresses); returns the
 * number of ops that wrote their block */
API int64_t ffref_vp8_mc_frame(int bilinear, int mb_width, int mb_height, int nrefs, const B200Vp8McRef *refs, int64_t nops,
                               const B200Vp8McOp *ops, uint8_t *const dst[3], ptrdiff_t ls_y, ptrdiff_t ls_uv)
{
    static uint8_t edge_emu_buffer[21 * EDGE_EMU_LINESIZE];
    VP8DSPContext *c = ref_vp8dsp(0);
    int64_t done = 0;
    for (int64_t i = 0; i < nops; i++) {
        const B200Vp8McOp *op = &ops[i];
        const int pc = op->plane, block_w = op->w, block_h = op->h, mx = op->mx, my = op->my;
        if (pc > 1 || size_idx(block_w) < 0 || block_h < 1 || block_h > 16 || mx > 7 || my > 7 || op->ref >= nrefs) continue;
        if (!bilinear && block_w == 16 && ((mx | my) & 1)) continue;
        const int width = (pc ? 8 : 16) * mb_width, height = (pc ? 8 : 16) * mb_height;
        if ((op->dst_x & 3) || op->dst_x < 0 || op->dst_y < 0 || op->dst_x > width - block_w || op->dst_y > height - block_h) continue;
        vp8_mc_func (*mc_func)[3] = bilinear ? c->put_vp8_bilinear_pixels_tab[size_idx(block_w)] : c->put_vp8_epel_pixels_tab[size_idx(block_w)];
        const int mx_idx = subpel_idx[0][mx], my_idx = subpel_idx[0][my], x_off = op->src_x, y_off = op->src_y;
        const ptrdiff_t linesize = pc ? ls_uv : ls_y;
        for (int p = 0; p < (pc ? 2 : 1); p++) {
            const uint8_t *plane = pc == 0 ? refs[op->ref].y : p ? refs[op->ref].v : refs[op->ref].u;
            const ptrdiff_t ref_ls = pc ? refs[op->ref].ls_uv : refs[op->ref].ls_y;
            uint8_t *d = dst[pc ? 1 + p : 0] + (ptrdiff_t)op->dst_y * linesize + op->dst_x;
            const uint8_t *src = plane + (ptrdiff_t)y_off * ref_ls + x_off;
            ptrdiff_t src_linesize = ref_ls;
            if (x_off < mx_idx || x_off >= width - block_w - subpel_idx[2][mx] ||
                y_off < my_idx || y_off >= height - block_h - subpel_idx[2][my]) {
                ffref_emulated_edge_mc(edge_emu_buffer, src - my_idx * ref_ls - mx_idx, EDGE_EMU_LINESIZE, ref_ls,
                                       block_w + subpel_idx[1][mx], block_h + subpel_idx[1][my], x_off - mx_idx, y_off - my_idx, width, height);
                src = edge_emu_buffer + mx_idx + EDGE_EMU_LINESIZE * my_idx;
                src_linesize = EDGE_EMU_LINESIZE;
            }
            mc_func[my_idx][mx_idx](d, linesize, src, src_linesize, block_h, mx, my);
        }
        done++;
    }
    return done;
}

/* the residual of each macroblock as the decoder reaches it: the WHT member on block_dc, then idct_mb's member calls */
API int64_t ffref_vp8_residual_frame(int is_vp7, int64_t nops, const B200Vp8ResidualOp *ops, const int16_t *coef, uint8_t *const dst[3],
                                     ptrdiff_t ls_y, ptrdiff_t ls_uv)
{
    VP8DSPContext *s = ref_vp8dsp(is_vp7);
    int64_t done = 0;
    if (!s) return -1;
    for (int64_t i = 0; i < nops; i++) {
        const B200Vp8ResidualOp *op = &ops[i];
        if (op->mb_x < 0 || op->mb_y < 0 || op->coef_off < 0 || (op->coef_off & 7)) continue;
        DECLARE_ALIGNED(16, int16_t, block)[6][4][16];
        DECLARE_ALIGNED(16, int16_t, block_dc)[16];
        memcpy(block, coef + op->coef_off, sizeof(block));
        memcpy(block_dc, coef + op->coef_off + 384, sizeof(block_dc));
        if (op->y2_nnz) {
            if (op->y2_nnz == 1) s->vp8_luma_dc_wht_dc(block, block_dc);
            else s->vp8_luma_dc_wht(block, block_dc);
        }
        uint8_t *const mbdst[3] = { dst[0] + (ptrdiff_t)op->mb_y * 16 * ls_y + (ptrdiff_t)op->mb_x * 16,
                                    dst[1] + (ptrdiff_t)op->mb_y * 8 * ls_uv + (ptrdiff_t)op->mb_x * 8,
                                    dst[2] + (ptrdiff_t)op->mb_y * 8 * ls_uv + (ptrdiff_t)op->mb_x * 8 };
        int x, y, ch;
        if (op->flags & B200_VP8_RESIDUAL_LUMA) {
            uint8_t *y_dst = mbdst[0];
            for (y = 0; y < 4; y++) {
                uint32_t nnz4 = AV_RL32(op->nnz[y]);
                if (nnz4) {
                    if (nnz4 & ~0x01010101) {
                        for (x = 0; x < 4; x++) {
                            if ((uint8_t)nnz4 == 1) s->vp8_idct_dc_add(y_dst + 4 * x, block[y][x], ls_y);
                            else if ((uint8_t)nnz4 > 1) s->vp8_idct_add(y_dst + 4 * x, block[y][x], ls_y);
                            nnz4 >>= 8;
                            if (!nnz4) break;
                        }
                    } else {
                        s->vp8_idct_dc_add4y(y_dst, block[y], ls_y);
                    }
                }
                y_dst += 4 * ls_y;
            }
        }
        for (ch = 0; ch < 2; ch++) {
            uint32_t nnz4 = AV_RL32(op->nnz[4 + ch]);
            if (nnz4) {
                uint8_t *ch_dst = mbdst[1 + ch];
                if (nnz4 & ~0x01010101) {
                    for (y = 0; y < 2; y++) {
                        for (x = 0; x < 2; x++) {
                            if ((uint8_t)nnz4 == 1) s->vp8_idct_dc_add(ch_dst + 4 * x, block[4 + ch][(y << 1) + x], ls_uv);
                            else if ((uint8_t)nnz4 > 1) s->vp8_idct_add(ch_dst + 4 * x, block[4 + ch][(y << 1) + x], ls_uv);
                            nnz4 >>= 8;
                            if (!nnz4) goto chroma_idct_end;
                        }
                        ch_dst += 4 * ls_uv;
                    }
                } else {
                    s->vp8_idct_dc_add4uv(ch_dst, block[4 + ch], ls_uv);
                }
            }
chroma_idct_end:
            ;
        }
        done++;
    }
    return done;
}
