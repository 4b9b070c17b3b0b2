/* TEST INFRASTRUCTURE — the reference's VC-1 DSP (libavcodec/vc1dsp.c, compiled unmodified where it lies by oracle/ref/vc1dsp.mk into
 * oracle/_ref/libffref_vc1dsp.so, next to libffref.so which it links against for hpeldsp, h264chroma, emulated_edge_mc and
 * add_pixels_clamped) exposed through a flat C ABI: one member per call of the context ff_vc1dsp_init fills, its pointers, and the
 * decoder's two sequences for the frame entries of include/b200dsp.h: the progressive MC of ff_vc1_mc_1mv / ff_vc1_mc_4mv_luma /
 * ff_vc1_mc_4mv_chroma / ff_vc1_interp_mc (vc1_mc.c:172-836, :1004-1230) from the point where the source positions are known — the
 * edge test, the emulated_edge_mc windows in an EDGE_PITCH buffer, range reduction, the IC LUTs, the member calls — and the transform
 * dispatch of vc1_decode_p_block (vc1_block.c:1124-1240) on a copy of the coefficients.  Plus the compile-time proof that
 * B200VC1DSPContext can be copied member for member into VC1DSPContext.  tests/vc1dsplib.py loads it and reads the marker below. */
#include <stdint.h>
#include <stddef.h>
#include <string.h>

#include "config.h"
#include "libavcodec/vc1dsp.h"
#include "../../include/b200dsp.h"

#define API __attribute__((visibility("default")))

#define SAME_OFF(A, B, m)  _Static_assert(offsetof(A, m) == offsetof(B, m), "offset of " #m " in " #A " / " #B)
#define SAME_TYPE(A, B, m) _Static_assert(__builtin_types_compatible_p(__typeof__(((A *)0)->m), __typeof__(((B *)0)->m)), "type of " #m " in " #A " / " #B)
#define SAME(m)            SAME_OFF(VC1DSPContext, B200VC1DSPContext, m); SAME_TYPE(VC1DSPContext, B200VC1DSPContext, m)

/* VC1DSPContext, libavcodec/vc1dsp.h:37-97 */
_Static_assert(sizeof(VC1DSPContext) == sizeof(B200VC1DSPContext) && sizeof(VC1DSPContext) == 95 * sizeof(void *), "size of VC1DSPContext");
SAME(vc1_inv_trans_8x8); SAME(vc1_inv_trans_8x4); SAME(vc1_inv_trans_4x8); SAME(vc1_inv_trans_4x4);
SAME(vc1_inv_trans_8x8_dc); SAME(vc1_inv_trans_8x4_dc); SAME(vc1_inv_trans_4x8_dc); SAME(vc1_inv_trans_4x4_dc);
SAME(vc1_v_overlap); SAME(vc1_h_overlap); SAME(vc1_v_s_overlap); SAME(vc1_h_s_overlap);
SAME(vc1_v_loop_filter4); SAME(vc1_h_loop_filter4); SAME(vc1_v_loop_filter8); SAME(vc1_h_loop_filter8);
SAME(vc1_v_loop_filter16); SAME(vc1_h_loop_filter16);
SAME(put_vc1_mspel_pixels_tab); SAME(avg_vc1_mspel_pixels_tab);
SAME(put_no_rnd_vc1_chroma_pixels_tab); SAME(avg_no_rnd_vc1_chroma_pixels_tab);
SAME(sprite_h); SAME(sprite_v_single); SAME(sprite_v_double_noscale); SAME(sprite_v_double_onescale); SAME(sprite_v_double_twoscale);
SAME(startcode_find_candidate); SAME(vc1_unescape_buffer);

API const char ffref_vc1dsp_layout_check[] = "b200dsp.h B200VC1DSPContext matches VC1DSPContext";

/* libffref.so (oracle/ref/ref_shim.c) */
int ffref_hpel(int tab, int size_idx, int xy, uint8_t *block, const uint8_t *pixels, ptrdiff_t line_size, int h);
int ffref_h264chroma(int avg, int idx, uint8_t *dst, const uint8_t *src, ptrdiff_t stride, int h, int x, int y);
void ffref_emulated_edge_mc(uint8_t *buf, const uint8_t *src, ptrdiff_t buf_linesize, ptrdiff_t src_linesize, int block_w, int block_h,
                            int src_x, int src_y, int w, int h);
void ffref_pixels_clamped(int kind, const int16_t *block, uint8_t *pixels, ptrdiff_t line_size);

static VC1DSPContext *ref_vc1dsp(void)
{
    static VC1DSPContext c;
    static int ok;
    if (!ok) {
        memset(&c, 0, sizeof(c));
        ff_vc1dsp_init(&c);
        ok = 1;
    }
    return &c;
}

/* the 95 pointers of the context, in member order */
API void ffref_vc1_pointers(void **out) { memcpy(out, ref_vc1dsp(), sizeof(VC1DSPContext)); }

API int ffref_vc1_mspel(int avg, int size, int dxy, uint8_t *dst, const uint8_t *src, ptrdiff_t stride, int rnd)
{
    if (size < 0 || size > 1 || dxy < 0 || dxy > 15) return -1;
    (avg ? ref_vc1dsp()->avg_vc1_mspel_pixels_tab : ref_vc1dsp()->put_vc1_mspel_pixels_tab)[size][dxy](dst, src, stride, rnd);
    return 0;
}

API int ffref_vc1_chroma(int avg, int idx, uint8_t *dst, const uint8_t *src, ptrdiff_t stride, int h, int x, int y)
{
    if (idx < 0 || idx > 1 || x < 0 || x > 7 || y < 0 || y > 7 || h < 0) return -1;
    (avg ? ref_vc1dsp()->avg_no_rnd_vc1_chroma_pixels_tab : ref_vc1dsp()->put_no_rnd_vc1_chroma_pixels_tab)[idx](dst, src, stride, h, x, y);
    return 0;
}

/* tt: 0 8x8, 1 8x4, 2 4x8, 3 4x4 */
API int ffref_vc1_itx(int tt, int dc, uint8_t *dest, ptrdiff_t stride, int16_t *block)
{
    VC1DSPContext *c = ref_vc1dsp();
    if (tt < 0 || tt > 3) return -1;
    if (tt == 0 && !dc) { c->vc1_inv_trans_8x8(block); return 0; }
    void (*f)(uint8_t *, ptrdiff_t, int16_t *) =
        dc ? (tt == 0 ? c->vc1_inv_trans_8x8_dc : tt == 1 ? c->vc1_inv_trans_8x4_dc : tt == 2 ? c->vc1_inv_trans_4x8_dc : c->vc1_inv_trans_4x4_dc)
           : (tt == 1 ? c->vc1_inv_trans_8x4 : tt == 2 ? c->vc1_inv_trans_4x8 : c->vc1_inv_trans_4x4);
    f(dest, stride, block);
    return 0;
}

/* ---------------------------------------------------------------- the decoder's MC sequence (progressive: field_mode 0, interlace 0) */
enum { EDGE_PITCH = 64 };

static void scale_rr(uint8_t *p, int k)                          /* vc1_scale_luma / vc1_scale_chroma */
{
    for (int j = 0; j < k; j++)
        for (int i = 0; i < k; i++) p[j * EDGE_PITCH + i] = ((p[j * EDGE_PITCH + i] - 128) >> 1) + 128;
}

static void scale_lut(uint8_t *p, const uint8_t *lut1, const uint8_t *lut2, int k)   /* vc1_lut_scale_luma / _chroma */
{
    for (int j = 0; j < k; j += 2) {
        for (int i = 0; i < k; i++) p[i] = lut1[p[i]];
        p += EDGE_PITCH;
        if (j + 1 == k) break;
        for (int i = 0; i < k; i++) p[i] = lut2[p[i]];
        p += EDGE_PITCH;
    }
}

/* The members take one stride, the decoder's linesize, for source and destination.  Here the window and the destination block are
 * both held at EDGE_PITCH: the window is emulated_edge_mc's output (with range reduction and the LUTs) where the edge test fires and
 * a copy of the plane where it does not, and the destination block is copied in and back out. */
static void load_window(uint8_t *buf, const uint8_t *plane, ptrdiff_t ls, int k, int x0, int y0, int emu, int w, int h, int rr,
                        const uint8_t (*lut)[256])
{
    const uint8_t *org = plane + y0 * ls + x0;
    if (!emu) {
        for (int j = 0; j < k; j++) memcpy(buf + j * EDGE_PITCH, org + j * ls, k);
        return;
    }
    ffref_emulated_edge_mc(buf, org, EDGE_PITCH, ls, k, k, x0, y0, w, h);
    if (rr) scale_rr(buf, k);
    if (lut) scale_lut(buf, lut[(0 + y0) & 1], lut[(1 + y0) & 1], k);
}

static void block_io(uint8_t *blk, uint8_t *d, ptrdiff_t ls, int n, int out)
{
    for (int j = 0; j < n; j++) {
        if (out) memcpy(d + j * ls, blk + j * EDGE_PITCH, n);
        else memcpy(blk + j * EDGE_PITCH, d + j * ls, n);
    }
}

/* the chroma pair of an op at ((uvmx & 3) << 1, (uvmy & 3) << 1): put_h264_chroma (rnd 0) or put_no_rnd_vc1_chroma (rnd 1), avg_ forms */
static void chroma_pair(const B200Vc1McRef *R, const B200Vc1McSrc *S, int emu, int avg, int rnd, uint8_t *du, uint8_t *dv, ptrdiff_t ls_uv,
                        int H, int V)
{
    const int x = (S->uvmx & 3) << 1, y = (S->uvmy & 3) << 1;
    for (int p = 0; p < 2; p++) {
        uint8_t win[9 * EDGE_PITCH], blk[8 * EDGE_PITCH];
        load_window(win, p ? R->v : R->u, R->ls_uv, 9, S->uvx, S->uvy, emu, H >> 1, V >> 1, R->rangeredfrm, R->use_ic ? R->lutuv : NULL);
        uint8_t *d = p ? dv : du;
        block_io(blk, d, ls_uv, 8, 0);
        if (!rnd) ffref_h264chroma(avg, 0, blk, win, EDGE_PITCH, 8, x, y);
        else (avg ? ref_vc1dsp()->avg_no_rnd_vc1_chroma_pixels_tab : ref_vc1dsp()->put_no_rnd_vc1_chroma_pixels_tab)[0](blk, win, EDGE_PITCH, 8, x, y);
        block_io(blk, d, ls_uv, 8, 1);
    }
}

API int64_t ffref_vc1_mc_frame(int nrefs, const B200Vc1McRef *refs, uint8_t *const dst[3], ptrdiff_t ls_y, ptrdiff_t ls_uv, int mbw, int mbh,
                               int H, int V, int64_t nops, const B200Vc1McOp *ops)
{
    VC1DSPContext *c = ref_vc1dsp();
    int64_t wrote = 0;
    for (int64_t i = 0; i < nops; i++) {
        const B200Vc1McOp *op = &ops[i];
        const int nsrc = op->flags & B200_VC1_MC_AVG ? 2 : 1, ms = !!(op->flags & B200_VC1_MC_MSPEL), rnd = !!(op->flags & B200_VC1_MC_RND);
        int ok = op->kind <= B200_VC1_MC_CHROMA8 && !(nsrc == 2 && op->kind != B200_VC1_MC_1MV);
        for (int s = 0; s < nsrc && ok; s++)
            ok = op->src[s].ref < nrefs && op->src[s].mx < 4 && op->src[s].my < 4 && op->src[s].uvmx < 4 && op->src[s].uvmy < 4;
        const int n = op->kind == B200_VC1_MC_1MV ? 16 : 8, sc = op->kind == B200_VC1_MC_CHROMA8 ? 8 : 16;
        if (!ok || op->dst_x < 0 || op->dst_y < 0 || op->dst_x % 8 || op->dst_y % 8 || op->dst_x + n > sc * mbw || op->dst_y + n > sc * mbh)
            continue;
        for (int s = 0; s < nsrc; s++) {
            const B200Vc1McSrc *S = &op->src[s];
            const B200Vc1McRef *R = &refs[S->ref];
            const int mx = S->mx, my = S->my, src_x = S->x, src_y = S->y;
            if (op->kind == B200_VC1_MC_CHROMA8) {                    /* ff_vc1_mc_4mv_chroma, vc1_mc.c:735-831 */
                const int emu = R->rangeredfrm || R->use_ic || H < 18 || V < 18 || (unsigned)S->uvx > (H >> 1) - 9 ||
                                (unsigned)S->uvy > (V >> 1) - 9;
                chroma_pair(R, S, emu, 0, rnd, dst[1] + op->dst_y * ls_uv + op->dst_x, dst[2] + op->dst_y * ls_uv + op->dst_x, ls_uv, H, V);
                continue;
            }
            int emu;
            const int k = (op->kind == B200_VC1_MC_1MV ? 17 : 9) + ms * 2;
            if (op->kind == B200_VC1_MC_LUMA8)                         /* vc1_mc.c:563-566 */
                emu = R->rangeredfrm || R->use_ic || H < 13 || V < 23 || (unsigned)(src_x - ms) > H - (mx & 3) - 8 - ms * 2 ||
                      (unsigned)(src_y - ms) > V - (my & 3) - (8 + ms * 2);
            else if (s == 0)                                           /* ff_vc1_mc_1mv, vc1_mc.c:299-302 */
                emu = R->rangeredfrm || R->use_ic || H < 22 || V < 22 || (unsigned)(src_x - ms) > H - (mx & 3) - 16 - ms * 3 ||
                      (unsigned)(src_y - 1) > V - (my & 3) - 16 - 3;
            else                                                       /* ff_vc1_interp_mc, vc1_mc.c:1066-1068 */
                emu = R->rangeredfrm || H < 22 || V < 22 || R->use_ic || (unsigned)(src_x - 1) > H - (mx & 3) - 16 - 3 ||
                      (unsigned)(src_y - 1) > V - (my & 3) - 16 - 3;
            uint8_t win[19 * EDGE_PITCH], blk[16 * EDGE_PITCH];
            load_window(win, R->y, R->ls_y, k, src_x - ms, src_y - ms, emu, H, V, R->rangeredfrm, R->use_ic ? R->luty : NULL);
            uint8_t *d = dst[0] + op->dst_y * ls_y + op->dst_x;
            block_io(blk, d, ls_y, n, 0);
            const uint8_t *sp = win + ms * (1 + EDGE_PITCH);
            const int size = op->kind == B200_VC1_MC_1MV ? 0 : 1;
            if (ms)
                (s ? c->avg_vc1_mspel_pixels_tab : c->put_vc1_mspel_pixels_tab)[size][((my & 3) << 2) | (mx & 3)](blk, sp, EDGE_PITCH, rnd);
            else
                ffref_hpel(s ? (rnd ? 3 : 1) : (rnd ? 2 : 0), size, (my & 2) | ((mx & 2) >> 1), blk, sp, EDGE_PITCH, n);
            block_io(blk, d, ls_y, n, 1);
            if (op->kind == B200_VC1_MC_1MV)
                chroma_pair(R, S, emu, s, rnd, dst[1] + op->dst_y / 2 * ls_uv + op->dst_x / 2, dst[2] + op->dst_y / 2 * ls_uv + op->dst_x / 2,
                            ls_uv, H, V);
        }
        wrote++;
    }
    return wrote;
}

/* ---------------------------------------------------------------- vc1_decode_p_block's transform dispatch */
API int64_t ffref_vc1_residual_frame(uint8_t *const planes[3], ptrdiff_t ls_y, ptrdiff_t ls_uv, int mbw, int mbh, const int16_t *coef,
                                     int64_t nops, const B200Vc1ResidualOp *ops)
{
    VC1DSPContext *c = ref_vc1dsp();
    int64_t wrote = 0;
    for (int64_t i = 0; i < nops; i++) {
        const B200Vc1ResidualOp *op = &ops[i];
        const int sc = op->plane ? 8 : 16;
        if (op->plane > 2 || op->ttblk > 3 || op->coef_off < 0 || op->coef_off % 8 || op->x < 0 || op->y < 0 || op->x % 8 || op->y % 8 ||
            op->x + 8 > sc * mbw || op->y + 8 > sc * mbh)
            continue;
        int16_t block[64];
        memcpy(block, coef + op->coef_off, sizeof(block));
        const ptrdiff_t linesize = op->plane ? ls_uv : ls_y;
        uint8_t *dst = planes[op->plane] + op->y * linesize + op->x;
        const int subblkpat = op->subblkpat;
        switch (op->ttblk) {
        case 0:
            if (op->dc & 1)
                c->vc1_inv_trans_8x8_dc(dst, linesize, block);
            else {
                c->vc1_inv_trans_8x8(block);
                ffref_pixels_clamped(2, block, dst, linesize);
            }
            break;
        case 3:
            for (int j = 0; j < 4; j++) {
                const int off = (j & 1) * 4 + (j & 2) * 16;
                if (!(subblkpat & (1 << (3 - j)))) {
                    if ((op->dc >> j) & 1) c->vc1_inv_trans_4x4_dc(dst + (j & 1) * 4 + (j & 2) * 2 * linesize, linesize, block + off);
                    else c->vc1_inv_trans_4x4(dst + (j & 1) * 4 + (j & 2) * 2 * linesize, linesize, block + off);
                }
            }
            break;
        case 1:
            for (int j = 0; j < 2; j++) {
                const int off = j * 32;
                if (!(subblkpat & (1 << (1 - j)))) {
                    if ((op->dc >> j) & 1) c->vc1_inv_trans_8x4_dc(dst + j * 4 * linesize, linesize, block + off);
                    else c->vc1_inv_trans_8x4(dst + j * 4 * linesize, linesize, block + off);
                }
            }
            break;
        case 2:
            for (int j = 0; j < 2; j++) {
                const int off = j * 4;
                if (!(subblkpat & (1 << (1 - j)))) {
                    if ((op->dc >> j) & 1) c->vc1_inv_trans_4x8_dc(dst + j * 4, linesize, block + off);
                    else c->vc1_inv_trans_4x8(dst + j * 4, linesize, block + off);
                }
            }
            break;
        }
        wrote++;
    }
    return wrote;
}
