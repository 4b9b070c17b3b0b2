/*
 * vp8dsp_oracle.c — TEST INFRASTRUCTURE ONLY.  CPU restatement of VP8 / VP7 motion compensation and residual reconstruction: the
 * functions behind put_vp8_epel_pixels_tab, put_vp8_bilinear_pixels_tab and the six residual members of VP8DSPContext
 * (libavcodec/vp8dsp.h:37-82) as ff_vp78dsp_init, ff_vp8dsp_init and ff_vp7dsp_init install them (vp8dsp.c:641-760), and the semantics
 * of b200_vp8_mc_frame_device / b200_vp8_residual_frame_device (include/b200dsp.h).
 *
 * Follows (behaviour, not text) libavcodec/vp8dsp.c:56-639 in the reference's own form: the running 4-tap / 6-tap / bilinear loops
 * with their tmp arrays (4-tap with taps F[1..4] of whatever row the phase picks), the VP8 WHT / IDCT (column pass first, int16
 * intermediates) and the VP7 ones (row pass first, unsigned products).  The frame entries restate the decoder: vp8_mc_luma /
 * vp8_mc_chroma (vp8.c:1831-1929) from the point where the source position and phase are known — its edge test, a window of clamped
 * samples where the test says the block's window leaves the plane (what emulated_edge_mc gives), and the member call — and, per
 * macroblock, the WHT of decode_mb_coeffs (vp8.c:1517-1524) followed by idct_mb (vp8.c:2085-2146) with its early break / goto.
 */
#include <string.h>
#include "vp8dsp_oracle.h"

static const uint8_t SF[7][6] = {
    { 0, 6, 123, 12, 1, 0 }, { 2, 11, 108, 36, 8, 1 }, { 0, 9, 93, 50, 6, 0 }, { 3, 16, 77, 77, 16, 3 },
    { 0, 6, 50, 93, 9, 0 }, { 1, 8, 36, 108, 11, 2 }, { 0, 1, 12, 123, 6, 0 },
};
const uint8_t *orc_vp8_subpel_filters(void) { return &SF[0][0]; }

static uint8_t clip8(int v) { return v < 0 ? 0 : v > 255 ? 255 : (uint8_t)v; }

static uint8_t tap6(const uint8_t *s, ptrdiff_t st, const uint8_t *F)
{
    return clip8((F[2] * s[0] - F[1] * s[-st] + F[0] * s[-2 * st] + F[3] * s[st] - F[4] * s[2 * st] + F[5] * s[3 * st] + 64) >> 7);
}
static uint8_t tap4(const uint8_t *s, ptrdiff_t st, const uint8_t *F)
{
    return clip8((F[2] * s[0] - F[1] * s[-st] + F[3] * s[st] - F[4] * s[2 * st] + 64) >> 7);
}
static uint8_t taps(int n, const uint8_t *s, ptrdiff_t st, const uint8_t *F) { return n == 6 ? tap6(s, st, F) : tap4(s, st, F); }

/* the member at any h 1..16 (the frame entry's ops may be taller than the reference's tmp_array allows) */
static void mc(int bilinear, int w, int v, int hi, uint8_t *dst, ptrdiff_t ds, const uint8_t *src, ptrdiff_t ss, int h, int mx, int my)
{
    uint8_t tmp[(32 + 5) * 16];
    if (!v && !hi) {
        for (int y = 0; y < h; y++, dst += ds, src += ss) memcpy(dst, src, w);
        return;
    }
    if (bilinear) {
        const int a = 8 - mx, b = mx, c = 8 - my, d = my;
        if (!v) {
            for (int y = 0; y < h; y++, dst += ds, src += ss)
                for (int x = 0; x < w; x++) dst[x] = (a * src[x] + b * src[x + 1] + 4) >> 3;
        } else if (!hi) {
            for (int y = 0; y < h; y++, dst += ds, src += ss)
                for (int x = 0; x < w; x++) dst[x] = (c * src[x] + d * src[x + ss] + 4) >> 3;
        } else {
            uint8_t *t = tmp;
            for (int y = 0; y < h + 1; y++, t += w, src += ss)
                for (int x = 0; x < w; x++) t[x] = (a * src[x] + b * src[x + 1] + 4) >> 3;
            t = tmp;
            for (int y = 0; y < h; y++, dst += ds, t += w)
                for (int x = 0; x < w; x++) dst[x] = (c * t[x] + d * t[x + w] + 4) >> 3;
        }
        return;
    }
    const int ht = hi == 1 ? 4 : 6, vt = v == 1 ? 4 : 6;
    if (!v) {
        for (int y = 0; y < h; y++, dst += ds, src += ss)
            for (int x = 0; x < w; x++) dst[x] = taps(ht, src + x, 1, SF[mx - 1]);
    } else if (!hi) {
        for (int y = 0; y < h; y++, dst += ds, src += ss)
            for (int x = 0; x < w; x++) dst[x] = taps(vt, src + x, ss, SF[my - 1]);
    } else {
        uint8_t *t = tmp;
        src -= (2 - (vt == 4)) * ss;
        for (int y = 0; y < h + vt - 1; y++, t += w, src += ss)
            for (int x = 0; x < w; x++) t[x] = taps(ht, src + x, 1, SF[mx - 1]);
        t = tmp + (2 - (vt == 4)) * w;
        for (int y = 0; y < h; y++, dst += ds, t += w)
            for (int x = 0; x < w; x++) dst[x] = taps(vt, t + x, w, SF[my - 1]);
    }
}

int orc_vp8_mc(int bilinear, int w, int v, int hi, uint8_t *dst, ptrdiff_t ds, const uint8_t *src, ptrdiff_t ss, int h, int mx, int my)
{
    if ((w != 16 && w != 8 && w != 4) || v < 0 || v > 2 || hi < 0 || hi > 2 || h < 1 || h > 2 * w) return -1;
    if (!bilinear && w == 16 && (v == 1 || hi == 1)) return -1;                 /* NULL in put_vp8_epel_pixels_tab[0] */
    const int lo = bilinear ? 0 : 1;
    if ((hi && (mx < lo || mx > 7)) || (v && (my < lo || my > 7))) return -1;
    mc(bilinear, w, v, hi, dst, ds, src, ss, h, mx, my);
    return 0;
}

/* ---------------------------------------------------------------- residual members */
static void vp7_wht(int16_t block[4][4][16], int16_t dc[16])
{
    unsigned a1, b1, c1, d1;
    int16_t tmp[16];
    for (int i = 0; i < 4; i++) {
        a1 = (dc[i * 4 + 0] + dc[i * 4 + 2]) * 23170;
        b1 = (dc[i * 4 + 0] - dc[i * 4 + 2]) * 23170;
        c1 = dc[i * 4 + 1] * 12540 - dc[i * 4 + 3] * 30274;
        d1 = dc[i * 4 + 1] * 30274 + dc[i * 4 + 3] * 12540;
        tmp[i * 4 + 0] = (int)(a1 + d1) >> 14;
        tmp[i * 4 + 3] = (int)(a1 - d1) >> 14;
        tmp[i * 4 + 1] = (int)(b1 + c1) >> 14;
        tmp[i * 4 + 2] = (int)(b1 - c1) >> 14;
    }
    for (int i = 0; i < 4; i++) {
        a1 = (tmp[i + 0] + tmp[i + 8]) * 23170;
        b1 = (tmp[i + 0] - tmp[i + 8]) * 23170;
        c1 = tmp[i + 4] * 12540 - tmp[i + 12] * 30274;
        d1 = tmp[i + 4] * 30274 + tmp[i + 12] * 12540;
        memset(dc + i * 4, 0, 4 * sizeof(int16_t));
        block[0][i][0] = (int)(a1 + d1 + 0x20000) >> 18;
        block[3][i][0] = (int)(a1 - d1 + 0x20000) >> 18;
        block[1][i][0] = (int)(b1 + c1 + 0x20000) >> 18;
        block[2][i][0] = (int)(b1 - c1 + 0x20000) >> 18;
    }
}

static void vp8_wht(int16_t block[4][4][16], int16_t dc[16])
{
    int t0, t1, t2, t3;
    for (int i = 0; i < 4; i++) {
        t0 = dc[0 * 4 + i] + dc[3 * 4 + i];
        t1 = dc[1 * 4 + i] + dc[2 * 4 + i];
        t2 = dc[1 * 4 + i] - dc[2 * 4 + i];
        t3 = dc[0 * 4 + i] - dc[3 * 4 + i];
        dc[0 * 4 + i] = t0 + t1;
        dc[1 * 4 + i] = t3 + t2;
        dc[2 * 4 + i] = t0 - t1;
        dc[3 * 4 + i] = t3 - t2;
    }
    for (int i = 0; i < 4; i++) {
        t0 = dc[i * 4 + 0] + dc[i * 4 + 3] + 3;
        t1 = dc[i * 4 + 1] + dc[i * 4 + 2];
        t2 = dc[i * 4 + 1] - dc[i * 4 + 2];
        t3 = dc[i * 4 + 0] - dc[i * 4 + 3] + 3;
        memset(dc + i * 4, 0, 4 * sizeof(int16_t));
        block[i][0][0] = (t0 + t1) >> 3;
        block[i][1][0] = (t3 + t2) >> 3;
        block[i][2][0] = (t0 - t1) >> 3;
        block[i][3][0] = (t3 - t2) >> 3;
    }
}

static int vp7_dc(int v) { return (23170 * (23170 * v >> 14) + 0x20000) >> 18; }

static void wht_dc(int is_vp7, int16_t block[4][4][16], int16_t dc[16])
{
    const int val = is_vp7 ? vp7_dc(dc[0]) : (dc[0] + 3) >> 3;
    dc[0] = 0;
    for (int i = 0; i < 4; i++)
        for (int j = 0; j < 4; j++) block[i][j][0] = val;
}

void orc_vp8_wht(int is_vp7, int dc_only, int16_t *block, int16_t *dc)
{
    int16_t (*b)[4][16] = (int16_t (*)[4][16])block;
    if (dc_only) wht_dc(is_vp7, b, dc);
    else if (is_vp7) vp7_wht(b, dc);
    else vp8_wht(b, dc);
}

static void vp7_idct_add(uint8_t *dst, int16_t block[16], ptrdiff_t stride)
{
    unsigned a1, b1, c1, d1;
    int16_t tmp[16];
    for (int i = 0; i < 4; i++) {
        a1 = (block[i * 4 + 0] + block[i * 4 + 2]) * 23170;
        b1 = (block[i * 4 + 0] - block[i * 4 + 2]) * 23170;
        c1 = block[i * 4 + 1] * 12540 - block[i * 4 + 3] * 30274;
        d1 = block[i * 4 + 1] * 30274 + block[i * 4 + 3] * 12540;
        memset(block + i * 4, 0, 4 * sizeof(int16_t));
        tmp[i * 4 + 0] = (int)(a1 + d1) >> 14;
        tmp[i * 4 + 3] = (int)(a1 - d1) >> 14;
        tmp[i * 4 + 1] = (int)(b1 + c1) >> 14;
        tmp[i * 4 + 2] = (int)(b1 - c1) >> 14;
    }
    for (int i = 0; i < 4; i++) {
        a1 = (tmp[i + 0] + tmp[i + 8]) * 23170;
        b1 = (tmp[i + 0] - tmp[i + 8]) * 23170;
        c1 = tmp[i + 4] * 12540 - tmp[i + 12] * 30274;
        d1 = tmp[i + 4] * 30274 + tmp[i + 12] * 12540;
        dst[0 * stride + i] = clip8(dst[0 * stride + i] + ((int)(a1 + d1 + 0x20000) >> 18));
        dst[3 * stride + i] = clip8(dst[3 * stride + i] + ((int)(a1 - d1 + 0x20000) >> 18));
        dst[1 * stride + i] = clip8(dst[1 * stride + i] + ((int)(b1 + c1 + 0x20000) >> 18));
        dst[2 * stride + i] = clip8(dst[2 * stride + i] + ((int)(b1 - c1 + 0x20000) >> 18));
    }
}

#define MUL_20091(a) ((((a) * 20091) >> 16) + (a))
#define MUL_35468(a)  (((a) * 35468) >> 16)

static void vp8_idct_add(uint8_t *dst, int16_t block[16], ptrdiff_t stride)
{
    int t0, t1, t2, t3;
    int16_t tmp[16];
    for (int i = 0; i < 4; i++) {
        t0 = block[0 * 4 + i] + block[2 * 4 + i];
        t1 = block[0 * 4 + i] - block[2 * 4 + i];
        t2 = MUL_35468(block[1 * 4 + i]) - MUL_20091(block[3 * 4 + i]);
        t3 = MUL_20091(block[1 * 4 + i]) + MUL_35468(block[3 * 4 + i]);
        block[0 * 4 + i] = block[1 * 4 + i] = block[2 * 4 + i] = block[3 * 4 + i] = 0;
        tmp[i * 4 + 0] = t0 + t3;
        tmp[i * 4 + 1] = t1 + t2;
        tmp[i * 4 + 2] = t1 - t2;
        tmp[i * 4 + 3] = t0 - t3;
    }
    for (int i = 0; i < 4; i++, dst += stride) {
        t0 = tmp[0 * 4 + i] + tmp[2 * 4 + i];
        t1 = tmp[0 * 4 + i] - tmp[2 * 4 + i];
        t2 = MUL_35468(tmp[1 * 4 + i]) - MUL_20091(tmp[3 * 4 + i]);
        t3 = MUL_20091(tmp[1 * 4 + i]) + MUL_35468(tmp[3 * 4 + i]);
        dst[0] = clip8(dst[0] + ((t0 + t3 + 4) >> 3));
        dst[1] = clip8(dst[1] + ((t1 + t2 + 4) >> 3));
        dst[2] = clip8(dst[2] + ((t1 - t2 + 4) >> 3));
        dst[3] = clip8(dst[3] + ((t0 - t3 + 4) >> 3));
    }
}

static void dc_add(int is_vp7, uint8_t *dst, int16_t block[16], ptrdiff_t stride)
{
    const int dc = is_vp7 ? vp7_dc(block[0]) : (block[0] + 4) >> 3;
    block[0] = 0;
    for (int i = 0; i < 4; i++, dst += stride)
        for (int j = 0; j < 4; j++) dst[j] = clip8(dst[j] + dc);
}

static void idct_add(int is_vp7, uint8_t *dst, int16_t block[16], ptrdiff_t stride)
{
    if (is_vp7) vp7_idct_add(dst, block, stride);
    else vp8_idct_add(dst, block, stride);
}

static void dc_add4y(int is_vp7, uint8_t *dst, int16_t block[4][16], ptrdiff_t stride)
{
    for (int k = 0; k < 4; k++) dc_add(is_vp7, dst + 4 * k, block[k], stride);
}

static void dc_add4uv(int is_vp7, uint8_t *dst, int16_t block[4][16], ptrdiff_t stride)
{
    dc_add(is_vp7, dst, block[0], stride);
    dc_add(is_vp7, dst + 4, block[1], stride);
    dc_add(is_vp7, dst + 4 * stride, block[2], stride);
    dc_add(is_vp7, dst + 4 * stride + 4, block[3], stride);
}

void orc_vp8_idct(int is_vp7, int which, uint8_t *dst, int16_t *block, ptrdiff_t stride)
{
    switch (which) {
    case 0: idct_add(is_vp7, dst, block, stride); break;
    case 1: dc_add(is_vp7, dst, block, stride); break;
    case 2: dc_add4y(is_vp7, dst, (int16_t (*)[16])block, stride); break;
    case 3: dc_add4uv(is_vp7, dst, (int16_t (*)[16])block, stride); break;
    }
}

/* ---------------------------------------------------------------- frame entries */
static const uint8_t subpel_idx[3][8] = {
    { 0, 1, 2, 1, 2, 1, 2, 1 },
    { 0, 3, 5, 3, 5, 3, 5, 3 },
    { 0, 2, 3, 2, 3, 2, 3, 2 },
};

int64_t orc_vp8_mc_frame(int bilinear, int mb_width, int mb_height, int nrefs, const B200Vp8McRef *refs, int64_t nops, const B200Vp8McOp *ops,
                         uint8_t *const dst[3], ptrdiff_t ls_y, ptrdiff_t ls_uv)
{
    uint8_t buf[21 * 32];                                       /* td->edge_emu_buffer, EDGE_EMU_LINESIZE 32 (vp8.h:147-148) */
    int64_t done = 0;
    for (int64_t i = 0; i < nops; i++) {
        const B200Vp8McOp *op = &ops[i];
        const int c = op->plane, bw = op->w, bh = op->h, mx = op->mx, my = op->my;
        if (c > 1 || (bw != 16 && bw != 8 && bw != 4) || bh < 1 || bh > 16 || mx > 7 || my > 7 || op->ref >= nrefs) continue;
        if (!bilinear && bw == 16 && ((mx | my) & 1)) continue;
        const int width = (c ? 8 : 16) * mb_width, height = (c ? 8 : 16) * mb_height;
        if ((op->dst_x & 3) || op->dst_x < 0 || op->dst_y < 0 || op->dst_x > width - bw || op->dst_y > height - bh) continue;
        const int mx_idx = subpel_idx[0][mx], my_idx = subpel_idx[0][my], x_off = op->src_x, y_off = op->src_y;
        const ptrdiff_t ls = c ? ls_uv : ls_y;
        for (int p = 0; p < (c ? 2 : 1); p++) {
            const uint8_t *plane = c == 0 ? refs[op->ref].y : p ? refs[op->ref].v : refs[op->ref].u;
            const ptrdiff_t rls = c ? refs[op->ref].ls_uv : refs[op->ref].ls_y;
            const uint8_t *src;
            ptrdiff_t src_ls = rls;
            if (x_off < mx_idx || x_off >= width - bw - subpel_idx[2][mx] || y_off < my_idx || y_off >= height - bh - subpel_idx[2][my]) {
                const int bwe = bw + subpel_idx[1][mx], bhe = bh + subpel_idx[1][my];
                for (int y = 0; y < bhe; y++)
                    for (int x = 0; x < bwe; x++) {
                        long long yy = (long long)y_off - my_idx + y, xx = (long long)x_off - mx_idx + x;
                        yy = yy < 0 ? 0 : yy >= height ? height - 1 : yy;
                        xx = xx < 0 ? 0 : xx >= width ? width - 1 : xx;
                        buf[y * 32 + x] = plane[yy * rls + xx];
                    }
                src = buf + mx_idx + 32 * my_idx;
                src_ls = 32;
            } else {
                src = plane + (ptrdiff_t)y_off * rls + x_off;
            }
            uint8_t *d = dst[c ? 1 + p : 0] + (ptrdiff_t)op->dst_y * ls + op->dst_x;
            mc(bilinear, bw, my_idx, mx_idx, d, ls, src, src_ls, bh, mx, my);
        }
        done++;
    }
    return done;
}

static uint32_t rl32(const uint8_t *p) { return p[0] | (uint32_t)p[1] << 8 | (uint32_t)p[2] << 16 | (uint32_t)p[3] << 24; }

int64_t orc_vp8_residual_frame(int is_vp7, int64_t nops, const B200Vp8ResidualOp *ops, const int16_t *coef, uint8_t *const dst[3],
                               ptrdiff_t ls_y, ptrdiff_t ls_uv)
{
    int64_t done = 0;
    for (int64_t i = 0; i < nops; i++) {
        const B200Vp8ResidualOp *op = &ops[i];
        if (op->mb_x < 0 || op->mb_y < 0 || op->coef_off < 0 || (op->coef_off & 7)) continue;
        int16_t block[6][4][16], block_dc[16];
        memcpy(block, coef + op->coef_off, sizeof(block));
        memcpy(block_dc, coef + op->coef_off + 384, sizeof(block_dc));
        if (op->y2_nnz) orc_vp8_wht(is_vp7, op->y2_nnz == 1, &block[0][0][0], block_dc);
        if (op->flags & B200_VP8_RESIDUAL_LUMA) {
            uint8_t *y_dst = dst[0] + (ptrdiff_t)op->mb_y * 16 * ls_y + (ptrdiff_t)op->mb_x * 16;
            for (int y = 0; y < 4; y++) {
                uint32_t nnz4 = rl32(op->nnz[y]);
                if (nnz4) {
                    if (nnz4 & ~0x01010101) {
                        for (int x = 0; x < 4; x++) {
                            if ((uint8_t)nnz4 == 1) dc_add(is_vp7, y_dst + 4 * x, block[y][x], ls_y);
                            else if ((uint8_t)nnz4 > 1) idct_add(is_vp7, y_dst + 4 * x, block[y][x], ls_y);
                            nnz4 >>= 8;
                            if (!nnz4) break;
                        }
                    } else {
                        dc_add4y(is_vp7, y_dst, block[y], ls_y);
                    }
                }
                y_dst += 4 * ls_y;
            }
        }
        for (int ch = 0; ch < 2; ch++) {
            uint32_t nnz4 = rl32(op->nnz[4 + ch]);
            if (nnz4) {
                uint8_t *ch_dst = dst[1 + ch] + (ptrdiff_t)op->mb_y * 8 * ls_uv + (ptrdiff_t)op->mb_x * 8;
                if (nnz4 & ~0x01010101) {
                    for (int y = 0; y < 2; y++) {
                        for (int x = 0; x < 2; x++) {
                            if ((uint8_t)nnz4 == 1) dc_add(is_vp7, ch_dst + 4 * x, block[4 + ch][(y << 1) + x], ls_uv);
                            else if ((uint8_t)nnz4 > 1) idct_add(is_vp7, ch_dst + 4 * x, block[4 + ch][(y << 1) + x], ls_uv);
                            nnz4 >>= 8;
                            if (!nnz4) goto chroma_idct_end;
                        }
                        ch_dst += 4 * ls_uv;
                    }
                } else {
                    dc_add4uv(is_vp7, ch_dst, block[4 + ch], ls_uv);
                }
            }
chroma_idct_end:
            ;
        }
        done++;
    }
    return done;
}
