/*
 * hevcsao_oracle.c — TEST INFRASTRUCTURE ONLY.  CPU restatement of the SAO members of HEVCDSPContext (libavcodec/hevc/dsp.h:47-125:
 * sao_band_filter, sao_edge_filter, sao_edge_restore[0 / 1]) as ff_hevc_dsp_init installs them for depth 8, 9, 10 and 12
 * (hevc/dsp.c:217-228), and of the picture-level semantics of b200_hevc_sao_plane_device (include/b200dsp.h): per CTB, what the
 * decoder's sao_filter_CTB (hevc/filter.c:269-478) does for one component when every neighbour sample it reads is the deblocked
 * one, including restore_tqb_pixels' PU loop with the luma CTB origin and the component's CTB size.
 *
 * Follows (behaviour, not text) h26x/h2656_sao_template.c.  Counters (cnt, may be NULL) show which outcomes an input reaches:
 *   cnt[0] band samples changed          cnt[1..4] edge samples filtered, class 0..3     cnt[5] picture-border samples
 *   cnt[6..9] samples put back by vert_edge[0], vert_edge[1], horiz_edge[0], horiz_edge[1]
 *   cnt[10..13] corner samples put back by diag_edge[0..3]
 *   cnt[14..17] corner saves (save_upper_left, _upper_right, _lower_right, _lower_left) that kept a sample filtered
 *   cnt[18] samples put back by the keep map   cnt[19] marked PUs of a CTB's luma area the keep loop does not visit (chroma quirk)
 *   cnt[20] / cnt[21] results clipped at 0 / at the maximum
 */
#include <stdint.h>
#include <stddef.h>
#include <string.h>
#include "../include/b200dsp.h"

#define NCNT 22
static int64_t *g_cnt;
static int64_t g_dummy[NCNT];

static int rd(const uint8_t *p, int bps) { return bps == 1 ? *p : *(const uint16_t *)p; }
static void wr(uint8_t *p, int bps, int v)
{
    if (bps == 1) *p = (uint8_t)v;
    else *(uint16_t *)p = (uint16_t)v;
}
static int clip_count(int v, int depth)
{
    const int maxv = (1 << depth) - 1;
    if (v < 0) { g_cnt[20]++; return 0; }
    if (v > maxv) { g_cnt[21]++; return maxv; }
    return v;
}
#define AT(base, stride, x, y) ((base) + (ptrdiff_t)(y) * (stride) + (ptrdiff_t)(x) * bps)

/* sao_band_filter: a 32-entry table, offsets at (k + left_class) mod 32 */
static void band(int depth, uint8_t *dst, const uint8_t *src, ptrdiff_t sd, ptrdiff_t ss, const int16_t *off, int left_class, int w, int h)
{
    const int bps = depth > 8 ? 2 : 1;
    int table[32] = { 0 };
    for (int k = 0; k < 4; k++) table[(unsigned)(k + left_class) % 32u] = off[k + 1];
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++) {
            const int s = rd(AT(src, ss, x, y), bps), t = table[s >> (depth - 5)];
            if (t) g_cnt[0]++;
            wr(AT(dst, sd, x, y), bps, clip_count(s + t, depth));
        }
}

/* sao_edge_filter: src at the 192-byte stride */
static void edge(int depth, uint8_t *dst, const uint8_t *src, ptrdiff_t sd, const int16_t *off, int eo, int w, int h)
{
    static const int dx[4] = { -1, 0, -1, 1 }, dy[4] = { 0, -1, -1, -1 };      /* neighbour a; b = -a */
    static const int idx[5] = { 1, 2, 0, 3, 4 };
    const int bps = depth > 8 ? 2 : 1;
    const ptrdiff_t ss = 192;
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++) {
            const int s = rd(AT(src, ss, x, y), bps);
            const int a = rd(AT(src, ss, x + dx[eo], y + dy[eo]), bps), b = rd(AT(src, ss, x - dx[eo], y - dy[eo]), bps);
            const int d = (s > a) - (s < a) + (s > b) - (s < b);
            g_cnt[1 + eo]++;
            wr(AT(dst, sd, x, y), bps, clip_count(s + off[idx[d + 2]], depth));
        }
}

static void put_border(int depth, uint8_t *dst, const uint8_t *src, ptrdiff_t sd, ptrdiff_t ss, int x, int y, int off0)
{
    const int bps = depth > 8 ? 2 : 1;
    g_cnt[5]++;
    wr(AT(dst, sd, x, y), bps, clip_count(rd(AT(src, ss, x, y), bps) + off0, depth));
}
static void put_src(int depth, uint8_t *dst, const uint8_t *src, ptrdiff_t sd, ptrdiff_t ss, int x, int y, int which)
{
    const int bps = depth > 8 ? 2 : 1;
    g_cnt[which]++;
    wr(AT(dst, sd, x, y), bps, rd(AT(src, ss, x, y), bps));
}

/* sao_edge_restore_0 (r1 = 0) and _1 (r1 = 1) */
static void restore(int depth, int r1, uint8_t *dst, const uint8_t *src, ptrdiff_t sd, ptrdiff_t ss, const B200SAOParams *sao,
                    const int *borders, int W, int H, int c_idx, const uint8_t *ve, const uint8_t *he, const uint8_t *de)
{
    const int off0 = sao->offset_val[c_idx][0], eo = sao->eo_class[c_idx];
    int x0 = 0, y0 = 0, w = W, h = H;
    if (eo != 1) {                                            /* not vertical: the left and right columns */
        if (borders[0]) { for (int y = 0; y < h; y++) put_border(depth, dst, src, sd, ss, 0, y, off0); x0 = 1; }
        if (borders[2]) { for (int y = 0; y < h; y++) put_border(depth, dst, src, sd, ss, w - 1, y, off0); w--; }
    }
    if (eo != 0) {                                            /* not horizontal: the top and bottom rows */
        if (borders[1]) { for (int x = x0; x < w; x++) put_border(depth, dst, src, sd, ss, x, 0, off0); if (r1) y0 = 1; }
        if (borders[3]) { for (int x = x0; x < w; x++) put_border(depth, dst, src, sd, ss, x, h - 1, off0); h--; }
    }
    if (!r1) return;
    const int ul = !de[0] && eo == 2 && !borders[0] && !borders[1];
    const int ur = !de[1] && eo == 3 && !borders[1] && !borders[2];
    const int lr = !de[2] && eo == 2 && !borders[2] && !borders[3];
    const int ll = !de[3] && eo == 3 && !borders[0] && !borders[3];
    if ((ul && (ve[0] || he[0])) ) g_cnt[14]++;
    if ((ur && (ve[1] || he[0])) ) g_cnt[15]++;
    if ((lr && (ve[1] || he[1])) ) g_cnt[16]++;
    if ((ll && (ve[0] || he[1])) ) g_cnt[17]++;
    if (ve[0] && eo != 1) for (int y = y0 + ul; y < h - ll; y++) put_src(depth, dst, src, sd, ss, 0, y, 6);
    if (ve[1] && eo != 1) for (int y = y0 + ur; y < h - lr; y++) put_src(depth, dst, src, sd, ss, w - 1, y, 7);
    if (he[0] && eo != 0) for (int x = x0 + ul; x < w - ur; x++) put_src(depth, dst, src, sd, ss, x, 0, 8);
    if (he[1] && eo != 0) for (int x = x0 + ll; x < w - lr; x++) put_src(depth, dst, src, sd, ss, x, h - 1, 9);
    if (de[0] && eo == 2) put_src(depth, dst, src, sd, ss, 0, 0, 10);
    if (de[1] && eo == 3) put_src(depth, dst, src, sd, ss, w - 1, 0, 11);
    if (de[2] && eo == 2) put_src(depth, dst, src, sd, ss, w - 1, h - 1, 12);
    if (de[3] && eo == 3) put_src(depth, dst, src, sd, ss, 0, h - 1, 13);
}

static void set_cnt(int64_t *cnt) { g_cnt = cnt ? cnt : g_dummy; }

void orc_hevc_sao_band(int depth, uint8_t *dst, const uint8_t *src, ptrdiff_t sd, ptrdiff_t ss, const int16_t *off, int left_class, int w,
                       int h, int64_t *cnt)
{
    set_cnt(cnt);
    band(depth, dst, src, sd, ss, off, left_class, w, h);
}

void orc_hevc_sao_edge(int depth, uint8_t *dst, const uint8_t *src, ptrdiff_t sd, const int16_t *off, int eo, int w, int h, int64_t *cnt)
{
    set_cnt(cnt);
    edge(depth, dst, src, sd, off, eo, w, h);
}

void orc_hevc_sao_restore(int depth, int which, uint8_t *dst, const uint8_t *src, ptrdiff_t sd, ptrdiff_t ss, const B200SAOParams *sao,
                          const int *borders, int w, int h, int c_idx, const uint8_t *ve, const uint8_t *he, const uint8_t *de, int64_t *cnt)
{
    set_cnt(cnt);
    restore(depth, which, dst, src, sd, ss, sao, borders, w, h, c_idx, ve, he, de);
}

typedef void (*restore_fn)(uint8_t *, const uint8_t *, ptrdiff_t, ptrdiff_t, const void *, const int *, int, int, int, const uint8_t *,
                           const uint8_t *, const uint8_t *);

/* Every eo_class 0..3 x borders[4] (16) x, for which = 1, the eight edge flags (256) x c_idx 0..2 on a w x h block (w, h >= 2) with
 * off0 = offset_val[c_idx][0] (non-zero, different per component): fn (a member's address; NULL = this checker) on seeded src / dst
 * buffers with a margin of 2 samples; returns the FNV-1a 64 digest of every dst buffer, margins included. */
uint64_t orc_hevc_sao_restore_sweep(int depth, int which, void *fn, int w, int h, uint32_t seed)
{
    const int bps = depth > 8 ? 2 : 1, maxv = (1 << depth) - 1, M = 2;
    const ptrdiff_t ss = (ptrdiff_t)(w + 2 * M + 3) * bps, sd = (ptrdiff_t)(w + 2 * M) * bps;
    uint8_t src[72 * 72 * 2], dst[72 * 72 * 2];
    uint64_t hsh = 1469598103934665603ull;
    uint32_t r = seed;
    B200SAOParams sao;
    memset(&sao, 0, sizeof(sao));
    set_cnt(NULL);
    for (int c = 0; c < 3; c++) sao.offset_val[c][0] = (int16_t)(c == 0 ? 7 : c == 1 ? -5 : (depth == 12 ? 124 : 31));
    for (int eo = 0; eo < 4; eo++)
        for (int bd = 0; bd < 16; bd++)
            for (int fl = 0; fl < (which ? 256 : 1); fl++)
                for (int c = 0; c < 3; c++) {
                    for (size_t i = 0; i < sizeof(src) / bps; i++) {     /* samples at 0 / the maximum among random ones */
                        r = r * 1664525u + 1013904223u;
                        const int v = (int)((r >> 8) % 5u) == 0 ? ((r >> 12) & 1 ? maxv : 0) : (int)((r >> 4) & (unsigned)maxv);
                        wr(src + i * bps, bps, v);
                        wr(dst + i * bps, bps, v ^ 0x5A);               /* stands for the edge filter's output */
                    }
                    sao.eo_class[c] = eo;
                    const int borders[4] = { bd & 1, (bd >> 1) & 1, (bd >> 2) & 1, (bd >> 3) & 1 };
                    const uint8_t ve[2] = { fl & 1, (fl >> 1) & 1 }, he[2] = { (fl >> 2) & 1, (fl >> 3) & 1 };
                    const uint8_t de[4] = { (fl >> 4) & 1, (fl >> 5) & 1, (fl >> 6) & 1, (fl >> 7) & 1 };
                    uint8_t *d0 = dst + M * sd + M * bps;
                    const uint8_t *s0 = src + M * ss + M * bps;
                    if (fn) ((restore_fn)fn)(d0, s0, sd, ss, &sao, borders, w, h, c, ve, he, de);
                    else restore(depth, which, d0, s0, sd, ss, &sao, borders, w, h, c, ve, he, de);
                    for (ptrdiff_t i = 0; i < (h + 2 * M) * sd; i++) { hsh ^= dst[i]; hsh *= 1099511628211ull; }
                }
    return hsh;
}

/* The plane entry's semantics: dst = SAO of src per CTB (CTBs visited in raster order, or reversed when `reverse`: the result is the
 * same because only src is read).  keep NULL = no PCM / bypass restoration.  Returns 0; cnt[NCNT] outcome counts (may be NULL). */
int orc_hevc_sao_plane(int depth, uint8_t *dst, ptrdiff_t sd, const uint8_t *src, ptrdiff_t ss, int width, int height, int log2_ctb,
                       int hs, int vs, const B200HevcSaoCtb *ctb, int64_t cstride, const uint8_t *keep, int64_t kstride, int log2_pu,
                       int reverse, int64_t *cnt)
{
    const int bps = depth > 8 ? 2 : 1, cw = (1 << log2_ctb) >> hs, ch = (1 << log2_ctb) >> vs;
    const int ncx = (width + cw - 1) / cw, ncy = (height + ch - 1) / ch;
    uint8_t buf[(64 + 2) * 192 + 64];                            /* the decoder's edge buffer: 192-byte rows, block at row 1 */
    set_cnt(cnt);
    for (int t = 0; t < ncx * ncy; t++) {
        const int k = reverse ? ncx * ncy - 1 - t : t, i = k % ncx, j = k / ncx;
        const B200HevcSaoCtb *r = &ctb[(int64_t)j * cstride + i];
        const int x0 = i * cw, y0 = j * ch, w = width - x0 < cw ? width - x0 : cw, h = height - y0 < ch ? height - y0 : ch;
        uint8_t *d = AT(dst, sd, x0, y0);
        const uint8_t *s = AT(src, ss, x0, y0);
        for (int y = 0; y < h; y++) memcpy(d + (ptrdiff_t)y * sd, s + (ptrdiff_t)y * ss, (size_t)w * bps);
        if (r->type == B200_HEVC_SAO_BAND) {
            band(depth, d, s, sd, ss, r->offset_val, r->cls & 31, w, h);
        } else if (r->type == B200_HEVC_SAO_EDGE && r->cls <= 3) {
            const int edges[4] = { i == 0, j == 0, i == ncx - 1, j == ncy - 1 };
            uint8_t *b = buf + 192 + 32;                         /* sample (0, 0) of the block */
            memset(buf, 0, sizeof(buf));
            for (int y = -1; y <= h; y++)                        /* deblocked neighbours, inside the plane */
                for (int x = -1; x <= w; x++)
                    if (x0 + x >= 0 && x0 + x < width && y0 + y >= 0 && y0 + y < height)
                        wr(AT(b, 192, x, y), bps, rd(AT(src, ss, x0 + x, y0 + y), bps));
            edge(depth, d, b, sd, r->offset_val, r->cls, w, h);
            /* the restore member and its flags as sao_filter_CTB computes them (0 where a side is a picture border) */
            const int rest = r->flags & B200_HEVC_SAO_RESTORE, f = rest ? r->flags : 0;
            const uint8_t ve[2] = { !edges[0] && (f & B200_HEVC_SAO_VERT_L), !edges[2] && (f & B200_HEVC_SAO_VERT_R) };
            const uint8_t he[2] = { !edges[1] && (f & B200_HEVC_SAO_HORIZ_T), !edges[3] && (f & B200_HEVC_SAO_HORIZ_B) };
            const uint8_t de[4] = { !edges[0] && !edges[1] && (f & B200_HEVC_SAO_DIAG_TL), !edges[1] && !edges[2] && (f & B200_HEVC_SAO_DIAG_TR),
                                    !edges[2] && !edges[3] && (f & B200_HEVC_SAO_DIAG_BR), !edges[0] && !edges[3] && (f & B200_HEVC_SAO_DIAG_BL) };
            B200SAOParams sao;
            memset(&sao, 0, sizeof(sao));
            sao.offset_val[0][0] = r->offset_val[0];
            sao.eo_class[0] = r->cls;
            restore(depth, rest != 0, d, b, sd, 192, &sao, edges, w, h, 0, ve, he, de);
        } else {
            continue;
        }
        if (!keep) continue;
        /* restore_tqb_pixels: PUs x_min..x_max-1 / y_min..y_max-1 from the luma origin and the component's width / height */
        const int X = i << log2_ctb, Y = j << log2_ctb, pu = 1 << log2_pu;
        const int x_min = X >> log2_pu, y_min = Y >> log2_pu, x_max = (X + w) >> log2_pu, y_max = (Y + h) >> log2_pu;
        const int len = pu >> hs;
        for (int py = y_min; py < y_max; py++)
            for (int px = x_min; px < x_max; px++) {
                if (!keep[(int64_t)py * kstride + px]) continue;
                const int cy = ((py << log2_pu) - Y) >> vs, cx = ((px << log2_pu) - X) >> hs;
                for (int n = 0; n < (pu >> vs); n++) {
                    memcpy(AT(d, sd, cx, cy + n), AT(s, ss, cx, cy + n), (size_t)len * bps);
                    g_cnt[18] += len;
                }
            }
        /* marked PUs of the CTB's whole luma area that the loop above does not visit */
        const int lx_max = (X + (w << hs)) >> log2_pu, ly_max = (Y + (h << vs)) >> log2_pu;
        for (int py = y_min; py < ly_max; py++)
            for (int px = x_min; px < lx_max; px++)
                if ((px >= x_max || py >= y_max) && keep[(int64_t)py * kstride + px]) g_cnt[19]++;
    }
    return 0;
}
