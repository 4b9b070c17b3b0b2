/*
 * vp9mc_oracle.c — TEST INFRASTRUCTURE ONLY.  CPU restatement of VP9 motion compensation: the functions behind the mc[5][4][2][2][2]
 * and smc[5][4][2] tables of VP9DSPContext (libavcodec/vp9dsp.h:40-122) as ff_vp9dsp_init installs them for depth 8, 10 and 12
 * (vp9dsp_template.c:2302-2361, :2540-2569), and the batch semantics of b200_vp9_mc_batch_device (include/b200dsp.h).
 *
 * Follows (behaviour, not text) libavcodec/vp9dsp_template.c:1971-2569:
 *   8-tap     clip((sum F[k] S[-3 + k] + 64) >> 7), F the bank's row of the phase; in two dimensions the horizontal results, clipped
 *             samples, for rows -3 .. h + 3, then the vertical filter over those
 *   bilinear  S[0] + ((m (S[1] - S[0]) + 8) >> 4), not clipped; in two dimensions the horizontal results for rows 0 .. h
 *   put       dst = v;   avg  dst = (dst + v + 1) >> 1
 *   scaled    always two passes; the phase walks along a row as imx += dx, ioff += imx >> 4, imx &= 15 and down the rows in the same
 *             way (the running form of the reference; the kernel uses the closed form (mx + x dx) >> 4, & 15)
 * The filter rows are the subpel_filters of the VP9 bitstream specification, in FilterMode order (smooth, regular, sharp).
 * Batch op: the decoder's sequence (vp9_mc_template.c, vp9recon.c:299-551): the put member of table position [!!mx][!!my] (the scaled
 * put member for a reference whose steps are not 16, 16) from slot 0, for a compound op then the avg member from slot 1; source
 * samples through coordinates clamped to the reference plane (what emulated_edge_mc's windows give).
 */
#include <string.h>
#include "vp9mc_oracle.h"

static const int16_t SF[3][16][8] = {
    {   /* smooth */
      { 0, 0, 0, 128, 0, 0, 0, 0 }, { -3, -1, 32, 64, 38, 1, -3, 0 }, { -2, -2, 29, 63, 41, 2, -3, 0 }, { -2, -2, 26, 63, 43, 4, -4, 0 },
      { -2, -3, 24, 62, 46, 5, -4, 0 }, { -2, -3, 21, 60, 49, 7, -4, 0 }, { -1, -4, 18, 59, 51, 9, -4, 0 }, { -1, -4, 16, 57, 53, 12, -4, -1 },
      { -1, -4, 14, 55, 55, 14, -4, -1 }, { -1, -4, 12, 53, 57, 16, -4, -1 }, { 0, -4, 9, 51, 59, 18, -4, -1 }, { 0, -4, 7, 49, 60, 21, -3, -2 },
      { 0, -4, 5, 46, 62, 24, -3, -2 }, { 0, -4, 4, 43, 63, 26, -2, -2 }, { 0, -3, 2, 41, 63, 29, -2, -2 }, { 0, -3, 1, 38, 64, 32, -1, -3 },
    },
    {   /* regular */
      { 0, 0, 0, 128, 0, 0, 0, 0 }, { 0, 1, -5, 126, 8, -3, 1, 0 }, { -1, 3, -10, 122, 18, -6, 2, 0 }, { -1, 4, -13, 118, 27, -9, 3, -1 },
      { -1, 4, -16, 112, 37, -11, 4, -1 }, { -1, 5, -18, 105, 48, -14, 4, -1 }, { -1, 5, -19, 97, 58, -16, 5, -1 }, { -1, 6, -19, 88, 68, -18, 5, -1 },
      { -1, 6, -19, 78, 78, -19, 6, -1 }, { -1, 5, -18, 68, 88, -19, 6, -1 }, { -1, 5, -16, 58, 97, -19, 5, -1 }, { -1, 4, -14, 48, 105, -18, 5, -1 },
      { -1, 4, -11, 37, 112, -16, 4, -1 }, { -1, 3, -9, 27, 118, -13, 4, -1 }, { 0, 2, -6, 18, 122, -10, 3, -1 }, { 0, 1, -3, 8, 126, -5, 1, 0 },
    },
    {   /* sharp */
      { 0, 0, 0, 128, 0, 0, 0, 0 }, { -1, 3, -7, 127, 8, -3, 1, 0 }, { -2, 5, -13, 125, 17, -6, 3, -1 }, { -3, 7, -17, 121, 27, -10, 5, -2 },
      { -4, 9, -20, 115, 37, -13, 6, -2 }, { -4, 10, -23, 108, 48, -16, 8, -3 }, { -4, 10, -24, 100, 59, -19, 9, -3 }, { -4, 11, -24, 90, 70, -21, 10, -4 },
      { -4, 11, -23, 80, 80, -23, 11, -4 }, { -4, 10, -21, 70, 90, -24, 11, -4 }, { -3, 9, -19, 59, 100, -24, 10, -4 }, { -3, 8, -16, 48, 108, -23, 10, -4 },
      { -2, 6, -13, 37, 115, -20, 9, -4 }, { -2, 5, -10, 27, 121, -17, 7, -3 }, { -1, 3, -6, 17, 125, -13, 5, -2 }, { 0, 1, -3, 8, 127, -7, 3, -1 },
    },
};

/* the three 8-tap banks as [3][16][8] int16, in FilterMode order */
const int16_t *orc_vp9_subpel_filters(void) { return &SF[0][0][0]; }

static int sample(const uint8_t *src, ptrdiff_t stride, int hbd, int x, int y)
{
    const uint8_t *row = src + y * stride;
    return hbd ? ((const uint16_t *)row)[x] : row[x];
}
static int clipd(int v, int depth) { return v < 0 ? 0 : v > (1 << depth) - 1 ? (1 << depth) - 1 : v; }

/* one filtered sample from eight (8-tap: s[0..7] = positions -3..+4) or two (bilinear: s[3], s[4] = positions 0, +1) */
static int filt(int bank, int phase, const int *s, int depth)
{
    if (bank == 3) return s[3] + ((phase * (s[4] - s[3]) + 8) >> 4);
    int acc = 64;
    for (int k = 0; k < 8; k++) acc += SF[bank][phase][k] * s[k];
    return clipd(acc >> 7, depth);
}

static void store(void *dst, ptrdiff_t stride, int hbd, int x, int y, int v, int avg)
{
    uint8_t *row = (uint8_t *)dst + y * stride;
    if (hbd) ((uint16_t *)row)[x] = (uint16_t)(avg ? (((uint16_t *)row)[x] + v + 1) >> 1 : v);
    else row[x] = (uint8_t)(avg ? (row[x] + v + 1) >> 1 : v);
}

static int args_ok(int depth, int bank, int w, int h, int mx, int my)
{
    return (depth == 8 || depth == 10 || depth == 12) && bank >= 0 && bank <= 3 && (w == 4 || w == 8 || w == 16 || w == 32 || w == 64) &&
           h >= 1 && h <= 64 && mx >= 0 && mx <= 15 && my >= 0 && my <= 15;
}

/* mc[size of w][bank][avg][hdir][vdir](dst, dst_stride, src, src_stride, h, mx, my); strides in bytes; -1 for arguments outside the
 * reference's contract.  Reads only what the reference function reads: bilinear samples 0, +1 in a filtered direction, 8-tap -3..+4. */
int orc_vp9_mc(int depth, int bank, int avg, int hdir, int vdir, void *dst, ptrdiff_t dst_stride, const void *src_, ptrdiff_t src_stride,
               int w, int h, int mx, int my)
{
    const uint8_t *src = src_;
    const int hbd = depth > 8, lo = bank == 3 ? 3 : 0, hi = bank == 3 ? 5 : 8;     /* taps read: s[lo .. hi - 1] */
    static int tmp[(64 + 7) * 64];
    if (!args_ok(depth, bank, w, h, mx, my)) return -1;
    if (hdir && vdir)
        for (int y = lo - 3; y < h + hi - 4; y++)
            for (int x = 0; x < w; x++) {
                int s[8] = { 0 };
                for (int k = lo; k < hi; k++) s[k] = sample(src, src_stride, hbd, x - 3 + k, y);
                tmp[(y + 3) * 64 + x] = filt(bank, mx, s, depth);
            }
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++) {
            int s[8] = { 0 }, v;
            if (hdir && vdir) {
                for (int k = lo; k < hi; k++) s[k] = tmp[(y + k) * 64 + x];
                v = filt(bank, my, s, depth);
            } else if (hdir) {
                for (int k = lo; k < hi; k++) s[k] = sample(src, src_stride, hbd, x - 3 + k, y);
                v = filt(bank, mx, s, depth);
            } else if (vdir) {
                for (int k = lo; k < hi; k++) s[k] = sample(src, src_stride, hbd, x, y - 3 + k);
                v = filt(bank, my, s, depth);
            } else {
                v = sample(src, src_stride, hbd, x, y);
            }
            store(dst, dst_stride, hbd, x, y, v, avg);
        }
    return 0;
}

/* smc[size of w][bank][avg](dst, dst_stride, src, src_stride, h, mx, my, dx, dy), steps 1..32 */
int orc_vp9_smc(int depth, int bank, int avg, void *dst, ptrdiff_t dst_stride, const void *src_, ptrdiff_t src_stride, int w, int h, int mx,
                int my, int dx, int dy)
{
    const uint8_t *src = src_;
    const int hbd = depth > 8, lo = bank == 3 ? 3 : 0, hi = bank == 3 ? 5 : 8;
    static int tmp[135 * 64];
    if (!args_ok(depth, bank, w, h, mx, my) || dx < 1 || dx > 32 || dy < 1 || dy > 32) return -1;
    const int rows = (((h - 1) * dy + my) >> 4) + hi - lo;                          /* source rows lo - 3 .. */
    for (int y = 0; y < rows; y++) {
        int imx = mx, ioff = 0;
        for (int x = 0; x < w; x++) {
            int s[8] = { 0 };
            for (int k = lo; k < hi; k++) s[k] = sample(src, src_stride, hbd, ioff - 3 + k, y + lo - 3);
            tmp[y * 64 + x] = filt(bank, imx, s, depth);
            imx += dx;
            ioff += imx >> 4;
            imx &= 15;
        }
    }
    int row = 0;
    for (int y = 0; y < h; y++) {
        for (int x = 0; x < w; x++) {
            int s[8] = { 0 };
            for (int k = lo; k < hi; k++) s[k] = tmp[(row + k - lo) * 64 + x];
            store(dst, dst_stride, hbd, x, y, filt(bank, my, s, depth), avg);
        }
        my += dy;
        row += my >> 4;
        my &= 15;
    }
    return 0;
}

/* b200_vp9_mc_batch_device on host memory (refs[].data host addresses); returns the number of ops that wrote their block */
int64_t orc_vp9_mc_batch(int depth, int nrefs, const B200Vp9McRef *refs, int64_t nops, const B200Vp9McOp *ops, uint8_t *dst, ptrdiff_t dst_stride)
{
    const int bps = depth > 8 ? 2 : 1;
    static uint8_t win[(126 + 8) * (126 + 8) * 2];
    int64_t done = 0;
    for (int64_t i = 0; i < nops; i++) {
        const B200Vp9McOp *op = &ops[i];
        const int nslot = op->kind == B200_VP9_MC_COMPOUND ? 2 : 1;
        int ok = op->kind <= 1 && args_ok(depth, op->filter, op->w, op->h, 0, 0) && !(op->dst_off % bps);
        for (int r = 0; r < nslot; r++) ok = ok && op->ref[r] < nrefs && op->mx[r] <= 15 && op->my[r] <= 15;
        if (!ok) continue;
        for (int r = 0; r < nslot; r++) {
            const B200Vp9McRef *f = &refs[op->ref[r]];
            const int scaled = f->dx != 16 || f->dy != 16, mx = op->mx[r], my = op->my[r];
            /* the 8-tap window of the call, whatever the bank: the functions read a part of it */
            const int wc = (((op->w - 1) * f->dx + mx) >> 4) + 8, wr = (((op->h - 1) * f->dy + my) >> 4) + 8, wp = wc * bps;
            for (int y = 0; y < wr; y++)
                for (int x = 0; x < wc; x++) {
                    long long yy = (long long)op->y[r] - 3 + y, xx = (long long)op->x[r] - 3 + x;
                    yy = yy < 0 ? 0 : yy >= f->h ? f->h - 1 : yy;
                    xx = xx < 0 ? 0 : xx >= f->w ? f->w - 1 : xx;
                    memcpy(win + y * wp + x * bps, f->data + yy * f->stride + xx * bps, bps);
                }
            const uint8_t *src = win + 3 * wp + 3 * bps;
            if (scaled) orc_vp9_smc(depth, op->filter, r, dst + op->dst_off, dst_stride, src, wp, op->w, op->h, mx, my, f->dx, f->dy);
            else orc_vp9_mc(depth, op->filter, r, !!mx, !!my, dst + op->dst_off, dst_stride, src, wp, op->w, op->h, mx, my);
        }
        done++;
    }
    return done;
}
