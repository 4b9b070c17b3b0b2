/* TEST INFRASTRUCTURE — the reference's VP9 intra reconstruction (libavcodec/vp9recon.c with vp9data.c and the predictors and
 * inverse transforms of vp9dsp.c, vp9dsp_8bpp.c, vp9dsp_10bpp.c, vp9dsp_12bpp.c, compiled unmodified where they lie by
 * oracle/ref/vp9intra.mk into oracle/_ref/libffref_vp9intra.so) exposed through a flat C ABI: one intra_pred member of
 * ff_vp9dsp_init(.., bpp, 0) per call, and ff_vp9_intra_recon_{8,16}bpp block by block over a frame on a hand-set VP9Context /
 * VP9TileData / VP9Block, the way decode_b and decode_tiles drive it: dst or the tmp_* buffers by the emu rule of vp9block.c:1368-1386
 * with the copy-back of :1399-1430, and intra_pred_data copied at the end of each superblock row as vp9.c:1387-1398 does.
 * tests/vp9intralib.py loads it. */
#include <stdint.h>
#include <stddef.h>
#include <stdlib.h>
#include <string.h>

#include "config.h"
#include "libavutil/frame.h"
#include "libavcodec/avcodec.h"
#include "libavcodec/vp9dec.h"
#include "libavcodec/vp9data.h"
#include "../../include/b200dsp.h"

#define API __attribute__((visibility("default")))

_Static_assert(offsetof(VP9DSPContext, intra_pred) == offsetof(B200VP9DSPContext, intra_pred), "intra_pred offset");
_Static_assert(sizeof(((VP9DSPContext *)0)->intra_pred) == sizeof(((B200VP9DSPContext *)0)->intra_pred), "intra_pred size");

/* vp9recon.c's inter_recon refers to it; intra_recon never calls it */
void ff_progress_frame_await(const ProgressFrame *f, int progress) { (void)f; (void)progress; }

static VP9Context ctx;
static VP9TileData td;
static VP9Block blk;
static AVFrame frame;

API int ffref_vp9_intra_pred(int depth, int tx, int mode, uint8_t *dst, ptrdiff_t stride, const uint8_t *left, const uint8_t *top)
{
    static VP9DSPContext dsp;
    if ((depth != 8 && depth != 10 && depth != 12) || tx < 0 || tx > 3 || mode < 0 || mode >= N_INTRA_PRED_MODES) return -1;
    ff_vp9dsp_init(&dsp, depth, 0);
    dsp.intra_pred[tx][mode](dst, stride, left, top);
    return 0;
}

/* 1 if intra_pred[tx][mode] at `depth` is the same function as at depth 10 */
API int ffref_vp9_intra_shared10(int depth, int tx, int mode)
{
    static VP9DSPContext a, b;
    ff_vp9dsp_init(&a, depth, 0);
    ff_vp9dsp_init(&b, 10, 0);
    return a.intra_pred[tx][mode] == b.intra_pred[tx][mode];
}

/* One block per 16 ints of `blocks`, in decode order: row, col (8x8 units), bs, tx, uvtx, skip, mode[0..3], uvmode, tile_col_start,
 * intra, coefficient offsets (elements) of the luma, U and V blocks in `coef`.  eobs: 3 x 256 bytes per block (td->eob, uveob[0],
 * uveob[1], 16-bit little-endian values for transforms above 8x8).  Inter blocks (intra == 0) are skipped.  HOST planes; their line
 * sizes decide the emu path as in the decoder. */
API int ffref_vp9_intra_frame(int depth, int ss_h, int ss_v, int width, int height, uint8_t *const planes[3], ptrdiff_t ls_y, ptrdiff_t ls_uv,
                              int lossless, int nblocks, const int32_t *blocks, void *coef, uint8_t *eobs)
{
    if (depth != 8 && depth != 10 && depth != 12) return -1;
    const int bps = depth > 8 ? 2 : 1;
    memset(&ctx, 0, sizeof(ctx));
    memset(&td, 0, sizeof(td));
    ff_vp9dsp_init(&ctx.dsp, depth, 0);
    ctx.bytesperpixel = bps;
    ctx.ss_h = ss_h;
    ctx.ss_v = ss_v;
    ctx.cols = (width + 7) >> 3;
    ctx.rows = (height + 7) >> 3;
    ctx.s.h.bpp = depth;
    ctx.s.h.lossless = lossless;
    ctx.s.frames[CUR_FRAME].tf.f = &frame;
    for (int p = 0; p < 3; p++) frame.data[p] = planes[p];
    frame.linesize[0] = (int)ls_y;
    frame.linesize[1] = frame.linesize[2] = (int)ls_uv;
    for (int p = 0; p < 3; p++) ctx.intra_pred_data[p] = calloc((size_t)ctx.cols * 64 * bps + 64, 1);
    td.s = &ctx;
    td.b = &blk;
    const int cs = depth > 8 ? 4 : 2;
    for (int k = 0; k < nblocks; k++) {
        const int32_t *r = blocks + 16 * k;
        const int row = r[0], col = r[1];
        if (r[12]) {
            memset(&blk, 0, sizeof(blk));
            blk.bs = r[2];
            blk.tx = r[3];
            blk.uvtx = r[4];
            blk.skip = r[5];
            for (int i = 0; i < 4; i++) blk.mode[i] = r[6 + i];
            blk.uvmode = r[10];
            blk.intra = 1;
            td.tile_col_start = r[11];
            td.row = row;
            td.row7 = row & 7;
            td.col = col;
            td.col7 = col & 7;
            td.block = (int16_t *)((uint8_t *)coef + (size_t)r[13] * cs);
            td.uvblock[0] = (int16_t *)((uint8_t *)coef + (size_t)r[14] * cs);
            td.uvblock[1] = (int16_t *)((uint8_t *)coef + (size_t)r[15] * cs);
            td.eob = eobs + (size_t)k * 768;
            td.uveob[0] = td.eob + 256;
            td.uveob[1] = td.eob + 512;
            /* vp9block.c:1368-1386 */
            const int w4 = ff_vp9_bwh_tab[1][blk.bs][0], h4 = ff_vp9_bwh_tab[1][blk.bs][1];
            const ptrdiff_t yoff = (ptrdiff_t)row * 8 * ls_y + (ptrdiff_t)col * 8 * bps;
            const ptrdiff_t uvoff = (ptrdiff_t)row * (8 >> ss_v) * ls_uv + (ptrdiff_t)col * (8 >> ss_h) * bps;
            int emu[2];
            emu[0] = (col + w4) * 8 * bps > frame.linesize[0] || (row + h4) > (int)ctx.rows;
            emu[1] = ((col + w4) * 8 >> ss_h) * bps > frame.linesize[1] || (row + h4) > (int)ctx.rows;
            if (emu[0]) {
                td.dst[0] = td.tmp_y;
                td.y_stride = 128;
            } else {
                td.dst[0] = frame.data[0] + yoff;
                td.y_stride = frame.linesize[0];
            }
            if (emu[1]) {
                td.dst[1] = td.tmp_uv[0];
                td.dst[2] = td.tmp_uv[1];
                td.uv_stride = 128;
            } else {
                td.dst[1] = frame.data[1] + uvoff;
                td.dst[2] = frame.data[2] + uvoff;
                td.uv_stride = frame.linesize[1];
            }
            if (bps > 1) ff_vp9_intra_recon_16bpp(&td, yoff, uvoff);
            else ff_vp9_intra_recon_8bpp(&td, yoff, uvoff);
            /* the copy-back of vp9block.c:1399-1430: whole rows of the visible part (the mc[n][0][0][0][0] copies, put with no filter) */
            if (emu[0]) {
                const int w = FFMIN((int)ctx.cols - col, w4) * 8, h = FFMIN((int)ctx.rows - row, h4) * 8;
                for (int y = 0; y < h; y++) memcpy(frame.data[0] + yoff + (ptrdiff_t)y * ls_y, td.tmp_y + y * 128, (size_t)w * bps);
            }
            if (emu[1]) {
                const int w = FFMIN((int)ctx.cols - col, w4) * 8 >> ss_h, h = FFMIN((int)ctx.rows - row, h4) * 8 >> ss_v;
                for (int p = 0; p < 2; p++)
                    for (int y = 0; y < h; y++)
                        memcpy(frame.data[1 + p] + uvoff + (ptrdiff_t)y * ls_uv, td.tmp_uv[p] + y * 128, (size_t)w * bps);
            }
        }
        /* vp9.c:1387-1398 at the end of a superblock row */
        const int sbr = row >> 3;
        if (k + 1 == nblocks || (blocks[16 * (k + 1)] >> 3) != sbr) {
            const int r8 = sbr * 8;
            if (r8 + 8 < (int)ctx.rows) {
                const ptrdiff_t yo = (ptrdiff_t)r8 * 8 * ls_y, uvo = (ptrdiff_t)r8 * (8 >> ss_v) * ls_uv;
                memcpy(ctx.intra_pred_data[0], frame.data[0] + yo + 63 * ls_y, 8 * ctx.cols * bps);
                memcpy(ctx.intra_pred_data[1], frame.data[1] + uvo + ((64 >> ss_v) - 1) * ls_uv, 8 * ctx.cols * bps >> ss_h);
                memcpy(ctx.intra_pred_data[2], frame.data[2] + uvo + ((64 >> ss_v) - 1) * ls_uv, 8 * ctx.cols * bps >> ss_h);
            }
        }
    }
    for (int p = 0; p < 3; p++) free(ctx.intra_pred_data[p]);
    return 0;
}
