/* TEST INFRASTRUCTURE — the reference's VP9 inverse transforms (libavcodec/vp9dsp.c, vp9dsp_8bpp.c, vp9dsp_10bpp.c, vp9dsp_12bpp.c,
 * compiled unmodified where they lie by oracle/ref/vp9itxfm.mk into oracle/_ref/libffref_vp9itxfm.so) exposed through a flat C ABI:
 * one itxfm_add member of ff_vp9dsp_init(.., bpp, 1) per call, the decoder's residual sequence for a batch of B200Vp9TxOp (the member
 * on a copy of each op's coefficients, so the batch's coefficient buffer stays as it was, like the product's read-only entry), and
 * the pointer-sharing facts of the table (vp9dsp_template.c:1755-1778).  tests/vp9itxfmlib.py loads it. */
#include <stdint.h>
#include <stddef.h>
#include <string.h>

#include "config.h"
#include "libavcodec/vp9dsp.h"
#include "../../include/b200dsp.h"

#define API __attribute__((visibility("default")))

_Static_assert(DCT_DCT == 0 && DCT_ADST == 1 && ADST_DCT == 2 && ADST_ADST == 3, "TxfmType order");
_Static_assert(TX_4X4 == 0 && TX_8X8 == 1 && TX_16X16 == 2 && TX_32X32 == 3, "TxfmMode order");

static VP9DSPContext *ref_vp9dsp(int depth)
{
    static VP9DSPContext c[13];
    static int ok[13];
    if (depth != 8 && depth != 10 && depth != 12) return NULL;
    if (!ok[depth]) { ff_vp9dsp_init(&c[depth], depth, 1); ok[depth] = 1; }
    return &c[depth];
}

/* itxfm_add[tx][type] of ff_vp9dsp_init(depth); block holds int16 (8 bit) / int32 (10 / 12 bit) coefficients */
API int ffref_vp9_itxfm(int depth, int tx, int type, uint8_t *dst, ptrdiff_t stride, void *block, int eob)
{
    VP9DSPContext *c = ref_vp9dsp(depth);
    if (!c || tx < 0 || tx > 4 || type < 0 || type > 3) return -1;
    c->itxfm_add[tx][type](dst, stride, (int16_t *)block, eob);
    return 0;
}

/* 1 if [0..2][*] are 12 distinct functions and every slot of [3] and of [4] is one function each (distinct from all others) */
API int ffref_vp9_itxfm_shared(int depth)
{
    VP9DSPContext *c = ref_vp9dsp(depth);
    if (!c) return -1;
    for (int tx = 3; tx < 5; tx++)
        for (int t = 1; t < 4; t++)
            if (c->itxfm_add[tx][t] != c->itxfm_add[tx][0]) return 0;
    for (int a = 0; a < 20; a++)
        for (int b = 0; b < a; b++) {
            const int same_row = a / 4 == b / 4 && a / 4 >= 3;
            if ((c->itxfm_add[a / 4][a % 4] == c->itxfm_add[b / 4][b % 4]) != same_row) return 0;
        }
    return 1;
}

/* the decoder's sequence for each op of a batch (the same op guard as the product; coef is a host address and stays unchanged: each
 * member call works on a copy of its op's coefficients); returns the number of ops that wrote their block */
API int64_t ffref_vp9_itxfm_batch(int depth, int64_t nops, const B200Vp9TxOp *ops, const void *coef, uint8_t *dst, ptrdiff_t dst_stride)
{
    VP9DSPContext *c = ref_vp9dsp(depth);
    const int bps = depth > 8 ? 2 : 1, cs = depth > 8 ? 4 : 2;
    int64_t done = 0;
    static int32_t block[32 * 32];
    if (!c) return -1;
    for (int64_t i = 0; i < nops; i++) {
        const B200Vp9TxOp *op = &ops[i];
        if (op->tx > 4 || op->type > 3 || (op->coef_off & 15) || (op->dst_off % (4 * bps))) continue;
        const int n = op->tx == 4 ? 4 : 4 << op->tx;
        memcpy(block, (const uint8_t *)coef + op->coef_off * cs, (size_t)n * n * cs);
        c->itxfm_add[op->tx][op->type](dst + op->dst_off, dst_stride, (int16_t *)block, op->eob);
        done++;
    }
    return done;
}
