/* TEST INFRASTRUCTURE — the reference's HEVC residual members (libavcodec/hevc/dsp.c, compiled unmodified where it lies by
 * oracle/ref/Makefile into oracle/_ref/libffref_hevcidct.so) exposed through a flat C ABI: one member per call, and the decoder's
 * per-transform-unit sequence (hevc/cabac.c:1550-1592, then add_residual) for a batch of B200HevcTuOp, each op on a copy of its
 * coefficients.  tests/hevcidctlib.py loads it. */
#include <stdint.h>
#include <stddef.h>
#include <string.h>

#include "config.h"
#include "libavcodec/hevc/dsp.h"
#include "../../include/b200dsp.h"

#define API __attribute__((visibility("default")))

_Static_assert(sizeof(B200HevcTuOp) == 32, "B200HevcTuOp");

static HEVCDSPContext *ref_hevcdsp(int depth)
{
    static HEVCDSPContext c[13];
    static int ok[13];
    if (depth != 8 && depth != 9 && depth != 10 && depth != 12) return NULL;
    if (!ok[depth]) { ff_hevc_dsp_init(&c[depth], depth); ok[depth] = 1; }
    return &c[depth];
}

/* fn: 0 idct[log2 - 2](c, arg), 1 idct_dc[log2 - 2], 2 transform_4x4_luma, 3 dequant(c, log2), 4 transform_rdpcm(c, log2, arg) */
API int ffref_hevc_tx(int depth, int fn, int log2, int16_t *c, int arg)
{
    HEVCDSPContext *h = ref_hevcdsp(depth);
    if (!h || log2 < 2 || log2 > 5 || (fn == 2 && log2 != 2)) return -1;
    switch (fn) {
    case 0: h->idct[log2 - 2](c, arg); return 0;
    case 1: h->idct_dc[log2 - 2](c); return 0;
    case 2: h->transform_4x4_luma(c); return 0;
    case 3: h->dequant(c, log2); return 0;
    case 4: h->transform_rdpcm(c, log2, arg); return 0;
    }
    return -1;
}

API int ffref_hevc_add_residual(int depth, int log2, uint8_t *dst, const int16_t *res, ptrdiff_t stride)
{
    HEVCDSPContext *h = ref_hevcdsp(depth);
    if (!h || log2 < 2 || log2 > 5) return -1;
    h->add_residual[log2 - 2](dst, res, stride);
    return 0;
}

/* the decoder's calls for each op of a batch (the same op guard as the product); returns the number of ops that wrote their block */
API int64_t ffref_hevc_tu_batch(int depth, int64_t nops, const B200HevcTuOp *ops, const int16_t *coef, uint8_t *dst, ptrdiff_t dst_stride)
{
    HEVCDSPContext *h = ref_hevcdsp(depth);
    const int bps = depth > 8 ? 2 : 1;
    int16_t coeffs[32 * 32];
    int64_t done = 0;
    if (!h) return -1;
    for (int64_t i = 0; i < nops; i++) {
        const B200HevcTuOp *op = &ops[i];
        const int log2 = op->log2_size, kind = op->kind, f = op->flags;
        if (log2 < 2 || log2 > 5 || kind > B200_HEVC_TU_BYPASS || (kind == B200_HEVC_TU_DST4 && log2 != 2) || (op->coef_off & 7) ||
            (op->dst_off % (4 * bps)))
            continue;
        memcpy(coeffs, coef + op->coef_off, sizeof(int16_t) << (2 * log2));
        switch (kind) {
        case B200_HEVC_TU_BYPASS:                                            /* cabac.c:1550-1556 */
            if (f & B200_HEVC_TU_RDPCM) h->transform_rdpcm(coeffs, log2, !!(f & B200_HEVC_TU_RDPCM_VER));
            break;
        case B200_HEVC_TU_SKIP:                                              /* cabac.c:1558-1575 */
            if ((f & B200_HEVC_TU_ROTATE) && log2 == 2)
                for (int j = 0; j < 8; j++) { const int16_t t = coeffs[j]; coeffs[j] = coeffs[16 - j - 1]; coeffs[16 - j - 1] = t; }
            h->dequant(coeffs, log2);
            if (f & B200_HEVC_TU_RDPCM) h->transform_rdpcm(coeffs, log2, !!(f & B200_HEVC_TU_RDPCM_VER));
            break;
        case B200_HEVC_TU_DST4: h->transform_4x4_luma(coeffs); break;       /* cabac.c:1576-1577 */
        case B200_HEVC_TU_IDCT_DC: h->idct_dc[log2 - 2](coeffs); break;     /* cabac.c:1579-1580 */
        default: h->idct[log2 - 2](coeffs, op->col_limit); break;           /* cabac.c:1581-1582 */
        }
        h->add_residual[log2 - 2](dst + op->dst_off, coeffs, dst_stride);  /* cabac.c:1592 */
        done++;
    }
    return done;
}
