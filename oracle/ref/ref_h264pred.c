/* TEST INFRASTRUCTURE — the reference's H.264 intra prediction (libavcodec/h264pred.c, compiled unmodified where it lies by
 * oracle/ref/Makefile into oracle/_ref/libffref_h264pred.so, next to libffref.so which it links against for ff_crop_tab and
 * libavutil) exposed through a flat C ABI, plus the compile-time proof that include/b200dsp.h's B200H264PredContext can be copied
 * member for member into H264PredContext (same size, member offsets and function-pointer types) and that B200_CODEC_ID_H264 is
 * AV_CODEC_ID_H264.  tests/h264predlib.py loads it and reads the marker below. */
#include <stdint.h>
#include <stddef.h>
#include <string.h>

#include "config.h"
#include "libavcodec/codec_id.h"
#include "libavcodec/h264pred.h"
#include "../../include/b200dsp.h"

#define API __attribute__((visibility("default")))

#define SAME_OFF(A, B, m)  _Static_assert(offsetof(A, m) == offsetof(B, m), "offset of " #m " in " #A " / " #B)
#define SAME_TYPE(A, B, m) _Static_assert(__builtin_types_compatible_p(__typeof__(((A *)0)->m), __typeof__(((B *)0)->m)), "type of " #m " in " #A " / " #B)
#define SAME(A, B, m)      SAME_OFF(A, B, m); SAME_TYPE(A, B, m)

/* H264PredContext, libavcodec/h264pred.h:94-114 */
_Static_assert(sizeof(H264PredContext) == sizeof(B200H264PredContext), "size of H264PredContext / B200H264PredContext");
SAME(H264PredContext, B200H264PredContext, pred4x4);
SAME(H264PredContext, B200H264PredContext, pred8x8l);
SAME(H264PredContext, B200H264PredContext, pred8x8);
SAME(H264PredContext, B200H264PredContext, pred16x16);
SAME(H264PredContext, B200H264PredContext, pred4x4_add);
SAME(H264PredContext, B200H264PredContext, pred8x8l_add);
SAME(H264PredContext, B200H264PredContext, pred8x8l_filter_add);
SAME(H264PredContext, B200H264PredContext, pred8x8_add);
SAME(H264PredContext, B200H264PredContext, pred16x16_add);
_Static_assert(AV_CODEC_ID_H264 == B200_CODEC_ID_H264, "codec id of H.264");

API const char ffref_h264pred_layout_check[] = "b200dsp.h B200H264PredContext matches H264PredContext";

/* ------------------------------------------------------------------ H.264 intra prediction ----------------------- */

static H264PredContext *ref_h264pred(int depth, int idc)
{
    static H264PredContext c[15][4];
    static int ok[15][4];
    if ((depth != 8 && depth != 9 && depth != 10 && depth != 12 && depth != 14) || idc < 0 || idc > 3) return NULL;
    if (!ok[depth][idc]) {
        memset(&c[depth][idc], 0, sizeof(H264PredContext));      /* ff_h264_pred_init only sets the members it fills */
        ff_h264_pred_init(&c[depth][idc], AV_CODEC_ID_H264, depth, idc);
        ok[depth][idc] = 1;
    }
    return &c[depth][idc];
}

/* one member of ff_h264_pred_init(AV_CODEC_ID_H264, depth, idc); table numbering as orc_h264_pred (oracle/oracle.h): 0 pred4x4,
 * 1 pred8x8l, 2 pred8x8, 3 pred16x16, 4 pred4x4_add, 5 pred8x8l_add, 6 pred8x8l_filter_add, 7 pred8x8_add, 8 pred16x16_add.
 * flags bit 0 / 1 become the decoder's has_topleft 0x8000 / has_topright 0x4000.  -1 for a NULL member. */
API int ffref_h264_pred(int depth, int idc, int table, int mode, uint8_t *pix, const uint8_t *topright, int flags, int16_t *block,
                        const int *block_offset, ptrdiff_t stride)
{
    H264PredContext *h = ref_h264pred(depth, idc);
    const int tl = flags & 1 ? 0x8000 : 0, tr = flags & 2 ? 0x4000 : 0;
    if (!h || mode < 0) return -1;
    switch (table) {
    case 0: if (mode >= 15 || !h->pred4x4[mode]) return -1; h->pred4x4[mode](pix, topright, stride); return 0;
    case 1: if (mode >= 12 || !h->pred8x8l[mode]) return -1; h->pred8x8l[mode](pix, tl, tr, stride); return 0;
    case 2: if (mode >= 11 || !h->pred8x8[mode]) return -1; h->pred8x8[mode](pix, stride); return 0;
    case 3: if (mode >= 9 || !h->pred16x16[mode]) return -1; h->pred16x16[mode](pix, stride); return 0;
    case 4: if (mode >= 2 || !h->pred4x4_add[mode]) return -1; h->pred4x4_add[mode](pix, block, stride); return 0;
    case 5: if (mode >= 2 || !h->pred8x8l_add[mode]) return -1; h->pred8x8l_add[mode](pix, block, stride); return 0;
    case 6: if (mode >= 2 || !h->pred8x8l_filter_add[mode]) return -1; h->pred8x8l_filter_add[mode](pix, block, tl, tr, stride); return 0;
    case 7: if (mode >= 3 || !h->pred8x8_add[mode]) return -1; h->pred8x8_add[mode](pix, block_offset, block, stride); return 0;
    case 8: if (mode >= 3 || !h->pred16x16_add[mode]) return -1; h->pred16x16_add[mode](pix, block_offset, block, stride); return 0;
    }
    return -1;
}

/* which members ff_h264_pred_init(AV_CODEC_ID_H264, depth, idc) fills: mask[i] = 0 / 1 for the 63 function pointers in member order */
API int ffref_h264_pred_members(int depth, int idc, uint8_t *mask)
{
    H264PredContext *h = ref_h264pred(depth, idc);
    if (!h) return -1;
    void **p = (void **)h;
    for (size_t i = 0; i < sizeof(*h) / sizeof(void *); i++) mask[i] = p[i] != NULL;
    return (int)(sizeof(*h) / sizeof(void *));
}
