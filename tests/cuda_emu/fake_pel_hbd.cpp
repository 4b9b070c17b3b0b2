// fake_pel_hbd.cpp — TEST INFRASTRUCTURE ONLY: pel_hbd.cu's tables are installed by b200_h264qpel_init() in pel.cu (inline PTX, not part of
// the emulated build); this is the same call with the table lookup spelled out.
#include "common.h"
#include "pel_hbd.h"
extern "C" int emu_host_qpel_hbd_tab(int depth, int avg, int size_idx, int pos, uint8_t *dst, const uint8_t *src, long long stride)
{
    B200H264QpelContext c;
    memset(&c, 0, sizeof(c));
    if (!pel_hbd_fill(&c, depth)) return -38;
    (avg ? c.avg_h264_qpel_pixels_tab : c.put_h264_qpel_pixels_tab)[size_idx][pos](dst, src, (ptrdiff_t)stride);
    return 0;
}
extern "C" int emu_host_chroma_hbd_tab(int avg, int idx, uint8_t *dst, const uint8_t *src, long long stride, int h, int x, int y)
{
    B200H264ChromaContext c;
    pel_hbd_fill_chroma(&c);
    if (c.put_h264_chroma_pixels_tab[3] || c.avg_h264_chroma_pixels_tab[3]) return -1;        // stays NULL like the reference's
    (avg ? c.avg_h264_chroma_pixels_tab : c.put_h264_chroma_pixels_tab)[idx](dst, src, (ptrdiff_t)stride, h, x, y);
    return 0;
}
