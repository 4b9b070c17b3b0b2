// pel_hbd.h — h264qpel tables for 9 / 10 / 12 / 14 bit samples (pel_hbd.cu), installed by b200_h264qpel_init() in pel.cu
#pragma once
#include "common.h"

// fills both tables of c with the functions of that depth; false when the depth has none (ff_h264qpel_init knows 8, 9, 10, 12, 14)
bool pel_hbd_fill(B200H264QpelContext *c, int bit_depth);
// the 16-bit tables of ff_h264chroma_init (h264chroma.c:45-50)
void pel_hbd_fill_chroma(B200H264ChromaContext *c);
