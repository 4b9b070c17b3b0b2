# Builds oracle/_ref/libffref_vc1dsp.so (`make -f vc1dsp.mk vc1dsp`, after Makefile's `all`): the reference's VC-1 DSP,
# libavcodec/vc1dsp.c compiled unmodified where it lies, with startcode.c for ff_startcode_find_candidate_c, plus the shim ref_vc1dsp.c;
# hpeldsp.c, h264chroma.c, videodsp.c and idctdsp.c (the members the decoder's MC and residual sequences call besides VC1DSPContext's)
# come from libffref.so, which every feature library links against.  The same `feature` recipe, shared config.h and output layout as
# every library of Makefile.
include Makefile

vc1dsp_SRCS := libavcodec/vc1dsp.c libavcodec/startcode.c
vc1dsp_SHIMS := ref_vc1dsp.c
$(eval $(call feature,vc1dsp))

.PHONY: vc1dsp
vc1dsp: $(OUT)/libffref_vc1dsp.so
