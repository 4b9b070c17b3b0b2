# Builds oracle/_ref/libffref_vp8dsp.so (`make -f vp8dsp.mk vp8dsp`, after Makefile's `all`): the reference's VP8 / VP7 DSP,
# libavcodec/vp8dsp.c compiled unmodified where it lies, with mathtables.c for ff_crop_tab, plus the shim ref_vp8dsp.c; the same
# `feature` recipe, shared config.h and output layout as every library of Makefile.
# vp8dsp.c builds its VP7 and VP8 functions only under CONFIG_VP7_DECODER / CONFIG_VP8_DECODER.  The shared $(INC)/config.h does not
# define them (gen_config.sh would define them to 0 for a config.h made from a list naming vp8dsp.c), so this library's objects get
# both on their compile line; no other library's compile line changes.
include Makefile

vp8dsp_SRCS := libavcodec/vp8dsp.c libavcodec/mathtables.c
vp8dsp_SHIMS := ref_vp8dsp.c
$(eval $(call feature,vp8dsp))
$(vp8dsp_REFOBJS) $(vp8dsp_SHIMOBJS): CFLAGS += -DCONFIG_VP7_DECODER=1 -DCONFIG_VP8_DECODER=1

.PHONY: vp8dsp
vp8dsp: $(OUT)/libffref_vp8dsp.so
