# Builds oracle/_ref/libffref_vp8lf.so (`make -f vp8lf.mk vp8lf`, after Makefile's `all`): the reference's VP8 / VP7 loop filter,
# libavcodec/vp8dsp.c compiled unmodified where it lies, with mathtables.c for ff_crop_tab, plus the shim ref_vp8lf.c (the ten
# loop-filter members of each context, the decoder's per-macroblock filter sequence around them, the contexts' pointers); the same
# `feature` recipe, shared config.h and output layout as every library of Makefile.  Like vp8dsp.mk, it puts CONFIG_VP7_DECODER and
# CONFIG_VP8_DECODER on this library's compile lines only, because the shared $(INC)/config.h does not define them.
include Makefile

vp8lf_SRCS := libavcodec/vp8dsp.c libavcodec/mathtables.c
vp8lf_SHIMS := ref_vp8lf.c
$(eval $(call feature,vp8lf))
$(vp8lf_REFOBJS) $(vp8lf_SHIMOBJS): CFLAGS += -DCONFIG_VP7_DECODER=1 -DCONFIG_VP8_DECODER=1

.PHONY: vp8lf
vp8lf: $(OUT)/libffref_vp8lf.so
