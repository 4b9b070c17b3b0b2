# Builds oracle/_ref/libffref_vp9lf.so: the UNMODIFIED reference libavcodec/vp9lpf.c (the decoder's per-superblock loop-filter driver),
# vp9dsp.c, vp9dsp_8bpp.c, vp9dsp_10bpp.c and vp9dsp_12bpp.c (the loop-filter functions it calls), compiled where they lie under $(REF)
# with a generic-C configuration, plus ref_vp9lf.c (flat C ABI for the tests: one loop-filter member per call, and ff_vp9_loopfilter_sb
# over a frame's superblocks in raster or wavefront order on a hand-set VP9Context).  vp9lpf.c includes vp9dec.h, which reaches
# get_bits.h and other libavcodec headers, so this build writes its own config.h from a file list that includes them (gen_config.sh
# defines every symbol the listed files mention).  libffref.so provides libavutil, so `make -C oracle/ref` runs first.  Nothing is
# written into $(REF), no reference source is copied into this repository; output goes to oracle/_ref/ (git-ignored).
#     make -C oracle/ref -f vp9lf.mk
REF ?= /root/reference
OUT ?= ../_ref
CC  ?= gcc
INC := $(OUT)/include_vp9lf
CFLAGS := -std=c17 -O3 -fPIC -w -fno-math-errno -fno-signed-zeros -pthread \
  -D_ISOC11_SOURCE -D_FILE_OFFSET_BITS=64 -D_POSIX_C_SOURCE=200112 -D_XOPEN_SOURCE=600 -D_GNU_SOURCE \
  -DHAVE_AV_CONFIG_H -I$(INC) -I$(REF)
CFG_FILES := libavcodec/vp9lpf.c libavcodec/vp9dsp.c libavcodec/vp9dsp_template.c libavcodec/vp9dec.h libavcodec/vp9shared.h \
  libavcodec/vp9dsp.h libavcodec/vp9.h libavcodec/get_bits.h libavcodec/mathops.h libavcodec/videodsp.h libavcodec/vpx_rac.h \
  libavcodec/vp89_rac.h libavcodec/cbs_vp9.h libavcodec/cbs.h libavcodec/progressframe.h libavcodec/avcodec.h libavcodec/codec_id.h \
  libavcodec/bit_depth_template.c libavcodec/rnd_avg.h libavcodec/internal.h libavcodec/thread.h libavcodec/vlc.h

all: $(OUT)/libffref_vp9lf.so

$(INC)/config.h: gen_config.sh vp9lf.mk
	@./gen_config.sh $(REF) $(INC) $(CFG_FILES)

$(OUT)/obj/vp9lf/%.o: $(REF)/libavcodec/%.c $(INC)/config.h
	@mkdir -p $(dir $@)
	@$(CC) $(CFLAGS) -c $< -o $@

$(OUT)/obj/vp9lf/ref_vp9lf.o: ref_vp9lf.c ../../include/b200dsp.h $(INC)/config.h
	@mkdir -p $(dir $@)
	@$(CC) $(CFLAGS) -c $< -o $@

VP9LF_OBJS := $(addprefix $(OUT)/obj/vp9lf/, vp9lpf.o vp9dsp.o vp9dsp_8bpp.o vp9dsp_10bpp.o vp9dsp_12bpp.o ref_vp9lf.o)

$(OUT)/libffref_vp9lf.so: $(VP9LF_OBJS) $(OUT)/libffref.so
	@$(CC) -shared -o $@ $(VP9LF_OBJS) -L$(OUT) -lffref -lm -pthread \
	   -Wl,-rpath,'$$ORIGIN' -Wl,-Bsymbolic -Wl,--no-undefined

clean:
	rm -rf $(OUT)/obj/vp9lf $(OUT)/include_vp9lf $(OUT)/libffref_vp9lf.so
