# Builds oracle/_ref/libffref_vp9intra.so: the UNMODIFIED reference libavcodec/vp9recon.c (the decoder's intra_recon and
# check_intra_mode, reached through ff_vp9_intra_recon_8bpp / _16bpp), vp9data.c (ff_vp9_bwh_tab, ff_vp9_intra_txfm_type), vp9dsp.c,
# vp9dsp_8bpp.c, vp9dsp_10bpp.c and vp9dsp_12bpp.c (the intra predictors and inverse transforms it calls), compiled where they lie under
# $(REF) with a generic-C configuration, plus ref_vp9intra.c (flat C ABI for the tests: one intra_pred member per call, and intra_recon
# block by block over a frame on a hand-set VP9Context / VP9TileData / VP9Block).  vp9recon.c includes vp9dec.h, which reaches
# get_bits.h and other libavcodec headers, so this build writes its own config.h from a file list that includes them (gen_config.sh
# defines every symbol the listed files mention).  libffref.so provides libavutil, so `make -C oracle/ref` runs first.  Nothing is
# written into $(REF), no reference source is copied into this repository; output goes to oracle/_ref/ (git-ignored).
#     make -C oracle/ref -f vp9intra.mk
REF ?= /root/reference
OUT ?= ../_ref
CC  ?= gcc
INC := $(OUT)/include_vp9intra
CFLAGS := -std=c17 -O3 -fPIC -w -fno-math-errno -fno-signed-zeros -pthread \
  -D_ISOC11_SOURCE -D_FILE_OFFSET_BITS=64 -D_POSIX_C_SOURCE=200112 -D_XOPEN_SOURCE=600 -D_GNU_SOURCE \
  -DHAVE_AV_CONFIG_H -I$(INC) -I$(REF)
CFG_FILES := libavcodec/vp9recon.c libavcodec/vp9data.c libavcodec/vp9data.h libavcodec/vp9dsp.c libavcodec/vp9dsp_template.c libavcodec/vp9dec.h libavcodec/vp9shared.h \
  libavcodec/vp9dsp.h libavcodec/vp9.h libavcodec/get_bits.h libavcodec/mathops.h libavcodec/videodsp.h libavcodec/vpx_rac.h \
  libavcodec/vp89_rac.h libavcodec/cbs_vp9.h libavcodec/cbs.h libavcodec/progressframe.h libavcodec/avcodec.h libavcodec/codec_id.h \
  libavcodec/bit_depth_template.c libavcodec/rnd_avg.h libavcodec/internal.h libavcodec/thread.h libavcodec/vlc.h

all: $(OUT)/libffref_vp9intra.so

$(INC)/config.h: gen_config.sh vp9intra.mk
	@./gen_config.sh $(REF) $(INC) $(CFG_FILES)

$(OUT)/obj/vp9intra/%.o: $(REF)/libavcodec/%.c $(INC)/config.h
	@mkdir -p $(dir $@)
	@$(CC) $(CFLAGS) -c $< -o $@

$(OUT)/obj/vp9intra/ref_vp9intra.o: ref_vp9intra.c ../../include/b200dsp.h $(INC)/config.h
	@mkdir -p $(dir $@)
	@$(CC) $(CFLAGS) -c $< -o $@

VP9INTRA_OBJS := $(addprefix $(OUT)/obj/vp9intra/, vp9recon.o vp9data.o vp9dsp.o vp9dsp_8bpp.o vp9dsp_10bpp.o vp9dsp_12bpp.o ref_vp9intra.o)

$(OUT)/libffref_vp9intra.so: $(VP9INTRA_OBJS) $(OUT)/libffref.so
	@$(CC) -shared -o $@ $(VP9INTRA_OBJS) -L$(OUT) -lffref -lm -pthread \
	   -Wl,-rpath,'$$ORIGIN' -Wl,-Bsymbolic -Wl,--no-undefined

clean:
	rm -rf $(OUT)/obj/vp9intra $(OUT)/include_vp9intra $(OUT)/libffref_vp9intra.so
