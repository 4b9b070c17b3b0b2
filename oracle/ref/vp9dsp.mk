# Builds oracle/_ref/libffref_vp9dsp.so: the UNMODIFIED reference libavcodec/vp9dsp.c, vp9dsp_8bpp.c, vp9dsp_10bpp.c and
# vp9dsp_12bpp.c (each of the last three includes vp9dsp_template.c for its bit depth), compiled where they lie under $(REF) with the
# generic-C configuration of oracle/ref/Makefile, plus ref_vp9dsp.c (flat C ABI for the tests, the decoder's batch sequence, and the
# layout check of B200VP9DSPContext).  emulated_edge_mc comes from libffref.so, so `make -C oracle/ref` runs first (it also writes the
# config.h used here).  Nothing is written into $(REF), no reference source is copied into this repository; output goes to
# oracle/_ref/ (git-ignored).
#     make -C oracle/ref -f vp9dsp.mk
REF ?= /root/reference
OUT ?= ../_ref
CC  ?= gcc
INC := $(OUT)/include
CFLAGS := -std=c17 -O3 -fPIC -w -fno-math-errno -fno-signed-zeros -pthread \
  -D_ISOC11_SOURCE -D_FILE_OFFSET_BITS=64 -D_POSIX_C_SOURCE=200112 -D_XOPEN_SOURCE=600 -D_GNU_SOURCE \
  -DHAVE_AV_CONFIG_H -I$(INC) -I$(REF)

all: $(OUT)/libffref_vp9dsp.so

$(OUT)/obj/vp9dsp/%.o: $(REF)/libavcodec/%.c $(INC)/config.h
	@mkdir -p $(dir $@)
	@$(CC) $(CFLAGS) -c $< -o $@

$(OUT)/obj/vp9dsp/ref_vp9dsp.o: ref_vp9dsp.c ../../include/b200dsp.h $(INC)/config.h
	@mkdir -p $(dir $@)
	@$(CC) $(CFLAGS) -c $< -o $@

VP9DSP_OBJS := $(addprefix $(OUT)/obj/vp9dsp/, vp9dsp.o vp9dsp_8bpp.o vp9dsp_10bpp.o vp9dsp_12bpp.o ref_vp9dsp.o)

$(OUT)/libffref_vp9dsp.so: $(VP9DSP_OBJS) $(OUT)/libffref.so
	@$(CC) -shared -o $@ $(VP9DSP_OBJS) -L$(OUT) -lffref -lm -pthread \
	   -Wl,-rpath,'$$ORIGIN' -Wl,-Bsymbolic -Wl,--no-undefined

clean:
	rm -rf $(OUT)/obj/vp9dsp $(OUT)/libffref_vp9dsp.so
