# Builds oracle/_ref/libffref_vp9itxfm.so: the UNMODIFIED reference libavcodec/vp9dsp.c, vp9dsp_8bpp.c, vp9dsp_10bpp.c and
# vp9dsp_12bpp.c (each of the last three includes vp9dsp_template.c for its bit depth), compiled where they lie under $(REF) with the
# generic-C configuration of oracle/ref/Makefile, plus ref_vp9itxfm.c (flat C ABI for the tests: one itxfm_add member per call, the
# decoder's residual sequence for a batch, the table's pointer sharing).  libffref.so provides libavutil, so `make -C oracle/ref` runs
# first (it also writes the config.h used here).  Nothing is written into $(REF), no reference source is copied into this repository;
# output goes to oracle/_ref/ (git-ignored).
#     make -C oracle/ref -f vp9itxfm.mk
REF ?= /root/reference
OUT ?= ../_ref
CC  ?= gcc
INC := $(OUT)/include
CFLAGS := -std=c17 -O3 -fPIC -w -fno-math-errno -fno-signed-zeros -pthread \
  -D_ISOC11_SOURCE -D_FILE_OFFSET_BITS=64 -D_POSIX_C_SOURCE=200112 -D_XOPEN_SOURCE=600 -D_GNU_SOURCE \
  -DHAVE_AV_CONFIG_H -I$(INC) -I$(REF)

all: $(OUT)/libffref_vp9itxfm.so

$(OUT)/obj/vp9itxfm/%.o: $(REF)/libavcodec/%.c $(INC)/config.h
	@mkdir -p $(dir $@)
	@$(CC) $(CFLAGS) -c $< -o $@

$(OUT)/obj/vp9itxfm/ref_vp9itxfm.o: ref_vp9itxfm.c ../../include/b200dsp.h $(INC)/config.h
	@mkdir -p $(dir $@)
	@$(CC) $(CFLAGS) -c $< -o $@

VP9ITXFM_OBJS := $(addprefix $(OUT)/obj/vp9itxfm/, vp9dsp.o vp9dsp_8bpp.o vp9dsp_10bpp.o vp9dsp_12bpp.o ref_vp9itxfm.o)

$(OUT)/libffref_vp9itxfm.so: $(VP9ITXFM_OBJS) $(OUT)/libffref.so
	@$(CC) -shared -o $@ $(VP9ITXFM_OBJS) -L$(OUT) -lffref -lm -pthread \
	   -Wl,-rpath,'$$ORIGIN' -Wl,-Bsymbolic -Wl,--no-undefined

clean:
	rm -rf $(OUT)/obj/vp9itxfm $(OUT)/libffref_vp9itxfm.so
