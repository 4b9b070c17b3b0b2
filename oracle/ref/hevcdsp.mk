# Builds oracle/_ref/libffref_hevcdsp.so: the UNMODIFIED reference libavcodec/hevc/dsp.c (which includes hevc/dsp_template.c and
# h26x/h2656_inter_template.c once per bit depth), compiled where it lies under $(REF) with the generic-C configuration of
# oracle/ref/Makefile, plus ref_hevcdsp.c (flat C ABI for the tests, the decoder's batch sequence, and the layout check of
# B200HEVCDSPContext).  emulated_edge_mc comes from libffref.so, so `make -C oracle/ref` runs first (it also writes the config.h
# used here).  Nothing is written into $(REF), no reference source is copied into this repository; output goes to oracle/_ref/
# (git-ignored).
#     make -C oracle/ref -f hevcdsp.mk
REF ?= /root/reference
OUT ?= ../_ref
CC  ?= gcc
INC := $(OUT)/include
CFLAGS := -std=c17 -O3 -fPIC -w -fno-math-errno -fno-signed-zeros -pthread \
  -D_ISOC11_SOURCE -D_FILE_OFFSET_BITS=64 -D_POSIX_C_SOURCE=200112 -D_XOPEN_SOURCE=600 -D_GNU_SOURCE \
  -DHAVE_AV_CONFIG_H -I$(INC) -I$(REF)

all: $(OUT)/libffref_hevcdsp.so

$(OUT)/obj/hevcdsp/dsp.o: $(REF)/libavcodec/hevc/dsp.c $(INC)/config.h
	@mkdir -p $(dir $@)
	@$(CC) $(CFLAGS) -c $< -o $@

$(OUT)/obj/hevcdsp/ref_hevcdsp.o: ref_hevcdsp.c ../../include/b200dsp.h $(INC)/config.h
	@mkdir -p $(dir $@)
	@$(CC) $(CFLAGS) -c $< -o $@

HEVCDSP_OBJS := $(addprefix $(OUT)/obj/hevcdsp/, dsp.o ref_hevcdsp.o)

$(OUT)/libffref_hevcdsp.so: $(HEVCDSP_OBJS) $(OUT)/libffref.so
	@$(CC) -shared -o $@ $(HEVCDSP_OBJS) -L$(OUT) -lffref -lm -pthread \
	   -Wl,-rpath,'$$ORIGIN' -Wl,-Bsymbolic -Wl,--no-undefined

clean:
	rm -rf $(OUT)/obj/hevcdsp $(OUT)/libffref_hevcdsp.so
