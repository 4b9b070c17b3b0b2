# Builds oracle/_ref/libffref_hevcdbk.so: the UNMODIFIED reference libavcodec/hevc/dsp.c (its loop-filter members: hevc/dsp_template.c
# once per bit depth), compiled where it lies under $(REF) with the generic-C configuration of oracle/ref/Makefile, plus
# ref_hevcdbk.c (flat C ABI for the tests and the decoder's CTB-by-CTB deblocking order).  `make -C oracle/ref` runs first (it writes
# the config.h used here and libffref.so, which dsp.c's other members link against).  Nothing is written into $(REF), no reference
# source is copied into this repository; output goes to oracle/_ref/ (git-ignored).
#     make -C oracle/ref -f hevcdbk.mk
REF ?= /root/reference
OUT ?= ../_ref
CC  ?= gcc
INC := $(OUT)/include
CFLAGS := -std=c17 -O3 -fPIC -w -fno-math-errno -fno-signed-zeros -pthread \
  -D_ISOC11_SOURCE -D_FILE_OFFSET_BITS=64 -D_POSIX_C_SOURCE=200112 -D_XOPEN_SOURCE=600 -D_GNU_SOURCE \
  -DHAVE_AV_CONFIG_H -I$(INC) -I$(REF)

all: $(OUT)/libffref_hevcdbk.so

$(OUT)/obj/hevcdbk/dsp.o: $(REF)/libavcodec/hevc/dsp.c $(INC)/config.h
	@mkdir -p $(dir $@)
	@$(CC) $(CFLAGS) -c $< -o $@

$(OUT)/obj/hevcdbk/ref_hevcdbk.o: ref_hevcdbk.c ../../include/b200dsp.h $(INC)/config.h
	@mkdir -p $(dir $@)
	@$(CC) $(CFLAGS) -c $< -o $@

HEVCDBK_OBJS := $(addprefix $(OUT)/obj/hevcdbk/, dsp.o ref_hevcdbk.o)

$(OUT)/libffref_hevcdbk.so: $(HEVCDBK_OBJS) $(OUT)/libffref.so
	@$(CC) -shared -o $@ $(HEVCDBK_OBJS) -L$(OUT) -lffref -lm -pthread \
	   -Wl,-rpath,'$$ORIGIN' -Wl,-Bsymbolic -Wl,--no-undefined

clean:
	rm -rf $(OUT)/obj/hevcdbk $(OUT)/libffref_hevcdbk.so
