# Builds oracle/_ref/libffref_hevcpred.so: the UNMODIFIED reference libavcodec/hevc/pred.c (HEVCPredContext: intra_pred and the
# members it calls, hevc/pred_template.c once per bit depth) and libavcodec/hevc/dsp.c (for add_residual), compiled where they lie
# under $(REF) with the generic-C configuration of oracle/ref/Makefile, plus ref_hevcpred.c (flat C ABI for the tests, the minimal
# decoder contexts intra_pred reads, and the compile-time layout check of B200HEVCPredContext).  `make -C oracle/ref` runs first (it
# writes the config.h used here and libffref.so, which dsp.c's other members link against).  Nothing is written into $(REF), no
# reference source is copied into this repository; output goes to oracle/_ref/ (git-ignored).
#     make -C oracle/ref -f hevcpred.mk
REF ?= /root/reference
OUT ?= ../_ref
CC  ?= gcc
INC := $(OUT)/include
CFLAGS := -std=c17 -O3 -fPIC -w -fno-math-errno -fno-signed-zeros -pthread \
  -D_ISOC11_SOURCE -D_FILE_OFFSET_BITS=64 -D_POSIX_C_SOURCE=200112 -D_XOPEN_SOURCE=600 -D_GNU_SOURCE \
  -DHAVE_AV_CONFIG_H -I$(INC) -I$(REF)

all: $(OUT)/libffref_hevcpred.so

$(OUT)/obj/hevcpred/pred.o: $(REF)/libavcodec/hevc/pred.c $(INC)/config.h
	@mkdir -p $(dir $@)
	@$(CC) $(CFLAGS) -c $< -o $@

$(OUT)/obj/hevcpred/dsp.o: $(REF)/libavcodec/hevc/dsp.c $(INC)/config.h
	@mkdir -p $(dir $@)
	@$(CC) $(CFLAGS) -c $< -o $@

$(OUT)/obj/hevcpred/ref_hevcpred.o: ref_hevcpred.c ../../include/b200dsp.h $(INC)/config.h
	@mkdir -p $(dir $@)
	@$(CC) $(CFLAGS) -c $< -o $@

HEVCPRED_OBJS := $(addprefix $(OUT)/obj/hevcpred/, pred.o dsp.o ref_hevcpred.o)

$(OUT)/libffref_hevcpred.so: $(HEVCPRED_OBJS) $(OUT)/libffref.so
	@$(CC) -shared -o $@ $(HEVCPRED_OBJS) -L$(OUT) -lffref -lm -pthread \
	   -Wl,-rpath,'$$ORIGIN' -Wl,-Bsymbolic -Wl,--no-undefined

clean:
	rm -rf $(OUT)/obj/hevcpred $(OUT)/libffref_hevcpred.so
