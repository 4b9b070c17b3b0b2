# Builds oracle/_ref/libffref_hevcintra.so: the UNMODIFIED reference libavcodec/hevc/pred.c (intra_pred) and libavcodec/hevc/dsp.c (the
# residual members), compiled where they lie under $(REF) with the generic-C configuration of oracle/ref/Makefile, plus ref_hevcidct.c
# (its ffref_hevc_tu_batch: the decoder's per-transform-unit sequence) and ref_hevcintra.c (the whole picture in decode order over minimal
# decoder contexts).  `make -C oracle/ref` runs first (it writes the config.h used here and libffref.so, which dsp.c's other members link
# against).  Nothing is written into $(REF), no reference source is copied into this repository; output goes to oracle/_ref/ (git-ignored).
#     make -C oracle/ref -f hevcintra.mk
REF ?= /root/reference
OUT ?= ../_ref
CC  ?= gcc
INC := $(OUT)/include
CFLAGS := -std=c17 -O3 -fPIC -w -fno-math-errno -fno-signed-zeros -pthread \
  -D_ISOC11_SOURCE -D_FILE_OFFSET_BITS=64 -D_POSIX_C_SOURCE=200112 -D_XOPEN_SOURCE=600 -D_GNU_SOURCE \
  -DHAVE_AV_CONFIG_H -I$(INC) -I$(REF)

all: $(OUT)/libffref_hevcintra.so

$(OUT)/obj/hevcintra/pred.o: $(REF)/libavcodec/hevc/pred.c $(INC)/config.h
	@mkdir -p $(dir $@)
	@$(CC) $(CFLAGS) -c $< -o $@

$(OUT)/obj/hevcintra/dsp.o: $(REF)/libavcodec/hevc/dsp.c $(INC)/config.h
	@mkdir -p $(dir $@)
	@$(CC) $(CFLAGS) -c $< -o $@

$(OUT)/obj/hevcintra/%.o: %.c ../../include/b200dsp.h $(INC)/config.h
	@mkdir -p $(dir $@)
	@$(CC) $(CFLAGS) -c $< -o $@

HEVCINTRA_OBJS := $(addprefix $(OUT)/obj/hevcintra/, pred.o dsp.o ref_hevcidct.o ref_hevcintra.o)

$(OUT)/libffref_hevcintra.so: $(HEVCINTRA_OBJS) $(OUT)/libffref.so
	@$(CC) -shared -o $@ $(HEVCINTRA_OBJS) -L$(OUT) -lffref -lm -pthread \
	   -Wl,-rpath,'$$ORIGIN' -Wl,-Bsymbolic -Wl,--no-undefined

clean:
	rm -rf $(OUT)/obj/hevcintra $(OUT)/libffref_hevcintra.so
