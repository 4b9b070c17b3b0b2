# Builds oracle/_ref/libffref_h264pred.so: the UNMODIFIED reference libavcodec/h264pred.c (which includes h264pred_template.c once
# per bit depth), compiled where it lies under $(REF) with the generic-C configuration of oracle/ref/Makefile, plus ref_h264pred.c
# (flat C ABI for the tests, and the layout check of B200H264PredContext).  libavcodec/mathtables.c comes along for ff_crop_tab (a
# hidden symbol, so it cannot come from libffref.so); libavutil comes from libffref.so, so `make -C oracle/ref` runs first (it writes the config.h used here).  Nothing is written into $(REF), no reference
# source is copied into this repository; output goes to oracle/_ref/ (git-ignored).
#     make -C oracle/ref -f h264pred.mk
REF ?= /root/reference
OUT ?= ../_ref
CC  ?= gcc
INC := $(OUT)/include
CFLAGS := -std=c17 -O3 -fPIC -w -fno-math-errno -fno-signed-zeros -pthread \
  -D_ISOC11_SOURCE -D_FILE_OFFSET_BITS=64 -D_POSIX_C_SOURCE=200112 -D_XOPEN_SOURCE=600 -D_GNU_SOURCE \
  -DHAVE_AV_CONFIG_H -I$(INC) -I$(REF)

all: $(OUT)/libffref_h264pred.so

$(OUT)/obj/h264pred/h264pred.o: $(REF)/libavcodec/h264pred.c $(INC)/config.h
	@mkdir -p $(dir $@)
	@$(CC) $(CFLAGS) -c $< -o $@

$(OUT)/obj/h264pred/mathtables.o: $(REF)/libavcodec/mathtables.c $(INC)/config.h
	@mkdir -p $(dir $@)
	@$(CC) $(CFLAGS) -c $< -o $@

$(OUT)/obj/h264pred/ref_h264pred.o: ref_h264pred.c ../../include/b200dsp.h $(INC)/config.h
	@mkdir -p $(dir $@)
	@$(CC) $(CFLAGS) -c $< -o $@

H264PRED_OBJS := $(addprefix $(OUT)/obj/h264pred/, h264pred.o mathtables.o ref_h264pred.o)

$(OUT)/libffref_h264pred.so: $(H264PRED_OBJS) $(OUT)/libffref.so
	@$(CC) -shared -o $@ $(H264PRED_OBJS) -L$(OUT) -lffref -lm -pthread \
	   -Wl,-rpath,'$$ORIGIN' -Wl,-Bsymbolic -Wl,--no-undefined

clean:
	rm -rf $(OUT)/obj/h264pred $(OUT)/libffref_h264pred.so
