# Builds oracle/_ref/libffref_hevcsao.so: the UNMODIFIED reference libavcodec/hevc/dsp.c (its SAO members:
# h26x/h2656_sao_template.c once per bit depth) and libavcodec/hevc/filter.c (the decoder's loop filter: sao_filter_CTB,
# restore_tqb_pixels, ff_hevc_hls_filter), compiled where they lie under $(REF) with the generic-C configuration of oracle/ref/Makefile,
# plus ref_hevcsao.c (flat C ABI for the tests, the minimal decoder contexts filter.c reads, and stubs for the two symbols it links
# against that are not reached).  `make -C oracle/ref` runs first (it writes the config.h used here and libffref.so, which dsp.c's
# other members link against).  Nothing is written into $(REF), no reference source is copied into this repository; output goes to
# oracle/_ref/ (git-ignored).
#     make -C oracle/ref -f hevcsao.mk
REF ?= /root/reference
OUT ?= ../_ref
CC  ?= gcc
INC := $(OUT)/include
CFLAGS := -std=c17 -O3 -fPIC -w -fno-math-errno -fno-signed-zeros -pthread \
  -D_ISOC11_SOURCE -D_FILE_OFFSET_BITS=64 -D_POSIX_C_SOURCE=200112 -D_XOPEN_SOURCE=600 -D_GNU_SOURCE \
  -DHAVE_AV_CONFIG_H -I$(INC) -I$(REF)

all: $(OUT)/libffref_hevcsao.so

$(OUT)/obj/hevcsao/dsp.o: $(REF)/libavcodec/hevc/dsp.c $(INC)/config.h
	@mkdir -p $(dir $@)
	@$(CC) $(CFLAGS) -c $< -o $@

$(OUT)/obj/hevcsao/filter.o: $(REF)/libavcodec/hevc/filter.c $(INC)/config.h
	@mkdir -p $(dir $@)
	@$(CC) $(CFLAGS) -c $< -o $@

$(OUT)/obj/hevcsao/ref_hevcsao.o: ref_hevcsao.c ../../include/b200dsp.h $(INC)/config.h
	@mkdir -p $(dir $@)
	@$(CC) $(CFLAGS) -c $< -o $@

HEVCSAO_OBJS := $(addprefix $(OUT)/obj/hevcsao/, dsp.o filter.o ref_hevcsao.o)

$(OUT)/libffref_hevcsao.so: $(HEVCSAO_OBJS) $(OUT)/libffref.so
	@$(CC) -shared -o $@ $(HEVCSAO_OBJS) -L$(OUT) -lffref -lm -pthread \
	   -Wl,-rpath,'$$ORIGIN' -Wl,-Bsymbolic -Wl,--no-undefined

clean:
	rm -rf $(OUT)/obj/hevcsao $(OUT)/libffref_hevcsao.so
