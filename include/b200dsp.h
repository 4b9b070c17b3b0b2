/*
 * b200dsp.h — C ABI of libb200dsp.so: H100-native (sm_90a) implementations of FFmpeg's DSP hot paths.
 *
 * Every entry point replaces (and cites) one interface of the reference; paths are relative to the FFmpeg tree.
 * Two levels per path:
 *   drop-in level  : the reference's own signature, HOST pointers.  Used by un-modified callers and by the parity
 *                    tests; each call stages through the device (H2D, kernel, D2H) and is therefore latency-bound.
 *   batched level  : many frames / blocks / transforms per call, DEVICE pointers (or pinned host buffers for the
 *                    *_host variants, which pipeline copies and kernels).  This is where the throughput is.
 * There is no CPU fallback: every function fails with a negative B200_E* code if no CUDA device is usable.
 * No function retains caller pointers after it returns (stream-ordered work is finished or the documented
 * b200_device_sync() point applies).  Contexts are not thread-safe; use one per thread like the reference's.
 */
#ifndef B200DSP_H
#define B200DSP_H

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200DSP_ABI_VERSION 1

/* error codes: negative errno values, mirroring AVERROR(x) = -(x) (libavutil/error.h) */
#define B200_EINVAL   (-22)
#define B200_ENOMEM   (-12)
#define B200_ENOSYS   (-38)   /* AVERROR(ENOSYS): combination not implemented (the reference's PATCHWELCOME/ENOTSUP cases) */
#define B200_ENODEV   (-19)   /* no CUDA device / CUDA runtime failure */
#define B200_EEXTERNAL (-5)   /* CUDA error during execution (see b200_last_error) */

int         b200_abi_version(void);
const char *b200_last_error(void);          /* thread-local, human readable */

/* ------------------------------------------------------------------------------------------------ device
 * Plays the role of AVHWDeviceContext/AVCUDADeviceContext {CUcontext, CUstream}
 * (libavutil/hwcontext_cuda.h, libavutil/hwcontext_cuda.c:932-956): one device ordinal + one stream on which all
 * work of the contexts created from it is ordered.  `cu_stream` may be a caller-owned CUstream/cudaStream_t
 * (e.g. AVCUDADeviceContext.stream, or torch's current stream) or NULL to let the library create one. */
typedef struct B200Device B200Device;

int   b200_device_open(B200Device **dev, int ordinal, void *cu_stream);
void  b200_device_close(B200Device *dev);
int   b200_device_sync(B200Device *dev);
int   b200_device_ordinal(const B200Device *dev);
void *b200_device_stream(const B200Device *dev);
int   b200_device_sm_count(const B200Device *dev);
/* process-wide default device used by the pointer tables that have no context argument
 * (IDCTDSPContext, MECmpContext, H264QpelContext, HpelDSPContext).  Opened lazily on ordinal 0 if unset. */
int   b200_set_default_device(B200Device *dev);
/* memory helpers so that C callers need no CUDA headers */
void *b200_malloc_device(B200Device *dev, size_t bytes);
void  b200_free_device(B200Device *dev, void *p);
void *b200_malloc_host(size_t bytes);                 /* pinned */
void  b200_free_host(void *p);
int   b200_memcpy_h2d(B200Device *dev, void *dst_dev, const void *src_host, size_t bytes);  /* async on the stream */
int   b200_memcpy_d2h(B200Device *dev, void *dst_host, const void *src_dev, size_t bytes);  /* async on the stream */
/* number of kernels this library has launched in this process (bench.py's gpu_launches) */
uint64_t b200_launch_count(void);

/* ------------------------------------------------------------------------------------------------ libswscale
 * Replaces the legacy scaler for AV_PIX_FMT_YUV420P -> packed 8-bit RGB (rgb24, bgr24, rgba, bgra, argb, abgr) and
 * AV_PIX_FMT_YUV420P -> AV_PIX_FMT_YUV420P (scaling):
 *   sws_getContext / sws_init_context ....... libswscale/utils.c:1919,1884 (ff_sws_init_single_context :1137)
 *   sws_setColorspaceDetails ................ libswscale/utils.c:849
 *   sws_scale ............................... libswscale/swscale.h:583, swscale.c:1626
 *   SwsFunc (convert_unscaled / ff_swscale).. libswscale/swscale_internal.h:99-101, swscale.c:263
 * Flags keep the reference's values (libswscale/swscale.h:88-118).  Output is bit-identical to the reference's
 * C path (the one FATE pins with accurate_rnd+bitexact, and yuv2rgb_c_24_rgb without accurate_rnd).  */
#define B200_PIX_FMT_YUV420P 0     /* AV_PIX_FMT_YUV420P, libavutil/pixfmt.h */
#define B200_PIX_FMT_NV12    23    /* AV_PIX_FMT_NV12: source only; src[1] is the interleaved U,V plane, src[2] is ignored */
#define B200_PIX_FMT_NV21    24    /* AV_PIX_FMT_NV21: same with V,U */
#define B200_PIX_FMT_RGB24   2     /* AV_PIX_FMT_RGB24 */
#define B200_PIX_FMT_BGR24   3     /* AV_PIX_FMT_BGR24 */
#define B200_PIX_FMT_ARGB    25    /* AV_PIX_FMT_ARGB  (alpha byte = 255, the source has no alpha plane) */
#define B200_PIX_FMT_RGBA    26    /* AV_PIX_FMT_RGBA  */
#define B200_PIX_FMT_ABGR    27    /* AV_PIX_FMT_ABGR  */
#define B200_PIX_FMT_BGRA    28    /* AV_PIX_FMT_BGRA  */

#define B200_SWS_FAST_BILINEAR 0x1
#define B200_SWS_BILINEAR      0x2
#define B200_SWS_BICUBIC       0x4
#define B200_SWS_X             0x8
#define B200_SWS_POINT         0x10
#define B200_SWS_AREA          0x20
#define B200_SWS_BICUBLIN      0x40
#define B200_SWS_GAUSS         0x80     /* X, GAUSS, SINC, LANCZOS, SPLINE: default parameters (param[] = SWS_PARAM_DEFAULT) */
#define B200_SWS_SINC          0x100
#define B200_SWS_LANCZOS       0x200
#define B200_SWS_SPLINE        0x400
#define B200_SWS_FULL_CHR_H_INT 0x2000
#define B200_SWS_FULL_CHR_H_INP 0x4000   /* packed RGB source: chroma from every pixel instead of every other one */
#define B200_SWS_ACCURATE_RND  0x40000
#define B200_SWS_BITEXACT      0x80000

typedef struct B200SwsContext B200SwsContext;

/* like sws_getContext(); srcFilter/dstFilter/param are not supported (must be the defaults). NULL on failure.
 * Sources: yuv420p, nv12, nv21 (-> packed 8-bit RGB or yuv420p / nv12 / nv21) and rgb24 / bgr24 / rgba / bgra / argb / abgr (-> yuv420p /
 * nv12 / nv21, or, when the size changes and alpha is not carried from source to destination, -> packed 8-bit RGB; the input
 * readers of libswscale/input.c:264-393,1068-1172, hScale16To15_c, and the bgr24ToYv12Wrapper special converter,
 * libswscale/swscale_unscaled.c:2453-2457); a packed RGB source is passed as plane 0 (src[1], src[2] unused).
 * Destinations nv12 / nv21 (what NVENC reads) are yuv420p with the chroma planes interleaved: planarToNv12Wrapper
 * (libswscale/swscale_unscaled.c:147-165) unscaled, yuv2nv12cX_c (libswscale/output.c:495-528) through the scaler; dst[1] is the
 * interleaved plane, dst[2] unused. */
B200SwsContext *b200_sws_getContext(B200Device *dev, int srcW, int srcH, int srcFormat,
                                    int dstW, int dstH, int dstFormat, int flags);
/* The same with SwsContext.src_range / .dst_range (libswscale/swscale.h, AVOption "src_range" / "dst_range"; 0 = limited,
 * 1 = full) set before sws_init_context(), the way vf_scale's in_range / out_range reach the scaler (libswscale/utils.c:
 * 1164-1167).  With a yuv420p destination and different ranges the 15-bit lines are range-converted between the horizontal
 * and the vertical pass (lumRangeToJpeg_c ... chrRangeFromJpeg_c, libswscale/swscale.c:163-209, :577-660) and the same-size
 * case goes through the scaler instead of planarCopyWrapper (utils.c:1623-1626).  For RGB destinations dstRange is ignored
 * and srcRange selects the look-up tables, as in the reference. */
B200SwsContext *b200_sws_getContext_range(B200Device *dev, int srcW, int srcH, int srcFormat, int srcRange,
                                          int dstW, int dstH, int dstFormat, int dstRange, int flags);
/* The same with SwsContext.scaler_params — the `param` argument of sws_getContext() (libswscale/swscale.h; utils.c:312-360):
 * bicubic B / C (default 0 / 0.6), Gaussian exponent (3), Lanczos width (3), the experimental scaler's power (1).  NULL, or
 * 123456 (SWS_PARAM_DEFAULT) in either slot, selects the default. */
B200SwsContext *b200_sws_getContext_params(B200Device *dev, int srcW, int srcH, int srcFormat, int srcRange,
                                           int dstW, int dstH, int dstFormat, int dstRange, int flags, const double *param);
/* sws_getContext's srcFilter / dstFilter (SwsFilter / SwsVector, libswscale/swscale.h:187-204): initFilter convolves the source vector of
 * each direction into that direction's filter bank; of a destination vector only the length counts (the reference never applies it,
 * "FIXME dstFilter", utils.c:384-413); any vector longer than one tap rules out the unscaled special converters (utils.c:1256-1263).
 * NULL pointers = no filter.  The vectors are copied. */
typedef struct B200SwsVector { const double *coeff; int length; } B200SwsVector;
typedef struct B200SwsFilter { const B200SwsVector *lumH, *lumV, *chrH, *chrV; } B200SwsFilter;
B200SwsContext *b200_sws_getContext_filters(B200Device *dev, int srcW, int srcH, int srcFormat, int srcRange, int dstW, int dstH, int dstFormat,
                                            int dstRange, int flags, const B200SwsFilter *srcFilter, const B200SwsFilter *dstFilter,
                                            const double *param);
void b200_sws_freeContext(B200SwsContext *c);
/* like sws_setColorspaceDetails() (libswscale/utils.c:849-1004).  RGB destination: `table` / dstRange are accepted and
 * ignored like the reference.  yuv420p destination: the ranges are stored and the range conversion is re-selected
 * (brightness / contrast / saturation do not apply); a context that was initialised as a plain copy (same size, equal
 * ranges) stays one, as in the reference, where convert_unscaled is chosen once at init.  inv_table != table for
 * yuv -> yuv makes the reference cascade through bgr24: not implemented, B200_ENOSYS. */
int  b200_sws_setColorspaceDetails(B200SwsContext *c, const int inv_table[4], int srcRange,
                                   const int table[4], int dstRange, int brightness, int contrast, int saturation);
/* drop-in for sws_scale(): HOST pointers, strides in bytes (negative allowed), returns output lines.
 * Top-down slice sequences are supported (bands uploaded into a device copy of the picture, lines emitted as soon as
 * their vertical taps are complete, same return values as the reference) from planar / semi-planar and packed RGB sources, into packed RGB and
 * into yuv420p / nv12 / nv21 destinations; a sequence whose first band touches the last line runs bottom-up (the picture is flipped internally like
 * scale_internal, swscale.c:1096-1159; even heights, yuv sources). */
int  b200_sws_scale(B200SwsContext *c, const uint8_t *const srcSlice[], const int srcStride[],
                    int srcSliceY, int srcSliceH, uint8_t *const dst[], const int dstStride[]);
/* SwsFunc-shaped entry (first argument is the context): what a maintainer installs as convert_unscaled */
int  b200_sws_func(void *c, const uint8_t *const src[], const int srcStride[], int srcSliceY, int srcSliceH,
                   uint8_t *const dst[], const int dstStride[]);
/* batched, DEVICE pointers: frame f's plane p starts at src[p] + f*srcFrameStride[p]; rgb at dst + f*dstFrameStride.
 * Asynchronous on the device's stream. */
int  b200_sws_scale_batch_device(B200SwsContext *c, const uint8_t *const src[3], const int srcStride[3],
                                 const int64_t srcFrameStride[3], uint8_t *dst, int dstStride,
                                 int64_t dstFrameStride, int nframes);
/* yuv420p -> yuv420p (context created with dstFormat = B200_PIX_FMT_YUV420P; the reference's yuv2planeX_8_c / yuv2plane1_8_c
 * writers, libswscale/output.c:468-493, and planarCopyWrapper at same size): three destination planes.
 * b200_sws_scale() takes them as dst[0..2] / dstStride[0..2] like the reference; the single-plane batch entry points
 * return B200_EINVAL for such a context and this one returns B200_EINVAL for a packed-RGB context. */
int  b200_sws_scale_batch_device_planar(B200SwsContext *c, const uint8_t *const src[3], const int srcStride[3],
                                        const int64_t srcFrameStride[3], uint8_t *const dst[3], const int dstStride[3],
                                        const int64_t dstFrameStride[3], int nframes);
/* batched, HOST pointers (pinned memory recommended): chunks of frames are copied in, converted and copied back
 * on rotating streams so that H2D, kernels and D2H overlap.  Synchronous: returns when dst is complete. */
int  b200_sws_scale_batch_host(B200SwsContext *c, const uint8_t *const src[3], const int srcStride[3],
                               const int64_t srcFrameStride[3], uint8_t *dst, int dstStride,
                               int64_t dstFrameStride, int nframes);
/* introspection for tests: same layout as the shim used on the reference (16 ints) */
int  b200_sws_info(const B200SwsContext *c, int *out16);
/* diagnostics: which kernels the launches since the previous call used (scaled path: bit 0 two passes through 15-bit line planes,
 * bit 1 fused CUDA-core kernels, bit 2 fused kernels with the tensor-core horizontal pass; same size: bit 3 the line-pair kernel);
 * reading clears it. */
int  b200_sws_last_path(B200SwsContext *c);
/* which: 0 hLum 1 hChr 2 vLum 3 vChr — host copies of the generated filter tables */
int  b200_sws_get_filter(const B200SwsContext *c, int which, int16_t *filter, int32_t *pos, int cap);

/* host-only: build the set-up tables for a configuration WITHOUT touching a GPU (used by the CPU test tier to check
 * the filter generation against the reference).  info16 as b200_sws_info; filter/pos may be NULL. Returns n or <0. */
int  b200_sws_plan_probe(int srcW, int srcH, int dstW, int dstH, int flags, int which,
                         int16_t *filter, int32_t *pos, int cap, int *info16);
/* the general form: cfg = { srcW, srcH, srcFormat, srcRange, dstW, dstH, dstFormat, dstRange, flags }; details = NULL or the 13
 * ints of a sws_setColorspaceDetails() call made after initialisation { inv_table[4], srcRange, table[4], dstRange,
 * brightness, contrast, saturation }.  info32: [0..15] as b200_sws_info ([12] = vertical chroma shift of the destination),
 * [16] plain-copy context, [17] range conversion (0 none, 1 limited->full, 2 full->limited), [18..21] its luma coefficient,
 * luma offset, chroma coefficient, chroma offset (libswscale/swscale.c:577-624), [22] fast-bilinear horizontal pass,
 * [23] semi-planar source kind, [24] return value of the details call, [25] src_range, [26] dst_range, [27] packed RGB source
 * (bytes per pixel), [28] / [29] horizontal / vertical chroma shift of the source as the scaler sees it, [30] bgr24 -> yv12
 * converter installed, [31] semi-planar destination kind (1 nv12, 2 nv21), [32..40] input_rgb2yuv_table.  The array must hold 48 ints. */
int  b200_sws_plan_probe2(const int cfg[9], const int *details, int which, int16_t *filter, int32_t *pos, int cap, int *info48);
/* host-only: a horizontal filter bank (n outputs x size taps, first-tap positions) regrouped into the operands of the tensor-core
 * horizontal pass (csrc/sws_mma.cuh): ginfo = (ceil(n / 8) + 1) pairs { first source column of the group's window, first chunk index },
 * bfrag = 128 words per chunk (32 lanes x { hi b0, hi b1, lo b0, lo b1 } of mma.m16n8k32's B operand), pitch[2] = staged-line byte
 * pitches for 128- and 64-column tiles.  Returns the number of bfrag words or <0.  Replaces nothing in the reference: the tables
 * hold libswscale's hLumFilter / hLumFilterPos (swscale_internal.h:437-448) in another order. */
int  b200_sws_mma_probe(const int16_t *coef, const int32_t *pos, int n, int size, int32_t *ginfo, int ginfo_cap,
                        uint32_t *bfrag, int bfrag_cap, int *pitch);

/* ------------------------------------------------------------------------------------------------ idctdsp
 * Replaces IDCTDSPContext (libavcodec/idctdsp.h:43-91) as filled by ff_idctdsp_init (libavcodec/idctdsp.c:228-314)
 * for idct_algo = FF_IDCT_SIMPLE / AUTO, 8 bit: ff_simple_idct_{put,add,}_int16_8bit
 * (libavcodec/simple_idct_template.c:329-368) and the clamp helpers (libavcodec/idctdsp.c:73-165).
 * The struct below has the reference's member order so that a maintainer can memcpy / alias it. */
typedef struct B200IDCTDSPContext {
    void (*put_pixels_clamped)(const int16_t *block, uint8_t *pixels, ptrdiff_t line_size);
    void (*put_signed_pixels_clamped)(const int16_t *block, uint8_t *pixels, ptrdiff_t line_size);
    void (*add_pixels_clamped)(const int16_t *block, uint8_t *pixels, ptrdiff_t line_size);
    void (*idct)(int16_t *block);
    void (*idct_put)(uint8_t *dest, ptrdiff_t line_size, int16_t *block);
    void (*idct_add)(uint8_t *dest, ptrdiff_t line_size, int16_t *block);
    uint8_t idct_permutation[64];
    int perm_type;                 /* enum idct_permutation_type: FF_IDCT_PERM_NONE = 0 */
    int mpeg4_studio_profile;
} B200IDCTDSPContext;

/* like ff_idctdsp_init(c, avctx) with avctx->idct_algo / bits_per_raw_sample / lowres passed explicitly.
 * Returns 0, or B200_ENOSYS for algorithms other than simple/auto at 8 bit, lowres 0. */
int  b200_idctdsp_init(B200IDCTDSPContext *c, int idct_algo, int bits_per_raw_sample, int lowres);

#define B200_IDCT      0   /* in place on the coefficient blocks */
#define B200_IDCT_PUT  1
#define B200_IDCT_ADD  2
/* batched, DEVICE pointers.  blocks: nblocks x int16[64] natural order (FF_IDCT_PERM_NONE), 16-byte aligned.
 * Block i goes to dest + dest_off[i] with line size line_size[i] (line_size NULL -> uniform_line_size).
 * For B200_IDCT the result replaces the coefficients and dest/dest_off are ignored.
 * Unlike the reference the coefficient blocks are NOT clobbered by put/add. */
int  b200_idct_batch_device(B200Device *dev, int kind, int16_t *blocks, int64_t nblocks, uint8_t *dest,
                            const int64_t *dest_off, const int32_t *line_size, int uniform_line_size);
/* batched macroblock stream, DEVICE pointers: nframes frames of mb_w x mb_h 4:2:0 macroblocks, 6 blocks each in the
 * decoder's order Y0 Y1 Y2 Y3 Cb Cr (libavcodec/mpegvideo_dec.c:940-1128 put_dct/add_dct calls); destinations are
 * implied: luma (16*mbx + 8*(b&1), 16*mby + 8*(b>>1)), chroma (8*mbx, 8*mby).  Planes of frame f start at
 * plane + f*frame_stride[p]. */
int  b200_idct_mb420_device(B200Device *dev, int kind, const int16_t *blocks, int mb_w, int mb_h, int nframes,
                            uint8_t *const planes[3], const int linesize[3], const int64_t frame_stride[3]);
/* same from HOST memory (copies in/out, pipelined). */
int  b200_idct_mb420_host(B200Device *dev, int kind, const int16_t *blocks, int mb_w, int mb_h, int nframes,
                          uint8_t *const planes[3], const int linesize[3], const int64_t frame_stride[3]);

/* The same table for bits_per_raw_sample 9 / 10 / 12: ff_simple_idct_{,put_,add_}int16_10bit resp. _12bit
 * (libavcodec/idctdsp.c:248-266, libavcodec/simple_idct_template.c:63-104,329-368); uint16 pixels, line sizes in bytes.  Kept as a
 * separate entry until it has run on hardware, then b200_idctdsp_init() takes the depth.  The clamp helpers stay the 8-bit ones
 * like the reference's.  As with the 8-bit batch call the coefficient blocks are NOT clobbered by put / add. */
int  b200_idctdsp_init_hbd(B200IDCTDSPContext *c, int idct_algo, int bits_per_raw_sample, int lowres);
/* batched, DEVICE pointers: as b200_idct_batch_device with depth 10 (9 maps to it) or 12; dest_off / line sizes in bytes, even */
int  b200_idct_hbd_batch_device(B200Device *dev, int depth, int kind, int16_t *blocks, int64_t nblocks, uint8_t *dest,
                                const int64_t *dest_off, const int32_t *line_size, int uniform_line_size);

/* ProresDSPContext (libavcodec/proresdsp.h:28-35) as ff_proresdsp_init(dsp, bits_per_raw_sample) fills it for 10 and 12 bit
 * (libavcodec/proresdsp.c:56-82,102-194): idct_put = dequantise by qmat + inverse transform + bias + clip to [4, 2^bits - 5], the
 * fused "dequant + IDCT" of the ProRes decoder (libavcodec/proresdec.c:559-598).  Same member order as the reference struct;
 * idct_put_bayer (ProRes RAW) is left NULL. */
typedef struct B200ProresDSPContext {
    int idct_permutation_type;             /* FF_IDCT_PERM_NONE */
    uint8_t idct_permutation[64];
    void (*idct_put)(uint16_t *out, ptrdiff_t linesize, int16_t *block, const int16_t *qmat);     /* HOST pointers; block is not clobbered */
    void (*idct_put_bayer)(uint16_t *out, ptrdiff_t linesize, int32_t *block, const int16_t *qmat, const uint16_t *lin_curve);
} B200ProresDSPContext;
int  b200_proresdsp_init(B200ProresDSPContext *c, int bits_per_raw_sample);
/* batched, DEVICE pointers: block i = blocks + 64*i goes, dequantised by qmat[64] (device), to dest + dest_off[i] (bytes; uint16 pixels)
 * with line size line_size[i] or uniform_line_size (bytes, even) */
int  b200_prores_idct_put_batch_device(B200Device *dev, int bits, const int16_t *blocks, int64_t nblocks, const int16_t *qmat,
                                       uint8_t *dest, const int64_t *dest_off, const int32_t *line_size, int uniform_line_size);

/* H.264 in-loop deblocking, 8 bit: the loop-filter members of H264DSPContext (libavcodec/h264dsp.h:48-73) in the reference's order,
 * as ff_h264dsp_init(c, 8, chroma_format_idc) installs them (libavcodec/h264dsp.c:109-132; functions libavcodec/h264dsp_template.c:
 * 103-340).  pix points at the first pixel on the far side of the edge, like the reference; HOST pointers. */
typedef struct B200H264LoopFilterContext {
    void (*v_loop_filter_luma)(uint8_t *pix, ptrdiff_t stride, int alpha, int beta, int8_t *tc0);
    void (*h_loop_filter_luma)(uint8_t *pix, ptrdiff_t stride, int alpha, int beta, int8_t *tc0);
    void (*h_loop_filter_luma_mbaff)(uint8_t *pix, ptrdiff_t stride, int alpha, int beta, int8_t *tc0);
    void (*v_loop_filter_luma_intra)(uint8_t *pix, ptrdiff_t stride, int alpha, int beta);
    void (*h_loop_filter_luma_intra)(uint8_t *pix, ptrdiff_t stride, int alpha, int beta);
    void (*h_loop_filter_luma_mbaff_intra)(uint8_t *pix, ptrdiff_t stride, int alpha, int beta);
    void (*v_loop_filter_chroma)(uint8_t *pix, ptrdiff_t stride, int alpha, int beta, int8_t *tc0);
    void (*h_loop_filter_chroma)(uint8_t *pix, ptrdiff_t stride, int alpha, int beta, int8_t *tc0);
    void (*h_loop_filter_chroma_mbaff)(uint8_t *pix, ptrdiff_t stride, int alpha, int beta, int8_t *tc0);
    void (*v_loop_filter_chroma_intra)(uint8_t *pix, ptrdiff_t stride, int alpha, int beta);
    void (*h_loop_filter_chroma_intra)(uint8_t *pix, ptrdiff_t stride, int alpha, int beta);
    void (*h_loop_filter_chroma_mbaff_intra)(uint8_t *pix, ptrdiff_t stride, int alpha, int beta);
} B200H264LoopFilterContext;
int  b200_h264_loop_filter_init(B200H264LoopFilterContext *c, int bit_depth, int chroma_format_idc);     /* 8, or 9 / 10 / 12 / 14 (uint16 samples) */
/* kinds for the batched call: 0 v_luma, 1 h_luma, 2 h_luma_mbaff, 3-5 their _intra forms, 6 v_chroma, 7 h_chroma, 8 h_chroma_mbaff,
 * 9-11 their _intra forms, 12 / 13 h_chroma / h_chroma_mbaff of 4:2:2 content, 14 / 15 their _intra forms */
/* batched, DEVICE pointers: edge e of kind kinds[e] at pix + pix_off[e] with alpha[e], beta[e] and tc0[4*e .. 4*e+3] (ignored by the
 * intra kinds).  The edges of one call must not read or write each other's pixels (p3..q3 across, the edge's lines along): the
 * decoder's sequential order becomes one call per independent set of edges. */
int  b200_h264_loop_filter_batch_device(B200Device *dev, int64_t nedges, const uint8_t *kinds, uint8_t *pix, const int64_t *pix_off,
                                        ptrdiff_t stride, const uint8_t *alpha, const uint8_t *beta, const int8_t *tc0);
/* the same for 9 / 10 / 12 / 14 bit samples (uint16): pix_off and stride in BYTES; alpha, beta and tc0 are the 8-bit table values the
 * reference's callers pass (the functions scale them to the sample depth, h264dsp_template.c:109-112,241-246) */
int  b200_h264_loop_filter_hbd_batch_device(B200Device *dev, int bit_depth, int64_t nedges, const uint8_t *kinds, uint8_t *pix,
                                            const int64_t *pix_off, ptrdiff_t stride, const uint8_t *alpha, const uint8_t *beta, const int8_t *tc0);

/* H.264 intra prediction: H264PredContext (libavcodec/h264pred.h:94-114) in the reference's member order and table sizes, as
 * ff_h264_pred_init(h, AV_CODEC_ID_H264, bit_depth, chroma_format_idc) fills it (libavcodec/h264pred.c:437-539; functions
 * libavcodec/h264pred_template.c).  HOST pointers, the reference's signatures: samples are uint8 at 8 bit and uint16 above, strides in
 * bytes, coefficients (`block`) int16 at 8 bit and int32 above; the _add members clear their coefficients.  Members the reference
 * leaves NULL for H.264 stay NULL.  pred4x4's topright may point anywhere (the decoder passes a stack word, h264_mb.c:676-691). */
#define B200_CODEC_ID_H264 27           /* AV_CODEC_ID_H264 */
typedef struct B200H264PredContext {
    void (*pred4x4[9 + 3 + 3])(uint8_t *src, const uint8_t *topright, ptrdiff_t stride);
    void (*pred8x8l[9 + 3])(uint8_t *src, int topleft, int topright, ptrdiff_t stride);
    void (*pred8x8[4 + 3 + 4])(uint8_t *src, ptrdiff_t stride);
    void (*pred16x16[4 + 3 + 2])(uint8_t *src, ptrdiff_t stride);
    void (*pred4x4_add[2])(uint8_t *pix, int16_t *block, ptrdiff_t stride);
    void (*pred8x8l_add[2])(uint8_t *pix, int16_t *block, ptrdiff_t stride);
    void (*pred8x8l_filter_add[2])(uint8_t *pix, int16_t *block, int topleft, int topright, ptrdiff_t stride);
    void (*pred8x8_add[3])(uint8_t *pix, const int *block_offset, int16_t *block, ptrdiff_t stride);
    void (*pred16x16_add[3])(uint8_t *pix, const int *block_offset, int16_t *block, ptrdiff_t stride);
} B200H264PredContext;
/* 0, or B200_ENOSYS for other codec ids (the SVQ3 / RV40 / VP7 / VP8 replacements) and depths other than 8 / 9 / 10 / 12 / 14,
 * B200_EINVAL for h == NULL or chroma_format_idc outside 0..3, B200_ENODEV.  chroma_format_idc <= 1 selects the 8x8 chroma functions,
 * 2 and 3 the 8x16 ones. */
int  b200_h264_pred_init(B200H264PredContext *h, int codec_id, int bit_depth, int chroma_format_idc);
/* Batched, DEVICE pointers.  Op i predicts the block whose top-left sample is at pix + pix_off[i] (bytes; stride in bytes; uint8 samples at
 * 8 bit, uint16 above).  kinds[i] = table << 4 | mode, mode being the index into the reference's table:
 *   b200_h264_pred_batch_device:      0 pred4x4 (modes 0-11), 1 pred8x8l (0-11), 2 pred8x8 as 8x8 (0-10), 3 pred8x8 as 8x16 (0-10),
 *                                     4 pred16x16 (0-6)
 *   b200_h264_pred_add_batch_device:  0 pred4x4_add, 1 pred8x8l_add, 2 pred8x8l_filter_add (modes 0 VERT, 1 HOR), 3 pred8x8_add as 8x8,
 *                                     4 pred8x8_add as 8x16, 5 pred16x16_add (modes 1 HOR, 2 VERT)
 * An op whose kind names a member the reference leaves NULL changes nothing.  flags[i]: bit 0 has_topleft, bit 1 has_topright for
 * pred8x8l and pred8x8l_filter_add; for pred4x4, bit 1 set reads the four top-right samples at src + 4 - stride, clear uses four
 * copies of src[3 - stride] (the decoder's substitute); other tables ignore it.
 * The add forms wrap (modulo 2^8 at 8 bit, 2^16 above; no clipping) and clear the coefficients they read.  Op i's coefficients start
 * at coef + coef_off[i] (in coefficients: int16 at 8 bit, int32 above); 4x4 sub-block k of the 8x8 / 8x16 / 16x16 add forms is at
 * + 16 k and sits where h264_slice.c:554-563 puts block k (scan8 order; 8x16: the 4x4 rows 0-3 in pairs), relative to the call's
 * stride.  The sub-blocks chain as in the reference: each predicts from its neighbour's already added samples.
 * The ops of one call must be independent: no op may write samples another op of the same call reads or writes.  The decoder's
 * sequential order (macroblocks in raster order, the 4x4 / 8x8 blocks of one in scan order) becomes one call per wavefront step.
 * Returns 0, or B200_EINVAL (launching nothing) for NULL pointers, a negative nops or stride, an odd stride or pix above 8 bit, or a
 * depth other than 8 / 9 / 10 / 12 / 14; nops == 0 returns 0. */
int  b200_h264_pred_batch_device(B200Device *dev, int bit_depth, int64_t nops, const uint8_t *kinds, const uint8_t *flags, uint8_t *pix,
                                 const int64_t *pix_off, ptrdiff_t stride);
int  b200_h264_pred_add_batch_device(B200Device *dev, int bit_depth, int64_t nops, const uint8_t *kinds, const uint8_t *flags, uint8_t *pix,
                                     const int64_t *pix_off, ptrdiff_t stride, void *coef, const int64_t *coef_off);

/* HEVC motion compensation: HEVCDSPContext (libavcodec/hevc/dsp.h:47-125) in the reference's member order and types.
 * b200_hevc_dsp_init() fills the six inter-prediction tables put_hevc_{q,e}pel, _uni, _uni_w, _bi, _bi_w ([10][2][2] each, every
 * width index) as ff_hevc_dsp_init does (hevc/dsp.c:140-196, :230-235); every other member stays NULL.  HOST pointers, the
 * reference's signatures: samples uint8 at 8 bit and uint16 above, strides in bytes, the int16 `dst` of put_hevc_?pel and `src2` of
 * the _bi forms at the MAX_PB_SIZE (64) element stride, 1 <= width, height <= 64, mx / my 0..3 (qpel) or 0..7 (epel); the width
 * index is ignored, as the reference does.  A member reads exactly the samples its reference function reads: columns -3..+4 (qpel) /
 * -1..+2 (epel) around the block only where it filters horizontally, the same rows only where it filters vertically. */
struct GetBitContext;
struct SAOParams;
typedef struct B200HEVCDSPContext {
    void (*put_pcm)(uint8_t *_dst, ptrdiff_t _stride, int width, int height, struct GetBitContext *gb, int pcm_bit_depth);
    void (*add_residual[4])(uint8_t *dst, const int16_t *res, ptrdiff_t stride);
    void (*dequant)(int16_t *coeffs, int16_t log2_size);
    void (*transform_rdpcm)(int16_t *coeffs, int16_t log2_size, int mode);
    void (*transform_4x4_luma)(int16_t *coeffs);
    void (*idct[4])(int16_t *coeffs, int col_limit);
    void (*idct_dc[4])(int16_t *coeffs);
    void (*sao_band_filter[5])(uint8_t *_dst, const uint8_t *_src, ptrdiff_t _stride_dst, ptrdiff_t _stride_src,
                               const int16_t *sao_offset_val, int sao_left_class, int width, int height);
    void (*sao_edge_filter[5])(uint8_t *_dst, const uint8_t *_src, ptrdiff_t stride_dst, const int16_t *sao_offset_val,
                               int sao_eo_class, int width, int height);
    void (*sao_edge_restore[2])(uint8_t *_dst, const uint8_t *_src, ptrdiff_t _stride_dst, ptrdiff_t _stride_src,
                                const struct SAOParams *sao, const int *borders, int _width, int _height, int c_idx,
                                const uint8_t *vert_edge, const uint8_t *horiz_edge, const uint8_t *diag_edge);
    void (*put_hevc_qpel[10][2][2])(int16_t *dst, const uint8_t *src, ptrdiff_t srcstride, int height, intptr_t mx, intptr_t my, int width);
    void (*put_hevc_qpel_uni[10][2][2])(uint8_t *dst, ptrdiff_t dststride, const uint8_t *src, ptrdiff_t srcstride, int height,
                                        intptr_t mx, intptr_t my, int width);
    void (*put_hevc_qpel_uni_w[10][2][2])(uint8_t *_dst, ptrdiff_t _dststride, const uint8_t *_src, ptrdiff_t _srcstride, int height,
                                          int denom, int wx, int ox, intptr_t mx, intptr_t my, int width);
    void (*put_hevc_qpel_bi[10][2][2])(uint8_t *dst, ptrdiff_t dststride, const uint8_t *_src, ptrdiff_t _srcstride, const int16_t *src2,
                                       int height, intptr_t mx, intptr_t my, int width);
    void (*put_hevc_qpel_bi_w[10][2][2])(uint8_t *dst, ptrdiff_t dststride, const uint8_t *_src, ptrdiff_t _srcstride, const int16_t *src2,
                                         int height, int denom, int wx0, int wx1, int ox, intptr_t mx, intptr_t my, int width);
    void (*put_hevc_epel[10][2][2])(int16_t *dst, const uint8_t *src, ptrdiff_t srcstride, int height, intptr_t mx, intptr_t my, int width);
    void (*put_hevc_epel_uni[10][2][2])(uint8_t *dst, ptrdiff_t dststride, const uint8_t *_src, ptrdiff_t _srcstride, int height,
                                        intptr_t mx, intptr_t my, int width);
    void (*put_hevc_epel_uni_w[10][2][2])(uint8_t *_dst, ptrdiff_t _dststride, const uint8_t *_src, ptrdiff_t _srcstride, int height,
                                          int denom, int wx, int ox, intptr_t mx, intptr_t my, int width);
    void (*put_hevc_epel_bi[10][2][2])(uint8_t *dst, ptrdiff_t dststride, const uint8_t *_src, ptrdiff_t _srcstride, const int16_t *src2,
                                       int height, intptr_t mx, intptr_t my, int width);
    void (*put_hevc_epel_bi_w[10][2][2])(uint8_t *dst, ptrdiff_t dststride, const uint8_t *_src, ptrdiff_t _srcstride, const int16_t *src2,
                                         int height, int denom, int wx0, int wx1, int ox, intptr_t mx, intptr_t my, int width);
    void (*hevc_h_loop_filter_luma)(uint8_t *pix, ptrdiff_t stride, int beta, const int32_t *tc, const uint8_t *no_p, const uint8_t *no_q);
    void (*hevc_v_loop_filter_luma)(uint8_t *pix, ptrdiff_t stride, int beta, const int32_t *tc, const uint8_t *no_p, const uint8_t *no_q);
    void (*hevc_h_loop_filter_chroma)(uint8_t *pix, ptrdiff_t stride, const int32_t *tc, const uint8_t *no_p, const uint8_t *no_q);
    void (*hevc_v_loop_filter_chroma)(uint8_t *pix, ptrdiff_t stride, const int32_t *tc, const uint8_t *no_p, const uint8_t *no_q);
    void (*hevc_h_loop_filter_luma_c)(uint8_t *pix, ptrdiff_t stride, int beta, const int32_t *tc, const uint8_t *no_p, const uint8_t *no_q);
    void (*hevc_v_loop_filter_luma_c)(uint8_t *pix, ptrdiff_t stride, int beta, const int32_t *tc, const uint8_t *no_p, const uint8_t *no_q);
    void (*hevc_h_loop_filter_chroma_c)(uint8_t *pix, ptrdiff_t stride, const int32_t *tc, const uint8_t *no_p, const uint8_t *no_q);
    void (*hevc_v_loop_filter_chroma_c)(uint8_t *pix, ptrdiff_t stride, const int32_t *tc, const uint8_t *no_p, const uint8_t *no_q);
} B200HEVCDSPContext;
/* 0; B200_EINVAL for c == NULL; B200_ENOSYS for depths other than 8, 9, 10 and 12 (the reference installs its 8-bit functions for
 * those, but its decoder refuses such streams before it initialises the context, hevc/ps.c:1193-1215); B200_ENODEV. */
int  b200_hevc_dsp_init(B200HEVCDSPContext *c, int bit_depth);

/* One prediction unit of b200_hevc_mc_batch_device.  Reference r (0, 1) is the picture whose sample (0, 0) is at ref + ref_off[r]
 * (bytes, may be negative); the block's integer-sample position in it is (x[r], y[r]) (any value), its phase (mx[r], my[r]) (0..3
 * for qpel, 0..7 for epel).  The block is w x h samples at dst + dst_off (bytes).  kind:
 *   B200_HEVC_MC_UNI    put_hevc_?pel_uni[idx][!!my0][!!mx0] on reference 0
 *   B200_HEVC_MC_UNI_W  put_hevc_?pel_uni_w[..] on reference 0 with (denom, wx0, ox)
 *   B200_HEVC_MC_BI     put_hevc_?pel[..](tmp, reference 0), then put_hevc_?pel_bi[idx][!!my1][!!mx1](dst, reference 1, tmp)
 *   B200_HEVC_MC_BI_W   the same with put_hevc_?pel_bi_w[..](denom, wx0, wx1, ox); ox = o0 + o1 (hevcdec.c:1853-1859)
 * ox is the slice header's 8-bit offset; the functions scale it by 1 << (depth - 8). */
enum { B200_HEVC_MC_UNI = 0, B200_HEVC_MC_UNI_W = 1, B200_HEVC_MC_BI = 2, B200_HEVC_MC_BI_W = 3 };
typedef struct B200HevcMcOp {
    int64_t dst_off;
    int64_t ref_off[2];
    int32_t x[2], y[2];
    uint8_t mx[2], my[2];
    uint8_t w, h, kind, denom;
    int32_t wx0, wx1, ox;
    uint8_t reserved[4];
} B200HevcMcOp;
#ifdef __cplusplus
static_assert(sizeof(B200HevcMcOp) == 64, "B200HevcMcOp is 64 bytes");
#else
_Static_assert(sizeof(B200HevcMcOp) == 64, "B200HevcMcOp is 64 bytes");
#endif
/* Batched HEVC inter prediction of one plane, DEVICE pointers: epel 0 = luma (8-tap qpel), 1 = chroma (4-tap epel).  Every op's
 * result is the reference's call sequence above, its source samples read with edge replication: coordinates clamped to
 * [0, pic_w) x [0, pic_h), which is what the decoder's emulated_edge_mc windows give (hevcdec.c:1813-1845, :1906-1923), so no
 * separate edge emulation pass is needed.  Both references share ref_stride and the picture size.  The caller guarantees that the
 * ops of one call write disjoint blocks and that no op reads samples another op of the call writes (the current-picture reference
 * of screen-content coding needs a call of its own).  An op whose w or h is outside 1..64, whose kind is undefined, whose phase is
 * out of range or whose dst_off / ref_off is not a multiple of the sample size writes nothing.
 * Returns 0, or B200_EINVAL (launching nothing) for NULL pointers, nops < 0, epel not 0 / 1, a stride not a multiple of the sample
 * size, pic_w or pic_h < 1, or a depth other than 8, 9, 10 or 12; nops == 0 returns 0. */
int  b200_hevc_mc_batch_device(B200Device *dev, int bit_depth, int epel, int64_t nops, const B200HevcMcOp *ops,
                               uint8_t *dst, ptrdiff_t dst_stride, const uint8_t *ref, ptrdiff_t ref_stride, int pic_w, int pic_h);

/* HEVC residual: fills the transform members of a B200HEVCDSPContext as ff_hevc_dsp_init does (hevc/dsp.c:198-215):
 * add_residual[0..3], dequant, transform_rdpcm, transform_4x4_luma, idct[0..3], idct_dc[0..3] (hevc/dsp_template.c:46-309).  It does
 * not clear the context and touches no other member: call b200_hevc_dsp_init() first, then this.  HOST pointers, the reference's
 * signatures: the members that take `coeffs` work in place on the int16 coefficients; add_residual clips to the sample depth
 * (samples uint8 at 8 bit, uint16 above, stride in bytes) and leaves `res` as it is.  idct[k](coeffs, col_limit) takes col_limit as
 * the reference does, as part of the function: odd inputs at or beyond the limit are not summed (so a block with non-zero
 * coefficients there does not get the full transform); any int value gives the reference's result.  dequant / transform_rdpcm with a
 * log2_size outside 2..5 (outside the reference's contract) write nothing and record the reason (b200_last_error()).
 * Returns 0; B200_EINVAL for c == NULL; B200_ENOSYS for depths other than 8, 9, 10 and 12; B200_ENODEV. */
int  b200_hevc_dsp_init_transform(B200HEVCDSPContext *c, int bit_depth);

/* One transform unit of b200_hevc_transform_add_batch_device: the (1 << log2_size)^2 coefficients at coef + coef_off (int16 elements,
 * row-major, as the parser leaves them: already scaled) and the block of samples at dst + dst_off (bytes).  The op's result is the
 * decoder's sequence (hevc/cabac.c:1550-1592) on a copy of the coefficients, then add_residual[log2_size - 2]:
 *   B200_HEVC_TU_IDCT     idct[log2_size - 2](c, col_limit)
 *   B200_HEVC_TU_IDCT_DC  idct_dc[log2_size - 2](c)
 *   B200_HEVC_TU_DST4     transform_4x4_luma(c)                     (4x4 only)
 *   B200_HEVC_TU_SKIP     the 180-degree swap of a 4x4 when B200_HEVC_TU_ROTATE is set, dequant(c, log2_size), then
 *                         transform_rdpcm(c, log2_size, B200_HEVC_TU_RDPCM_VER set) when B200_HEVC_TU_RDPCM is set
 *   B200_HEVC_TU_BYPASS   transform_rdpcm(c, log2_size, B200_HEVC_TU_RDPCM_VER set) when B200_HEVC_TU_RDPCM is set
 * The decoder's choices (DC when max_xy == 0, the implicit rdpcm direction, rotation) stay with the caller. */
enum { B200_HEVC_TU_IDCT = 0, B200_HEVC_TU_IDCT_DC = 1, B200_HEVC_TU_DST4 = 2, B200_HEVC_TU_SKIP = 3, B200_HEVC_TU_BYPASS = 4 };
enum { B200_HEVC_TU_RDPCM = 1, B200_HEVC_TU_RDPCM_VER = 2, B200_HEVC_TU_ROTATE = 4 };
typedef struct B200HevcTuOp {
    int64_t dst_off;      /* bytes, into dst */
    int64_t coef_off;     /* int16 elements, into coef */
    uint8_t log2_size;    /* 2..5 */
    uint8_t kind;         /* B200_HEVC_TU_* */
    uint8_t flags;        /* B200_HEVC_TU_RDPCM, B200_HEVC_TU_RDPCM_VER, B200_HEVC_TU_ROTATE */
    uint8_t reserved0;
    int32_t col_limit;    /* IDCT only, as the idct member receives it (cabac.c:1258-1265) */
    uint8_t reserved[8];
} B200HevcTuOp;
#ifdef __cplusplus
static_assert(sizeof(B200HevcTuOp) == 32, "B200HevcTuOp is 32 bytes");
#else
_Static_assert(sizeof(B200HevcTuOp) == 32, "B200HevcTuOp is 32 bytes");
#endif
/* Batched HEVC residual reconstruction of one plane, DEVICE pointers, asynchronous on the device's stream: every op's residual is
 * added to its block of dst, clipped to the sample depth.  Unlike the in-place members, `coef` is const: the batch never writes
 * coefficients.  The ops of one call write disjoint blocks.  An op whose log2_size is outside 2..5 or whose kind is undefined, a DST4
 * op on a block other than 4x4, and an op whose coef_off is not a multiple of 8 elements or whose dst_off is not a multiple of 4
 * samples write nothing (transform unit positions in a stream always satisfy these alignments).  Offsets are 64-bit; a call may have
 * more ops than one launch takes.
 * Returns 0, or B200_EINVAL (launching nothing) for NULL pointers, ops or coef not 16-byte aligned, dst not aligned to 4 samples,
 * nops < 0, a depth other than 8, 9, 10 or 12, or a dst_stride that is not a multiple of 4 samples; nops == 0 returns 0. */
int  b200_hevc_transform_add_batch_device(B200Device *dev, int bit_depth, int64_t nops, const B200HevcTuOp *ops, const int16_t *coef,
                                          uint8_t *dst, ptrdiff_t dst_stride);

/* HEVC deblocking: fills the eight loop-filter members of a B200HEVCDSPContext as ff_hevc_dsp_init does (hevc/dsp.c:237-244):
 * hevc_{h,v}_loop_filter_{luma,chroma} and their _c twins, each _c member the same function as its plain twin
 * (hevc/dsp_template.c:834-928).  It does not clear the context and touches no other member.  HOST pointers, the reference's
 * signatures: `pix` is Q0 of line 0, the stride in bytes, samples uint8 at 8 bit and uint16 above; two segments of 4 lines, tc[j],
 * no_p[j] and no_q[j] for lines 4j..4j+3 (any non-zero byte counts).  Domain: beta 0..255 and tc[j] <= 255 (the decoder's tables give
 * at most 64 and 24); a segment with tc[j] <= 0 is left as it is, as the reference leaves it.  A member reads only P3..Q3 (luma) or
 * P1..Q1 (chroma) of the lines of segments with tc[j] > 0, and writes only P2..Q2 / P0..Q0 of those lines.
 * Returns 0; B200_EINVAL for c == NULL; B200_ENOSYS for depths other than 8, 9, 10 and 12; B200_ENODEV. */
int  b200_hevc_dsp_init_deblock(B200HEVCDSPContext *c, int bit_depth);

/* One 4-sample edge segment of b200_hevc_deblock_plane_device: beta and tc as the members receive them (the 8-bit table values; the
 * kernel shifts them by depth - 8), flags B200_HEVC_DBK_NO_P / B200_HEVC_DBK_NO_Q (pcm / transquant-bypass sides left as they are).
 * Other flag bits and `reserved` are ignored. */
enum { B200_HEVC_DBK_NO_P = 1, B200_HEVC_DBK_NO_Q = 2 };
typedef struct B200HevcDbkSeg {
    uint8_t beta, tc, flags, reserved;
} B200HevcDbkSeg;
#ifdef __cplusplus
static_assert(sizeof(B200HevcDbkSeg) == 4, "B200HevcDbkSeg is 4 bytes");
#else
_Static_assert(sizeof(B200HevcDbkSeg) == 4, "B200HevcDbkSeg is 4 bytes");
#endif
/* Deblocks one width x height plane in place, DEVICE pointers, asynchronous on the device's stream.  chroma 0 selects the luma
 * filter, 1 the chroma (weak) filter.  Grids, in plane sample coordinates:
 *   vseg[(y / 4) * vseg_stride + x / 8]  rows y..y+3 of the vertical edge at column x   (x = 0, 8, ... < width; y = 0, 4, ... < height)
 *   hseg[(y / 8) * hseg_stride + x / 4]  columns x..x+3 of the horizontal edge at row y (y = 0, 8, ... < height; x = 0, 4, ... < width)
 * Entries at x = 0 (vertical) and y = 0 (horizontal) are picture edges and ignored.  The result is that of the member call for every
 * vertical segment (its beta, tc and flags; tc 0 for the member's other segment), then for every horizontal segment: the decoder's
 * CTB-by-CTB sequence of member calls (hevc/filter.c:501-676) gives the same picture.  64-bit offsets.
 * Returns 0, or B200_EINVAL (launching nothing) for NULL pointers, a depth other than 8, 9, 10 or 12, chroma other than 0 / 1, width or
 * height below 4 or not a multiple of 4, a stride shorter than a row or not a multiple of the sample size, pix not aligned to a sample,
 * vseg_stride < ceil(width / 8) or hseg_stride < width / 4. */
int  b200_hevc_deblock_plane_device(B200Device *dev, int bit_depth, int chroma, uint8_t *pix, ptrdiff_t stride, int width, int height,
                                    const B200HevcDbkSeg *vseg, int64_t vseg_stride, const B200HevcDbkSeg *hseg, int64_t hseg_stride);

/* HEVC sample adaptive offset: SAOParams (libavcodec/hevc/dsp.h:34-45) with the reference's layout, what sao_edge_restore[] reads
 * through its `const struct SAOParams *` (only offset_val[c_idx][0] and eo_class[c_idx]). */
typedef struct B200SAOParams {
    int32_t offset_abs[3][4];
    int32_t offset_sign[3][4];
    uint8_t band_position[3];
    int32_t eo_class[3];          /* 0 horizontal, 1 vertical, 2 = 135 degrees, 3 = 45 degrees */
    int16_t offset_val[3][5];     /* SaoOffsetVal: offset_abs << log2_sao_offset_scale with its sign (up to +-124 at 12 bit) */
    uint8_t type_idx[3];
} B200SAOParams;
#ifdef __cplusplus
static_assert(sizeof(B200SAOParams) == 148, "B200SAOParams is 148 bytes");
#else
_Static_assert(sizeof(B200SAOParams) == 148, "B200SAOParams is 148 bytes");
#endif

/* Fills the SAO members of a B200HEVCDSPContext as ff_hevc_dsp_init does (hevc/dsp.c:217-228): sao_band_filter[0..4] (one
 * function), sao_edge_filter[0..4] (one function), sao_edge_restore[0] and [1] (h26x/h2656_sao_template.c).  It does not clear the
 * context and touches no other member.  HOST pointers, the reference's signatures, samples uint8 at 8 bit and uint16 above, strides
 * in bytes:
 *   sao_band_filter   dst[x] = clip(src[x] + table[(src[x] >> (depth - 5)) & 31]), table[(k + sao_left_class) & 31] = offset_val[k + 1]
 *                     for k = 0..3 and 0 elsewhere, for any int sao_left_class.  Reads and writes exactly width x height; dst == src
 *                     with equal strides (the decoder's in-place call) works, as do separate buffers.
 *   sao_edge_filter   `src` at the implicit stride of 192 bytes (2 * MAX_PB_SIZE + AV_INPUT_BUFFER_PADDING_SIZE) at every depth;
 *                     reads the width x height block and only the ring its class's neighbours use (no rows -1 / height for the
 *                     horizontal class, no columns -1 / width for the vertical one); writes exactly width x height of dst.
 *   Domain of both: 1 <= width, height <= 64, sao_eo_class 0..3; outside it a member writes nothing and records the reason in
 *   b200_last_error().  Both run the plane kernel of b200_hevc_sao_plane_device on a scratch plane.
 *   sao_edge_restore  [0] / [1]: the picture-border samples (borders[4] = left, top, right, bottom) become clip(src + offset_val[0]);
 *                     [1] then puts back `src` where vert_edge[2], horiz_edge[2] and diag_edge[4] mark an edge that may not be
 *                     filtered, with the reference's corner exceptions, in the reference's order of writes.  They read only
 *                     sao->offset_val[c_idx][0] and sao->eo_class[c_idx] (any value, compared with the four classes as the
 *                     reference does); c_idx outside 0..2 or a size outside 1..64 writes nothing and records the reason.  They launch nothing: at most four lines of at most 64
 *                     samples are copied on the host, classified by the same per-sample function the kernel uses.  Where the
 *                     reference would write outside the width x height block (a 1-sample-wide block with a picture border and an
 *                     edge flag on the same side, which the decoder never passes), they do not.
 * Returns 0; B200_EINVAL for c == NULL; B200_ENOSYS for depths other than 8, 9, 10 and 12; B200_ENODEV. */
int  b200_hevc_dsp_init_sao(B200HEVCDSPContext *c, int bit_depth);

/* One CTB of one component for b200_hevc_sao_plane_device: what hls_sao_param parsed for it (offset_val = SaoOffsetVal[0..4], type,
 * band_position or eo_class) and what sao_filter_CTB computes from the slice and tile maps (hevc/filter.c:283-329): RESTORE = its
 * `restore` (sao_edge_restore[1] is used), VERT_L / VERT_R = vert_edge[0 / 1], HORIZ_T / HORIZ_B = horiz_edge[0 / 1], DIAG_TL / TR /
 * BR / BL = diag_edge[0..3].  The edge flags count only with RESTORE, and only where sao_filter_CTB can compute them: a flag on a side
 * (or a corner touching a side) that is a picture border is ignored.  Unknown flag bits and `reserved` are ignored. */
enum { B200_HEVC_SAO_NONE = 0, B200_HEVC_SAO_BAND = 1, B200_HEVC_SAO_EDGE = 2 };
enum {
    B200_HEVC_SAO_RESTORE = 1, B200_HEVC_SAO_VERT_L = 2, B200_HEVC_SAO_VERT_R = 4, B200_HEVC_SAO_HORIZ_T = 8, B200_HEVC_SAO_HORIZ_B = 16,
    B200_HEVC_SAO_DIAG_TL = 32, B200_HEVC_SAO_DIAG_TR = 64, B200_HEVC_SAO_DIAG_BR = 128, B200_HEVC_SAO_DIAG_BL = 256
};
typedef struct B200HevcSaoCtb {
    int16_t  offset_val[5];
    uint8_t  type;                /* B200_HEVC_SAO_NONE / _BAND / _EDGE */
    uint8_t  cls;                 /* band_position (BAND, used & 31) or eo_class (EDGE) */
    uint16_t flags;
    uint16_t reserved;
} B200HevcSaoCtb;
#ifdef __cplusplus
static_assert(sizeof(B200HevcSaoCtb) == 16, "B200HevcSaoCtb is 16 bytes");
#else
_Static_assert(sizeof(B200HevcSaoCtb) == 16, "B200HevcSaoCtb is 16 bytes");
#endif
/* Applies SAO to one width x height plane out of place, DEVICE pointers, asynchronous on the device's stream: `src` is the deblocked
 * plane and `dst` becomes what sao_filter_CTB (hevc/filter.c:269-478) makes of it for this component over every CTB, which depends
 * only on the deblocked plane whatever order the CTBs run in (neighbours always come from deblocked samples).  CTB (i, j) is
 * ctb[j * ctb_stride + i] and covers [i * cw, min((i + 1) * cw, width)) x [j * ch, min((j + 1) * ch, height)), cw = (1 << log2_ctb_size)
 * >> hshift, ch = (1 << log2_ctb_size) >> vshift (log2_ctb_size is the luma CTB size); the picture borders are the grid's outer
 * sides.  NONE CTBs, an unknown type and EDGE with cls > 3 are copied.
 * keep: NULL when the decoder's `transquant_bypass_enable_flag || (pcm_enabled && pcm_loop_filter_disabled)` is false; else its
 * is_pcm map (one byte per luma min PU, keep[py * keep_stride + px], 1 << log2_min_pu_size luma samples), and the samples
 * restore_tqb_pixels (hevc/filter.c:228-265) puts back are taken from src.  Reference quirk reproduced: it is called with the luma
 * CTB origin but the component's CTB width and height, so for 4:2:0 chroma only PCM / bypass blocks in the top-left quarter of a
 * chroma CTB are restored, for 4:2:2 only those in the left half (luma and 4:4:4: the whole CTB).
 * Reads nothing outside the src plane, writes nothing outside the dst plane; 64-bit offsets.
 * Returns 0, or B200_EINVAL (launching nothing) for NULL dst / src / ctb, a depth other than 8, 9, 10 or 12, width or height below 1,
 * log2_ctb_size outside 4..6, a shift outside {0, 1}, a stride shorter than a row or not a multiple of the sample size, dst / src
 * not aligned to a sample or ctb not aligned to 16 bytes, ctb_stride < ceil(width / cw), with keep given log2_min_pu_size outside
 * 2..log2_ctb_size - 1 or keep_stride < ((width << hshift) >> log2_min_pu_size), or dst and src byte ranges that overlap (the entry
 * does not work in place). */
int  b200_hevc_sao_plane_device(B200Device *dev, int bit_depth, uint8_t *dst, ptrdiff_t dst_stride, const uint8_t *src, ptrdiff_t src_stride,
                                int width, int height, int log2_ctb_size, int hshift, int vshift, const B200HevcSaoCtb *ctb,
                                int64_t ctb_stride, const uint8_t *keep, int64_t keep_stride, int log2_min_pu_size);

/* HEVC intra prediction: HEVCPredContext (libavcodec/hevc/pred.h) with the reference's layout and function types. */
struct HEVCLocalContext;
struct HEVCPPS;
typedef struct B200HEVCPredContext {
    void (*intra_pred[4])(struct HEVCLocalContext *lc, const struct HEVCPPS *pps, int x0, int y0, int c_idx);
    void (*pred_planar[4])(uint8_t *src, const uint8_t *top, const uint8_t *left, ptrdiff_t stride);
    void (*pred_dc)(uint8_t *src, const uint8_t *top, const uint8_t *left, ptrdiff_t stride, int log2_size, int c_idx);
    void (*pred_angular[4])(uint8_t *src, const uint8_t *top, const uint8_t *left, ptrdiff_t stride, int c_idx, int mode);
    void (*ref_filter_3tap[3])(uint8_t *filtered_left, uint8_t *filtered_top, const uint8_t *left, const uint8_t *top, int size);
    void (*ref_filter_strong)(uint8_t *filtered_top, uint8_t *left, const uint8_t *top);
} B200HEVCPredContext;

/* Fills every member of a B200HEVCPredContext that ff_hevc_pred_init fills (hevc/pred.c) except intra_pred[], which takes decoder
 * structs and is left NULL: the reference's own intra_pred calls everything else through s->hpc, so a decoder copies these members
 * over its HEVCPredContext.  HOST pointers, the reference's signatures, samples uint8 at 8 bit and uint16 above, and strides in SAMPLES
 * (intra_pred passes linesize / sizeof(pixel)):
 *   pred_planar[log2_size - 2], pred_dc, pred_angular[log2_size - 2]
 *                     stage the samples the reference function reads (planar top[0..size], left[0..size]; DC top[0..size - 1],
 *                     left[0..size - 1]; angular top[-1..2 * size - 1], left[-1..2 * size - 1]) onto the device, run the prediction stage
 *                     of the batch kernel and copy the size x size block back.  An angular mode outside 2..34 or a pred_dc log2_size
 *                     outside 2..5 writes nothing and records the reason (b200_last_error()).
 *   ref_filter_3tap[0..2] (one function), ref_filter_strong
 *                     run on the host (no launch) through the kernel's own filter functions, with the reference's writes:
 *                     the 3-tap filter writes filtered_left / filtered_top [-1..2 * size - 1]; the strong filter writes
 *                     filtered_top[-1..63] and left[0..62] in place.
 * Returns 0; B200_EINVAL for hpc == NULL; B200_ENOSYS for depths other than 8, 9, 10 and 12 (the reference installs its 8-bit functions
 * for them, but its decoder refuses such streams first); B200_ENODEV. */
int  b200_hevc_pred_init(B200HEVCPredContext *hpc, int bit_depth);

/* One transform block of b200_hevc_intra_pred_batch_device: what intra_pred (hevc/pred_template.c) reads for it at the call.
 * CAND_* = the five cand_* values as intra_pred has them after its z-scan checks (pred_template.c:154-158), before constrained
 * intra prediction; LUMA = (c_idx == 0); SMOOTH = !sps->intra_smoothing_disabled && (c_idx == 0 || chroma_format_idc == 3);
 * STRONG = sps->strong_intra_smoothing_enabled.  Unknown flag bits and `reserved` are ignored. */
enum {
    B200_HEVC_INTRA_CAND_BL = 1, B200_HEVC_INTRA_CAND_L = 2, B200_HEVC_INTRA_CAND_UL = 4, B200_HEVC_INTRA_CAND_U = 8,
    B200_HEVC_INTRA_CAND_UR = 16, B200_HEVC_INTRA_LUMA = 32, B200_HEVC_INTRA_SMOOTH = 64, B200_HEVC_INTRA_STRONG = 128
};
typedef struct B200HevcIntraOp {
    int32_t  x, y;        /* the TU's top-left in plane samples (x0 >> hshift, y0 >> vshift) */
    uint8_t  log2_size;   /* 2..5 */
    uint8_t  mode;        /* 0 planar, 1 DC, 2..34 angular: the mode intra_pred reads (tu.intra_pred_mode / _c, after the 4:2:2 remap) */
    uint16_t flags;       /* B200_HEVC_INTRA_* */
    uint8_t  reserved[4];
} B200HevcIntraOp;
#ifdef __cplusplus
static_assert(sizeof(B200HevcIntraOp) == 16, "B200HevcIntraOp is 16 bytes");
#else
_Static_assert(sizeof(B200HevcIntraOp) == 16, "B200HevcIntraOp is 16 bytes");
#endif
/* Batched HEVC intra prediction of one plane, DEVICE pointers, asynchronous on the device's stream: each op's block becomes what
 * intra_pred writes for that TU given the plane as it is at the call.  pix / stride: the component plane (bytes); width / height the
 * LUMA picture size (sps->width / height) and hshift / vshift the component's subsampling, so the plane is (width >> hshift) x
 * (height >> vshift).  intra_map: NULL when constrained_intra_pred_flag is 0; else one byte per luma min PU (1 << log2_min_pu_size
 * luma samples, (width >> log2_min_pu_size) x (height >> log2_min_pu_size) entries at map_stride bytes per row), non-zero where
 * pred_flag == PF_INTRA, and the constrained-intra branch (pred_template.c:165-295) is reproduced with its quirks.  Where that branch
 * reads a map entry outside the picture's map (the row above the picture, for a block on the top row whose left neighbours are all
 * inter), the kernel reads "not intra" and never reads outside the map.
 * The ops of one call must be independent: no op may write samples that another op of the call reads or writes; a decoder issues
 * one call per dependency level.  An op whose log2_size or mode is out of range, or whose block or neighbours (the row above when a
 * CAND_UL / U / UR flag is set, the column to the left when a CAND_BL / L / UL flag is set) fall outside the plane, writes nothing.
 * Offsets are 64-bit.  Returns 0, or B200_EINVAL (launching nothing) for NULL pix or ops, pix not aligned to a sample or ops not aligned to 16 bytes, an intra_map with map_stride <
 * (width >> log2_min_pu_size) or log2_min_pu_size outside 2..6, nops < 0, a depth other than 8, 9, 10 or 12, width or height below 1,
 * a shift outside {0, 1}, a stride shorter than a plane row, or an odd stride or pix above 8 bit; nops == 0 returns 0. */
int  b200_hevc_intra_pred_batch_device(B200Device *dev, int bit_depth, uint8_t *pix, ptrdiff_t stride, int width, int height, int hshift,
                                       int vshift, int64_t nops, const B200HevcIntraOp *ops, const uint8_t *intra_map, ptrdiff_t map_stride,
                                       int log2_min_pu_size);

/* mpegvideo inverse quantisers: the members of MPVUnquantDSPContext (libavcodec/mpegvideo_unquantize.h:31-44) as
 * ff_mpv_unquantize_init() installs them (libavcodec/mpegvideo_unquantize.c:50-290), i.e. what runs in front of the IDCT in
 * mpv_reconstruct_mb's put_dct / add_dequant_dct (libavcodec/mpegvideo_dec.c).  The reference functions take the whole
 * MPVContext; B200MpvUnquant carries the fields they read (mpegvideo.h:70-77 y/c_dc_scale, ac_pred, h263_aic, the scan
 * tables; :201-203 intra_matrix / inter_matrix; :258 q_scale_type).  variant 3 is the function the reference installs for
 * AV_CODEC_FLAG_BITEXACT (with mismatch control); variant 2 the plain one. */
#define B200_UNQUANT_MPEG1_INTRA          0
#define B200_UNQUANT_MPEG1_INTER          1
#define B200_UNQUANT_MPEG2_INTRA          2
#define B200_UNQUANT_MPEG2_INTRA_BITEXACT 3
#define B200_UNQUANT_MPEG2_INTER          4
#define B200_UNQUANT_H263_INTRA           5
#define B200_UNQUANT_H263_INTER           6
typedef struct B200MpvUnquant {
    uint16_t intra_matrix[64], inter_matrix[64];     /* raster order after the IDCT permutation, as MPVContext holds them */
    uint8_t  permutated[64], raster_end[64];         /* ScanTable (ff_init_scantable, mpegvideo_unquantize.c:36-48) of the scan in use */
    int32_t  y_dc_scale, c_dc_scale, q_scale_type, h263_aic, ac_pred;
} B200MpvUnquant;
/* batched, DEVICE pointers, in place: block i = blocks + 64*i (int16, 4-byte aligned), its number inside the macroblock
 * blk_n[i] (0-3 luma, 4+ chroma: selects the DC scale; NULL = macroblock stream order, i % 6), quantiser qscale[i] and
 * block_last_index last_index[i] (-1 = no coded coefficient; the H.263 variants need >= 0 like the reference asserts).
 * Coefficients beyond the coded part of the scan are left untouched, as by the reference. */
int  b200_mpv_unquantize_batch_device(B200Device *dev, int variant, const B200MpvUnquant *p, int16_t *blocks, int64_t nblocks,
                                      const uint8_t *blk_n, const uint8_t *qscale, const int8_t *last_index);

/* put_dct / add_dequant_dct of mpv_reconstruct_mb (libavcodec/mpegvideo_dec.c:907-922) for a whole 4:2:0 macroblock stream in one
 * kernel: inverse quantisation (variant, p, qscale[], last_index[] per block as in b200_mpv_unquantize_batch_device, block number
 * inside the macroblock = position in the stream % 6) straight into the simple IDCT put / add of b200_idct_mb420_device — the
 * dequantised coefficients stay in registers.  kind = B200_IDCT_ADD skips blocks whose last_index is < 0, like add_dequant_dct.
 * `blocks` is not modified.  Planes as for b200_idct_mb420_device, 16-byte (luma) / 8-byte (chroma) aligned.  Asynchronous on
 * the device's stream. */
int  b200_mpv_unquant_idct_mb420_device(B200Device *dev, int variant, const B200MpvUnquant *p, int kind, const int16_t *blocks,
                                        const uint8_t *qscale, const int8_t *last_index, int mb_w, int mb_h, int nframes,
                                        uint8_t *const planes[3], const int linesize[3], const int64_t frame_stride[3]);

/* ------------------------------------------------------------------------------------------------ float_dsp
 * Replaces AVFloatDSPContext (libavutil/float_dsp.h:24-210) as avpriv_float_dsp_alloc() fills it with the C functions
 * (libavutil/float_dsp.c:27-141, float_scalarproduct.c:25-33): the element-wise float work around the transforms, e.g.
 * vector_fmul_window after every iMDCT of the AAC decoder (libavcodec/aac/aacdec_dsp_template.c).  Same member order as the
 * reference struct.  The table entries take HOST pointers (copy in, kernel, copy out). */
typedef struct B200FloatDSPContext {
    void   (*vector_fmul)(float *dst, const float *src0, const float *src1, int len);
    void   (*vector_fmac_scalar)(float *dst, const float *src, float mul, int len);
    void   (*vector_dmac_scalar)(double *dst, const double *src, double mul, int len);
    void   (*vector_fmul_scalar)(float *dst, const float *src, float mul, int len);
    void   (*vector_dmul_scalar)(double *dst, const double *src, double mul, int len);
    void   (*vector_fmul_window)(float *dst, const float *src0, const float *src1, const float *win, int len);
    void   (*vector_fmul_add)(float *dst, const float *src0, const float *src1, const float *src2, int len);
    void   (*vector_fmul_reverse)(float *dst, const float *src0, const float *src1, int len);
    void   (*butterflies_float)(float *v1, float *v2, int len);
    float  (*scalarproduct_float)(const float *v1, const float *v2, int len);
    void   (*vector_dmul)(double *dst, const double *src0, const double *src1, int len);
    double (*scalarproduct_double)(const double *v1, const double *v2, size_t len);
} B200FloatDSPContext;
int  b200_float_dsp_init(B200FloatDSPContext *c);        /* like avpriv_float_dsp_alloc(), into caller storage */
/* ops, numbered in the struct's member order */
#define B200_FDSP_VECTOR_FMUL          0
#define B200_FDSP_VECTOR_FMAC_SCALAR   1
#define B200_FDSP_VECTOR_DMAC_SCALAR   2
#define B200_FDSP_VECTOR_FMUL_SCALAR   3
#define B200_FDSP_VECTOR_DMUL_SCALAR   4
#define B200_FDSP_VECTOR_FMUL_WINDOW   5
#define B200_FDSP_VECTOR_FMUL_ADD      6
#define B200_FDSP_VECTOR_FMUL_REVERSE  7
#define B200_FDSP_BUTTERFLIES_FLOAT    8
#define B200_FDSP_SCALARPRODUCT_FLOAT  9
#define B200_FDSP_VECTOR_DMUL          10
#define B200_FDSP_SCALARPRODUCT_DOUBLE 11
/* batched, DEVICE pointers: nvec vectors of len elements (float, or double for the D ops); vector v of each operand starts at
 * base + v*stride (strides in elements; 0 = one vector shared by all, e.g. the window).  Operand roles as in the reference:
 * vector_fmul_window: src2 = window of 2*len, dst gets 2*len; butterflies_float: dst = v1, src0 = v2, both rewritten;
 * the scalar products put one value per vector at dst[v*dst_stride] and, like the C loops, sum left to right (one thread per
 * vector: exact, not fast).  fmac / butterflies read dst; otherwise dst may alias an input only element for element. */
int  b200_float_dsp_batch_device(B200Device *dev, int op, int64_t nvec, int len, void *dst, int64_t dst_stride,
                                 const void *src0, int64_t src0_stride, const void *src1, int64_t src1_stride,
                                 const void *src2, int64_t src2_stride, double mul);

/* H.264 residual transforms, 8 bit: the IDCT members of H264DSPContext (libavcodec/h264dsp.h:81-88) as installed by
 * ff_h264dsp_init(c, 8, chroma_format_idc) (libavcodec/h264dsp.c:66-139): ff_h264_idct_add_8_c, ff_h264_idct8_add_8_c,
 * ff_h264_idct_dc_add_8_c, ff_h264_idct8_dc_add_8_c (libavcodec/h264idct_template.c:33-181).  The add16/add8/add4 wrappers
 * of the reference only dispatch to these four per 4x4/8x8 block and keep working on top of them. */
typedef void (*b200_h264_idct_fn)(uint8_t *dst, int16_t *block, ptrdiff_t stride);   /* block is cleared, like the reference */
typedef struct B200H264IDCTContext {
    b200_h264_idct_fn idct_add;        /* 4x4, dst 4-aligned */
    b200_h264_idct_fn idct8_add;       /* 8x8, dst 8-aligned */
    b200_h264_idct_fn idct_dc_add;     /* 4x4, only block[0] is read (and cleared) */
    b200_h264_idct_fn idct8_dc_add;
} B200H264IDCTContext;
int  b200_h264_idct_init(B200H264IDCTContext *c, int bit_depth, int chroma_format_idc);   /* 8, or 9 / 10 / 12 / 14: uint16 samples and
                                                                                              * int32 coefficients behind the int16_t * argument */
#define B200_H264_IDCT4    0
#define B200_H264_IDCT8    1
#define B200_H264_IDCT4_DC 2
#define B200_H264_IDCT8_DC 3
/* batched, DEVICE pointers, one kind per call: block i = blocks + blk_off[i] (int16 elements, 16-byte aligned blocks of
 * 16 or 64 coefficients; DC kinds touch block[0] only) is transformed, added to the 4x4 / 8x8 pixels at dst + dst_off[i]
 * and cleared.  dst + dst_off[i] and stride must be 4-aligned (8 for the 8x8 kinds), as the reference requires. */
int  b200_h264_idct_batch_device(B200Device *dev, int kind, int64_t n, int16_t *blocks, const int64_t *blk_off,
                                 uint8_t *dst, const int64_t *dst_off, ptrdiff_t stride);
/* the same for 9 / 10 / 12 / 14 bit samples: int32 coefficients (blk_off in int32 elements), uint16 samples (dst_off and stride in BYTES) */
int  b200_h264_idct_hbd_batch_device(B200Device *dev, int bit_depth, int kind, int64_t n, int32_t *blocks, const int64_t *blk_off,
                                     uint8_t *dst, const int64_t *dst_off, ptrdiff_t stride);

/* H.264 explicit weighted prediction, 8 bit: weight_pixels_tab / biweight_pixels_tab of H264DSPContext (libavcodec/h264dsp.h:33-45)
 * as installed by ff_h264dsp_init(c, 8, ...) (libavcodec/h264dsp.c:103-110; functions in h264dsp_template.c:30-99).
 * Index = width: [0] 16, [1] 8, [2] 4, [3] 2. */
typedef void (*b200_h264_weight_func)(uint8_t *block, ptrdiff_t stride, int height, int log2_denom, int weight, int offset);
typedef void (*b200_h264_biweight_func)(uint8_t *dst, uint8_t *src, ptrdiff_t stride, int height, int log2_denom,
                                        int weightd, int weights, int offset);
typedef struct B200H264WeightContext {
    b200_h264_weight_func   weight_pixels_tab[4];
    b200_h264_biweight_func biweight_pixels_tab[4];
} B200H264WeightContext;
int  b200_h264_weight_init(B200H264WeightContext *c, int bit_depth);            /* 8, or 9 / 10 / 12 / 14 (uint16 samples, stride in bytes) */
/* batched, DEVICE pointers.  params: 4 int32 per block (16-byte aligned array): [0] = width index | height << 8 | log2_denom << 16,
 * [1] = weight (the destination weight for biweight), [2] = source weight (biweight), [3] = offset.  src == NULL: weight
 * (in place on dst + dst_off[i]); src != NULL: biweight of dst + dst_off[i] with src + src_off[i].  One stride for both.
 * Destination blocks of one call must not overlap each other, and no op may read samples that another op of the same call writes. */
int  b200_h264_weight_batch_device(B200Device *dev, int64_t n, const int32_t *params, uint8_t *dst, const int64_t *dst_off,
                                   const uint8_t *src, const int64_t *src_off, ptrdiff_t stride);
/* the same for 9 / 10 / 12 / 14 bit samples (uint16): offsets and stride in BYTES (even) */
int  b200_h264_weight_hbd_batch_device(B200Device *dev, int bit_depth, int64_t n, const int32_t *params, uint8_t *dst, const int64_t *dst_off,
                                       const uint8_t *src, const int64_t *src_off, ptrdiff_t stride);

/* ------------------------------------------------------------------------------------------------ fdctdsp
 * Replaces FDCTDSPContext (libavcodec/fdctdsp.h:28-31) as filled by ff_fdctdsp_init(c, avctx) (libavcodec/fdctdsp.c:27-45): the forward
 * 8x8 DCT in place on 64 int16 (16-byte aligned), fdct248 = the 2-4-8 variant for interlaced blocks.  dct_algo / bits_per_raw_sample are
 * AVCodecContext's: 9 / 10 bit -> ff_jpeg_fdct_islow_10, else FF_DCT_FASTINT (1) -> ff_fdct_ifast, FF_DCT_FAAN (6) -> ENOSYS (keep the C
 * functions), anything else -> ff_jpeg_fdct_islow_8. */
typedef struct B200FDCTDSPContext {
    void (*fdct)(int16_t *block);       /* HOST pointer */
    void (*fdct248)(int16_t *block);
} B200FDCTDSPContext;
int  b200_fdctdsp_init(B200FDCTDSPContext *c, int dct_algo, int bits_per_raw_sample);
/* batched, DEVICE pointer: n blocks of 64 coefficients transformed in place (blocks 16-byte aligned) */
int  b200_fdct_batch_device(B200Device *dev, int dct_algo, int bits_per_raw_sample, int is248, int16_t *blocks, int64_t n);

/* ------------------------------------------------------------------------------------------------ me_cmp
 * Replaces MECmpContext (libavcodec/me_cmp.h:53-77) as filled by ff_me_cmp_init (libavcodec/me_cmp.c:961-1027) for the
 * SAD / SSE entries: sad[0..1] = pix_abs16_c / pix_abs8_c, sse[0..2] = sse16_c / sse8_c / sse4_c,
 * pix_abs[0..1][0..3] = full / x2 / y2 / xy2 (me_cmp.c:37-385), and hadamard8_diff, vsad, vsse, nsse, median_sad, dct_sad, dct_max,
 * dct264_sad ([0] 16 wide, [1] 8 wide; [4] / [5] the intra forms where upstream has them).  Entries this library does not implement
 * (quant_psnr, bit, rd: they run the encoder's quantiser and VLC tables; w53, w97: the snow wavelets) stay NULL.
 * me_cmp_func (me_cmp.h:47-51): the first argument (MPVEncContext *) is unused by these functions and may be NULL. */
typedef int (*b200_me_cmp_func)(void *c, const uint8_t *blk1, const uint8_t *blk2, ptrdiff_t stride, int h);
typedef struct B200MECmpContext {
    int (*sum_abs_dctelem)(const int16_t *block);
    b200_me_cmp_func sad[6];
    b200_me_cmp_func sse[6];
    b200_me_cmp_func hadamard8_diff[6];
    b200_me_cmp_func dct_sad[6];
    b200_me_cmp_func quant_psnr[6];
    b200_me_cmp_func bit[6];
    b200_me_cmp_func rd[6];
    b200_me_cmp_func vsad[6];
    b200_me_cmp_func vsse[6];
    b200_me_cmp_func nsse[6];
    b200_me_cmp_func w53[6];
    b200_me_cmp_func w97[6];
    b200_me_cmp_func dct_max[6];
    b200_me_cmp_func dct264_sad[6];
    b200_me_cmp_func pix_abs[2][4];
    b200_me_cmp_func median_sad[6];
} B200MECmpContext;
/* like ff_me_cmp_init(c, avctx); avctx->flags passed explicitly (only AV_CODEC_FLAG_BITEXACT matters upstream) */
int  b200_me_cmp_init(B200MECmpContext *c, int codec_flags);

#define B200_MECMP_SAD     0   /* idx 0: 16 wide, 1: 8 wide */
#define B200_MECMP_SSE     1   /* idx 0: 16, 1: 8, 2: 4 wide */
#define B200_MECMP_PIX_ABS 2   /* idx = 4*size(0:16,1:8) + (0 full, 1 x2, 2 y2, 3 xy2) */
#define B200_MECMP_HADAMARD8 3 /* hadamard8_diff (SATD, me_cmp.c:514-562,933-950): idx 0: 16 wide (h = 8 or 16), 1: 8x8 (h ignored);
                                * idx 4 / 5: hadamard8_intra16 / intra8x8 (me_cmp.c:564-612: the block blk1 itself, mean left out) */
#define B200_MECMP_VSAD    4   /* vsad[idx] (me_cmp.c:843-881): idx 0: 16 wide, 1: 8, 4: vsad_intra16, 5: vsad_intra8 */
#define B200_MECMP_VSSE    5   /* vsse[idx] (me_cmp.c:883-931): same indices */
#define B200_MECMP_NSSE    6   /* nsse[idx] (me_cmp.c:387-437): idx 0: 16, 1: 8; weight as set by b200_me_cmp_set_nsse_weight (default 8) */
#define B200_MECMP_MEDIAN_SAD 7 /* median_sad[idx] (me_cmp.c:145-183,292-330): idx 0: 16, 1: 8 */
#define B200_MECMP_DCT_SAD  8   /* dct_sad[idx] (me_cmp.c:614-622,952): sum |fdct(blk1 - blk2)|; idx 0: 16 wide (h = 8 or 16), 1: 8x8 */
#define B200_MECMP_DCT_MAX  9   /* dct_max[idx] (me_cmp.c:678-693,956): max |fdct(blk1 - blk2)| per 8x8 block, added up over the blocks */
#define B200_MECMP_DCT264_SAD 10 /* dct264_sad[idx] (me_cmp.c:624-675,954): the H.264 8x8 integer transform; upstream only in GPL builds */
/* dct_sad / dct_max run FDCTDSPContext.fdct of the encoder context they are handed (s->fdsp.fdct); the table entries cannot read it, so
 * the DCT is chosen here with AVCodecContext.dct_algo's values the way ff_fdctdsp_init does for 8-bit samples (fdctdsp.c:27-45):
 * FF_DCT_FASTINT (1) = ff_fdct_ifast, FF_DCT_FAAN (6) = not implemented (ENOSYS, setting unchanged), anything else = ff_jpeg_fdct_islow_8. */
int  b200_me_cmp_set_dct_algo(int dct_algo);
/* nsse multiplies its noise term by MPVEncContext.c.avctx->nsse_weight, or by 8 when the context argument is NULL (me_cmp.c:407-410).
 * The table entries cannot read the caller's context (its layout is private to the encoder): the weight is set here instead. */
void b200_me_cmp_set_nsse_weight(int weight);
/* sum_abs_dctelem_c (me_cmp.c:105-112) for n blocks of 64 coefficients, DEVICE pointers */
int  b200_sum_abs_dctelem_batch_device(B200Device *dev, const int16_t *blocks, int64_t n, int32_t *out);
/* batched, DEVICE pointers: out[i] = fn(frame1 + off1[i], frame2 + off2[i], stride, h) */
int  b200_me_cmp_batch_device(B200Device *dev, int fn, int idx, const uint8_t *frame1, const uint8_t *frame2,
                              ptrdiff_t stride, int h, const int64_t *off1, const int64_t *off2, int64_t n, int32_t *out);
/* exhaustive search over whole frames, DEVICE pointers: ff_me_search_esa (libavfilter/motion_estimation.c:78-97) driven
 * like vf_mestimate.c:85-127 — for every mb_size x mb_size block of every frame pair: cost of the zero vector first,
 * raster scan of the +-search_param window clipped to the frame, strict '<' (first minimum in raster order wins, the
 * zero vector wins ties against everything).  mb_size in {4, 8, 16}.  out_mv: 2 ints (absolute x, y of the best match)
 * per block in raster order per frame; out_cost: its SAD.  The window is staged in shared memory at its unclipped size, so
 * search_param >= 217 / 221 / 223 for mb_size 16 / 8 / 4 returns B200_ENOSYS and writes nothing, whatever the frame size
 * (vf_mestimate accepts any search_param >= 4). */
int  b200_me_esa_device(B200Device *dev, const uint8_t *cur, const uint8_t *ref, int linesize, int width, int height,
                        int64_t frame_stride, int nframes, int mb_size, int search_param, int32_t *out_mv, uint64_t *out_cost);
/* same on HOST buffers (vf_mestimate's frames live in host memory): chunks of frame pairs rotate over three streams, H2D of both luma
 * planes (frame_stride bytes per frame, frame_stride >= linesize * height), the search kernel, D2H of vectors and costs. */
int  b200_me_esa_host(B200Device *dev, const uint8_t *cur, const uint8_t *ref, int linesize, int width, int height,
                      int64_t frame_stride, int nframes, int mb_size, int search_param, int32_t *out_mv, uint64_t *out_cost);

/* libavutil's public block SAD: av_pixelutils_get_sad_fn (libavutil/pixelutils.h:31-52, pixelutils.c:43-111).  Square blocks of
 * 1 << w_bits pixels, w_bits = h_bits = 1 ... 5; NULL for anything else, like the reference (and when no device is set). */
typedef int (*b200_pixelutils_sad_fn)(const uint8_t *src1, ptrdiff_t stride1, const uint8_t *src2, ptrdiff_t stride2);   /* HOST pointers */
b200_pixelutils_sad_fn b200_pixelutils_get_sad_fn(int w_bits, int h_bits, int aligned, void *log_ctx);
/* batched, DEVICE pointers: out[i] = sad(frame1 + off1[i], stride1, frame2 + off2[i], stride2) over a (1 << w_bits)^2 block */
int  b200_pixelutils_sad_batch_device(B200Device *dev, int w_bits, const uint8_t *frame1, ptrdiff_t stride1, const uint8_t *frame2,
                                      ptrdiff_t stride2, const int64_t *off1, const int64_t *off2, int64_t n, int32_t *out);

/* ------------------------------------------------------------------------------------------------ h264qpel / hpeldsp
 * Replaces H264QpelContext (libavcodec/h264qpel.h:27-30) as filled by ff_h264qpel_init(c, 8) (libavcodec/h264qpel.c:50-120)
 * and HpelDSPContext (libavcodec/hpeldsp.h:39-97) as filled by ff_hpeldsp_init (libavcodec/hpeldsp.c:337-352), 8 bit.
 * qpel_mc_func (libavcodec/qpeldsp.h:65-67), op_pixels_func (libavcodec/hpeldsp.h:39-41). */
typedef void (*b200_qpel_mc_func)(uint8_t *dst, const uint8_t *src, ptrdiff_t stride);
typedef void (*b200_op_pixels_func)(uint8_t *block, const uint8_t *pixels, ptrdiff_t line_size, int h);
typedef struct B200H264QpelContext {
    b200_qpel_mc_func put_h264_qpel_pixels_tab[3][16];     /* [0:16x16, 1:8x8, 2:4x4][x + 4*y] */
    b200_qpel_mc_func avg_h264_qpel_pixels_tab[3][16];
} B200H264QpelContext;
typedef struct B200HpelDSPContext {
    b200_op_pixels_func put_pixels_tab[4][4];              /* [0:16, 1:8, 2:4, 3:2 wide][xhalf + 2*yhalf] */
    b200_op_pixels_func avg_pixels_tab[4][4];
    b200_op_pixels_func put_no_rnd_pixels_tab[3][4];       /* only [0..1] filled, like the reference */
    b200_op_pixels_func avg_no_rnd_pixels_tab[4];
} B200HpelDSPContext;
int  b200_h264qpel_init(B200H264QpelContext *c, int bit_depth);    /* bit_depth 8, or 9 / 10 / 12 / 14 (uint16 samples, stride in bytes:
                                                                     * h264qpel_template.c with BIT_DEPTH > 8); else B200_ENOSYS */
int  b200_hpeldsp_init(B200HpelDSPContext *c, int flags);

/* batched motion compensation, DEVICE pointers: operation i interpolates the block at src + src_off[i] into
 * dst + dst_off[i] (same stride for both, like the reference's single stride argument).
 * qpel op byte: bit0 avg, bits1-2 size index (0:16,1:8,2:4), bits3-6 position x+4*y.
 * hpel op byte: bits0-1 table (0 put, 1 avg, 2 put_no_rnd, 3 avg_no_rnd), bits2-3 size index (0:16,1:8,2:4,3:2),
 * bits4-5 xy; h[i] = block height. Destination blocks of one call must not overlap each other, and no op may read samples that
 * another op of the same call writes (ops run in any order, and the qpel kernel loads windows several ops ahead).
 * An op code naming a table entry the reference leaves NULL writes nothing: qpel size index 3; hpel put_no_rnd (table 2) at size
 * index 2 or 3, avg_no_rnd (table 3) at size index 1, 2 or 3.  n == 0 returns 0; NULL pointers or n < 0 return B200_EINVAL.
 * hpel writes exactly h rows for every h; the reference's xy2 functions step two rows at a time, so at an odd h (outside the
 * heights hpeldsp.h allows) they write one row more.
 * The qpel kernel may load the whole (size+5)^2 window of an operation whatever its position (unused taps never reach the
 * result): keep the planes edge-padded by 3 pixels / rows, as H.264 reference frames are (h264_mb.c mc_dir_part). */
int  b200_h264qpel_batch_device(B200Device *dev, int64_t n, const uint8_t *op, uint8_t *dst, const int64_t *dst_off,
                                const uint8_t *src, const int64_t *src_off, ptrdiff_t stride);
/* the same for 9 / 10 / 12 / 14 bit samples (uint16, native endian): op bytes as above, offsets and stride in BYTES (even) */
int  b200_h264qpel_hbd_batch_device(B200Device *dev, int bit_depth, int64_t n, const uint8_t *op, uint8_t *dst, const int64_t *dst_off,
                                    const uint8_t *src, const int64_t *src_off, ptrdiff_t stride);
int  b200_hpel_batch_device(B200Device *dev, int64_t n, const uint8_t *op, const uint8_t *h, uint8_t *dst,
                            const int64_t *dst_off, const uint8_t *src, const int64_t *src_off, ptrdiff_t stride);
/* HOST buffers, a stream of frames (mc_dir_part for every partition of every macroblock of a picture, h264_mb.c:210-330, collected per
 * frame): frame f occupies [f * frame_bytes, (f + 1) * frame_bytes) of `src` (its reference picture, edge-padded) and of `dst`; its
 * operations are op_begin[f] .. op_begin[f + 1] - 1 (op_begin has nframes + 1 entries), offsets counted from the start of dst / src
 * as in the device entry point, each operation staying inside its own frame.  Chunks of frames rotate over three streams: H2D of the
 * reference and destination pictures and of the lists, the kernel, D2H of the destination pictures. */
int  b200_h264qpel_frames_host(B200Device *dev, int nframes, int64_t frame_bytes, const int64_t *op_begin, const uint8_t *op,
                               uint8_t *dst, const int64_t *dst_off, const uint8_t *src, const int64_t *src_off, ptrdiff_t stride);

/* h264chroma: replaces H264ChromaContext (libavcodec/h264chroma.h:26-31) as filled by ff_h264chroma_init(c, 8)
 * (libavcodec/h264chroma.c:36-65): h264_chroma_mc_func (h264chroma.h:24), bilinear eighth-pel, x, y in 0..7. */
typedef void (*b200_h264_chroma_mc_func)(uint8_t *dst, const uint8_t *src, ptrdiff_t srcStride, int h, int x, int y);
typedef struct B200H264ChromaContext {
    b200_h264_chroma_mc_func put_h264_chroma_pixels_tab[4];   /* [0: 8 wide, 1: 4, 2: 2]; [3] is NULL like the reference's */
    b200_h264_chroma_mc_func avg_h264_chroma_pixels_tab[4];
} B200H264ChromaContext;
int  b200_h264chroma_init(B200H264ChromaContext *c, int bit_depth);   /* 9 ... 16: the uint16 tables (h264chroma.c:45-50); else 8 bit */
/* batched, DEVICE pointers.  op byte: bit0 avg, bits1-2 width index (0:8,1:4,2:2); h[i] = rows; xy[i] = x | y << 3.
 * Like the reference, x == 0 never reads the column right of the block and y == 0 never reads the row below it.  Destination blocks
 * of one call must not overlap each other, and no op may read samples that another op of the same call writes.  Width index 3 (the
 * reference's NULL entry) writes nothing.  n == 0 returns 0; NULL pointers or n < 0 return B200_EINVAL. */
int  b200_h264chroma_batch_device(B200Device *dev, int64_t n, const uint8_t *op, const uint8_t *h, const uint8_t *xy,
                                  uint8_t *dst, const int64_t *dst_off, const uint8_t *src, const int64_t *src_off,
                                  ptrdiff_t stride);
/* the same for 16-bit samples (any depth above 8): offsets and stride in BYTES (even) */
int  b200_h264chroma_hbd_batch_device(B200Device *dev, int64_t n, const uint8_t *op, const uint8_t *h, const uint8_t *xy,
                                      uint8_t *dst, const int64_t *dst_off, const uint8_t *src, const int64_t *src_off,
                                      ptrdiff_t stride);

/* videodsp: replaces VideoDSPContext (libavcodec/videodsp.h:32-69) as filled by ff_videodsp_init(ctx, 8)
 * (libavcodec/videodsp.c:32-62): emulated_edge_mc copies a block_w x block_h window whose top-left sample is picture
 * position (src_x, src_y) (src points AT that sample, inside or outside the picture) and replicates the border samples of
 * the w x h picture for everything outside it (videodsp_template.c:24-101).  prefetch is the reference's empty function. */
typedef struct B200VideoDSPContext {
    void (*emulated_edge_mc)(uint8_t *dst, const uint8_t *src, ptrdiff_t dst_linesize, ptrdiff_t src_linesize,
                             int block_w, int block_h, int src_x, int src_y, int w, int h);
    void (*prefetch)(const uint8_t *buf, ptrdiff_t stride, int h);
} B200VideoDSPContext;
int  b200_videodsp_init(B200VideoDSPContext *c, int bpc);             /* bpc <= 8: bytes; above: the 16-bit template (uint16 samples,
                                                                        * geometry in pixels, line sizes in bytes), videodsp.c:41-45 */
/* batched, DEVICE pointers: window i = geom[4i..4i+3] = {block_w, block_h, src_x, src_y} of the picture whose sample (0, 0)
 * is src + origin[i] (so one call can span many frames of equal w x h and linesize), written to buf + buf_off[i].
 * geom must be 16-byte aligned.  w == 0 or h == 0 writes nothing, like the reference. */
int  b200_emulated_edge_mc_batch_device(B200Device *dev, int64_t n, uint8_t *buf, const int64_t *buf_off,
                                        ptrdiff_t buf_linesize, const uint8_t *src, const int64_t *origin,
                                        ptrdiff_t src_linesize, const int32_t *geom, int w, int h);
/* the same for 16-bit samples: geom in pixels; buf_off, origin and the line sizes in BYTES (even) */
int  b200_emulated_edge_mc_hbd_batch_device(B200Device *dev, int64_t n, uint8_t *buf, const int64_t *buf_off,
                                            ptrdiff_t buf_linesize, const uint8_t *src, const int64_t *origin,
                                            ptrdiff_t src_linesize, const int32_t *geom, int w, int h);

/* ------------------------------------------------------------------------------------------------ libavutil/tx
 * Replaces av_tx_init / av_tx_uninit / av_tx_fn (libavutil/tx.h:151,202-208) for the types below, with the floating-point operation order
 * of the reference's C codelets (bit-identical results).
 * Inside FFmpeg the plug point is a codelet list with prio FF_TX_PRIO_MAX (libavutil/tx_priv.h:168, tx.c:340-351). */
#define B200_TX_FLOAT_FFT   0     /* AV_TX_FLOAT_FFT  */
#define B200_TX_FLOAT_MDCT  1     /* AV_TX_FLOAT_MDCT */
#define B200_TX_FLOAT_RDFT  6     /* AV_TX_FLOAT_RDFT: forward = real-to-complex (len floats -> len/2+1 complex), inverse =
                                   * complex-to-real; scale: const float *.  Like the reference's ff_tx_rdft_c2r
                                   * (tx_template.c:1655-1724) the host av_tx_fn rewrites its input on the inverse; the
                                   * batched device entry point leaves the input untouched.  AV_TX_REAL_TO_REAL /
                                   * AV_TX_REAL_TO_IMAGINARY are not implemented. */
#define B200_TX_DOUBLE_FFT  2     /* AV_TX_DOUBLE_FFT: AVComplexDouble in / out, power-of-two lengths up to 8192 (libavutil/tx_double.c) */
#define B200_TX_DOUBLE_MDCT 3     /* AV_TX_DOUBLE_MDCT: doubles, scale as const double *, power-of-two lengths */
#define B200_TX_INT32_FFT   4     /* AV_TX_INT32_FFT: AVComplexInt32 in / out, power-of-two lengths (libavutil/tx_int32.c) */
#define B200_TX_INT32_MDCT  5     /* AV_TX_INT32_MDCT: int32 samples, scale as const float *, power-of-two lengths (fixed-point AAC / AC-3) */
#define B200_TX_FLOAT_DCT   9     /* AV_TX_FLOAT_DCT: forward = DCT-II of len points, inverse = DCT-III of 2 * len points (the reference's
                                   * ff_tx_dct_init doubles the length it is given, libavutil/tx_template.c:1844-1848; callers pass N / 2).
                                   * ff_tx_dctII / ff_tx_dctIII (tx_template.c:1874-1968).  Input and output are N floats per transform;
                                   * unlike the reference neither the input is overwritten nor 2 floats of padding are needed. */
#define B200_TX_INPLACE     1     /* AV_TX_INPLACE: AV_TX_FLOAT_FFT only (power-of-two and compound); out == in is allowed (batch: out_step == in_step) */
#define B200_TX_UNALIGNED   2     /* AV_TX_UNALIGNED (accepted, no effect) */
#define B200_TX_FULL_IMDCT  4     /* AV_TX_FULL_IMDCT (libavutil/tx.h:175-180; ff_tx_mdct_inv_full, tx_template.c:1372-1413): inverse
                                   * AV_TX_FLOAT_MDCT only; 2 * len outputs, stride must be sizeof(float) */
typedef struct B200TXContext B200TXContext;
typedef void (*b200_tx_fn)(B200TXContext *s, void *out, void *in, ptrdiff_t stride);   /* av_tx_fn: HOST pointers */
/* like av_tx_init(); uses the process-wide default device.  scale: const float * (MDCT), ignored for FFT.
 * Lengths: powers of two, and for AV_TX_FLOAT_MDCT also 2 * N * 2^k with N = 15, 9, 7, 5 or 3: the compound transform av_tx_init() resolves
 * to for those (ff_tx_mdct_pfa_{15,9,7,5,3}xM_{inv,fwd}_float_c, libavutil/tx_template.c:1471-1599; 15 x M covers the Opus CELT sizes),
 * and for AV_TX_FLOAT_FFT also N * 2^k (2^k = 2 ... 512): the compound transform ff_tx_fft_pfa over fftN_ns and the split-radix
 * transform (libavutil/tx_template.c:948-1080; checkasm lengths 120 / 960 / 1920).  The compound FFT stores out[i * stride] like the
 * reference (stride in bytes, a multiple of 8); AV_TX_INPLACE is accepted for it.
 * Returns 0 or B200_ENOSYS (unsupported type / flags / length), B200_EINVAL, B200_ENODEV. */
int  b200_tx_init(B200TXContext **ctx, b200_tx_fn *tx, int type, int inv, int len, const void *scale, uint64_t flags);
/* host-only: the tables ff_tx_mdct_pfa_init() builds for a 15 x M MDCT, flattened into 32-bit words, for the CPU test tier
 * (layout8: word offsets of in_map, out_map, sub_map, exp, tab_53 + tab_7 + tab_9 (26 floats), cosine tables; then M and log2 M | N << 8).  Returns the word count. */
int  b200_tx_pfa_tables(int inv, int len, float scale, int32_t *words, int cap, int32_t *layout8);
/* host-only: the factor table of ff_tx_dct_init (N rotation factors, then N / 2 butterfly factors), for the CPU test tier */
int  b200_tx_dct_table(int inv, int len, float *tab, int cap);
/* host-only: the tables of an int32 transform flattened into words (layout4: offsets of map, exp, cosine tables; then log2 n) */
int  b200_tx_i32_tables(int type, int inv, int len, float scale, int32_t *words, int cap, int32_t *layout4);
/* host-only: the per-thread plan of the register-resident 512 ... 4096-point kernel (csrc/tx_r16.cu; word w of thread tg at
 * words[w * (n / 16) + tg]), for the CPU test tier, which replays the schedule in numpy and compares it with the checker.
 * Returns the word count, B200_ENOSYS for sizes the kernel does not cover. */
int  b200_tx_r16_plan(int n, int inv, uint32_t *words, int cap);
int  b200_tx_init_device(B200Device *dev, B200TXContext **ctx, b200_tx_fn *tx, int type, int inv, int len,
                         const void *scale, uint64_t flags);
void b200_tx_uninit(B200TXContext **ctx);
/* batched, DEVICE pointers: transform i reads in + i*in_step and writes out + i*out_step (bytes); `stride` as av_tx_fn
 * (bytes between MDCT input samples for the inverse / output samples for the forward transform; unused for FFT).
 * Alignment: the kernels move complex values as whole words, so a pointer and its step must both be multiples of
 *   FLOAT_FFT, FLOAT_RDFT (both directions): 8 for in and out (the real samples of r2c / c2r are read / written in pairs)
 *   FLOAT_MDCT power of two: in 4; out 8 for the inverse (AV_TX_FULL_IMDCT too), 4 for the forward; stride a multiple of 4
 *   FLOAT_MDCT compound: in 4; out 8 for the inverse, 4 for the forward (AV_TX_FULL_IMDCT: out + len / 2 floats 8-aligned)
 *   FLOAT_FFT compound: 8 for in, out and stride
 *   FLOAT_DCT: in 4; out 8 for the inverse (DCT-III), 4 for the forward
 *   INT32_FFT: 8 for in and out; INT32_MDCT: in 4, out 8 for the inverse and 4 for the forward
 *   DOUBLE_FFT: 16 for in and out; DOUBLE_MDCT: in 8, out 16 for the inverse and 8 for the forward, stride a multiple of 8
 * Other pointers or steps return B200_EINVAL (message in b200_last_error()) and launch nothing. */
int  b200_tx_batch_device(B200TXContext *ctx, void *out, const void *in, ptrdiff_t stride, int64_t count,
                          ptrdiff_t out_step, ptrdiff_t in_step);
/* same on HOST buffers (pinned memory for real overlap): chunks of transforms rotate over three streams, each chunk = one linear H2D
 * of [i * in_step, (i + n) * in_step), the kernels, one linear D2H; steps must be positive multiples of 16 bytes.  What a decoder that
 * keeps its coefficient buffers in host memory calls once per packet batch instead of count x av_tx_fn (aacdec_dsp_template.c:341-343). */
int  b200_tx_batch_host(B200TXContext *ctx, void *out, const void *in, ptrdiff_t stride, int64_t count,
                        ptrdiff_t out_step, ptrdiff_t in_step);

#ifdef __cplusplus
}
#endif
#endif /* B200DSP_H */
