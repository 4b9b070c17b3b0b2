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

/* One intra transform unit of b200_hevc_intra_recon_picture_device: a call of s->hpc.intra_pred[log2_size - 2] and the residual of
 * ff_hevc_hls_residual_coding that hls_transform_unit (hevc/hevcdec.c:1306-1513) adds after it.  plane, x, y, log2_size, mode and flags
 * mean what B200HevcIntraOp's fields mean for that plane (x / y multiples of 4).  The residual is B200HevcTuOp's: tu_kind, tu_flags
 * (B200_HEVC_TU_RDPCM / RDPCM_VER / ROTATE), col_limit and the (1 << log2_size)^2 coefficients at coef + coef_off (a multiple of 8);
 * tu_kind = B200_HEVC_TU_NONE for a TU whose cbf is 0 (prediction only, coef_off ignored). */
#define B200_HEVC_TU_NONE 0xFF
typedef struct B200HevcIntraReconOp {
    int64_t  coef_off;    /* int16 elements, into coef */
    int32_t  x, y;        /* the TU's top-left in plane samples */
    uint8_t  plane;       /* 0 luma, 1 Cb, 2 Cr */
    uint8_t  log2_size;   /* 2..5 */
    uint8_t  mode;        /* as B200HevcIntraOp.mode */
    uint8_t  tu_kind;     /* B200_HEVC_TU_* or B200_HEVC_TU_NONE */
    uint16_t flags;       /* B200_HEVC_INTRA_* */
    uint8_t  tu_flags;    /* B200_HEVC_TU_RDPCM, B200_HEVC_TU_RDPCM_VER, B200_HEVC_TU_ROTATE */
    uint8_t  reserved0;
    int32_t  col_limit;   /* B200_HEVC_TU_IDCT only */
    uint8_t  reserved[4];
} B200HevcIntraReconOp;
#ifdef __cplusplus
static_assert(sizeof(B200HevcIntraReconOp) == 32, "B200HevcIntraReconOp is 32 bytes");
#else
_Static_assert(sizeof(B200HevcIntraReconOp) == 32, "B200HevcIntraReconOp is 32 bytes");
#endif
/* Intra reconstruction of a whole HEVC picture in one call, DEVICE pointers (planes, ops, coef, intra_map), asynchronous on the device's
 * stream.  `ops` lists every intra TU of the picture, all components, in decode order (the order hls_transform_unit calls intra_pred).
 * The result is, for each op in that order, intra_pred as b200_hevc_intra_pred_batch_device defines it, then the residual as
 * b200_hevc_transform_add_batch_device defines it, on planes that already hold the picture's inter reconstruction and PCM samples: record
 * one op per TU and make this call after the inter MC and residual calls and before deblocking.  width / height: the luma picture size;
 * chroma_format_idc 0..3 gives the chroma planes' shifts (4:2:0, 4:2:2, 4:4:4; 0: luma only, planes[1] / [2] unused).  ls_y / ls_uv:
 * the line sizes in bytes.  intra_map, map_stride and log2_min_pu_size mean what they mean for the batch entry (one map for all
 * components).  `coef` (int16) is read only.
 * Not covered: cross-component prediction (4:4:4 range extensions, hevcdec.c:1398, where a chroma TU adds part of the luma residual) and
 * pictures whose PPS enables current-picture referencing; decode those with the batch entries.
 * The ops of one call write disjoint blocks (decode order gives that; where ops overlap, the samples of the overlap and of the ops
 * that read them are undefined).  An op waits for the earlier ops of its plane that write the samples it reads.  An op that the batch
 * entries would refuse writes nothing and holds up no later op: log2_size or mode out of range, an undefined tu_kind, DST4 on a TU other than 4x4, x / y not
 * multiples of 4, coef_off negative or not a multiple of 8 (with a residual), the block or its flagged neighbours outside the plane, a
 * plane index above 2 or above 0 with chroma_format_idc 0.
 * Returns 0, or B200_EINVAL (launching nothing) for NULL planes, a depth other than 8, 9, 10 or 12, chroma_format_idc outside 0..3,
 * width or height outside 1..65536, a line size shorter than a plane row or not a multiple of 4 samples, a plane not aligned to 4
 * samples, nops outside 0..2^30, an intra_map with map_stride < (width >> log2_min_pu_size) or log2_min_pu_size outside 2..6, or
 * (nops > 0) ops NULL or not aligned to 16 bytes, coef NULL or not aligned to 16 bytes; nops == 0 returns 0. */
int  b200_hevc_intra_recon_picture_device(B200Device *dev, int bit_depth, int chroma_format_idc, int width, int height,
                                          uint8_t *const planes[3], ptrdiff_t ls_y, ptrdiff_t ls_uv, int64_t nops,
                                          const B200HevcIntraReconOp *ops, const int16_t *coef, const uint8_t *intra_map,
                                          ptrdiff_t map_stride, int log2_min_pu_size);
/* The picture entry's waits are bounded by about one second each, after which the op runs anyway (wrong samples rather than a hung
 * GPU) and a per-device counter is incremented.  This waits for the device's stream and stores in *count the number of the picture
 * entry's waits that ran out on that device since the process started (the VP9 entries count theirs apart).  0; B200_EINVAL for
 * count == NULL; B200_ENODEV; B200_EEXTERNAL. */
int  b200_hevc_intra_timeouts(B200Device *dev, int64_t *count);

/* VP9 motion compensation: VP9DSPContext (libavcodec/vp9dsp.h:40-122) in the reference's member order and types.
 * b200_vp9_dsp_init() fills mc[5][4][2][2][2] and smc[5][4][2] completely, as ff_vp9dsp_init does through ff_vp9dsp_mc_init
 * (vp9dsp_template.c:2302-2361) and ff_vp9dsp_scaled_mc_init (:2540-2569): [size 0..4 = 64, 32, 16, 8, 4 columns][filter bank in
 * FilterMode order: smooth, regular, sharp, bilinear (vp9.h:64-71)][0 put, 1 avg][filters horizontally][filters vertically]; the four
 * [0][0] full-pel entries of a size and put / avg are one function, as in the reference (:2308-2322).  Every other member stays NULL.
 * HOST pointers, the reference's signatures: samples uint8 at 8 bit and uint16 at 10 / 12, strides in bytes, h 1..64, mx / my 0..15
 * (sixteenths), dx / dy 1..32 (sixteenths of a source sample per output sample: the range the reference's tmp[64 * 135] allows,
 * :2369-2370, a reference 2x larger to 16x smaller).
 *   8-tap banks  clip((sum F[k] * src[-3 + k] + 64) >> 7), F = ff_vp9_subpel_filters[bank][phase] (vp9dsp.c:32-85, the subpel_filters
 *                of the VP9 bitstream specification); in two dimensions the horizontal results are clipped samples for rows -3 .. h + 3
 *                and the vertical pass filters those (FILTER_8TAP :2026-2034, do_8tap_2d_c :2076-2113)
 *   bilinear     src[0] + ((m * (src[1] - src[0]) + 8) >> 4), no clip (:2150-2151), the horizontal results for rows 0 .. h
 *   put          dst = v;   avg: dst = (dst + v + 1) >> 1
 *   smc          source column of output column x is (mx + x * dx) >> 4 with phase (mx + x * dx) & 15, likewise rows with my, dy;
 *                always both passes (do_scaled_8tap_c :2363-2409, do_scaled_bilin_c :2439-2482)
 * A member filters in the directions its table position names, with the phase it is handed: phase 0 in a filtered direction is the
 * identity row { 0, 0, 0, 128, 0, 0, 0, 0 } / bilinear weight 0.  It reads exactly the samples its reference function reads: columns
 * -3..+4 around the block only where it filters horizontally with an 8-tap bank, 0..+1 for bilinear, the same for rows; an smc member
 * always the window of (((w - 1) * dx + mx) >> 4) + 8 columns by (((h - 1) * dy + my) >> 4) + 8 rows from (-3, -3) for an 8-tap bank,
 * + 2 from (0, 0) for bilinear.  A call with h, a phase or a step outside these ranges writes nothing and records the reason
 * (b200_last_error()). */
typedef void (*b200_vp9_mc_func)(uint8_t *dst, ptrdiff_t dst_stride, const uint8_t *ref, ptrdiff_t ref_stride, int h, int mx, int my);
typedef void (*b200_vp9_scaled_mc_func)(uint8_t *dst, ptrdiff_t dst_stride, const uint8_t *ref, ptrdiff_t ref_stride, int h, int mx, int my,
                                        int dx, int dy);
typedef struct B200VP9DSPContext {
    void (*intra_pred[4][15])(uint8_t *dst, ptrdiff_t stride, const uint8_t *left, const uint8_t *top);
    void (*itxfm_add[5][4])(uint8_t *dst, ptrdiff_t stride, int16_t *block, int eob);
    void (*loop_filter_8[3][2])(uint8_t *dst, ptrdiff_t stride, int mb_lim, int lim, int hev_thr);
    void (*loop_filter_16[2])(uint8_t *dst, ptrdiff_t stride, int mb_lim, int lim, int hev_thr);
    void (*loop_filter_mix2[2][2][2])(uint8_t *dst, ptrdiff_t stride, int mb_lim, int lim, int hev_thr);
    b200_vp9_mc_func mc[5][4][2][2][2];
    b200_vp9_scaled_mc_func smc[5][4][2];
} B200VP9DSPContext;
/* 0; B200_EINVAL for c == NULL; B200_ENOSYS for depths other than 8, 10 and 12 (the reference asserts there, vp9dsp.c:95);
 * B200_ENODEV. */
int  b200_vp9_dsp_init(B200VP9DSPContext *c, int bit_depth);

/* One reference plane of b200_vp9_mc_batch_device: `data` is the DEVICE address of its sample (0, 0), `stride` in bytes, w x h its size
 * in samples, dx / dy its scale steps in sixteenths (vp9.c: s->mvstep[ref]).  dx == dy == 16 is a reference of the current picture's
 * size, predicted through the mc table; any other pair in 1..32 goes through smc (the decoder's switch, vp9recon.c:426-429). */
typedef struct B200Vp9McRef {
    const uint8_t *data;
    ptrdiff_t stride;
    int32_t w, h;
    int32_t dx, dy;
} B200Vp9McRef;
/* One inter block of b200_vp9_mc_batch_device: w (4, 8, 16, 32, 64) x h (1..64) samples at dst + dst_off (bytes), filter bank 0..3
 * (FilterMode order).  Slot r (0; and 1 for COMPOUND) predicts from reference ref[r] of the call's array: integer sample position
 * (x[r], y[r]) in that plane (any value) and phase (mx[r], my[r]) in sixteenths, 0..15.  These are the values the decoder has after
 * its motion-vector arithmetic: mc_luma_unscaled (vp9recon.c:309-313, with mx << 1, my << 1 as at :336), mc_chroma_unscaled
 * (:349-356), and for scaled references the clipped and scaled vectors of mc_luma_scaled (:437-449) / mc_chroma_scaled (:497-520).
 *   B200_VP9_MC_SINGLE    mc[size][filter][0][!!mx0][!!my0] (smc[size][filter][0] for a scaled reference) from slot 0
 *   B200_VP9_MC_COMPOUND  the same, then mc[size][filter][1][!!mx1][!!my1] / smc[size][filter][1] from slot 1 into the same block
 *                         (vp9_mc_template.c); the two slots may name references of different size and steps */
enum { B200_VP9_MC_SINGLE = 0, B200_VP9_MC_COMPOUND = 1 };
typedef struct B200Vp9McOp {
    int64_t dst_off;
    int32_t x[2], y[2];
    uint8_t ref[2];
    uint8_t mx[2], my[2];
    uint8_t w, h, filter, kind;
    uint8_t reserved[6];
} B200Vp9McOp;
#ifdef __cplusplus
static_assert(sizeof(B200Vp9McOp) == 40, "B200Vp9McOp is 40 bytes");
#else
_Static_assert(sizeof(B200Vp9McOp) == 40, "B200Vp9McOp is 40 bytes");
#endif
/* Batched VP9 inter prediction of one plane: `refs` is a HOST array of 1 <= nrefs <= 8 planes (copied into the launch), `ops` and
 * `dst` are DEVICE pointers.  Every op's result is the reference's call sequence above with each output sample stored once, its
 * source samples read through coordinates clamped to [0, w) x [0, h) of that reference.  This is what the decoder's
 * emulated_edge_mc windows give, windows wholly outside the picture included, because whenever the decoder does not emulate, every
 * sample the function reads lies inside the picture (vp9recon.c:325-335, :460-468), so no separate edge emulation pass is needed.
 * The caller guarantees that the ops of one call write disjoint blocks and that no op reads samples another op of the call writes.
 * An op with an undefined kind, filter or width, a reference index >= nrefs, h outside 1..64, a phase above 15 or, at 10 / 12 bit,
 * an odd dst_off writes nothing.  Offsets are 64-bit; more ops than one launch takes are split inside the entry.
 * Returns 0, or B200_EINVAL (launching nothing) for NULL pointers, nops < 0, nrefs outside 1..8, a stride or pointer not a multiple
 * of the sample size, ops not aligned to 8 bytes, a reference with w or h < 1 or a step outside 1..32, or a depth other than 8, 10
 * or 12; nops == 0 returns 0. */
int  b200_vp9_mc_batch_device(B200Device *dev, int bit_depth, int nrefs, const B200Vp9McRef *refs, int64_t nops, const B200Vp9McOp *ops,
                              uint8_t *dst, ptrdiff_t dst_stride);

/* VP9 inverse transforms and residual add: b200_vp9_dsp_init_itxfm() fills the 20 itxfm_add[5][4] pointers of a B200VP9DSPContext as
 * vp9dsp_itxfm_init does (vp9dsp_template.c:1755-1778) and touches no other member (call it after b200_vp9_dsp_init, which leaves
 * them NULL): [tx 0..2 = 4x4, 8x8, 16x16][type in TxfmType order: DCT_DCT idct / idct, DCT_ADST iadst / idct, ADST_DCT idct / iadst,
 * ADST_ADST iadst / iadst] ("a / b" = the type of pass 1 / pass 2), [3][*] one function (32x32 idct / idct), [4][*] one function
 * (lossless: the Walsh-Hadamard transform).  HOST pointers and the reference's signature: `block` holds sz * sz int16 coefficients at
 * 8 bit and int32 ones at 10 / 12 bit (the int16_t * of the signature), the stride is in bytes.
 *   passes    pass 1 applies type a to every column i of the block (block[i + k sz]), giving row i of tmp; pass 2 applies type b to
 *             every column i of tmp, and its output j is added to dst row j, column i as clip(dst + ((int)(out + 2^(bits-1)) >> bits)),
 *             bits 4 / 5 / 6 / 6 for 4 / 8 / 16 / 32; the Walsh-Hadamard transform takes pass 1's inputs >> 2 and adds out unshifted
 *   storage   8 bit: tmp and out int16, arithmetic 32-bit; 10 / 12 bit: int32 and int64; every coefficient value is accepted
 *   DC only   idct / idct at 4..16 and every 32x32 slot with eob == 1: only block[0] is read and cleared; any other eob (0 included)
 *             runs the full transform, which clears all sz * sz coefficients.  Nothing else reads eob.
 * 0; B200_EINVAL for c == NULL; B200_ENOSYS for depths other than 8, 10 and 12; B200_ENODEV. */
int  b200_vp9_dsp_init_itxfm(B200VP9DSPContext *c, int bit_depth);

/* One transform block of b200_vp9_itxfm_add_batch_device: itxfm_add[tx][type](dst + dst_off, dst_stride, coef + coef_off, eob). */
typedef struct B200Vp9TxOp {
    int64_t dst_off;    /* bytes, into dst */
    int64_t coef_off;   /* coefficient elements (int16 at 8 bit, int32 at 10 / 12) into coef: the block's dense sz * sz coefficients */
    uint8_t tx;         /* itxfm_add's first index: 0..3 = 4x4..32x32, 4 = lossless */
    uint8_t type;       /* second index 0..3, TxfmType order (vp9.h) */
    uint16_t eob;       /* as the decoder passes it (vp9recon.c:624, :643) */
    uint8_t reserved[4];
} B200Vp9TxOp;
#ifdef __cplusplus
static_assert(sizeof(B200Vp9TxOp) == 24, "B200Vp9TxOp is 24 bytes");
#else
_Static_assert(sizeof(B200Vp9TxOp) == 24, "B200Vp9TxOp is 24 bytes");
#endif
/* Batched VP9 residual reconstruction of one plane (inter_recon's loop over transform blocks, vp9recon.c:608-652, as one call):
 * `ops`, `coef` and `dst` are DEVICE pointers; asynchronous on the device's stream.  Each op's block of dst becomes what the member
 * above makes of it.  `coef` is read only: the decoder clears its coefficient buffer itself.  The caller guarantees that the ops of
 * one call write disjoint blocks.  An op with tx > 4, type > 3, coef_off not a multiple of 16 or dst_off not a multiple of 4 samples
 * writes nothing.  Offsets are 64-bit; more ops than one launch takes are split inside the entry.
 * Returns 0, or B200_EINVAL (launching nothing) for NULL pointers, nops < 0, a depth other than 8, 10 or 12, ops not aligned to 8
 * bytes, coef not aligned to 16 bytes, dst not aligned to 4 samples or dst_stride not a multiple of 4 samples; nops == 0 returns 0. */
int  b200_vp9_itxfm_add_batch_device(B200Device *dev, int bit_depth, int64_t nops, const B200Vp9TxOp *ops, const void *coef, uint8_t *dst,
                                     ptrdiff_t dst_stride);

/* VP9 loop filter: b200_vp9_dsp_init_loopfilter() fills loop_filter_8[3][2], loop_filter_16[2] and loop_filter_mix2[2][2][2] of a
 * B200VP9DSPContext as vp9dsp_loopfilter_init does (vp9dsp_template.c:1947-1967): 16 distinct functions; it touches no other member.
 * The last index is the direction: 0 filters the edge between two columns (samples across the edge are dst[-8..7], the lines run down
 * the rows), 1 the edge between two rows (dst[-8 stride .. 7 stride], the lines run along the row).  HOST pointers and the reference's
 * signature (dst, stride in bytes, E, I, H); samples uint8 at 8 bit and uint16 at 10 / 12 bit.
 *   loop_filter_8[wd][dir]        8 lines of width 4 << wd (4, 8, 16) with E, I, H
 *   loop_filter_16[dir]           16 lines of width 16 with the same E, I, H
 *   loop_filter_mix2[a][b][dir]   8 lines of width 4 << a with E & 0xff, I & 0xff, H & 0xff, then the next 8 lines of width 4 << b with
 *                                 E >> 8, I >> 8, H >> 8 (:1926-1933)
 * Per line (:1780-1889): E, I and H are shifted left by depth - 8 and F = 1 << (depth - 8); nothing unless every neighbour difference
 * p3..q3 is <= I and 2 |p0 - q0| + |p1 - q1| / 2 <= E; width 16 with p7..q7 all within F of p0 / q0 and p3..q3 within F: the 15-tap
 * smoothing of p6..q6; width >= 8 with p3..q3 within F: the 7-tap smoothing of p2..q2; otherwise the 4-tap filter of p1..q1 (p0 / q0 only
 * when |p1 - p0| or |q1 - q0| exceeds H).  A member reads only dst[-4..3] across the edge for widths 4 / 8 and dst[-8..7] for width 16,
 * and writes only dst[-2..1], dst[-3..2] or dst[-7..6].
 * 0; B200_EINVAL for c == NULL; B200_ENOSYS for depths other than 8, 10 and 12; B200_ENODEV. */
int  b200_vp9_dsp_init_loopfilter(B200VP9DSPContext *c, int bit_depth);

/* One superblock's loop-filter record: VP9Filter's layout (libavcodec/vp9dec.h:79-83).  level[row * 8 + col] is the filter level of the
 * 8x8 luma block (row, col) of the superblock; mask[0 luma, 1 chroma][0 column edges, 1 row edges][8x8 luma row][0 16-wide, 1 8-wide,
 * 2 4-wide, 3 inner 4-wide], bit k = 8x8 luma column k, as the decoder's mask_edges leaves them (vp9block.c:1142-1262). */
typedef struct B200Vp9Filter {
    uint8_t level[8 * 8];
    uint8_t mask[2][2][8][4];
} B200Vp9Filter;
#ifdef __cplusplus
static_assert(sizeof(B200Vp9Filter) == 192, "B200Vp9Filter is 192 bytes");
#else
_Static_assert(sizeof(B200Vp9Filter) == 192, "B200Vp9Filter is 192 bytes");
#endif
/* Loop-filters a whole VP9 frame in place, DEVICE pointers (planes[0..2], lflvl), asynchronous on the device's stream.  The result is
 * ff_vp9_loopfilter_sb (vp9lpf.c:179-203) applied to every superblock in raster order, over Y, U and V: per plane all column edges of the
 * superblock in filter_plane_cols' order, then all its row edges in filter_plane_rows' order (vp9lpf.c:27-177), with that dispatch's
 * quirks, the chroma planes from mask[ss_h | ss_v] (4:4:4 uses the luma masks), the picture's left column and top row edges skipped,
 * E = mblim_lut[L], I = lim_lut[L], H = L >> 4 for the level L (lim_lut / mblim_lut are the decoder's s->filter_lut, HOST arrays copied
 * into the launch; levels index them modulo 64).
 * width and height are the luma picture size: cols = (width + 7) >> 3, rows = (height + 7) >> 3 8x8 blocks, and the superblock grid is
 * ((cols + 7) >> 3) x ((rows + 7) >> 3) records, lflvl[sb_row * lflvl_stride + sb_col].  The planes must cover the 8-aligned area: luma
 * cols * 8 x rows * 8 samples, chroma (cols * 8 >> ss_h) x (rows * 8 >> ss_v) rounded up to a multiple of 8 (the decoder's 8-line chroma
 * edges at an odd cols / rows reach that far).  Ignored, because mask_edges never sets them (vp9block.c:1436-1446, :1206-1225): mask
 * bits of 8x8 columns >= cols and rows >= rows, and the chroma 16-wide bits at column bit 7 (with ss_h) and in row 7 (with ss_v) of the
 * column / row masks, whose edges would reach into the next superblock.  No sample outside the area is read or written; a chroma
 * 16-wide edge whose 16 samples would leave the area (4 samples from its left or top edge, or past its right or bottom edge; the
 * decoder sets none) reads unspecified values for the missing ones.
 * The work runs as a wavefront: superblock (r, c) of a plane starts once (r, c - 1) and (r - 1, c + 1) are done, the order the result
 * depends on.  Offsets are 64-bit.
 * lflvl needs no alignment beyond a byte.
 * Returns 0, or B200_EINVAL (launching nothing) for NULL pointers, a depth other than 8, 10 or 12, ss_h / ss_v outside {0, 1}, width or
 * height < 1, a stride shorter than a plane row or not a multiple of the sample size, a plane not aligned to a sample, or lflvl_stride
 * below the superblock column count. */
int  b200_vp9_loopfilter_frame_device(B200Device *dev, int bit_depth, int ss_h, int ss_v, int width, int height, uint8_t *const planes[3],
                                      ptrdiff_t ls_y, ptrdiff_t ls_uv, const B200Vp9Filter *lflvl, int64_t lflvl_stride,
                                      const uint8_t lim_lut[64], const uint8_t mblim_lut[64]);
/* The frame entry's superblocks wait on the row above; every such wait is bounded by about one second, after which the superblock is
 * filtered anyway (wrong samples rather than a hung GPU) and a per-device counter is incremented.  This waits for the device's stream
 * and stores the number of waits that ran out on that device since the process started (0 unless something kept the row above from
 * running for a second) in *count.  0; B200_EINVAL for count == NULL; B200_ENODEV; B200_EEXTERNAL. */
int  b200_vp9_loopfilter_timeouts(B200Device *dev, int64_t *count);

/* VP9 intra prediction: b200_vp9_dsp_init_intrapred() fills the 60 intra_pred[4][15] pointers of a B200VP9DSPContext as
 * ff_vp9dsp_intrapred_init does (vp9dsp_template.c:1120-1152): [tx 0..3 = 4x4 .. 32x32][mode in IntraPredMode order, vp9.h:45-61];
 * at 12 bit every mode but TM_VP8 and DC_127 / 128 / 129 is the 10-bit function, as in the reference.  It touches no other member.
 * HOST pointers and the reference's signature (dst, stride in bytes, left, top); samples uint8 at 8 bit and uint16 at 10 / 12 bit.
 * `left` is the column bottom-to-top (left[size - 1] is the sample beside row 0) except for HOR_UP, which takes it top-to-bottom.
 * A member reads exactly the samples its reference function reads: top[-1] for TM, DIAG_DOWN_RIGHT, VERT_RIGHT and HOR_DOWN
 * (HOR_DOWN reads top[-1 .. size - 2]); top[0 .. 7] for the 4x4 DIAG_DOWN_LEFT and top[0 .. 6] for the 4x4 VERT_LEFT; left[1 .. size - 1]
 * for VERT_RIGHT; the DC_127 / 128 / 129 functions read nothing.  It writes only the size x size block.
 * 0; B200_EINVAL for c == NULL; B200_ENOSYS for depths other than 8, 10 and 12; B200_ENODEV. */
int  b200_vp9_dsp_init_intrapred(B200VP9DSPContext *c, int bit_depth);

/* One transform block of intra_recon (vp9recon.c:219-287) for b200_vp9_intra_recon_frame_device.  The flags are the call site's:
 *   B200_VP9_INTRA_HAVE_LEFT   col > td->tile_col_start || x > 0 (vp9recon.c:42)
 *   B200_VP9_INTRA_HAVE_RIGHT  x < w - 1 in 4x4 units of the block, w = w4 for luma and w4 >> ss_h for chroma (:43, :259)
 *   B200_VP9_INTRA_LOSSLESS    s->s.h.lossless: the residual goes through itxfm_add[4] (tx must be 0) */
enum { B200_VP9_INTRA_HAVE_LEFT = 1, B200_VP9_INTRA_HAVE_RIGHT = 2, B200_VP9_INTRA_LOSSLESS = 4 };
typedef struct B200Vp9IntraOp {
    int64_t coef_off;   /* element offset of td->block + 16 * n * bytesperpixel (or of td->uvblock[p] + ...) in coef: a multiple of 16 */
    int32_t x, y;       /* top-left sample of the transform block in its plane, multiples of 4 */
    uint16_t eob;       /* as intra_recon reads it: 0 when b->skip */
    uint8_t plane;      /* 0, 1, 2 */
    uint8_t tx;         /* b->tx or b->uvtx, 0..3: the intra_pred size index */
    uint8_t mode;       /* b->mode[...] or b->uvmode, 0..9, before mode_conv */
    uint8_t flags;      /* B200_VP9_INTRA_* */
    uint8_t reserved[10];
} B200Vp9IntraOp;
#ifdef __cplusplus
static_assert(sizeof(B200Vp9IntraOp) == 32, "B200Vp9IntraOp is 32 bytes");
#else
_Static_assert(sizeof(B200Vp9IntraOp) == 32, "B200Vp9IntraOp is 32 bytes");
#endif
/* Intra reconstruction of a whole VP9 frame in one call, DEVICE pointers (planes[0..2], ops, coef), asynchronous on the device's
 * stream.  `ops` lists every intra transform block of the frame, all three planes, in decode order: the order intra_recon visits them,
 * block after block (each block's luma, then U, then V).  The result is intra_recon's check_intra_mode, intra_pred[tx][mode] and, when
 * eob is non-zero, itxfm_add[4 * lossless + tx][txtp] (txtp = ff_vp9_intra_txfm_type[mode] for luma, DCT_DCT for chroma) applied to
 * every op in that order, on planes that already hold the frame's inter reconstruction.  The entry derives from each op: have_top =
 * y > 0; the top row's n_px_have = (cols * 8 >> ss_h) - x and the left column's (rows * 8 >> ss_v) - y (vp9recon.c:99, :188).
 * `coef` holds int16 coefficients at 8 bit and int32 ones at 10 / 12 bit and is read only (clearing stays with the decoder).
 * width and height are the luma picture size; cols = (width + 7) >> 3, rows = (height + 7) >> 3.  The planes must cover the 8-aligned
 * area: luma cols * 8 x rows * 8 samples, chroma (cols * 8 >> ss_h) x (rows * 8 >> ss_v).  Only samples inside it are read or written:
 * the part of a block that lies outside is not stored (the decoder's emulated-edge buffers drop it too, vp9block.c:1368-1430), and
 * nothing reads it.  The top row of a superblock row is read from the plane: run the loop filter after this call, so that the plane
 * row above still holds the decoder's intra_pred_data (vp9.c:1387-1398).
 * The ops of one call write disjoint blocks, and an op reads only samples of ops listed before it, of inter blocks or of earlier calls
 * (decode order guarantees both).  An op waits for the earlier ops that write the samples it reads; an op with plane > 2, tx > 3,
 * mode > 9, a negative or unaligned x, y or coef_off, or LOSSLESS with tx != 0, and an op outside the plane, writes nothing.
 * Returns 0, or B200_EINVAL (launching nothing) for NULL planes, a depth other than 8, 10 or 12, ss_h / ss_v outside {0, 1}, width or
 * height outside 1..65536, nops outside 0..2^30, a stride shorter than a plane row or not a multiple of the sample size, a plane not
 * aligned to a sample, or (nops > 0) ops NULL or not aligned to 8 bytes, coef NULL or not aligned to 16 bytes; nops == 0 returns 0. */
int  b200_vp9_intra_recon_frame_device(B200Device *dev, int bit_depth, int ss_h, int ss_v, int width, int height, uint8_t *const planes[3],
                                       ptrdiff_t ls_y, ptrdiff_t ls_uv, int64_t nops, const B200Vp9IntraOp *ops, const void *coef);
/* The frame entry's ops wait on earlier ops; every such wait is bounded by about one second, after which the op runs anyway (wrong
 * samples rather than a hung GPU) and a per-device counter is incremented.  This waits for the device's stream and stores the number of
 * the intra entry's waits that ran out on that device since the process started in *count (the loop filter's are counted apart, by
 * b200_vp9_loopfilter_timeouts).  0; B200_EINVAL for count == NULL; B200_ENODEV; B200_EEXTERNAL. */
int  b200_vp9_intra_timeouts(B200Device *dev, int64_t *count);

/* VP8 / VP7 motion compensation and residual: VP8DSPContext (libavcodec/vp8dsp.h:37-82) in the reference's member order and types.
 * b200_vp8_dsp_init() fills what ff_vp78dsp_init and ff_vp8dsp_init (is_vp7 = 0) / ff_vp7dsp_init (is_vp7 = 1) fill (vp8dsp.c:663-760)
 * except the ten loop-filter members, which it leaves NULL (b200_vp8_dsp_init_loopfilter fills them):
 *   vp8_luma_dc_wht, _wht_dc, vp8_idct_add, _dc_add, _dc_add4y, _dc_add4uv   the VP8 or the VP7 arithmetic
 *   put_vp8_epel_pixels_tab[size][v][h]       size 0..2 = 16, 8, 4 columns; v / h: 0 none, 1 4-tap, 2 6-tap; [0][1][*] and [0][*][1]
 *                                             NULL, as in the reference
 *   put_vp8_bilinear_pixels_tab[size][v][h]   v / h: 0 none, 1 and 2 bilinear
 * Shared as in the reference: [i][0][0] is one function in both tables; in the bilinear table [i][0][1] / [i][0][2] are one function,
 * [i][1][0] / [i][2][0] are one, and the four 2-D positions are one.  HOST pointers, the reference's signatures; MC source and
 * destination are uint8, strides in bytes.
 *   6-tap     clip((F0 s[-2] - F1 s[-1] + F2 s[0] + F3 s[1] - F4 s[2] + F5 s[3] + 64) >> 7), F = subpel_filters[phase - 1] (vp8dsp.c:459-490)
 *   4-tap     clip((- F1 s[-1] + F2 s[0] + F3 s[1] - F4 s[2] + 64) >> 7) of the same row, whatever the phase's parity
 *   bilinear  ((8 - m) s[0] + m s[1] + 4) >> 3
 *   2-D       the horizontal pass, clipped to uint8, over rows -2 .. h + 2 (6-tap vertical) or -1 .. h + 1 (4-tap) / 0 .. h (bilinear),
 *             then the vertical pass over it
 * A member reads exactly the samples its reference function reads.  It writes nothing and records the reason (b200_last_error()) for h
 * outside 1 .. 2 * width (the reference's tmp_array), a phase above 7, or an epel member handed phase 0 in a direction it filters (the
 * reference indexes subpel_filters[-1] there).
 *   wht        VP8: column pass into int16 dc[], then (x + 3) >> 3 into block[i][j][0] (vp8dsp.c:152-180); VP7: row pass with the
 *              products in unsigned, (int) >> 14 into int16, then the column pass (+ 0x20000) >> 18 (:56-84); clears dc[0..15]
 *   wht_dc     VP8 (dc[0] + 3) >> 3, VP7 (23170 * (23170 * dc[0] >> 14) + 0x20000) >> 18 into all 16 block[i][j][0]; clears dc[0]
 *   idct_add   VP8: column pass with MUL_20091 / MUL_35468 into int16, row pass (+ 4) >> 3 added and clipped (:195-231); VP7 as wht with
 *              the add (:99-131); clears block[0..15]
 *   dc_add     VP8 (block[0] + 4) >> 3, VP7 as wht_dc, added to the 4x4 block; reads and clears block[0] only
 *   dc_add4y   dc_add on the four blocks at dst + 0, 4, 8, 12;  dc_add4uv: at dst, dst + 4, dst + 4 stride, dst + 4 stride + 4
 * 0; B200_EINVAL for c == NULL or is_vp7 not 0 / 1; B200_ENODEV. */
typedef void (*b200_vp8_mc_func)(uint8_t *dst, ptrdiff_t dst_stride, const uint8_t *src, ptrdiff_t src_stride, int h, int mx, int my);
typedef struct B200VP8DSPContext {
    void (*vp8_luma_dc_wht)(int16_t block[4][4][16], int16_t dc[16]);
    void (*vp8_luma_dc_wht_dc)(int16_t block[4][4][16], int16_t dc[16]);
    void (*vp8_idct_add)(uint8_t *dst, int16_t block[16], ptrdiff_t stride);
    void (*vp8_idct_dc_add)(uint8_t *dst, int16_t block[16], ptrdiff_t stride);
    void (*vp8_idct_dc_add4y)(uint8_t *dst, int16_t block[4][16], ptrdiff_t stride);
    void (*vp8_idct_dc_add4uv)(uint8_t *dst, int16_t block[4][16], ptrdiff_t stride);
    void (*vp8_v_loop_filter16y)(uint8_t *dst, ptrdiff_t stride, int flim_E, int flim_I, int hev_thresh);
    void (*vp8_h_loop_filter16y)(uint8_t *dst, ptrdiff_t stride, int flim_E, int flim_I, int hev_thresh);
    void (*vp8_v_loop_filter8uv)(uint8_t *dstU, uint8_t *dstV, ptrdiff_t stride, int flim_E, int flim_I, int hev_thresh);
    void (*vp8_h_loop_filter8uv)(uint8_t *dstU, uint8_t *dstV, ptrdiff_t stride, int flim_E, int flim_I, int hev_thresh);
    void (*vp8_v_loop_filter16y_inner)(uint8_t *dst, ptrdiff_t stride, int flim_E, int flim_I, int hev_thresh);
    void (*vp8_h_loop_filter16y_inner)(uint8_t *dst, ptrdiff_t stride, int flim_E, int flim_I, int hev_thresh);
    void (*vp8_v_loop_filter8uv_inner)(uint8_t *dstU, uint8_t *dstV, ptrdiff_t stride, int flim_E, int flim_I, int hev_thresh);
    void (*vp8_h_loop_filter8uv_inner)(uint8_t *dstU, uint8_t *dstV, ptrdiff_t stride, int flim_E, int flim_I, int hev_thresh);
    void (*vp8_v_loop_filter_simple)(uint8_t *dst, ptrdiff_t stride, int flim);
    void (*vp8_h_loop_filter_simple)(uint8_t *dst, ptrdiff_t stride, int flim);
    b200_vp8_mc_func put_vp8_epel_pixels_tab[3][3][3];
    b200_vp8_mc_func put_vp8_bilinear_pixels_tab[3][3][3];
} B200VP8DSPContext;
int  b200_vp8_dsp_init(B200VP8DSPContext *c, int is_vp7);

/* One reference frame of b200_vp8_mc_frame_device: DEVICE addresses of sample (0, 0) of its three planes, line sizes in bytes. */
typedef struct B200Vp8McRef {
    const uint8_t *y, *u, *v;
    ptrdiff_t ls_y, ls_uv;
} B200Vp8McRef;
/* One inter block of b200_vp8_mc_frame_device.  plane LUMA writes a w x h block of Y at (dst_x, dst_y); CHROMA writes the same block
 * of U and of V, as vp8_mc_chroma does.  (src_x, src_y) is the integer source position and mx / my the eighth-sample phase (0..7), as
 * the decoder has them after its motion-vector arithmetic: x_off + (mv >> 2) with phase (mv * 2) & 7 for luma, x_off + (mv >> 3) with
 * mv & 7 for chroma (vp8.c:1844-1848, :1900-1904).  Split-MV chroma averaging, profile-3 full-pel chroma and MV clamping stay with the
 * caller. */
enum { B200_VP8_MC_LUMA = 0, B200_VP8_MC_CHROMA = 1 };
typedef struct B200Vp8McOp {
    int32_t src_x, src_y;   /* any value */
    int32_t dst_x, dst_y;   /* top-left sample of the block in its plane; dst_x a multiple of 4 */
    uint8_t plane;          /* B200_VP8_MC_LUMA / B200_VP8_MC_CHROMA */
    uint8_t w, h;           /* w 16, 8 or 4; h 1..16 */
    uint8_t ref;            /* index into the call's refs */
    uint8_t mx, my;         /* 0..7 */
    uint8_t reserved[2];
} B200Vp8McOp;
#ifdef __cplusplus
static_assert(sizeof(B200Vp8McOp) == 24, "B200Vp8McOp is 24 bytes");
#else
_Static_assert(sizeof(B200Vp8McOp) == 24, "B200Vp8McOp is 24 bytes");
#endif
/* Inter prediction of a whole VP8 / VP7 frame in one call: `refs` is a HOST array of 1 <= nrefs <= 3 frames (copied into the launch),
 * `ops` and the dst[0..2] planes are DEVICE pointers; asynchronous on the device's stream.  bilinear selects
 * put_vp8_bilinear_pixels_tab, else put_vp8_epel_pixels_tab (the decoder's put_pixels_tab: epel for VP7 and for VP8 profile 0,
 * vp8.c:601, :757-762).  Each op's result is put_pixels_tab[size of w][subpel_idx[0][my]][subpel_idx[0][mx]] (odd phase 4-tap, even
 * non-zero phase 6-tap, vp8.c:1809-1814), its source samples read through coordinates clamped to the plane: 16 mb_width x 16 mb_height
 * for luma, 8 mb_width x 8 mb_height for chroma.  That is what the decoder's emulated_edge_mc windows give, and where the decoder does
 * not emulate its own test (vp8.c:1853-1854, :1910-1911) keeps every read inside the plane, so no edge emulation pass is needed.
 * The caller guarantees that the ops of one call write disjoint blocks and that no op reads what another op of the call writes.
 * An op writes nothing if its plane class or width is undefined, h is outside 1..16, a phase is above 7, ref >= nrefs, it is a
 * 16-wide epel op with an odd phase (the reference table is NULL there), dst_x is not a multiple of 4, or its block is not inside the
 * plane.  Offsets are 64-bit; more ops than one launch takes are split inside the entry.
 * Returns 0, or B200_EINVAL (launching nothing) for NULL pointers, nops < 0, nrefs outside 1..3, mb_width or mb_height outside
 * 1..65536, ops not aligned to 4 bytes, or a dst plane or line size that is not a multiple of 4; nops == 0 returns 0. */
int  b200_vp8_mc_frame_device(B200Device *dev, int bilinear, int mb_width, int mb_height, int nrefs, const B200Vp8McRef *refs, int64_t nops,
                              const B200Vp8McOp *ops, uint8_t *const dst[3], ptrdiff_t ls_y, ptrdiff_t ls_uv);

/* One macroblock of b200_vp8_residual_frame_device: the state decode_mb_coeffs leaves for idct_mb (vp8.c:1493-1566, :2085-2146). */
enum { B200_VP8_RESIDUAL_LUMA = 1 };    /* flags: the luma residual is present (mode != MODE_I4x4) */
typedef struct B200Vp8ResidualOp {
    int64_t coef_off;       /* element offset in coef of the MB's 400 int16: td->block[6][4][16], then block_dc[16]; a multiple of 8 */
    int32_t mb_x, mb_y;     /* >= 0 */
    uint8_t nnz[6][4];      /* td->non_zero_count_cache */
    uint8_t y2_nnz;         /* 0 none, 1 vp8_luma_dc_wht_dc, > 1 vp8_luma_dc_wht */
    uint8_t flags;          /* B200_VP8_RESIDUAL_* */
    uint8_t reserved[6];
} B200Vp8ResidualOp;
#ifdef __cplusplus
static_assert(sizeof(B200Vp8ResidualOp) == 48, "B200Vp8ResidualOp is 48 bytes");
#else
_Static_assert(sizeof(B200Vp8ResidualOp) == 48, "B200Vp8ResidualOp is 48 bytes");
#endif
/* The residual of every macroblock of a VP8 / VP7 frame in one call, DEVICE pointers (ops, coef, dst[0..2]), asynchronous on the
 * device's stream.  Per op: with y2_nnz > 0 the WHT (or WHT_DC) of block_dc replaces coefficient 0 of the 16 luma blocks, then idct_mb
 * with idct_mb's own decisions: in a luma row (and a chroma plane) whose four nnz bytes are all <= 1 and not all 0, dc_add4y (dc_add4uv)
 * adds the DC of all four blocks, nnz-0 blocks included; otherwise each block alone: nnz 1 dc_add (reads coefficient 0 only), nnz > 1
 * idct_add, 0 nothing.  Luma only with B200_VP8_RESIDUAL_LUMA.  is_vp7 selects the VP7 arithmetic.  Every int16 value is accepted.
 * `coef` is read only: clearing it stays with the decoder.  The ops of one call write disjoint macroblocks.  An op with a negative
 * mb_x / mb_y or coef_off, or coef_off not a multiple of 8, writes nothing.  Offsets are 64-bit; more ops than one launch takes are
 * split inside the entry.
 * Returns 0, or B200_EINVAL (launching nothing) for NULL pointers, nops < 0, is_vp7 not 0 / 1, ops not aligned to 8 bytes, coef not
 * aligned to 16 bytes, or a dst plane or line size that is not a multiple of 4; nops == 0 returns 0. */
int  b200_vp8_residual_frame_device(B200Device *dev, int is_vp7, int64_t nops, const B200Vp8ResidualOp *ops, const int16_t *coef,
                                    uint8_t *const dst[3], ptrdiff_t ls_y, ptrdiff_t ls_uv);

/* VP8 / VP7 loop filter: b200_vp8_dsp_init_loopfilter() fills the ten loop-filter members of a B200VP8DSPContext (vp8_v_loop_filter16y
 * .. vp8_h_loop_filter_simple) as ff_vp8dsp_init (is_vp7 = 0) / ff_vp7dsp_init (is_vp7 = 1) fill them (vp8dsp.c:702-713, :733-744):
 * ten distinct functions per codec, twenty in all; it touches no other member.  v filters the edge between two rows (samples across it
 * are dst[-4 stride .. 3 stride], the lines run along the row), h the edge between two columns (dst[-4..3], the lines run down).  HOST
 * pointers and the reference's signatures; 16y filters 16 lines, 8uv 8 lines of U and 8 of V in one call, simple 16 lines.
 * Per line (vp8dsp.c:263-457): the simple limit is 2 |p0 - q0| + (|p1 - q1| >> 1) <= E for VP8 and |p0 - q0| <= E for VP7; the normal
 * limit adds every neighbour difference of p3..q3 <= I; hev is |p1 - p0| > H or |q1 - q0| > H.
 *   common     a = clip_int8(3 (q0 - p0) + clip_int8(p1 - q1)) (the 4-tap form; without it the p1 - q1 term is left out), f1 = min(a + 4,
 *              127) >> 3, f2 = min(a + 3, 127) >> 3 for VP8 and f1 - ((a & 7) == 4) for VP7; p0 += f2, q0 -= f1, and without the 4-tap
 *              form p1 += (f1 + 1) >> 1, q1 -= (f1 + 1) >> 1, each clipped to 0..255
 *   mbedge     w = clip_int8(clip_int8(p1 - q1) + 3 (q0 - p0)); p2 / q2, p1 / q1, p0 / q0 moved by (9 w + 63) >> 7, (18 w + 63) >> 7,
 *              (27 w + 63) >> 7
 *   16y, 8uv          normal limit, then hev ? common 4-tap : mbedge; reads dst[-4..3] across, writes dst[-3..2]
 *   16y_inner, 8uv_inner   normal limit, then hev ? common 4-tap : common without it; reads dst[-4..3], writes dst[-2..1]
 *   simple     simple limit, then common 4-tap; reads dst[-2..1], writes dst[-1..0]
 * 0; B200_EINVAL for c == NULL or is_vp7 not 0 / 1; B200_ENODEV. */
int  b200_vp8_dsp_init_loopfilter(B200VP8DSPContext *c, int is_vp7);

/* One macroblock's loop-filter strength: VP8FilterStrength's layout (libavcodec/vp8.h:90-94), 3 bytes, byte alignment, as
 * filter_level_for_mb leaves it (vp8.c:2149-2179). */
typedef struct B200Vp8FilterStrength {
    uint8_t filter_level;   /* 0: the MB is not filtered; above 63: left untouched (the decoder clips the level to 6 bits) */
    uint8_t inner_limit;    /* I, and part of the VP8 edge limits */
    uint8_t inner_filter;   /* nonzero: the inner edges are filtered */
} B200Vp8FilterStrength;
#ifdef __cplusplus
static_assert(sizeof(B200Vp8FilterStrength) == 3, "B200Vp8FilterStrength is 3 bytes");
#else
_Static_assert(sizeof(B200Vp8FilterStrength) == 3, "B200Vp8FilterStrength is 3 bytes");
#endif
/* Loop-filters a whole VP8 / VP7 frame in place, DEVICE pointers (planes[0..2], f), asynchronous on the device's stream.  The result is
 * what filter_mb_row (vp8.c:2523-2574) gives run over every MB row in order: per macroblock (mb_x, mb_y) with record
 * f[mb_y * f_stride + mb_x] of level L, inner limit I and inner filter F,
 *   normal (simple = 0)  filter_mb (vp8.c:2181-2266): VP8 edge limits bedge = 2 L + I, mbedge = bedge + 4; VP7 bedge_y = L,
 *                        bedge_uv = 2 L, mbedge = L + 2; hev_thresh 1 from L = 15, one more from 40, and on inter frames (keyframe = 0)
 *                        one more from 20.  h_loop_filter16y / 8uv at the left MB edge when mb_x > 0; with F the inner column edges
 *                        (4, 8, 12 in luma, 4 in chroma); v_loop_filter16y / 8uv at the top MB edge when mb_y > 0; with F the inner
 *                        row edges.  VP7 filters its inner column edges after the row edges (vp8.c:2265), VP8 before them.
 *   simple (simple = 1)  filter_mb_simple (vp8.c:2268-2299) on luma only, the chroma planes untouched: the same edges with the simple
 *                        members, and the VP8 limits 2 L + I / + 4 for VP7 too (with the VP7 members).
 * An MB with L = 0 is skipped; an MB with L > 63 is left untouched too (the reference would index hev_thresh_lut out of bounds; the
 * decoder clips L to 6 bits).  A nonzero inner_filter counts as true.
 * Filtering the fully reconstructed frame once is exact: the decoder filters row r - 1 before it decodes row r, but row r's intra
 * prediction reads the unfiltered top border that backup_mb_border / xchg_mb_border saved (vp8.c:1701-1706, :2556-2561), and its left
 * neighbours unfiltered too, so this gives the single-threaded decoder's picture.  Call it after b200_vp8_residual_frame_device.
 * The work runs as a wavefront: MB (r, c) starts once (r, c - 1) and (r - 1, c + 1) are done (the decoder's own check_thread_pos rule),
 * the order the result depends on: a frame-wide order (all column edges, then all row edges) or a slope-1 wavefront give other pictures.
 * Only the 16 mb_width x 16 mb_height luma and 8 mb_width x 8 mb_height chroma samples are read or written.  f needs no alignment
 * beyond a byte.  Offsets are 64-bit.
 * Returns 0, or B200_EINVAL (launching nothing) for NULL pointers, is_vp7, simple or keyframe not 0 / 1, mb_width or mb_height < 1,
 * ls_y < 16 mb_width, ls_uv < 8 mb_width, or f_stride < mb_width. */
int  b200_vp8_loopfilter_frame_device(B200Device *dev, int is_vp7, int simple, int keyframe, int mb_width, int mb_height,
                                      uint8_t *const planes[3], ptrdiff_t ls_y, ptrdiff_t ls_uv, const B200Vp8FilterStrength *f,
                                      int64_t f_stride);
/* The frame entry's MB rows wait on the row above; every such wait is bounded by about one second, after which the MB is filtered
 * anyway (wrong samples rather than a hung GPU) and a per-device counter is incremented.  This waits for the device's stream and stores
 * the number of the VP8 loop filter's waits that ran out on that device since the process started in *count.  0; B200_EINVAL for
 * count == NULL; B200_ENODEV; B200_EEXTERNAL. */
int  b200_vp8_loopfilter_timeouts(B200Device *dev, int64_t *count);

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
/* the same for 9 / 10 / 12 / 14 bit samples (uint16): offsets and stride in BYTES (even); params must be 4-byte aligned (B200_EINVAL
 * otherwise) */
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
/* the same for 9 / 10 / 12 / 14 bit samples (uint16, native endian): op bytes as above (size index 3 writes nothing), offsets and stride
 * in BYTES (even) */
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
/* the same for 16-bit samples (any depth above 8): op bytes as above (width index 3 writes nothing), offsets and stride in BYTES (even) */
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
/* the same for 16-bit samples: geom in pixels; buf_off, origin and the line sizes in BYTES (even); geom must be 4-byte aligned
 * (B200_EINVAL otherwise) */
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

/* VC-1 / WMV3 motion compensation and inverse transforms: VC1DSPContext (libavcodec/vc1dsp.h:37-97) in the reference's member order and
 * types.  b200_vc1_dsp_init() fills what ff_vc1dsp_init fills (vc1dsp.c:968-1017) of these members, sharing functions as it does:
 *   vc1_inv_trans_{8x8,8x4,4x8,4x4} and their _dc forms            the eight transforms
 *   put_vc1_mspel_pixels_tab[size][dxy], avg_vc1_mspel_pixels_tab    size 0 = 16x16, 1 = 8x8; dxy = hmode + 4 vmode (mx & 3, my & 3);
 *                                                                    [size][0] is the plain copy (put_pixels16x16_c / 8x8_c), which
 *                                                                    ignores its last argument
 *   put_no_rnd_vc1_chroma_pixels_tab[0..1], avg_no_rnd_...[0..1]    8 and 4 wide; [2] NULL as in the reference
 * The overlap members, the six loop filters, the five sprite members, startcode_find_candidate and vc1_unescape_buffer stay NULL.  HOST
 * pointers, the reference's signatures; a member reads only what its reference function reads and writes only what it writes.
 *   mspel      4-tap rows {-4, 53, 18, -3}, {-1, 9, 9, -1}, {-3, 18, 53, -4} for modes 1..3 (vc1dsp.c:542-584); horizontal only
 *              (taps + 32 - rnd) >> 6 (+ 8 - rnd >> 4 at mode 2); vertical only the same with 1 - rnd for rnd; both: vertical pass over
 *              columns -1 .. w + 1 with shift (s[h] + s[v]) >> 1, s = {0, 5, 1, 5}, rounding (1 << (shift - 1)) + rnd - 1, into int16,
 *              then the horizontal pass (+ 64 - rnd) >> 7; clipped to 0..255; avg (dst + x + 1) >> 1
 *   chroma     (A s00 + B s01 + C s10 + D s11 + 28) >> 6 with A = (8 - x)(8 - y), B = x (8 - y), C = (8 - x) y, D = x y over h rows; avg
 *              (dst + x + 1) >> 1; x, y 0..7, h 0..4096 (outside: the member writes nothing and records why in b200_last_error())
 *   8x8        in place on block: column pass (+ 4) >> 3 into int16, row pass (+ 64) >> 7, + 1 on outputs 4..7, into int16 block
 *   8x4, 4x8, 4x4   row pass (+ 4) >> 3 written back into block (int16), column pass (+ 64) >> 7 added to dest and clipped
 *   _dc        dest += the DC of block[0] (vc1dsp.c:241-260, :332-351, :409-424, :482-497); block untouched
 * 0; B200_EINVAL for c == NULL; B200_ENODEV. */
typedef void (*b200_vc1op_pixels_func)(uint8_t *block, const uint8_t *pixels, ptrdiff_t line_size, int round);
typedef struct B200VC1DSPContext {
    void (*vc1_inv_trans_8x8)(int16_t *b);
    void (*vc1_inv_trans_8x4)(uint8_t *dest, ptrdiff_t stride, int16_t *block);
    void (*vc1_inv_trans_4x8)(uint8_t *dest, ptrdiff_t stride, int16_t *block);
    void (*vc1_inv_trans_4x4)(uint8_t *dest, ptrdiff_t stride, int16_t *block);
    void (*vc1_inv_trans_8x8_dc)(uint8_t *dest, ptrdiff_t stride, int16_t *block);
    void (*vc1_inv_trans_8x4_dc)(uint8_t *dest, ptrdiff_t stride, int16_t *block);
    void (*vc1_inv_trans_4x8_dc)(uint8_t *dest, ptrdiff_t stride, int16_t *block);
    void (*vc1_inv_trans_4x4_dc)(uint8_t *dest, ptrdiff_t stride, int16_t *block);
    void (*vc1_v_overlap)(uint8_t *src, ptrdiff_t stride);
    void (*vc1_h_overlap)(uint8_t *src, ptrdiff_t stride);
    void (*vc1_v_s_overlap)(int16_t *top, int16_t *bottom);
    void (*vc1_h_s_overlap)(int16_t *left, int16_t *right, ptrdiff_t left_stride, ptrdiff_t right_stride, int flags);
    void (*vc1_v_loop_filter4)(uint8_t *src, ptrdiff_t stride, int pq);
    void (*vc1_h_loop_filter4)(uint8_t *src, ptrdiff_t stride, int pq);
    void (*vc1_v_loop_filter8)(uint8_t *src, ptrdiff_t stride, int pq);
    void (*vc1_h_loop_filter8)(uint8_t *src, ptrdiff_t stride, int pq);
    void (*vc1_v_loop_filter16)(uint8_t *src, ptrdiff_t stride, int pq);
    void (*vc1_h_loop_filter16)(uint8_t *src, ptrdiff_t stride, int pq);
    b200_vc1op_pixels_func put_vc1_mspel_pixels_tab[2][16];
    b200_vc1op_pixels_func avg_vc1_mspel_pixels_tab[2][16];
    b200_h264_chroma_mc_func put_no_rnd_vc1_chroma_pixels_tab[3];
    b200_h264_chroma_mc_func avg_no_rnd_vc1_chroma_pixels_tab[3];
    void (*sprite_h)(uint8_t *dst, const uint8_t *src, int offset, int advance, int count);
    void (*sprite_v_single)(uint8_t *dst, const uint8_t *src1a, const uint8_t *src1b, int offset, int width);
    void (*sprite_v_double_noscale)(uint8_t *dst, const uint8_t *src1a, const uint8_t *src2a, int alpha, int width);
    void (*sprite_v_double_onescale)(uint8_t *dst, const uint8_t *src1a, const uint8_t *src1b, int offset1, const uint8_t *src2a, int alpha,
                                     int width);
    void (*sprite_v_double_twoscale)(uint8_t *dst, const uint8_t *src1a, const uint8_t *src1b, int offset1, const uint8_t *src2a,
                                     const uint8_t *src2b, int offset2, int alpha, int width);
    int (*startcode_find_candidate)(const uint8_t *buf, int size);
    int (*vc1_unescape_buffer)(const uint8_t *src, int size, uint8_t *dst);
} B200VC1DSPContext;
int  b200_vc1_dsp_init(B200VC1DSPContext *c);

/* One reference picture of b200_vc1_mc_frame_device: DEVICE addresses of sample (0, 0) of its three planes, line sizes in bytes, and
 * the state the decoder keeps per reference (v->last_* / v->next_*): rangeredfrm, use_ic with luty / lutuv indexed by source-row
 * parity, and whether the reference is interlaced (refused: interlaced MC is not implemented). */
typedef struct B200Vc1McRef {
    const uint8_t *y, *u, *v;
    ptrdiff_t ls_y, ls_uv;
    int32_t rangeredfrm, use_ic, interlaced, reserved;
    uint8_t luty[2][256], lutuv[2][256];
} B200Vc1McRef;
/* One prediction source of an op: reference index, the luma position src_x / src_y after the decoder's clip (vc1_mc.c:258-273) with
 * mx & 3 / my & 3, and the chroma position uvsrc_x / uvsrc_y with uvmx & 3 / uvmy & 3 (after fastuvmc).  An op reads the fields of
 * the planes it writes. */
typedef struct B200Vc1McSrc {
    int16_t x, y;           /* luma: src_x, src_y */
    int16_t uvx, uvy;       /* chroma: uvsrc_x, uvsrc_y */
    uint8_t ref;            /* index into the call's refs */
    uint8_t mx, my;         /* mx & 3, my & 3 */
    uint8_t uvmx, uvmy;     /* uvmx & 3, uvmy & 3 */
    uint8_t reserved[3];
} B200Vc1McSrc;
/* One op of b200_vc1_mc_frame_device.  kind 1MV is one call of ff_vc1_mc_1mv (vc1_mc.c:172-449): Y 16x16 at (dst_x, dst_y) and U, V
 * 8x8 at (dst_x / 2, dst_y / 2), the chroma window copied exactly when the luma edge test fires; with B200_VC1_MC_AVG src[1] is then
 * averaged in as ff_vc1_interp_mc does (vc1_mc.c:1004-1230, B-frame interpolation, its own edge test).  LUMA8 is ff_vc1_mc_4mv_luma
 * (:452-631, avg 0): Y 8x8 at (dst_x, dst_y).  CHROMA8 is the MC half of ff_vc1_mc_4mv_chroma (:634-836): U and V 8x8 at (dst_x, dst_y)
 * in chroma samples, from the uv fields.  The chroma vector averaging of 4MV stays with the caller. */
enum { B200_VC1_MC_1MV = 0, B200_VC1_MC_LUMA8 = 1, B200_VC1_MC_CHROMA8 = 2 };
enum { B200_VC1_MC_MSPEL = 1, B200_VC1_MC_RND = 2, B200_VC1_MC_AVG = 4 };   /* flags: s->mspel, v->rnd, src[1] averaged in (1MV only) */
typedef struct B200Vc1McOp {
    int16_t dst_x, dst_y;   /* top-left sample of the block in the plane it writes; multiples of 8 */
    uint8_t kind;           /* B200_VC1_MC_* kind */
    uint8_t flags;          /* B200_VC1_MC_MSPEL | B200_VC1_MC_RND | B200_VC1_MC_AVG */
    uint8_t reserved[2];
    B200Vc1McSrc src[2];
} B200Vc1McOp;
#ifdef __cplusplus
static_assert(sizeof(B200Vc1McSrc) == 16 && sizeof(B200Vc1McOp) == 40, "B200Vc1McOp is 40 bytes");
static_assert(sizeof(B200Vc1McRef) == 1080, "B200Vc1McRef is 1080 bytes");
#else
_Static_assert(sizeof(B200Vc1McSrc) == 16 && sizeof(B200Vc1McOp) == 40, "B200Vc1McOp is 40 bytes");
_Static_assert(sizeof(B200Vc1McRef) == 1080, "B200Vc1McRef is 1080 bytes");
#endif
/* Inter prediction of a whole progressive VC-1 picture in one call: `refs` is a HOST array of 1 <= nrefs <= 2 references (copied into
 * the launch), `ops` and the dst planes are DEVICE pointers; asynchronous on the device's stream.  Each op's result is the reference
 * sequence for progressive pictures (field_mode 0, interlace 0):
 *   1. the decoder's edge test, on the luma fields for 1MV (ff_vc1_mc_1mv: x against mspel, y against 1; src[1] as ff_vc1_interp_mc:
 *      both against 1) and LUMA8, on the uv fields for CHROMA8; rangeredfrm or use_ic of the op's reference always fire it;
 *   2. where it fires, the emulated_edge_mc window: 17 + 2 mspel (1MV) / 9 + 2 mspel (LUMA8) samples square from (x - mspel,
 *      y - mspel), 9 x 9 from (uvx, uvy), coordinates clamped to h_edge_pos x v_edge_pos (chroma: halves); where it does not, the
 *      plane is read directly (so planes must be readable wherever the decoder reads them);
 *   3. in the window, range reduction ((s - 128) >> 1) + 128 when rangeredfrm, then with use_ic luty / lutuv of the window row's
 *      source-row parity;
 *   4. the member: with MSPEL put_vc1_mspel_pixels_tab[size][dxy] (avg_ for src[1]); else hpeldsp put_pixels_tab / put_no_rnd_ (avg_ /
 *      avg_no_rnd_ for src[1]) as rnd is 0 / 1 at dxy = (my & 2) | (mx & 2) >> 1; chroma put_h264_chroma_pixels_tab[0] (avg_ for
 *      src[1]) with rnd 0 and put_no_rnd_vc1_chroma_pixels_tab[0] (avg_no_rnd_) with rnd 1, at ((uvmx & 3) << 1, (uvmy & 3) << 1).
 * The caller guarantees that the ops of one call write disjoint blocks and that no op reads what another op of the call writes.
 * An op writes nothing if its kind is undefined, a phase is above 3, a reference index is >= nrefs, AVG is set on a kind other than
 * 1MV, dst_x or dst_y is not a multiple of 8, or its blocks are not inside 16 mb_width x 16 mb_height luma / 8 mb_width x 8 mb_height
 * chroma.  More ops than one launch takes are split inside the entry.
 * Returns 0, or B200_EINVAL (launching nothing) for NULL pointers, nops < 0, nrefs outside 1..2, mb_width or mb_height outside 1..2047,
 * h_edge_pos or v_edge_pos outside 1..32767, ops not aligned to 4 bytes, or a dst plane or line size that is not a multiple of 4;
 * B200_ENOSYS (launching nothing) for an interlaced reference; nops == 0 returns 0. */
int  b200_vc1_mc_frame_device(B200Device *dev, int nrefs, const B200Vc1McRef *refs, uint8_t *const dst[3], ptrdiff_t ls_y, ptrdiff_t ls_uv,
                              int mb_width, int mb_height, int h_edge_pos, int v_edge_pos, int64_t nops, const B200Vc1McOp *ops);

/* One inter 8x8 block of b200_vc1_residual_frame_device: the transform calls vc1_decode_p_block makes (vc1_block.c:1124-1240). */
enum { B200_VC1_TT_8X8 = 0, B200_VC1_TT_8X4 = 1, B200_VC1_TT_4X8 = 2, B200_VC1_TT_4X4 = 3 };
typedef struct B200Vc1ResidualOp {
    int64_t coef_off;       /* element offset in coef of the block's 64 int16, dequantised, raster order as in block[]; a multiple of 8 */
    int16_t x, y;           /* top-left sample of the block in its plane; multiples of 8 */
    uint8_t plane;          /* 0 Y, 1 U, 2 V */
    uint8_t ttblk;          /* B200_VC1_TT_*: the generic type after the decoder's TT_8X4_TOP / ... conversion */
    uint8_t subblkpat;      /* 8x4 / 4x8: bit 1 - j skips sub-block j; 4x4: bit 3 - j skips sub-block j (j in raster order) */
    uint8_t dc;             /* bit j: sub-block j takes the _dc form (the decoder's i == 1) */
} B200Vc1ResidualOp;
#ifdef __cplusplus
static_assert(sizeof(B200Vc1ResidualOp) == 16, "B200Vc1ResidualOp is 16 bytes");
#else
_Static_assert(sizeof(B200Vc1ResidualOp) == 16, "B200Vc1ResidualOp is 16 bytes");
#endif
/* The inter residual of a whole picture in one call, DEVICE pointers (ops, coef, dst[0..2]), asynchronous on the device's stream.  Per
 * op, for every sub-block j that subblkpat does not mask: with dc bit j vc1_inv_trans_<tt>_dc, else vc1_inv_trans_<tt> (8x8:
 * vc1_inv_trans_8x8 followed by add_pixels_clamped), at the sub-block's place; int16 truncation exactly where the reference stores, so
 * every int16 coefficient value is accepted.  `coef` is read only.  The ops of one call write disjoint blocks.  An op writes nothing if
 * its plane or ttblk is undefined, coef_off is negative or not a multiple of 8, x or y is not a multiple of 8, or its block is not
 * inside 16 mb_width x 16 mb_height luma / 8 mb_width x 8 mb_height chroma.  Intra blocks are not covered.
 * Returns 0, or B200_EINVAL (launching nothing) for NULL pointers, nops < 0, mb_width or mb_height outside 1..2047, ops not aligned
 * to 8 bytes, coef not aligned to 16 bytes, or a dst plane or line size that is not a multiple of 4; nops == 0 returns 0. */
int  b200_vc1_residual_frame_device(B200Device *dev, uint8_t *const dst[3], ptrdiff_t ls_y, ptrdiff_t ls_uv, int mb_width, int mb_height,
                                    const int16_t *coef, int64_t nops, const B200Vc1ResidualOp *ops);

#ifdef __cplusplus
}
#endif
#endif /* B200DSP_H */
