"""Shared case lists and synthetic-input generators for the parity tests and scripts/gen_golden.py."""
import numpy as np

SWS_BILINEAR, SWS_BICUBIC, SWS_POINT, SWS_AREA, SWS_BICUBLIN = 2, 4, 0x10, 0x20, 0x40
SWS_FULL_CHR_H_INT, SWS_ACCURATE_RND, SWS_BITEXACT = 0x2000, 0x40000, 0x80000
FATE = SWS_BICUBIC | SWS_ACCURATE_RND | SWS_BITEXACT      # tests/fate-run.sh:262-265 sws_flags

# (srcW, srcH, dstW, dstH, flags, input kind) — small: inputs and reference outputs are stored in tests/golden
SWS_SMALL_CASES = [
    (64, 48, 64, 48, FATE, "random"),            # same size, FATE flags: _X writer, 4-tap vertical chroma
    (64, 48, 64, 48, SWS_BICUBIC, "random"),     # same size, plain bicubic: unscaled LUT converter
    (64, 48, 128, 96, FATE, "smooth"),           # 2x up
    (64, 48, 32, 24, FATE, "random"),            # 2x down
    (64, 48, 37, 21, FATE, "random"),            # odd output width: full-chroma writer
    (34, 18, 34, 18, SWS_BICUBIC, "random"),     # width % 16 != 0 on the LUT path (tails 2 wide)
    (38, 20, 38, 20, FATE, "limited"),
    (64, 48, 100, 60, SWS_BILINEAR, "random"),   # _2 writer
    (64, 48, 64, 48, SWS_BILINEAR | SWS_ACCURATE_RND, "random"),  # _1 writer with uvalpha
    (64, 48, 80, 33, SWS_POINT, "random"),
    (64, 48, 40, 30, SWS_AREA, "random"),
    (64, 48, 96, 72, SWS_AREA, "random"),
    (64, 48, 90, 50, SWS_BICUBLIN, "smooth"),
    (64, 48, 64, 48, FATE | SWS_FULL_CHR_H_INT, "random"),
    (16, 16, 16, 16, FATE, "random"),
    (8, 8, 8, 8, SWS_BICUBIC, "random"),
    (2, 2, 2, 2, FATE, "random"),
    (4, 4, 8, 8, FATE, "random"),
    (64, 48, 64, 47, SWS_BICUBIC, "random"),     # odd height: no LUT converter even without accurate_rnd
    (33, 17, 64, 40, FATE, "random"),            # odd source size
]

# larger: only sha256 of the reference output is stored (inputs regenerated from the seed, input hash checked too)
SWS_HASH_CASES = [
    (352, 288, 352, 288, FATE, "random"),        # the FATE filter-pixfmts geometry (vsynth1 is 352x288)
    (352, 288, 352, 288, SWS_BICUBIC, "random"),
    (352, 288, 200, 100, FATE, "smooth"),        # filter-pixfmts-scale geometry
    (640, 360, 640, 360, FATE, "random"),        # BASELINE.json configs[0]
    (640, 360, 640, 360, SWS_BICUBIC, "limited"),
    (640, 360, 1280, 720, FATE, "random"),
    (1920, 1080, 1280, 720, FATE, "random"),
    (352, 288, 351, 288, FATE, "random"),
    (720, 576, 1000, 563, SWS_BILINEAR | SWS_BITEXACT, "smooth"),
]


def idct_blocks(kind, n, seed=0):
    """Coefficient blocks like the reference's tests generate them."""
    rng = np.random.default_rng(seed)
    if kind == "dense":      # tests/checkasm/idctdsp.c:40-48: rnd() % 0x201 - 0x100
        return rng.integers(-256, 257, (n, 64)).astype(np.int16)
    if kind == "wide":
        return rng.integers(-2048, 2048, (n, 64)).astype(np.int16)
    if kind == "extreme":
        return rng.integers(-32768, 32768, (n, 64)).astype(np.int16)
    b = np.zeros((n, 64), np.int16)
    if kind == "sparse":     # libavcodec/tests/dct.c:144-150: 1..10 non-zero coefficients
        for i in range(n):
            k = int(rng.integers(1, 11))
            b[i, rng.integers(0, 64, k)] = rng.integers(-1024, 1024, k)
    elif kind == "dc63":     # libavcodec/tests/dct.c:151-154
        b[:, 0] = rng.integers(-1024, 1024, n)
        b[:, 63] = rng.integers(-3, 4, n)
    elif kind == "dconly":
        b[:, 0] = rng.integers(-2048, 2048, n)
    else:
        raise ValueError(kind)
    return b


# (dstW, dstH, flags, [(srcSliceY, srcSliceH), ...]) on a 64x48 source: sws_scale() called band by band
SWS_SLICE_CASES = [
    (64, 48, FATE, [(0, 16), (16, 16), (32, 16)]),
    (64, 48, FATE, [(0, 2), (2, 46)]),
    (64, 48, SWS_BICUBIC, [(0, 16), (16, 32)]),                    # unscaled LUT converter
    (100, 60, SWS_BILINEAR, [(0, 8), (8, 8), (16, 8), (24, 24)]),
    (32, 24, FATE, [(0, 24), (24, 24)]),
    (37, 21, FATE, [(0, 10), (10, 20), (30, 18)]),                  # odd width: full-chroma writer
    (64, 96, FATE, [(0, 4), (4, 4), (8, 40)]),
]


# emulated_edge_mc fixture: picture 37 x 29 (linesize 48); (block_w, block_h, src_x, src_y) — inside, each edge, each corner,
# fully outside on every side (the reference's src_y >= h / <= -block_h / src_x >= w / <= -block_w clamps), 1-wide windows
EDGE_PIC = (37, 29, 48)
EDGE_CASES = [(9, 9, 5, 5), (21, 21, -3, 4), (21, 21, 30, 4), (21, 21, 8, -2), (21, 21, 8, 20), (21, 21, -5, -5), (21, 21, 25, 15),
              (9, 9, -3, 25), (9, 9, 33, -4), (17, 9, -17, 3), (17, 9, -40, 3), (17, 9, 37, 3), (17, 9, 90, 3), (9, 17, 3, -17),
              (9, 17, 3, -50), (9, 17, 3, 29), (9, 17, 3, 77), (23, 23, -60, -60), (23, 23, 60, 60), (1, 1, -1, -1), (1, 5, 36, 27),
              (5, 1, 36, 28), (23, 23, -10, -10), (4, 4, 0, 0), (4, 4, 33, 25), (2, 13, 36, -6)]


# other packed RGB writers of the same pipeline (SURVEY 8f row 2): (w, h, dw, dh, flags, input kind) run for every format of
# cpulibs.PACKED_RGB_FORMATS except rgb24 — the _X writer same-size (FATE flags), the unscaled LUT converter, a rescale
# through the int16 line planes, full chroma (odd width forces it), widths that leave scalar tails, and a vector-width case
SWS_FORMAT_CASES = [(64, 48, 64, 48, FATE, "random"), (64, 48, 64, 48, SWS_BICUBIC, "random"), (64, 48, 100, 70, FATE, "limited"),
                    (64, 48, 33, 21, SWS_BILINEAR, "random"), (38, 22, 38, 22, SWS_BICUBIC, "random"), (70, 30, 70, 30, FATE, "smooth"),
                    (64, 48, 64, 48, FATE | SWS_FULL_CHR_H_INT, "random"), (352, 288, 352, 288, FATE, "random"),
                    (352, 288, 352, 288, SWS_BICUBIC, "limited"), (352, 288, 200, 100, FATE, "random")]


# yuv420p -> yuv420p (SURVEY 8f row 2: yuv2planeX / yuv2plane1 writers, planarCopyWrapper): (w, h, dw, dh, flags, kind)
SWS_PLANAR_CASES = [(64, 48, 64, 48, FATE, "random"), (64, 48, 100, 70, FATE, "random"), (64, 48, 33, 21, SWS_BILINEAR, "limited"),
                    (66, 50, 40, 96, SWS_BICUBIC, "random"), (64, 48, 128, 96, SWS_BILINEAR, "smooth"), (64, 48, 64, 30, FATE, "random"),
                    (64, 48, 32, 48, SWS_BICUBIC, "random"), (352, 288, 200, 100, FATE, "random"), (100, 50, 37, 21, FATE, "limited"),
                    (64, 48, 64, 47, SWS_POINT, "random"), (64, 48, 31, 17, SWS_AREA, "random"), (352, 288, 640, 360, SWS_BICUBLIN, "random"),
                    (63, 47, 80, 60, SWS_BICUBIC, "random"), (352, 288, 176, 144, FATE, "smooth")]


# SWS_FAST_BILINEAR (ff_hyscale_fast_c / ff_hcscale_fast_c horizontal pass): (w, h, dw, dh, flags, kind); run for rgb24 and yuv420p
SWS_FAST_BILINEAR = 1
SWS_FASTBIL_CASES = [(64, 48, 64, 48, 1 | SWS_ACCURATE_RND, "random"), (64, 48, 64, 48, 1, "random"), (64, 48, 100, 70, 1, "limited"),
                     (64, 48, 33, 21, 1, "random"), (352, 288, 640, 360, 1, "random"), (352, 288, 200, 100, 1 | SWS_ACCURATE_RND | SWS_BITEXACT, "random"),
                     (66, 50, 40, 96, 1, "smooth"), (7, 48, 64, 30, 1, "random"), (64, 48, 8, 48, 1, "random"), (100, 50, 37, 21, 1, "random"),
                     (640, 360, 1280, 720, 1, "random")]


# nv12 / nv21 sources (plane 1 = interleaved chroma; the reference de-interleaves with nvXXtoUV_c and, having no LUT converter
# for them, always runs the scaler): (w, h, dw, dh, flags, kind), each for nv12 and nv21, to rgb24, bgra and yuv420p
SWS_NV_CASES = [(64, 48, 64, 48, FATE, "random"), (64, 48, 64, 48, SWS_BICUBIC, "random"), (64, 48, 100, 70, FATE, "limited"),
                (64, 48, 33, 21, SWS_BILINEAR, "random"), (352, 288, 200, 100, FATE, "random"), (66, 50, 66, 50, SWS_BICUBIC, "random"),
                (63, 47, 63, 47, SWS_BICUBIC, "smooth"), (64, 48, 128, 96, 1, "random"), (352, 288, 352, 288, FATE, "random")]


# yuv -> yuv range conversion (SURVEY 8f row 2: lum/chrRangeToJpeg_c, FromJpeg_c between the two passes, swscale.c:163-209):
# (w, h, dw, dh, flags, kind, (src_range, dst_range) at init, sws_setColorspaceDetails() call after init or None)
# details = (src_cs, src_range, dst_cs, dst_range, brightness, contrast, saturation), cs = SWS_CS_* index
_ID = (5, 0, 5, 0, 0, 1 << 16, 1 << 16)
SWS_RANGE_CASES = [
    (352, 288, 352, 288, FATE, "random", (0, 1), None),              # the geometry of FATE's sws-yuv-range: same size, through the scaler
    (352, 288, 352, 288, FATE, "limited", (1, 0), None),
    (64, 48, 100, 70, FATE, "random", (0, 1), None),
    (64, 48, 100, 70, FATE, "random", (1, 0), None),
    (66, 50, 40, 96, SWS_BILINEAR, "limited", (0, 1), None),
    (352, 288, 200, 100, SWS_BICUBIC, "smooth", (1, 0), None),
    (64, 48, 33, 21, SWS_FAST_BILINEAR, "random", (0, 1), None),
    (64, 48, 128, 96, SWS_FAST_BILINEAR, "random", (1, 0), None),
    (64, 48, 64, 48, SWS_BICUBIC, "random", (1, 1), None),           # equal ranges: plain copy
    (64, 48, 100, 70, FATE, "random", (0, 0), (5, 0, 5, 1, 0, 1 << 16, 1 << 16)),       # ranges changed after init: conversion switched on
    (64, 48, 100, 70, FATE, "random", (0, 1), (5, 1, 5, 1, 0, 1 << 16, 1 << 16)),       # ... and off
    (64, 48, 100, 70, FATE, "random", (0, 1), (5, 1, 5, 0, 2000, 70000, 80000)),        # direction flipped; brightness etc. do not apply
    (64, 48, 64, 48, FATE, "random", (0, 0), (5, 0, 5, 1, 0, 1 << 16, 1 << 16)),        # initialised as a copy: stays a copy
    (64, 48, 64, 48, FATE, "random", (0, 1), _ID),                                       # initialised through the scaler: stays there
]


# packed RGB sources (SURVEY 8f row 2: the input readers rgb24ToY_c / ...ToUV_c / ...ToUV_half_c and the 32-bit templates,
# input.c:264-393,1068-1172; hScale16To15_c; bgr24ToYv12Wrapper): (w, h, dw, dh, flags, kind); every case runs for the six source
# byte orders -> yuv420p, and (when the size changes) -> rgb24 for the 3-byte sources
SWS_FULL_CHR_H_INP = 0x4000
SWS_RGBSRC_CASES = [(64, 48, 64, 48, FATE, "random"), (64, 48, 64, 48, SWS_BICUBIC, "random"), (64, 48, 100, 70, FATE, "smooth"),
                    (64, 48, 33, 21, SWS_BILINEAR, "random"), (352, 288, 200, 100, FATE, "random"), (63, 47, 63, 47, SWS_BICUBIC, "random"),
                    (63, 47, 80, 60, FATE, "random"), (64, 48, 128, 96, SWS_BICUBIC | SWS_FULL_CHR_H_INP, "random"),
                    (64, 48, 40, 30, SWS_POINT, "random"), (64, 48, 100, 70, SWS_FAST_BILINEAR, "random"),
                    (64, 48, 40, 30, SWS_FAST_BILINEAR, "smooth"), (352, 288, 640, 360, SWS_BICUBLIN, "random"),
                    (66, 50, 66, 50, FATE | SWS_FULL_CHR_H_INP, "random"), (64, 48, 64, 30, FATE, "random"), (64, 48, 32, 48, SWS_AREA, "random")]


# the scalers initFilter evaluates in double precision (libswscale/utils.c:325-368): experimental, Gaussian, sinc, Lanczos, spline
SWS_X, SWS_GAUSS, SWS_SINC, SWS_LANCZOS, SWS_SPLINE = 0x8, 0x80, 0x100, 0x200, 0x400
SWS_FLOAT_KERNEL_CASES = [(w, h, dw, dh, fl | extra, "random")
                          for fl in (SWS_X, SWS_GAUSS, SWS_SINC, SWS_LANCZOS, SWS_SPLINE)
                          for (w, h, dw, dh, extra) in ((64, 48, 100, 30, 0), (100, 50, 32, 64, 0xc0000), (352, 288, 200, 100, 0xc0000),
                                                        (34, 16, 200, 151, 0x2000), (130, 98, 17, 8, 0))]

# sws_getContext's `param` (SwsContext.scaler_params; 123456 = SWS_PARAM_DEFAULT): (scaler flag, (param0, param1))
SWS_PARAM_CASES = [(4, (0.0, 0.5)), (4, (1 / 3, 1 / 3)), (4, (1.0, 0.0)), (4, (123456.0, 0.75)), (0x40, (0.0, 0.75)), (0x80, (2.0, 123456.0)),
                   (0x80, (4.5, 123456.0)), (0x200, (2.0, 123456.0)), (0x200, (5.0, 123456.0)), (0x8, (0.5, 123456.0)), (0x8, (2.0, 123456.0)), (2, (0.3, 0.3))]


# yuv -> yuv with two different matrices: (w, h, dw, dh, flags, src format, dst format, ranges before init, details).  The reference cascades
# through a bgr24 picture of the smaller size (utils.c:914-989).  Cases whose first context would be the unscaled LUT converter on an odd
# width are left out: it never writes the last column and the reference then reads uninitialised memory there.
SWS_CASCADE_CASES = [
    (64, 48, 100, 70, 4 | 0x80000 | 0x40000, 0, 0, (0, 0), (1, 0, 5, 0, 0, 1 << 16, 1 << 16)),
    (100, 70, 64, 48, 4, 0, 0, (0, 0), (5, 0, 1, 0, 0, 1 << 16, 1 << 16)),
    (64, 48, 64, 48, 4, 0, 0, (0, 0), (1, 1, 9, 0, 1 << 12, 70000, 80000)),
    (66, 34, 66, 34, 2, 23, 0, (1, 0), (9, 1, 7, 1, 0, 1 << 16, 80000)),
    (87, 66, 87, 66, 4 | 0x40000, 0, 0, (0, 0), (1, 0, 5, 0, -(1 << 13), 1 << 16, 80000)),
    (77, 28, 90, 63, 1 | 0x40000, 0, 23, (1, 1), (1, 1, 9, 1, 0, 70000, 80000)),
    (50, 40, 25, 20, 0x10, 24, 24, (0, 1), (7, 0, 1, 1, 0, 1 << 16, 1 << 16)),
    (33, 21, 64, 40, 0x20 | 0x40000, 0, 23, (0, 0), (5, 0, 9, 0, 0, 50000, 1 << 16)),
    (128, 64, 96, 80, 4 | 0x2000, 23, 0, (0, 0), (9, 0, 5, 1, 1 << 12, 1 << 16, 40000)),
]


# sws_getContext with srcFilter / dstFilter: (w, h, dw, dh, flags, destination 'rgb24' / 'bgra' / 'yuv420p', source vectors (lumH, lumV, chrH,
# chrV; None = no vector), destination vector lengths)
def _gauss(sigma, n):
    import math
    v = [math.exp(-((i - (n - 1) / 2) ** 2) / (2 * sigma * sigma)) for i in range(n)]
    t = sum(v)
    return [x / t for x in v]


SWS_FILTER_CASES = [
    (64, 48, 100, 70, 4 | 0x80000 | 0x40000, "rgb24", (_gauss(0.8, 5), _gauss(0.8, 5), None, None), (0, 0, 0, 0)),
    (100, 70, 64, 48, 4, "rgb24", (None, None, _gauss(1.5, 9), _gauss(1.5, 9)), (0, 0, 0, 0)),
    (64, 48, 64, 48, 4, "bgra", ([-0.25, 1.5, -0.25], [-0.25, 1.5, -0.25], None, None), (0, 0, 0, 0)),        # same size: the LUT converter is ruled out
    (66, 34, 66, 34, 2, "yuv420p", ([0.25, 0.5, 0.25], None, [0.25, 0.5, 0.25], None), (0, 0, 0, 0)),            # same size: no plane copy
    (87, 66, 120, 90, 4 | 0x40000, "yuv420p", (_gauss(1.0, 7), _gauss(1.0, 7), _gauss(1.0, 7), _gauss(1.0, 7)), (3, 3, 3, 3)),
    (77, 28, 90, 63, 1, "rgb24", ([0.3, 0.7], [0.3, 0.7], None, None), (0, 5, 0, 0)),                            # fast bilinear ignores the horizontal bank
    (50, 40, 25, 20, 0x10, "bgra", (None, None, None, None), (3, 0, 3, 0)),                                      # destination vectors only: wider rows, same taps
    (128, 64, 96, 80, 0x20, "yuv420p", ([1.0], [1.0], [1.0], [1.0]), (1, 1, 1, 1)),                              # one-tap vectors: nothing changes
]


# The scaled path's three kernels (csrc/sws.cu launch_batch / launch_planar3), as b200_sws_last_path reports them: 4 the fused tensor-core
# kernels (csrc/sws_mma.cuh), 2 the fused CUDA-core kernels, 1 two passes through int16 line planes; a yuv420p destination ORs the bits of
# its three planes.  Each row: geometry, flags, optional `param` / `src_filter` (lumH, lumV, chrH, chrV) / nv12 or nv21 `src_fmt`, the
# kernels expected for each destination in the three memory layouts of tests/test_sws_scaled_paths_gpu.py (A: everything 16-byte aligned;
# B: source planes at base + 1 with odd strides; C: destination at base + 1 with an odd stride), and what the row is there to reach
# (tests/test_sws_mma_plan.py REACHES says what each name means and checks it on the host).
_SHARPEN = [-0.5, 2.0, -0.5]
_P = (4, 2, 1)                  # tensor-core kernel where aligned, CUDA-core fused kernel from misaligned sources, two passes into a misaligned destination
_TWO = (1, 1, 1)
_STD = {"rgb24": _P, "bgra": _P, "yuv420p": _P}
SWS_PATH_CASES = [
    dict(geom=(3840, 2160, 1920, 1080), flags=FATE, paths=_STD, reaches=("nch=1", "dstH%TR")),
    dict(geom=(1920, 1080, 3840, 2160), flags=FATE, paths=_STD, reaches=("up2x",)),
    dict(geom=(3840, 2160, 1280, 720), flags=FATE, paths=_STD, reaches=("nch=1",)),
    dict(geom=(3840, 2160, 960, 540), flags=FATE, paths=_STD, reaches=("nch=2", "smem>75K", "ngc<8")),
    dict(geom=(1920, 1080, 240, 540), flags=FATE, paths={"rgb24": (4, 1, 1), "bgra": (4, 1, 1), "yuv420p": (4, 1, 1)},
         reaches=("nch>=3", "taps>16", "smem>75K", "dstH%TR")),
    dict(geom=(1920, 1080, 960, 540), flags=SWS_LANCZOS | SWS_ACCURATE_RND | SWS_BITEXACT, param=(5.0, 123456.0),
         paths={"rgb24": (4, 1, 1), "bgra": (4, 1, 1), "yuv420p": (4, 1, 1)}, reaches=("taps>16", "nch=2")),
    dict(geom=(1024, 608, 96, 64), flags=FATE, paths={"rgb24": _TWO, "bgra": _TWO, "yuv420p": _TWO}, reaches=("no tile fits",)),
    dict(geom=(1280, 720, 640, 360), flags=SWS_POINT, paths={"rgb24": _TWO, "bgra": _TWO, "yuv420p": _P}, reaches=("vfs=1",)),
    dict(geom=(1920, 1080, 1280, 1080), flags=FATE, paths=_STD, reaches=("vfs=1", "hscaled")),
    dict(geom=(1920, 1080, 640, 352), flags=SWS_AREA, paths=_STD, reaches=("rgb row tile of 1",)),
    dict(geom=(640, 360, 1280, 720), flags=SWS_AREA, paths={"rgb24": _TWO, "bgra": _TWO, "yuv420p": _P}, reaches=("2-tap",)),
    dict(geom=(1280, 720, 1920, 1080), flags=SWS_BILINEAR | SWS_ACCURATE_RND | SWS_BITEXACT, paths={"rgb24": _TWO, "bgra": _TWO, "yuv420p": _P},
         reaches=("2-tap",)),
    dict(geom=(1920, 1080, 1280, 720), flags=SWS_BICUBLIN, paths=_STD, reaches=("bicublin",)),
    dict(geom=(1366, 768, 1920, 1080), flags=FATE, paths=_STD, reaches=("srcW%16",)),
    dict(geom=(1365, 765, 640, 352), flags=FATE, paths=_STD, reaches=("srcW%16", "odd chroma")),
    dict(geom=(8, 6, 32, 24), flags=FATE, paths=_STD, reaches=("srcW<16", "2-tap")),
    dict(geom=(12, 2, 48, 8), flags=FATE, paths={"rgb24": _TWO, "bgra": _TWO, "yuv420p": _P}, reaches=("srcW<16", "vfs=1")),
    dict(geom=(200, 120, 16, 16), flags=FATE, paths={"rgb24": (4, 1, 1), "bgra": (4, 1, 1), "yuv420p": (4, 1, 1)}, reaches=("one tile of 2 groups",)),
    dict(geom=(400, 300, 144, 100), flags=FATE, paths=_STD, reaches=("second tile of 2 groups",)),
    dict(geom=(2000, 64, 1040, 40), flags=FATE, paths=_STD, reaches=("partial column tile", "ngc<8")),
    dict(geom=(640, 360, 256, 161), flags=FATE, paths=_STD, reaches=("rgb row tile of 1",)),
    dict(geom=(640, 480, 512, 163), flags=FATE, paths=_STD, reaches=("luma row tile of 1",)),
    dict(geom=(400, 300, 136, 90), flags=FATE, paths={"yuv420p": (5, 3, 1)}, reaches=("chroma dstW%8",)),
    dict(geom=(1920, 1080, 1280, 720), flags=FATE, src_filter=(_SHARPEN, None, _SHARPEN, None), paths=_STD, reaches=("coef>16384", "clamp")),
    dict(geom=(1920, 1080, 1280, 720), flags=FATE, src_fmt=23, paths={"rgb24": _P, "bgra": _P, "yuv420p": (4, 6, 1)}, reaches=("nv",)),
    dict(geom=(1920, 1080, 1280, 720), flags=FATE, src_fmt=24, paths={"rgb24": _P, "bgra": _P, "yuv420p": (4, 6, 1)}, reaches=("nv",)),
    dict(geom=(1366, 768, 1024, 576), flags=FATE, src_fmt=23, paths={"rgb24": _P, "bgra": _P, "yuv420p": (4, 6, 1)}, reaches=("nv", "srcW%16")),
    dict(geom=(1366, 768, 1024, 576), flags=FATE, src_fmt=24, paths={"rgb24": _P, "bgra": _P, "yuv420p": (4, 6, 1)}, reaches=("nv", "srcW%16")),
    dict(geom=(640, 368, 320, 184), flags=FATE, paths=_STD, reaches=("nch=1",)),
    dict(geom=(1920, 1088, 1280, 720), flags=FATE, paths={k: _P for k in ("rgb24", "bgr24", "rgba", "bgra", "argb", "abgr", "yuv420p")},
         reaches=("nch=1",)),
    dict(geom=(704, 576, 1408, 1152), flags=SWS_BICUBIC, paths=_STD, reaches=("up2x",)),
]


# ---------------------------------------------------------------- exhaustive motion search (csrc/mecmp.cu launch_esa)
B200_ENOSYS = -38


def esa_kernel_for(mb, search):
    """Which kernel b200_me_esa_device runs for (mb, search), restating launch_esa<MB>'s shared-memory sizes: "esa2" while the four
    byte-phase copies of a two-macroblock window fit in 100 KB, "esa" while one window fits in 200 KB, else B200_ENOSYS."""
    wc = 2 * search + 2 * mb
    pitch = (wc + 3) // 4 + 1
    copy_words = (2 * search + mb + 7) * pitch + 1
    copy_words += (8 - (copy_words & 31) + 32) & 31
    if (2 * mb * (mb // 4) + 4 * copy_words) * 4 <= 100 * 1024:
        return "esa2"
    win_pitch = (2 * search + mb + 3) // 4 + 1
    return "esa" if (mb * (mb // 4) + (2 * search + mb) * win_pitch) * 4 <= 200 * 1024 else B200_ENOSYS


# Inputs of the search (esa_pictures): "flat" and the ties* kinds have several candidates of equal, minimal cost, spread over task groups of 8
# rows, lanes, warps and both macroblocks of an esa2 CTA.  "ties_zero_min": the zero vector's cost equals the minimum and is not 0;
# "ties_zero_0": it is 0 (the reference returns at once).  "extremes": inverse checkerboards (the zero vector costs 255 * mb^2, vectors of
# odd parity 0); "saturated": every candidate costs 255 * mb^2.
ESA_INPUTS_ALL = ("random", "shifted", "flat", "extremes", "saturated", "ties3", "ties8", "ties17", "ties_zero_min", "ties_zero_0")
ESA_INPUTS = ("random", "shifted", "flat", "extremes", "ties8", "ties_zero_min")


def _esa(w, h, mb, search, expect, note, nf=1, linesize=None, frame_stride=None, cur_off=0, ref_off=0, inputs=ESA_INPUTS, rows=None, group=None):
    linesize = linesize or w
    return dict(w=w, h=h, linesize=linesize, frame_stride=frame_stride or linesize * h, cur_off=cur_off, ref_off=ref_off, nf=nf, mb=mb,
                search=search, expect=expect, note=note, inputs=inputs, rows=rows, group=group)


def _boundary(mb, side, lo, last):
    """the searches just below and above the esa2 / esa boundary and esa's last one on a frame whose window both cover whole (identical
    outputs expected), and the first search that returns B200_ENOSYS"""
    g = f"boundary{mb}"
    return [_esa(side, side, mb, lo, "esa2", f"esa2_kernel<{mb}>, odd b_w, window = whole frame", inputs=ESA_INPUTS_ALL, group=g),
            _esa(side, side, mb, lo + 1, "esa", f"esa_kernel<{mb}> on the same case", inputs=ESA_INPUTS_ALL, group=g),
            _esa(side, side, mb, last, "esa", f"esa_kernel<{mb}>, its last search", inputs=ESA_INPUTS_ALL, group=g),
            _esa(side, side, mb, last + 1, B200_ENOSYS, "first search without a kernel: outputs untouched", inputs=("random",))]


_LS = 113                                                         # linesize = width + 13; frames at unaligned bases below
ESA_CASES = _boundary(16, 80, 64, 216) + _boundary(8, 72, 70, 220) + _boundary(4, 76, 74, 222) + [
    _esa(171, 107, 8, 75, "esa", "esa_kernel<8>, window inside the frame, size not a multiple of mb"),
    _esa(174, 102, 4, 80, "esa", "esa_kernel<4>, window inside the frame, size not a multiple of mb"),
    _esa(250, 170, 16, 70, "esa", "esa_kernel<16>, window inside the frame, size not a multiple of mb"),
    _esa(336, 200, 16, 32, "esa2", "odd b_w (21) at an everyday search, 8-row partial bottom band"),
    _esa(16, 200, 16, 32, "esa2", "b_w = 1"),
    _esa(200, 16, 16, 32, "esa2", "b_h = 1"),
    _esa(4, 4, 4, 3, "esa2", "one block"),
    _esa(100, 60, 8, 0, "esa2", "search 0"),
    _esa(37, 29, 4, 0, "esa2", "search 0, size not a multiple of mb"),
    _esa(48, 48, 16, 32, "esa2", "search beyond the frame on all four sides"),
    _esa(100, 70, 8, 12, "esa2", "linesize = width + 13, frame_stride odd, cur at base + 1, ref at base + 3: no word loads", nf=3,
         linesize=_LS, frame_stride=_LS * 70 + 5, cur_off=1, ref_off=3),
    _esa(100, 70, 16, 24, "esa2", "the same layout at mb 16", nf=3, linesize=_LS, frame_stride=_LS * 70 + 5, cur_off=1, ref_off=3),
    _esa(100, 70, 4, 80, "esa", "the same layout through esa_kernel<4>", nf=3, linesize=_LS, frame_stride=_LS * 70 + 5, cur_off=1, ref_off=3),
    _esa(101, 71, 16, 100, "esa", "the same layout through esa_kernel<16>", nf=2, linesize=_LS + 1, frame_stride=(_LS + 1) * 71 + 7,
         cur_off=3, ref_off=1),
    _esa(8, 8, 4, 4, "esa2", "65537 frames: the grid-z chunk loop, last chunk of two frames", nf=65537, linesize=9, frame_stride=75,
         inputs=("random", "ties3")),
    _esa(8, 8, 4, 75, "esa", "65537 frames through esa_kernel", nf=65537, linesize=9, frame_stride=75, inputs=("random", "ties3")),
    _esa(3840, 2160, 16, 32, "esa2", "BASELINE config 4: 4K pairs, +-32", nf=3, inputs=("shifted", "ties8"), rows=(0, 67, 134)),
    _esa(1920, 1080, 8, 16, "esa2", "1080p, mb 8", inputs=("shifted", "ties17"), rows=(0, 67, 134)),
    _esa(1920, 1080, 4, 7, "esa2", "1080p, mb 4", inputs=("shifted", "ties3"), rows=(0, 135, 269)),
]


def esa_pictures(kind, nf, h, w, seed):
    """(cur, ref): nf x h x w uint8 pictures of one input kind (see ESA_INPUTS_ALL)"""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    if kind == "random":
        return rng.integers(0, 256, (nf, h, w), dtype=np.uint8), rng.integers(0, 256, (nf, h, w), dtype=np.uint8)
    if kind == "shifted":                                        # a true vector exists, blurred by +-2 noise
        cur = rng.integers(0, 256, (nf, h, w), dtype=np.uint8)
        ref = np.stack([np.roll(cur[f], (int(rng.integers(-7, 8)), int(rng.integers(-7, 8))), (0, 1)) for f in range(nf)])
        return cur, (ref.astype(np.int16) + rng.integers(-2, 3, ref.shape)).clip(0, 255).astype(np.uint8)
    if kind == "flat":                                            # every candidate costs 2 * mb^2: the zero vector wins
        return np.full((nf, h, w), 99, np.uint8), np.full((nf, h, w), 97, np.uint8)
    if kind == "extremes":
        chk = ((xx + yy) % 2 * 255).astype(np.uint8)
        return np.broadcast_to(chk, (nf, h, w)).copy(), np.broadcast_to(255 - chk, (nf, h, w)).copy()
    if kind == "saturated":
        return np.full((nf, h, w), 255, np.uint8), np.zeros((nf, h, w), np.uint8)
    p, (sy, sx), plus = {"ties3": (3, (1, 2), 0), "ties8": (8, (3, 5), 0), "ties17": (17, (5, 11), 0),
                         "ties_zero_min": (5, (0, 0), 1), "ties_zero_0": (3, (0, 0), 0)}[kind]
    t = rng.integers(0, 255, (nf, p, p), dtype=np.uint8)           # periodic tiles: exact minima at every vector of the shift's class
    cur = t[:, yy % p, xx % p]
    return cur, t[:, (yy - sy) % p, (xx - sx) % p] + np.uint8(plus)


def esa_buffers(row, kind):
    """(cur buffer, ref buffer, cur pictures, ref pictures): the row's layout (offset, linesize, frame_stride) with the pictures of one
    input kind placed in it; padding bytes hold seeded noise, so a kernel that read them would change its result.  The seed depends on
    the picture size and the kind only: the rows of a boundary group search the same pictures."""
    w, h, ls, fs, nf = row["w"], row["h"], row["linesize"], row["frame_stride"], row["nf"]
    seed = (w * 10000 + h) * 16 + ESA_INPUTS_ALL.index(kind)
    cur, ref = esa_pictures(kind, nf, h, w, seed)
    rng = np.random.default_rng(seed + 1)
    bufs = []
    for pics, off in ((cur, row["cur_off"]), (ref, row["ref_off"])):
        b = rng.integers(0, 256, off + nf * fs + 64, dtype=np.uint8)
        frames = np.lib.stride_tricks.as_strided(b[off:], (nf, h, w), (fs, ls, 1), writeable=True)
        frames[...] = pics
        bufs.append(b)
    return bufs[0], bufs[1], cur, ref


def esa_expected(lib_fn, row, curbuf, refbuf, workers=None):
    """(mv [nf, blocks, 2] int32, cost [nf, blocks] uint64) of the CPU search `lib_fn` (orc_esa_frame / ffref_esa_frame) on the row's
    buffers, frames and macroblock-row ranges spread over threads (the C calls release the GIL).  Rows the case does not check stay 0."""
    import ctypes as C
    import os
    from concurrent.futures import ThreadPoolExecutor
    w, h, ls, fs, nf, mb, sp = (row[k] for k in ("w", "h", "linesize", "frame_stride", "nf", "mb", "search"))
    bw, bh = w // mb, h // mb
    mv, cost = np.zeros((nf, bh * bw, 2), np.int32), np.zeros((nf, bh * bw), np.uint64)
    spans = [(r, r + 1) for r in row["rows"]] if row["rows"] else [(r, min(r + 8, bh)) for r in range(0, bh, 8)]
    u8p, i32p, u64p = C.POINTER(C.c_uint8), C.POINTER(C.c_int32), C.POINTER(C.c_uint64)
    c0, r0 = curbuf.ctypes.data + row["cur_off"], refbuf.ctypes.data + row["ref_off"]

    def run(task):
        f0, f1, s = task
        for f in range(f0, f1):
            lib_fn(C.cast(c0 + f * fs, u8p), C.cast(r0 + f * fs, u8p), ls, w, h, mb, sp, s[0], s[1],
                   C.cast(mv[f].ctypes.data, i32p), C.cast(cost[f].ctypes.data, u64p))
    step = max(1, nf // 64)
    tasks = [(f, min(f + step, nf), s) for f in range(0, nf, step) for s in spans]
    with ThreadPoolExecutor(workers or os.cpu_count() or 1) as ex:
        list(ex.map(run, tasks))
    return mv, cost


# ---------------------------------------------------------------- motion compensation (csrc/pel.cu, csrc/pel_hbd.cu, csrc/h264weight.cu)
# Plane layouts of tests/test_pel_paths_gpu.py, tests/test_h264_hbd_paths_gpu.py and the checkers' pins on the reference.  A case's source
# and destination pictures have the same width and share one stride, like a decoder's reference and current pictures.  Each plane has an
# allocation of its own with PEL_SLACK bytes before its first and after its last sample: the kernels load the aligned 16-byte (qpel) or
# 8-byte (chroma) words around the bytes they need, so those words stay inside the allocation whatever the alignment of the base.
# Samples are bytes (bps = 1) or native-endian uint16 (bps = 2, depths 9 to 14); strides and offsets count bytes either way.
#   A  stride a multiple of 64 bytes (128 at bps 2), plane bases 64-byte aligned, block offsets as a decoder makes them (x a multiple of
#      the block width)
#   B  stride an odd number of samples (width + 37 or + 38): the rows of one block all have different alignments (at bps 2 they cycle
#      through 2, 4, 8 and 16 bytes); source base at +3 bytes (+2 at bps 2), destination base at +10, destination x jittered by 0..15
#      samples, so that 8- and 16-wide blocks take both the word and the sample store paths
#   C  the picture of A stored bottom-up: negative stride, the base (picture row 0) is the last row in memory and the offsets
#      y * stride + x * bps are negative
PEL_SLACK = 64
PEL_LAYOUTS = ("A", "B", "C")


class PelPlane:
    """One w x h picture in a layout.  buf: the whole allocation (uint8, seeded noise outside the picture); base: offset of sample
    (0, 0) in buf; stride: bytes from one picture row to the next (negative in layout C); bps: bytes per sample (1, or 2 for uint16
    samples).  Offsets handed to the kernels are relative to base: off(x, y) = y * stride + x * bps.  `pitch` / `mis` (bytes) replace
    the layout's row pitch / base misalignment."""

    def __init__(self, layout, w, h, role, seed, bps=1, pitch=None, mis=None):
        if layout == "B":
            lp, lm = (w + 37 if (w + 37) % 2 else w + 38) * bps, ((3 if bps == 1 else 2) if role == "src" else 10)
        else:
            lp, lm = (w * bps + 64 * bps - 1) // (64 * bps) * 64 * bps, 0
        pitch, mis = lp if pitch is None else pitch, lm if mis is None else mis
        self.layout, self.w, self.h, self.bps = layout, w, h, bps
        self.dtype = np.uint8 if bps == 1 else np.uint16
        self.stride = -pitch if layout == "C" else pitch
        self.base = PEL_SLACK + mis + ((h - 1) * pitch if layout == "C" else 0)
        size = PEL_SLACK + mis + (h - 1) * pitch + w * bps + PEL_SLACK
        self.buf = np.random.default_rng(seed).integers(0, 256, (size + 15) // 16 * 16, dtype=np.uint8)

    def off(self, x, y):
        return y * self.stride + x * self.bps

    def row(self, buf, y):
        """picture row y of the allocation `buf` (a copy of self.buf), as samples"""
        o = self.base + y * self.stride
        return buf[o:o + self.w * self.bps].view(self.dtype)

    def fill(self, pic):
        for y in range(self.h):
            self.row(self.buf, y)[:] = pic[y]
        return self

    def picture(self):
        return np.stack([self.row(self.buf, y).copy() for y in range(self.h)])


def pel_picture(kind, h, w, seed, depth=8):
    """'random', or 'extremes': 0 / max patterns in 24 x 24 tiles, cycling through vertical and horizontal stripes of periods 2, 3
    and 6, a checkerboard, flat 0 and flat max -- they drive the 6-tap sums, the centre sample and the weighted sums to both clip
    limits.  max = (1 << depth) - 1; uint8 samples at depth 8, uint16 above."""
    dt, mx = (np.uint8, 255) if depth == 8 else (np.uint16, (1 << depth) - 1)
    if kind == "random":
        return np.random.default_rng(seed).integers(0, mx + 1, (h, w), dtype=dt)
    yy, xx = np.mgrid[0:h, 0:w]
    pats = [xx % p < p // 2 for p in (2, 3, 6)] + [yy % p < p // 2 for p in (2, 3, 6)] + [(xx + yy) % 2 == 0, xx < 0, xx >= 0]
    tile = ((yy // 24) * 5 + xx // 24 + seed) % len(pats)
    return (np.select([tile == i for i in range(len(pats))], pats) * mx).astype(dt)


def pel_layout_case(layout, kind, blocks, seed, src_h=96, margin=(0, 0), cell=(16, 16), phases=None, cols=64, depth=8):
    """Source and destination planes and per-op offsets for a list of (block width, block height).  Op i reads its block at a seeded
    position of the source picture, `margin` = (samples before, samples after) it may read around the block staying inside the
    picture; with `phases`, the address of its sample (0, 0) is phases[i] mod 16 (bytes; even above depth 8).  It writes a block of
    its own cell (cell = (width, height)) of the destination picture, `cols` cells per row, at an x jitter the layout allows.
    depth 8: uint8 samples; 9 to 14: uint16 samples, offsets still in bytes.
    Returns dict(src=PelPlane, dst=PelPlane, soff=int64[n], doff=int64[n])."""
    rng = np.random.default_rng(seed)
    bps = 1 if depth == 8 else 2
    n = len(blocks)
    bw, bh = (np.array([b[k] for b in blocks], np.int64).reshape(n) for k in (0, 1))
    cw, ch = cell
    w = cols * cw
    rows = max(1, (n + cols - 1) // cols)
    src = PelPlane(layout, w, src_h, "src", seed + 1, bps).fill(pel_picture(kind, src_h, w, seed + 2, depth))
    dst = PelPlane(layout, w, rows * ch, "dst", seed + 3, bps).fill(pel_picture("random", rows * ch, w, seed + 4, depth))
    lo, hi = margin
    sy = rng.integers(lo, src_h - bh - hi + 1)
    sx = rng.integers(lo, w - bw - hi - 15 + 1)
    if phases is not None:
        assert bps == 1 or not (np.asarray(phases) % 2).any(), "uint16 samples sit at even byte phases"
        sx = sx + (np.asarray(phases, np.int64) - (src.base + src.off(sx, sy))) % 16 // bps
    if layout == "B":
        jx = rng.integers(0, np.minimum(15, cw - bw) + 1)
    else:
        jx = bw * rng.integers(0, (cw - bw) // bw + 1)
    i = np.arange(n, dtype=np.int64)
    return dict(src=src, dst=dst, soff=src.off(sx, sy).astype(np.int64), doff=dst.off((i % cols) * cw + jx, (i // cols) * ch).astype(np.int64))


# the (table, size index) pairs of HpelDSPContext the reference fills (hpeldsp.c:337-352): put / avg at 16, 8, 4 and 2 wide,
# put_no_rnd at 16 and 8, avg_no_rnd at 16; the other pairs are NULL there
HPEL_DEFINED = [(0, s) for s in range(4)] + [(1, s) for s in range(4)] + [(2, 0), (2, 1), (3, 0)]
HPEL_UNDEFINED = [(2, 2), (2, 3), (3, 1), (3, 2), (3, 3)]

EDGE_SIZES = ((1, 1), (80, 80), (71, 71), (33, 5), (5, 33), (21, 21), (9, 9), (64, 17), (17, 64))


def edge_windows(w, h):
    """(block_w, block_h, src_x, src_y): windows wholly outside each side and corner, straddling each border, and inside"""
    out = []
    for bw, bh in EDGE_SIZES:
        xs = sorted({-bw - 7, -bw, -bw + 1, -(bw // 2), 0, max(0, (w - bw) // 2), w - bw, w - 1, w, w + 9})
        ys = sorted({-bh - 7, -bh, -bh + 1, -(bh // 2), 0, max(0, (h - bh) // 2), h - bh, h - 1, h, h + 9})
        out += [(bw, bh, x, y) for x in xs for y in ys]
    return out
