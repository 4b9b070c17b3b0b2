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
