"""GPU tier: the same-size line-pair kernel (sws_vscale_rgb24_pair_kernel, FATE flags) against the oracle bit for bit, at the shapes
where its work split has edges: pair counts that do not fill the last band of a CTA, column strips whose last CTA or warp is only
partly covered, every output byte order from planar / nv12 / nv21 sources, slice sequences, bottom-up and padded strides, and a
batch of distinct frames through the device entry point, with positive and negative (bottom-up) strides.  Every case also checks
that the line-pair kernel ran (b200_sws_last_path bit 3)."""
import numpy as np
import pytest

import cpulibs as cl
from cases import FATE

pytestmark = pytest.mark.gpu

KINDS = [cl.PIX_FMT_RGB24, cl.PIX_FMT_BGR24, cl.PIX_FMT_RGBA, cl.PIX_FMT_BGRA, cl.PIX_FMT_ARGB, cl.PIX_FMT_ABGR]
SOURCES = [0, cl.PIX_FMT_NV12, cl.PIX_FMT_NV21]
PAIR_KERNEL = 8                                          # b200_sws_last_path: the same-size line-pair kernel ran


def planes(w, h, seed, src_fmt, kind="random"):
    """(y, u, v) for the oracle and what the context reads: (y, uv, uv) for the interleaved sources"""
    y, u, v = cl.yuv_frame(w, h, seed, kind)
    if src_fmt:
        uv = cl.nv_interleave(u, v, src_fmt, pad=16)
        return (y, uv, uv), (y, uv, uv)
    return (y, u, v), (y, u, v)


def check(device, w, h, fmt=cl.PIX_FMT_RGB24, src_fmt=0, seed=1, kind="random", dst_pad=0, pair=True):
    from ffmpeg_b200 import swscale as sw
    ref_in, gpu_in = planes(w, h, seed, src_fmt, kind)
    exp = cl.orc_sws(w, h, w, h, FATE, *ref_in, dst_pad=dst_pad, fmt=fmt, src_fmt=src_fmt)
    ctx = sw.sws_getContext(device, w, h, src_fmt, w, h, fmt, FATE)
    try:
        got = ctx.convert(*gpu_in, dst_pad=dst_pad)
        assert bool(ctx.last_path() & PAIR_KERNEL) == pair, "the line-pair kernel ran" if not pair else "the line-pair kernel did not run"
    finally:
        ctx.free()
    bpp = cl.fmt_bpp(fmt)
    assert np.array_equal(got[:, :w * bpp], exp[:, :w * bpp]), (w, h, fmt, src_fmt, int((got[:, :w * bpp] != exp[:, :w * bpp]).sum()))


@pytest.mark.parametrize("h", [12, 14, 32, 34, 36, 38, 64, 66, 68, 100, 102])
def test_pair_counts(device, h):
    """5 to 50 pairs: fewer than one band, one band, one more than a band, several bands with a short last one.  12 lines is the
    smallest height at which the host pairs the chroma windows of lines 2k+1 / 2k+2 (below, and at odd heights, the bicubic
    positions of the two lines differ)"""
    check(device, 336, h, seed=h)


@pytest.mark.parametrize("h", [4, 5, 8, 33, 35, 67, 101])
def test_unpaired_heights(device, h):
    """small and odd heights: the host keeps every line on the one-line kernel, with the same bytes"""
    check(device, 336, h, seed=h, pair=False)


@pytest.mark.parametrize("w", [16, 48, 3856, 4112])
def test_partial_strips(device, w):
    """one or three 16-px groups; a strip of whole warps plus a partial warp; two full strips plus a few groups"""
    for src_fmt in (0, cl.PIX_FMT_NV12):
        check(device, w, 38, src_fmt=src_fmt, seed=w)


@pytest.mark.parametrize("src_fmt", SOURCES)
@pytest.mark.parametrize("fmt", KINDS)
def test_kinds_and_sources(device, fmt, src_fmt):
    check(device, 1296, 70, fmt=fmt, src_fmt=src_fmt, seed=fmt + 100 * src_fmt, dst_pad=32)
    check(device, 208, 42, fmt=fmt, src_fmt=src_fmt, seed=7, kind="extremes")


@pytest.mark.parametrize("src_fmt", [0, cl.PIX_FMT_NV12])
@pytest.mark.parametrize("bands", [((0, 22), (22, 46), (68, 90), (158, 42)), ((0, 4), (4, 2), (6, 60), (66, 64), (130, 70)),
                                   ((0, 100), (100, 100))])
def test_slices(device, bands, src_fmt):
    """slice sequences whose edges fall inside the kernel's bands (a launch starts at an odd line and may start or end mid-band)"""
    from ffmpeg_b200 import swscale as sw
    w, h = 1040, 200
    ref_in, (y, u, v) = planes(w, h, 55, src_fmt)
    exp = cl.orc_sws(w, h, w, h, FATE, *ref_in, src_fmt=src_fmt)
    ctx = sw.sws_getContext(device, w, h, src_fmt, w, h, sw.AV_PIX_FMT_RGB24, FATE)
    out = np.full((h, w * 3), 0xA5, np.uint8)
    total = 0
    for sy, sh in bands:
        src = [y[sy:], u[sy // 2:]] + ([] if src_fmt else [v[sy // 2:]])
        total += ctx.scale(src, [a.strides[0] for a in src], sy, sh, [out], [w * 3])
    assert ctx.last_path() & PAIR_KERNEL
    ctx.free()
    assert total == h
    assert np.array_equal(out, exp), int((out != exp).sum())


@pytest.mark.parametrize("src_fmt", [0, cl.PIX_FMT_NV21])
def test_bottom_up_strides(device, src_fmt):
    """negative source strides (the picture is read upside down) and a negative destination stride"""
    from ffmpeg_b200 import swscale as sw
    w, h = 1296, 102
    ref_in, (y, u, v) = planes(w, h, 77, src_fmt)
    src = [y, u] + ([] if src_fmt else [v])
    flipped = [np.ascontiguousarray(a[::-1]) for a in ref_in]
    ctx = sw.sws_getContext(device, w, h, src_fmt, w, h, sw.AV_PIX_FMT_BGRA, FATE)
    out = np.zeros((h, w * 4), np.uint8)
    assert ctx.scale([a.ctypes.data + (a.shape[0] - 1) * a.strides[0] for a in src], [-a.strides[0] for a in src], 0, h, [out], [w * 4]) == h
    assert np.array_equal(out, cl.orc_sws(w, h, w, h, FATE, *flipped, fmt=cl.PIX_FMT_BGRA, src_fmt=src_fmt))
    out2 = np.zeros((h, w * 4), np.uint8)
    assert ctx.scale(src, [a.strides[0] for a in src], 0, h, [out2.ctypes.data + (h - 1) * w * 4], [-w * 4]) == h
    assert ctx.last_path() & PAIR_KERNEL
    ctx.free()
    assert np.array_equal(out2[::-1], cl.orc_sws(w, h, w, h, FATE, *ref_in, fmt=cl.PIX_FMT_BGRA, src_fmt=src_fmt))


@pytest.mark.parametrize("fmt", [cl.PIX_FMT_RGB24, cl.PIX_FMT_ARGB])
def test_batch_device_distinct_frames(device, fmt):
    """three distinct frames through scale_batch_device, padded source and destination strides"""
    import torch
    from ffmpeg_b200 import swscale as sw
    w, h, n, pad = 1920, 134, 3, 64
    frames = [cl.yuv_frame(w, h, 500 + i, ("random", "limited", "extremes")[i], pad=pad) for i in range(n)]
    bpp = cl.fmt_bpp(fmt)
    ds = w * bpp + pad
    ctx = sw.sws_getContext(device, w, h, 0, w, h, fmt, FATE)
    with torch.cuda.stream(torch.cuda.ExternalStream(device.stream)):
        dY, dU, dV = (torch.from_numpy(np.stack([f[k] for f in frames])).cuda() for k in range(3))
        out = torch.full((n, h, ds), 0xA5, dtype=torch.uint8, device="cuda")
        ctx.scale_batch_device([dY, dU, dV], [a.strides[0] for a in frames[0]], [a.size for a in frames[0]], out, ds, h * ds, n)
        device.sync()
        got = out.cpu().numpy()
    assert ctx.last_path() & PAIR_KERNEL
    ctx.free()
    for i in range(n):
        exp = cl.orc_sws(w, h, w, h, FATE, *frames[i], fmt=fmt)
        assert np.array_equal(got[i][:, :w * bpp], exp[:, :w * bpp]), i


@pytest.mark.parametrize("fmt", [cl.PIX_FMT_RGB24, cl.PIX_FMT_RGBA])
def test_batch_device_bottom_up(device, fmt):
    """scale_batch_device with negative strides, so that the kernel itself walks a picture bottom-up: the destination rows (each frame's
    pointer on its last row, negative row stride) and, in a second call, the source planes"""
    import torch
    from ffmpeg_b200 import swscale as sw
    w, h, n = 1296, 70, 3
    frames = [cl.yuv_frame(w, h, 610 + i, "random") for i in range(n)]
    bpp = cl.fmt_bpp(fmt)
    ds = w * bpp
    ctx = sw.sws_getContext(device, w, h, 0, w, h, fmt, FATE)
    ss = [w, w // 2, w // 2]
    sfs = [a.size for a in frames[0]]
    with torch.cuda.stream(torch.cuda.ExternalStream(device.stream)):
        dY, dU, dV = (torch.from_numpy(np.stack([f[k] for f in frames])).cuda() for k in range(3))
        out = torch.full((n, h, ds), 0xA5, dtype=torch.uint8, device="cuda")
        ctx.scale_batch_device([dY, dU, dV], ss, sfs, out.data_ptr() + (h - 1) * ds, -ds, h * ds, n)
        device.sync()
        got_dst = out.cpu().numpy()
        assert ctx.last_path() & PAIR_KERNEL
        out.fill_(0xA5)
        last = [p.data_ptr() + (p.shape[1] - 1) * p.stride(1) for p in (dY, dU, dV)]
        ctx.scale_batch_device(last, [-x for x in ss], sfs, out, ds, h * ds, n)
        device.sync()
        got_src = out.cpu().numpy()
        assert ctx.last_path() & PAIR_KERNEL
    ctx.free()
    for i in range(n):
        assert np.array_equal(got_dst[i][::-1], cl.orc_sws(w, h, w, h, FATE, *frames[i], fmt=fmt)), ("bottom-up destination", i)
        flipped = [np.ascontiguousarray(a[::-1]) for a in frames[i]]
        assert np.array_equal(got_src[i], cl.orc_sws(w, h, w, h, FATE, *flipped, fmt=fmt)), ("bottom-up source", i)
