"""GPU tier: the lane mapping of the same-size line-pair kernel for 24-bit rows (sws_vscale_rgb24_pair_kernel, FATE flags), where one
thread writes one 16-byte chunk of each line of its band: chunk r of a 16-px group lies at byte 16r of the group's 48.  Checked bit for
bit against the oracle over the whole destination buffer, not only the rows' pixels: pitch padding and the bytes before the first and
after the last frame hold a sentinel that must come back unchanged, so a lane that writes past its chunk is caught.  Widths put every
phase r at the end of a warp and of a CTA; destinations start at 16 mod 32 bytes, with pitches padded by 16 and 32 bytes; planar, nv12
and nv21 sources; top-down and bottom-up strides.  Every case also checks that the line-pair kernel ran (b200_sws_last_path bit 3)."""
import numpy as np
import pytest

import cpulibs as cl
from cases import FATE

pytestmark = pytest.mark.gpu

PAIR_KERNEL = 8                                          # b200_sws_last_path: the same-size line-pair kernel ran
SENTINEL = 0xA5
GUARD = 64                                               # sentinel bytes after the last frame


def frames(w, h, n, seed, src_fmt):
    """n distinct pictures: (oracle planes, planes the context reads) per frame; nv12 / nv21 as one interleaved plane"""
    out = []
    for i in range(n):
        y, u, v = cl.yuv_frame(w, h, seed + i, ("random", "extremes", "limited")[i % 3])
        if src_fmt:
            uv = cl.nv_interleave(u, v, src_fmt, pad=16)
            out.append(((y, uv, uv), [y, uv]))
        else:
            out.append(((y, u, v), [y, u, v]))
    return out


def run(device, w, h, fmt, src_fmt, *, n=2, seed=1, pitch_pad=0, base=0, src_up=False, dst_up=False):
    """n frames through scale_batch_device into one sentinel-filled buffer: destination `base` bytes into it, pitch w * bpp + pitch_pad.
    src_up / dst_up: the kernel walks the source planes / the destination rows bottom-up (pointer on the last row, negative stride)."""
    import torch
    from ffmpeg_b200 import swscale as sw
    bpp = cl.fmt_bpp(fmt)
    ds, pics = w * bpp + pitch_pad, frames(w, h, n, seed, src_fmt)
    exp = np.full(base + n * h * ds + GUARD, SENTINEL, np.uint8)
    for i, (ref_in, _) in enumerate(pics):
        ref = [np.ascontiguousarray(a[::-1]) for a in ref_in] if src_up else list(ref_in)
        img = cl.orc_sws(w, h, w, h, FATE, *ref, fmt=fmt, src_fmt=src_fmt)[:, :w * bpp]
        rows = exp[base + i * h * ds: base + (i + 1) * h * ds].reshape(h, ds)
        rows[:, :w * bpp] = img[::-1] if dst_up else img
    ctx = sw.sws_getContext(device, w, h, src_fmt, w, h, fmt, FATE)
    try:
        with torch.cuda.stream(torch.cuda.ExternalStream(device.stream)):
            planes = [torch.from_numpy(np.stack([p[1][k] for p in pics])).cuda() for k in range(len(pics[0][1]))]
            ss = [p.stride(1) for p in planes]
            sfs = [p.stride(0) for p in planes]
            src = planes
            if src_up:
                src = [p.data_ptr() + (p.shape[1] - 1) * p.stride(1) for p in planes]
                ss = [-s for s in ss]
            out = torch.full((exp.size,), SENTINEL, dtype=torch.uint8, device="cuda")
            assert out.data_ptr() % 32 == 0
            dst = out.data_ptr() + base + ((h - 1) * ds if dst_up else 0)
            ctx.scale_batch_device(src, ss, sfs, dst, -ds if dst_up else ds, h * ds, n)
            device.sync()
            got = out.cpu().numpy()
        assert ctx.last_path() & PAIR_KERNEL, "the line-pair kernel did not run"
    finally:
        ctx.free()
    bad = np.flatnonzero(got != exp)
    assert bad.size == 0, (w, h, fmt, src_fmt, pitch_pad, base, src_up, dst_up, int(bad.size), int(bad[0]))


# 16-px groups -> chunks per line (3 per group) -> where the last chunk falls: 1 -> 3, 2 -> 6, 11 -> 33 (one past a warp), 43 -> 129
# (one past a CTA of 128), 85 -> 255 (one short of two CTAs), 240 -> 720 (3840 px, the benchmark's width), 241 -> 723
@pytest.mark.parametrize("groups", [1, 2, 11, 43, 85, 240, 241])
@pytest.mark.parametrize("fmt", [cl.PIX_FMT_RGB24, cl.PIX_FMT_BGR24])
def test_chunk_counts(device, groups, fmt):
    """every phase of chunk at the end of a warp and of a CTA; tight pitch, so that the next line starts right after the last chunk"""
    run(device, 16 * groups, 36, fmt, 0, seed=groups)


@pytest.mark.parametrize("src_fmt", [0, cl.PIX_FMT_NV12, cl.PIX_FMT_NV21])
@pytest.mark.parametrize("pitch_pad,base", [(0, 16), (16, 0), (16, 16), (32, 16)])
def test_half_sector_destinations(device, src_fmt, pitch_pad, base):
    """a destination at 16 mod 32 bytes and pitches padded by 16 and 32 bytes: stores that are not whole sectors give the same bytes"""
    run(device, 16 * 43, 38, cl.PIX_FMT_RGB24, src_fmt, seed=3 + pitch_pad + base, pitch_pad=pitch_pad, base=base)


@pytest.mark.parametrize("src_fmt", [0, cl.PIX_FMT_NV12, cl.PIX_FMT_NV21])
@pytest.mark.parametrize("fmt", [cl.PIX_FMT_RGB24, cl.PIX_FMT_BGR24])
@pytest.mark.parametrize("src_up,dst_up", [(True, False), (False, True), (True, True)])
def test_bottom_up(device, src_fmt, fmt, src_up, dst_up):
    """negative source strides, a negative destination stride, or both, with a padded pitch and a base at 16 mod 32"""
    run(device, 16 * 85, 34, fmt, src_fmt, n=3, seed=40 + fmt, pitch_pad=16, base=16, src_up=src_up, dst_up=dst_up)
