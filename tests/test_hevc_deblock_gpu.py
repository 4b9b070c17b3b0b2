"""GPU tier for HEVC deblocking (ffmpeg_b200/csrc/hevcdbk.cu) on the H100: b200_hevc_deblock_plane_device against the reference's
fixture hashes and the checker at every depth, a 3840x2160 luma plane and its 4:2:0 chroma planes, a plane whose stride x height
exceeds 2^31 bytes, and every drop-in member of the context through host pointers.  Only committed fixtures and the checker are read."""
import numpy as np
import pytest

import hevcdbklib as hd

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    import ffmpeg_b200 as fb
    d = fb.Device(0)
    d.set_default()
    yield d


def _t(a):
    import torch
    a = np.ascontiguousarray(a)
    return torch.from_numpy(a.view(np.int16) if a.dtype == np.uint16 else a).cuda()


def on_device(dev, depth, chroma, buf, vg, hg, W, H):
    """one plane call on device copies of the buffer (plane at MARGIN, MARGIN) and the grids; returns the buffer as numpy"""
    import torch
    from ffmpeg_b200 import hevcdsp
    st = torch.cuda.ExternalStream(dev.stream)
    with torch.cuda.stream(st):
        db, dv, dh = _t(buf), _t(vg.view(np.uint8)), _t(hg.view(np.uint8))
        off = hd.MARGIN * buf.strides[0] + hd.MARGIN * buf.itemsize
        hevcdsp.hevc_deblock_plane_device(dev, depth, chroma, db.data_ptr() + off, buf.strides[0], W, H, dv, vg.shape[1], dh, hg.shape[1])
        dev.sync()
        return db.cpu().numpy().view(buf.dtype)


@pytest.mark.parametrize("depth", hd.DEPTHS)
@pytest.mark.parametrize("chroma", (0, 1), ids=("luma", "chroma"))
def test_plane_vs_fixture(dev, depth, chroma):
    """the fixture plane (every branch of the filters): the reference's result bit for bit, sentinels included"""
    (buf, vg, hg), W, H = hd.fixture_case(depth, chroma)
    got = on_device(dev, depth, chroma, buf, vg, hg, W, H)
    assert hd.digest(got) == hd.fixture_hashes()[(depth, bool(chroma))]
    assert np.array_equal(got, hd.orc_plane(depth, chroma, buf, vg, hg, W, H))


@pytest.mark.parametrize("depth", hd.DEPTHS)
@pytest.mark.parametrize("cls", hd.CLASSES)
def test_plane_vs_checker(dev, depth, cls):
    for chroma in (0, 1):
        W, H = (332, 188) if chroma else (516, 260)
        buf, vg, hg = hd.plane_case(2000 + 37 * depth + 5 * chroma + len(cls), depth, W, H, bool(chroma), cls)
        assert np.array_equal(on_device(dev, depth, chroma, buf, vg, hg, W, H), hd.orc_plane(depth, chroma, buf, vg, hg, W, H))


@pytest.mark.parametrize("depth", (8, 10))
def test_planes_3840x2160_420(dev, depth):
    """one decoder-shaped luma plane and both 4:2:0 chroma planes, one call each"""
    for seed, (W, H, chroma) in enumerate(((3840, 2160, 0), (1920, 1080, 1), (1920, 1080, 1))):
        buf, vg, hg = hd.plane_case(77 + depth + seed, depth, W, H, bool(chroma), ctb=64)
        got = on_device(dev, depth, chroma, buf, vg, hg, W, H)
        assert np.array_equal(got, hd.orc_plane(depth, chroma, buf, vg, hg, W, H))
        assert (got != buf).mean() > 0.02


def test_plane_beyond_2gb(dev):
    """a 10-bit plane whose stride x height exceeds 2^31 bytes (a 1 MiB stride): rows past 2^31 bytes are filtered where their
    64-bit offsets say, and nothing in the stride padding is written"""
    import torch
    from ffmpeg_b200 import hevcdsp
    W, H, stride = 136, 2052, 1 << 20
    buf, vg, hg = hd.plane_case(5, 10, W, H, False, "dense")
    plane = buf[hd.MARGIN:hd.MARGIN + H, hd.MARGIN:hd.MARGIN + W]
    assert stride * H > (1 << 31)
    st = torch.cuda.ExternalStream(dev.stream)
    with torch.cuda.stream(st):
        big = torch.full((H, stride // 2), 0x2A2A, dtype=torch.int16, device="cuda")
        big[:, :W] = torch.from_numpy(np.ascontiguousarray(plane).view(np.int16)).cuda()
        dv, dh = _t(vg.view(np.uint8)), _t(hg.view(np.uint8))
        hevcdsp.hevc_deblock_plane_device(dev, 10, 0, big, stride, W, H, dv, vg.shape[1], dh, hg.shape[1])
        dev.sync()
        got = big[:, :W].cpu().numpy().view(np.uint16)
        assert bool((big[:, W:] == 0x2A2A).all())
        del big
        torch.cuda.empty_cache()
    want = hd.orc_plane(10, 0, buf, vg, hg, W, H)[hd.MARGIN:hd.MARGIN + H, hd.MARGIN:hd.MARGIN + W]
    assert np.array_equal(got, want)
    assert not np.array_equal(got[-8:], plane[-8:])


@pytest.mark.parametrize("depth", hd.DEPTHS)
def test_dropin_members(dev, depth):
    """HEVCDSPContext from ff_hevc_dsp_init + ff_hevc_dsp_init_deblock: all eight loop-filter pointers (the _c pointers equal to the
    plain ones) called with host pointers against the checker on every input class; the MC tables the first init filled stay"""
    from ffmpeg_b200 import hevcdsp
    ctx = hevcdsp.ff_hevc_dsp_init(depth)
    mc = bytes(ctx.put_hevc_qpel)
    hevcdsp.ff_hevc_dsp_init_deblock(ctx, depth)
    assert bytes(ctx.put_hevc_qpel) == mc
    for n in ("h_loop_filter_luma", "v_loop_filter_luma", "h_loop_filter_chroma", "v_loop_filter_chroma"):
        assert getattr(ctx, "hevc_" + n) and getattr(ctx, "hevc_" + n) == getattr(ctx, "hevc_" + n + "_c")
    for cls in hd.CLASSES:
        for call in hd.member_calls(60 + depth + len(cls), depth, cls):
            want = hd.orc_member(depth, call)
            assert np.array_equal(hd.ctx_member(ctx, call), want), (cls, call[0], call[2:])
            assert np.array_equal(hd.ctx_member(ctx, call, twin=True), want)


def smoke(dev):
    """smoke(): a small decoder-shaped luma and chroma plane at 8 and 10 bit, bit-compared with the checker"""
    for depth in (8, 10):
        for chroma in (0, 1):
            W, H = (68, 36) if chroma else (132, 68)
            buf, vg, hg = hd.plane_case(11 + depth + chroma, depth, W, H, bool(chroma))
            got = on_device(dev, depth, chroma, buf, vg, hg, W, H)
            assert np.array_equal(got, hd.orc_plane(depth, chroma, buf, vg, hg, W, H)), ("hevc deblock mismatch", depth, chroma)
