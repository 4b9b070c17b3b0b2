"""GPU tier for HEVC sample adaptive offset (ffmpeg_b200/csrc/hevcsao.cu) on the H100: b200_hevc_sao_plane_device against the
reference's fixture hashes and the checker at every depth, a decoder-shaped 3840x2160 luma plane and two 1920x1080 chroma planes, a
plane whose stride x height exceeds 2^31 bytes, and every SAO member of the context through host pointers.  Only committed fixtures
and the checker are read."""
import numpy as np
import pytest

import hevcsaolib as hl

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


def on_device(dev, p, c, rec=None, keep="auto"):
    """component c through the plane entry on device copies of the framed src / dst buffers, records and keep map; returns the framed
    dst buffer as numpy (and checks that src was not written)"""
    import torch
    from ffmpeg_b200 import hevcdsp
    W, H, hs, vs = hl.comp_geometry(p, c)
    g = hl.records(p, c, garbage_seed=11 + c) if rec is None else rec
    k = hl.keep_map(p) if keep == "auto" else keep
    src = hl.framed(p.planes[c], p.depth)
    dst = np.full_like(src, hl.sentinel(p.depth))
    off = hl.MARGIN * src.strides[0] + hl.MARGIN * src.itemsize
    st = torch.cuda.ExternalStream(dev.stream)
    with torch.cuda.stream(st):
        ds, dd, dg = _t(src), _t(dst), _t(g.view(np.uint8))
        dk = None if k is None else _t(k)
        hevcdsp.hevc_sao_plane_device(dev, p.depth, dd.data_ptr() + off, dst.strides[0], ds.data_ptr() + off, src.strides[0], W, H, p.log2_ctb,
                                      hs, vs, dg, g.shape[1], dk, 0 if k is None else k.shape[1], p.log2_pu)
        dev.sync()
        assert np.array_equal(ds.cpu().numpy().view(src.dtype), src)
        return dd.cpu().numpy().view(dst.dtype)


@pytest.mark.parametrize("depth", hl.DEPTHS)
def test_plane_vs_fixture(dev, depth):
    """the fixture picture's luma and 4:2:0 chroma planes (every outcome): the reference's result bit for bit, sentinels included"""
    p = hl.fixture_case(depth)
    for c, name in ((0, "luma"), (1, "chroma420")):
        got = on_device(dev, p, c)
        assert hl.digest(got) == hl.fixture_hashes()[(depth, name)]
        assert np.array_equal(got, hl.orc_plane(p, c))


@pytest.mark.parametrize("depth", hl.DEPTHS)
@pytest.mark.parametrize("cfmt", (0, 1, 2, 3), ids=("luma", "420", "422", "444"))
def test_plane_vs_checker(dev, depth, cfmt):
    """CTB sizes 16 / 32 / 64, slices and tiles with and without filtering across, with and without a keep map"""
    for log2_ctb in (4, 5, 6):
        p = hl.picture_case(2000 + 37 * depth + 5 * cfmt + log2_ctb, depth, 520 + 8 * log2_ctb, 264 - 8 * cfmt, log2_ctb, cfmt, nslices=6,
                            tiles=(3, 2), lf_tiles=log2_ctb == 4, pcm=log2_ctb != 5, scatter=0.1)
        for c in range(len(p.planes)):
            assert np.array_equal(on_device(dev, p, c), hl.orc_plane(p, c)), (log2_ctb, c)


@pytest.mark.parametrize("depth", (8, 10))
def test_planes_3840x2160_420(dev, depth):
    """one decoder-shaped 4K picture (CTB 64, slices, PCM map): its luma plane and both 1920x1080 chroma planes, one call each"""
    p = hl.picture_case(77 + depth, depth, 3840, 2160, 6, 1, nslices=8, lf_slices=(1, 0), pcm=True)
    for c in range(3):
        got = on_device(dev, p, c)
        assert np.array_equal(got, hl.orc_plane(p, c)), c
        W, H, _, _ = hl.comp_geometry(p, c)
        assert (hl.inner(got, H, W) != p.planes[c]).mean() > 0.05


def test_plane_beyond_2gb(dev):
    """a 10-bit plane whose stride x height exceeds 2^31 bytes (a 1 MiB stride): rows past 2^31 bytes are filtered where their
    64-bit offsets say, and nothing in the stride padding of dst is written"""
    import torch
    from ffmpeg_b200 import hevcdsp
    W, H, stride = 136, 2056, 1 << 20
    p = hl.picture_case(5, 10, W, H, 5, 0, nslices=4, pcm=True)
    assert stride * H > (1 << 31)
    g, k = hl.records(p, 0), hl.keep_map(p)
    st = torch.cuda.ExternalStream(dev.stream)
    with torch.cuda.stream(st):
        src = torch.full((H, stride // 2), 0x1111, dtype=torch.int16, device="cuda")
        src[:, :W] = torch.from_numpy(p.planes[0].view(np.int16)).cuda()
        dst = torch.full((H, stride // 2), 0x2A2A, dtype=torch.int16, device="cuda")
        hevcdsp.hevc_sao_plane_device(dev, 10, dst, stride, src, stride, W, H, 5, 0, 0, _t(g.view(np.uint8)), g.shape[1], _t(k), k.shape[1], 2)
        dev.sync()
        got = dst[:, :W].cpu().numpy().view(np.uint16)
        assert bool((dst[:, W:] == 0x2A2A).all())
        del src, dst
        torch.cuda.empty_cache()
    want = hl.inner(hl.orc_plane(p, 0), H, W)
    assert np.array_equal(got, want)
    assert not np.array_equal(got[-8:], p.planes[0][-8:])


@pytest.mark.parametrize("depth", hl.DEPTHS)
def test_dropin_members(dev, depth):
    """HEVCDSPContext from ff_hevc_dsp_init + _init_transform + _init_deblock + _init_sao: every SAO pointer with host pointers against
    the checker (band in place and separate, edge at every class and size, both restore sweeps); the members the other inits filled
    stay as they were"""
    import ctypes as C
    from ffmpeg_b200 import hevcdsp
    ctx = hevcdsp.ff_hevc_dsp_init(depth)
    hevcdsp.ff_hevc_dsp_init_transform(ctx, depth)
    hevcdsp.ff_hevc_dsp_init_deblock(ctx, depth)
    first = type(ctx).sao_band_filter.offset
    raw = bytearray(C.string_at(C.addressof(ctx), C.sizeof(ctx)))
    hevcdsp.ff_hevc_dsp_init_sao(ctx, depth)
    after = bytearray(C.string_at(C.addressof(ctx), C.sizeof(ctx)))
    assert raw[:first] == after[:first] and raw[first + 96:] == after[first + 96:]
    assert raw[first:first + 96] == bytes(96) and all(ctx.sao_band_filter) and all(ctx.sao_edge_filter) and all(ctx.sao_edge_restore)
    from test_hevc_sao import check_members
    check_members(ctx, depth, 90 + depth)


def smoke(dev):
    """smoke(): a small picture's luma and 4:2:0 chroma planes at 8 and 10 bit, bit-compared with the checker"""
    for depth in (8, 10):
        p = hl.picture_case(11 + depth, depth, 136, 72, 5, 1, nslices=2, tiles=(2, 1), lf_tiles=False, pcm=True)
        for c in (0, 1):
            assert np.array_equal(on_device(dev, p, c), hl.orc_plane(p, c)), ("hevc sao mismatch", depth, c)
