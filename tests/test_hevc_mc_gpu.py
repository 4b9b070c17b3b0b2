"""GPU tier for HEVC motion compensation (ffmpeg_b200/csrc/hevcmc.cu) on the H100: b200_hevc_mc_batch_device against the checker and the
reference's fixture hashes at every depth for luma (qpel) and chroma (epel), one 3840x2160 call of mixed unit sizes, one call of more
ops than one launch takes, and every drop-in member of the HEVCDSPContext tables through host pointers.  Only committed fixtures and
the checker are read."""
import ctypes as C

import numpy as np
import pytest

import cpulibs as cl
import hevcmclib as hm

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    import ffmpeg_b200 as fb
    d = fb.Device(0)
    d.set_default()
    yield d


def on_device(dev, depth, epel, ref, dst, ops):
    """one batched call on device copies (ref = [2, h, w], the call's `ref` pointer at picture 1); returns dst as numpy"""
    import torch
    from ffmpeg_b200 import hevcdsp
    st = torch.cuda.ExternalStream(dev.stream)
    with torch.cuda.stream(st):
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.int16) if a.dtype == np.uint16 else np.ascontiguousarray(a)).cuda()
        dr, dd, do = t(ref), t(dst), t(ops.view(np.uint8))
        hevcdsp.hevc_mc_batch_device(dev, depth, epel, len(ops), do, dd, dst.strides[0], dr.data_ptr() + ref.strides[0], ref.strides[1],
                                     ref.shape[2], ref.shape[1])
        dev.sync()
        return dd.cpu().numpy().view(dst.dtype)


@pytest.mark.parametrize("depth", hm.DEPTHS)
@pytest.mark.parametrize("epel", (0, 1), ids=("luma", "chroma"))
def test_batch_vs_fixture(dev, depth, epel):
    """the fixture batch (every kind and width, edges, corners, windows wholly outside, mixed integer / fractional bi): the reference's
    destination picture bit for bit, sentinels around every block included"""
    case = hm.fixture_case(depth, epel)
    got = on_device(dev, depth, epel, *case)
    assert hm.digest(got) == hm.fixture_hashes()[(depth, bool(epel))]
    assert np.array_equal(got, hm.orc_batch(depth, epel, *case))


@pytest.mark.parametrize("depth", hm.DEPTHS)
@pytest.mark.parametrize("epel", (0, 1), ids=("luma", "chroma"))
@pytest.mark.parametrize("cls", (0, 1, 2, 3), ids=("noise", "zero", "max", "extremes"))
def test_batch_vs_checker(dev, depth, epel, cls):
    case = hm.batch_case(2000 + 37 * depth + 5 * epel + cls, 512, depth, epel, cls=cls)
    assert np.array_equal(on_device(dev, depth, epel, *case), hm.orc_batch(depth, epel, *case))


def frame_case(seed, depth, epel, W, H):
    """a W x H plane tiled with 8x8, 16x16, 32x32 and 64x64 units (64 x 64 CTUs, each split at random), every unit an op of a seeded
    kind and phases, motion within +-64 samples (so some windows leave the picture)"""
    rng = np.random.default_rng(seed)
    ref = np.stack([hm.picture(rng, H, W, depth, 0) for _ in range(2)])
    dst = np.zeros((H, W), hm.sdtype(depth))
    units = []

    def split(x, y, s):
        if s > 8 and rng.random() < 0.6:
            for dy in (0, s // 2):
                for dx in (0, s // 2):
                    split(x + dx, y + dy, s // 2)
        elif x < W and y < H:
            units.append((x, y, min(s, W - x), min(s, H - y)))
    for y in range(0, H, 64):
        for x in range(0, W, 64):
            split(x, y, 64)
    ops = np.zeros(len(units), hm.OP_DTYPE)
    u = np.array(units)
    bps, P = ref.itemsize, 8 if epel else 4
    ops["dst_off"] = u[:, 1] * dst.strides[0] + u[:, 0] * bps
    ops["w"], ops["h"] = u[:, 2], u[:, 3]
    ops["kind"] = rng.integers(0, 4, len(u))
    ops["ref_off"][:, 0] = -ref.strides[0]
    for r in (0, 1):
        ops["x"][:, r] = u[:, 0] + rng.integers(-64, 65, len(u))
        ops["y"][:, r] = u[:, 1] + rng.integers(-64, 65, len(u))
        ops["mx"][:, r] = rng.integers(0, P, len(u))
        ops["my"][:, r] = rng.integers(0, P, len(u))
    ops["denom"] = rng.integers(0, 8, len(u))
    ops["wx0"] = rng.integers(-128, 256, len(u))
    ops["wx1"] = rng.integers(-128, 256, len(u))
    ops["ox"] = rng.integers(-128, 128, len(u))
    return ref, dst, ops


@pytest.mark.parametrize("depth,epel", [(8, 0), (10, 0), (8, 1), (10, 1)], ids=("8-luma", "10-luma", "8-chroma", "10-chroma"))
def test_frame_3840x2160(dev, depth, epel):
    W, H = (3840, 2160) if not epel else (1920, 1080)
    case = frame_case(77 + depth + epel, depth, epel, W, H)
    got = on_device(dev, depth, epel, *case)
    exp = hm.orc_batch(depth, epel, *case)
    assert np.array_equal(got, exp)
    assert (got != 0).mean() > 0.5


def test_more_ops_than_one_launch(dev):
    """2^20 + 4099 chroma ops of 4x2 (more than one launch's 2^20): every block against the checker"""
    n, cols = (1 << 20) + 4099, 1024
    rng = np.random.default_rng(3)
    ref = np.stack([hm.picture(rng, 64, 96, 8, 0) for _ in range(2)])
    dst = np.zeros(((n + cols - 1) // cols * 2, cols * 4), np.uint8)
    ops = np.zeros(n, hm.OP_DTYPE)
    i = np.arange(n)
    ops["dst_off"] = (i // cols) * 2 * dst.strides[0] + (i % cols) * 4
    ops["w"], ops["h"], ops["kind"] = 4, 2, i % 4
    ops["ref_off"][:, 0] = -ref.strides[0]
    for r in (0, 1):
        ops["x"][:, r] = rng.integers(-8, 100, n)
        ops["y"][:, r] = rng.integers(-8, 70, n)
        ops["mx"][:, r] = rng.integers(0, 8, n)
        ops["my"][:, r] = rng.integers(0, 8, n)
    ops["denom"], ops["wx0"], ops["wx1"], ops["ox"] = 3, 20, 12, 5
    got = on_device(dev, 8, 1, ref, dst, ops)
    assert np.array_equal(got, hm.orc_batch(8, 1, ref, dst, ops))


@pytest.mark.parametrize("depth", hm.DEPTHS)
@pytest.mark.parametrize("epel", (0, 1), ids=("qpel", "epel"))
def test_dropin_members(dev, depth, epel):
    """HEVCDSPContext from ff_hevc_dsp_init through the library: every (form, [v][h], width) member called with host pointers
    against the checker, over the four content classes"""
    from ffmpeg_b200 import hevcdsp
    ctx = hevcdsp.ff_hevc_dsp_init(depth)
    for cls in range(4):
        pic, src2, dst0 = hm.member_case(60 + depth + cls, depth, epel, cls)
        for call in hm.member_calls(60 + depth + cls, depth, epel):
            exp = hm.run_member(cl.oracle(), "orc_hevc_mc", depth, epel, call, pic, src2, dst0)
            got = run_ctx_member(ctx, depth, epel, call, pic, src2, dst0)
            assert np.array_equal(got, exp), call


def run_ctx_member(ctx, depth, epel, call, pic, src2, dst0):
    """one call through the table entry [idx of width][v][h], HOST pointers, the reference's argument order"""
    form, v, h, width, height, mx, my, denom, wx0, wx1, ox = call
    fn = getattr(ctx, f"put_hevc_{'epel' if epel else 'qpel'}{hm.FORMS[form]}")[hm.WIDTHS.index(width)][v][h]
    src = pic.ctypes.data + 8 * pic.strides[0] + 8 * pic.itemsize
    ss = pic.strides[0]
    if form == 0:
        d = np.zeros((64, 64), np.int16)
        fn(d.ctypes.data, src, ss, height, mx, my, width)
        return d
    d = dst0.copy()
    ds = d.strides[0]
    if form == 1:
        fn(d.ctypes.data, ds, src, ss, height, mx, my, width)
    elif form == 2:
        fn(d.ctypes.data, ds, src, ss, height, denom, wx0, ox, mx, my, width)
    elif form == 3:
        fn(d.ctypes.data, ds, src, ss, src2.ctypes.data, height, mx, my, width)
    else:
        fn(d.ctypes.data, ds, src, ss, src2.ctypes.data, height, denom, wx0, wx1, ox, mx, my, width)
    return d


def smoke(dev):
    """smoke(): one small luma and chroma batch at 8 and 10 bit, bit-compared with the checker"""
    for depth in (8, 10):
        for epel in (0, 1):
            case = hm.batch_case(11 + depth + epel, 64, depth, epel)
            got = on_device(dev, depth, epel, *case)
            assert np.array_equal(got, hm.orc_batch(depth, epel, *case)), ("hevc mc mismatch", depth, epel)
