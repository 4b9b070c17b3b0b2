"""GPU tier for HEVC intra reconstruction of a whole picture (ffmpeg_b200/csrc/hevcintra.cu) on the H100:
b200_hevc_intra_recon_picture_device against the reference's fixture hashes and the checker, 1920x1080 and 3840x2160 4:2:0 pictures at
8 and 10 bit against the checker and against the per-level path of the batch entries, an inter picture with sparse intra TUs among
prefilled samples, constrained intra prediction, one call of more than 2^20 ops, invalid ops and the refusals.  After every test the
entry's wait-timeout counter is still 0.  Only committed fixtures and the checker are read."""
import ctypes as C

import numpy as np
import pytest

import hevcintralib as hl

pytestmark = pytest.mark.gpu
EINVAL = -22


@pytest.fixture(scope="module")
def dev():
    import ffmpeg_b200 as fb
    d = fb.Device(0)
    d.set_default()
    yield d


@pytest.fixture(autouse=True)
def no_timeouts(dev):
    yield
    from ffmpeg_b200 import hevcdsp
    assert hevcdsp.hevc_intra_timeouts(dev) == 0


def _t(a):
    import torch
    a = np.ascontiguousarray(a)
    return torch.from_numpy(a.view(np.int16) if a.dtype == np.uint16 else a).cuda()


def _back(t, like):
    return t.cpu().numpy().view(like.dtype)


def same(a, b):
    return len(a) == len(b) and all(np.array_equal(x, y) for x, y in zip(a, b))


def _ptrs(ts, bufs):
    return [t.data_ptr() + hl.MARGIN * b.strides[0] + hl.MARGIN * b.itemsize for t, b in zip(ts, bufs)]


def on_device(dev, p, ops=None, levels=False):
    """the picture entry (or, levels=True, the per-level path: per plane and dependency level one prediction batch and one residual
    batch) on device copies of the framed planes; returns the framed planes"""
    import torch
    from ffmpeg_b200 import hevcdsp
    bufs = p.framed()
    ops = np.ascontiguousarray(p.ops if ops is None else ops)
    st = torch.cuda.ExternalStream(dev.stream)
    with torch.cuda.stream(st):
        ts = [_t(b) for b in bufs]
        coef = _t(p.coef)
        m = None if p.map is None else _t(p.map)
        ms = 0 if p.map is None else p.map.strides[0]
        ptrs = _ptrs(ts, bufs)
        ls_y, ls_uv = p.strides(bufs)
        if not levels:
            hevcdsp.hevc_intra_recon_picture_device(dev, p.depth, p.cfmt, p.W, p.H, ptrs, ls_y, ls_uv, len(ops), _t(ops.view(np.uint8)), coef,
                                                    m, ms, p.log2_min_pu)
        else:
            for c, io, idx in hl.level_batches(p):
                hs, vs = p.shifts(c)
                s = bufs[c].strides[0]
                hevcdsp.hevc_intra_pred_batch_device(dev, p.depth, ptrs[c], s, p.W, p.H, hs, vs, len(io), _t(io.view(np.uint8)), m, ms,
                                                     p.log2_min_pu)
                tu = hl.level_tu_ops(p, idx, s)
                if len(tu):
                    hevcdsp.hevc_transform_add_batch_device(dev, p.depth, len(tu), _t(tu.view(np.uint8)), coef, ptrs[c], s)
        dev.sync()
        return [_back(t, b) for t, b in zip(ts, bufs)]


@pytest.mark.parametrize("name", hl.FIXTURE_NAMES)
def test_picture_vs_fixture(dev, name):
    """every fixture picture: the reference's hash and the checker, over the whole framed planes (sentinels unchanged)"""
    p = hl.fixture_case(name)
    got = on_device(dev, p)
    assert hl.digest(got) == hl.fixture_hashes()[name]
    assert same(got, hl.orc_picture(p))


LARGE = [(8, 1920, 1080), (10, 1920, 1080), (8, 3840, 2160), (10, 3840, 2160)]


@pytest.mark.parametrize("depth,W,H", LARGE, ids=[f"{d}-{h}p" for d, _, h in LARGE])
def test_large_pictures(dev, depth, W, H):
    """decoder-sized 4:2:0 intra pictures (CTB 64, slices, tiles): equal to the checker and to the per-level path"""
    p = hl.picture(50 + depth + H, depth, 1, W, H, 6, nslices=4, tiles=(2, 2), split=0.6)
    got = on_device(dev, p)
    assert same(got, hl.orc_picture(p))
    assert same(got, on_device(dev, p, levels=True))


def test_sparse_intra_in_inter_picture(dev):
    """an inter picture (prefilled samples) with a fifth of its CUs intra, constrained intra prediction on"""
    p = hl.picture(77, 10, 1, 1920, 1080, 6, cip=True, p_intra=0.2, nslices=2)
    got = on_device(dev, p)
    assert same(got, hl.orc_picture(p))
    assert same(got, on_device(dev, p, levels=True))


@pytest.mark.parametrize("cfmt", (2, 3))
def test_cip_pictures(dev, cfmt):
    """constrained intra prediction at 12 bit with 4:2:2 and 4:4:4 chroma"""
    p = hl.picture(80 + cfmt, 12, cfmt, 704, 576, 5, cip=True, tiles=(3, 2), nslices=3)
    assert same(on_device(dev, p), hl.orc_picture(p))


def many_ops_case():
    """a 4096x1440 4:4:4 picture of 4x4 TUs in raster order, luma, Cb and Cr at each position (1,105,920 ops > 2^20): left, up-left
    and up neighbours where they lie in the picture, every third TU with a DC residual from one shared block"""
    p = hl.picture(1, 8, 3, 32, 32, 4)                          # a template for the fields; its TUs are replaced
    W, H = 4096, 1440
    p.W, p.H = W, H
    rng = np.random.default_rng(9)
    ys, xs = np.meshgrid(np.arange(0, H, 4), np.arange(0, W, 4), indexing="ij")
    n = xs.size
    ops = np.zeros(3 * n, hl.RECON_DTYPE)
    for c in range(3):
        o = ops[c::3]
        o["x"], o["y"], o["plane"], o["log2_size"] = xs.ravel(), ys.ravel(), c, 2
        o["mode"] = rng.integers(0, 35, n)
        f = np.where(xs.ravel() > 0, hl.INTRA_CAND_L, 0) | np.where(ys.ravel() > 0, hl.INTRA_CAND_U, 0)
        f |= np.where((xs.ravel() > 0) & (ys.ravel() > 0), hl.INTRA_CAND_UL, 0)
        o["flags"] = f | (hl.INTRA_LUMA if c == 0 else 0)
        o["tu_kind"] = np.where(np.arange(n) % 3 == 0, 1, hl.TU_NONE)
    p.ops = ops
    p.coef = np.zeros(16, np.int16)
    p.coef[0] = 300
    import hevcpredlib as hp
    p.frames = [hl._frame(hp.content(rng, 8, H, W), 8) for _ in range(3)]
    p.map = None
    return p


def test_more_than_2_20_ops(dev):
    p = many_ops_case()
    assert len(p.ops) > 1 << 20
    assert same(on_device(dev, p), hl.orc_picture(p))


def test_invalid_ops(dev):
    """invalid ops mixed into a picture write nothing and hold up no later op"""
    import test_hevc_intra_recon as cpu
    p = hl.fixture_case("420-8")
    bad = cpu.bad_ops(p)
    mixed = np.insert(p.ops, np.sort(np.random.default_rng(4).integers(0, len(p.ops), len(bad))), bad)
    assert same(on_device(dev, p, mixed), hl.orc_picture(p))
    assert same(on_device(dev, p, bad), p.framed())


def test_refusals(dev):
    """B200_EINVAL cases launch nothing and write nothing on the device"""
    import ffmpeg_b200 as fb
    import torch
    L = fb.lib()
    buf = torch.zeros(1 << 16, dtype=torch.uint8, device="cuda")
    p = buf.data_ptr()
    before = fb.launch_count()

    def call(depth=8, cf=1, w=64, h=64, planes=(p, p + 8192, p + 12288), ls_y=64, ls_uv=32, nops=1, ops=p + 16384, coef=p + 32768):
        arr = (C.c_void_p * 3)(*planes)
        return L.b200_hevc_intra_recon_picture_device(dev.handle, depth, cf, w, h, arr, ls_y, ls_uv, nops, ops, coef, None, 0, 2)
    assert call(depth=11) == EINVAL and call(cf=4) == EINVAL and call(w=0) == EINVAL and call(nops=-1) == EINVAL
    assert call(ls_y=60) == EINVAL and call(ops=p + 16392) == EINVAL and call(coef=None) == EINVAL and call(planes=(p, None, p)) == EINVAL
    assert call(nops=0) == 0
    dev.sync()
    assert fb.launch_count() == before and not buf.any().item()


def smoke(dev):
    """one small 4:2:0 picture at 8 and 10 bit against the checker"""
    for depth in (8, 10):
        p = hl.picture(3 + depth, depth, 1, 96, 64, 5, nslices=2)
        assert same(on_device(dev, p), hl.orc_picture(p)), ("hevc intra picture mismatch", depth)
    from ffmpeg_b200 import hevcdsp
    assert hevcdsp.hevc_intra_timeouts(dev) == 0
