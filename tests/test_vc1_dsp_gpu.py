"""GPU tier for VC-1 motion compensation and inverse transforms (ffmpeg_b200/csrc/vc1mc.cu, vc1idct.cu) on the H100: both frame entries
against the reference's fixture hashes and the checker, seeded 1920x1088 and 3840x2160 P and B pictures (mspel and hpel, rnd 0 / 1, range
reduction and IC), arbitrary int16 coefficients, one call of more ops than one launch takes, every drop-in member through host pointers,
and the refusals.  Only committed fixtures and the checker are read."""
import ctypes as C

import numpy as np
import pytest

import cpulibs as cl
import vc1dsplib as v1

pytestmark = pytest.mark.gpu
EINVAL, ENOSYS = -22, -38


@pytest.fixture(scope="module")
def dev():
    import ffmpeg_b200 as fb
    d = fb.Device(0)
    d.set_default()
    yield d


def _t(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def same(a, b):
    return len(a) == len(b) and all(np.array_equal(x, y) for x, y in zip(a, b))


def mc_on_device(dev, mbw, mbh, H, V, refs, ops, dst):
    """one MC call on device copies of the reference buffers (poison included) and dst; returns the three planes as numpy"""
    import torch
    from ffmpeg_b200 import vc1dsp
    with torch.cuda.stream(torch.cuda.ExternalStream(dev.stream)):
        bufs = [[_t(p) for p in r.planes] for r in refs]
        descs = [r.desc([int(b.data_ptr()) for b in bb]) for r, bb in zip(refs, bufs)]
        dd, do = [_t(p) for p in dst], _t(np.ascontiguousarray(ops).view(np.uint8))
        vc1dsp.vc1_mc_frame_device(dev, descs, dd, dst[0].strides[0], dst[1].strides[0], mbw, mbh, H, V, len(ops), do)
        dev.sync()
        return [d.cpu().numpy() for d in dd]


def residual_on_device(dev, mbw, mbh, ops, coef, dst):
    import torch
    from ffmpeg_b200 import vc1dsp
    with torch.cuda.stream(torch.cuda.ExternalStream(dev.stream)):
        dd, do, dc = [_t(p) for p in dst], _t(np.ascontiguousarray(ops).view(np.uint8)), _t(coef)
        vc1dsp.vc1_residual_frame_device(dev, dd, dst[0].strides[0], dst[1].strides[0], mbw, mbh, dc, len(ops), do)
        dev.sync()
        return [d.cpu().numpy() for d in dd]


@pytest.mark.parametrize("name", [c[0] for c in v1.FIXTURE_CASES])
def test_fixture_frames(dev, name):
    """MC then residual on the fixture pictures: the reference's planes bit for bit, sentinels included"""
    mbw, mbh, H, V, refs, ops, dst, rops, coef = v1.fixture_case(name)
    mc = mc_on_device(dev, mbw, mbh, H, V, refs, ops, dst)
    assert same(mc, v1.orc_mc_frame(mbw, mbh, H, V, refs, ops, dst))
    got = residual_on_device(dev, mbw, mbh, rops, coef, mc)
    assert v1.digest(got) == v1.fixture_hashes()[name]


@pytest.mark.parametrize("w,h", ((1920, 1088), (3840, 2160)))
@pytest.mark.parametrize("b_frame,mspel,rnd,rr,ic", ((False, 1, 0, (0, 0), (0, 0)), (False, 0, 1, (1, 0), (0, 0)), (False, 1, 1, (0, 0), (1, 0)),
                                                    (True, 1, 0, (0, 0), (0, 1)), (True, 0, 1, (1, 1), (1, 1))),
                         ids=("p-mspel", "p-hpel-rr", "p-mspel-ic", "b-mspel-ic", "b-hpel-rr-ic"))
def test_large_frames(dev, w, h, b_frame, mspel, rnd, rr, ic):
    """seeded full-size pictures through both entries against the checker (2160 rows: the MB grid has 2160 / 16 = 135 rows exactly)"""
    mbw, mbh = w // 16, -(-h // 16)
    seed = w + h + 2 * mspel + rnd + 10 * b_frame
    refs, ops, dst, H, V = v1.mc_case(seed, mbw, mbh, w - 2, h - 4, b_frame, mspel, rnd, rr, ic)
    mc = mc_on_device(dev, mbw, mbh, H, V, refs, ops, dst)
    exp = v1.orc_mc_frame(mbw, mbh, H, V, refs, ops, dst)
    assert same(mc, exp)
    rops, coef = v1.residual_case(seed + 1, mbw, mbh, "decoder")
    assert same(residual_on_device(dev, mbw, mbh, rops, coef, mc), v1.orc_residual_frame(mbw, mbh, rops, coef, exp))


@pytest.mark.parametrize("kind", ("dense", "extreme"))
def test_arbitrary_coefficients(dev, kind):
    rng = np.random.default_rng(80 + len(kind))
    rops, coef = v1.residual_case(81 + len(kind), 40, 30, kind, skip=0.0)
    dst = [rng.integers(0, 256, p.shape).astype(np.uint8) for p in v1.dst_planes(40, 30)]
    assert same(residual_on_device(dev, 40, 30, rops, coef, dst), v1.orc_residual_frame(40, 30, rops, coef, dst))


def test_more_ops_than_one_launch(dev):
    """over 2^20 MC ops and 2^22 residual ops in one call each; the MC ops are one P picture's repeated, which write the same values"""
    refs, ops, dst, H, V = v1.mc_case(90, 8, 6)
    reps = (1 << 20) // len(ops) + 2
    big = np.tile(ops, reps)
    assert len(big) > 1 << 20
    assert same(mc_on_device(dev, 8, 6, H, V, refs, big, dst), v1.orc_mc_frame(8, 6, H, V, refs, ops, dst))
    rops, coef = v1.residual_case(91, 8, 6, "dense", skip=0.0)
    dst0 = [np.zeros_like(p) for p in dst]
    one = v1.orc_residual_frame(8, 6, rops, coef, dst0)
    # residual adds do not repeat idempotently: one copy of the ops, then ops the guard refuses (x beyond the grid) past 2^22
    pad = np.tile(rops[:1], (1 << 22) + 5 - len(rops))
    pad["x"] = 4096
    allops = np.concatenate([rops, pad])
    assert same(residual_on_device(dev, 8, 6, allops, coef, dst0), one)


def check_members(ctx, seed):
    """every mspel / chroma / transform member of ctx through host pointers against the checker"""
    from ffmpeg_b200._lib import VC1_MSPEL_FUNC, VC1_CHROMA_FUNC
    O = cl.oracle()
    pic, dst0 = v1.member_case(seed)
    stride = 40
    P = np.zeros((v1.MARGIN + 24, stride), np.uint8)
    P[:, :pic.shape[1]] = pic
    D0 = np.zeros((20, stride), np.uint8)
    D0[:, :20] = dst0
    src = P[v1.MARGIN:, v1.MARGIN:].ctypes.data
    mspel = v1._mspel_fn(O, "orc_vc1_mspel")
    for avg, size, dxy, rnd in v1.mspel_calls():
        d, e = D0.copy(), D0.copy()
        f = (ctx.avg_vc1_mspel_pixels_tab if avg else ctx.put_vc1_mspel_pixels_tab)[size][dxy]
        f(d.ctypes.data, src, stride, rnd)
        mspel(avg, size, dxy, e.ctypes.data, src, stride, rnd)
        assert np.array_equal(d, e), (avg, size, dxy, rnd)
    chroma = v1._chroma_fn(O, "orc_vc1_chroma")
    for avg, idx, h, x, y in v1.chroma_calls():
        d, e = D0.copy(), D0.copy()
        f = (ctx.avg_no_rnd_vc1_chroma_pixels_tab if avg else ctx.put_no_rnd_vc1_chroma_pixels_tab)[idx]
        f(d.ctypes.data, src, stride, h, x, y)
        chroma(avg, idx, e.ctypes.data, src, stride, h, x, y)
        assert np.array_equal(d, e), (avg, idx, h, x, y)
    for bad in ((8, 8, 3), (8, 3, -1), (-1, 0, 0), (4097, 0, 0)):
        d = D0.copy()
        ctx.put_no_rnd_vc1_chroma_pixels_tab[0](d.ctypes.data, src, stride, *bad)
        assert np.array_equal(d, D0), bad
    itx = v1._itx_fn(O, "orc_vc1_itx")
    rng = np.random.default_rng(seed)
    names = ("8x8", "8x4", "4x8", "4x4")
    for kind in ("decoder", "extreme"):
        for b in v1.coef_blocks(rng, 6, kind):
            for tt in range(4):
                for dc in (0, 1):
                    blk, eb = b.copy(), b.copy()
                    dest = rng.integers(0, 256, (8, 16)).astype(np.uint8)
                    ed = dest.copy()
                    if tt == 0 and not dc:
                        ctx.vc1_inv_trans_8x8(blk.ctypes.data)
                    else:
                        getattr(ctx, f"vc1_inv_trans_{names[tt]}{'_dc' if dc else ''}")(dest.ctypes.data, dest.strides[0], blk.ctypes.data)
                    itx(tt, dc, ed.ctypes.data, ed.strides[0], eb.ctypes.data)
                    assert np.array_equal(blk, eb) and np.array_equal(dest, ed), (kind, tt, dc)


def test_dropin_members(dev):
    from ffmpeg_b200 import vc1dsp
    check_members(vc1dsp.ff_vc1dsp_init(), 70)


def test_refusals_launch_nothing(dev):
    """interlaced references and an out-of-range nrefs are refused before any launch on the real device too"""
    import ffmpeg_b200 as fb
    from ffmpeg_b200._lib import Vc1McRef
    L = fb.lib()
    refs, ops, dst, H, V = v1.mc_case(95, 2, 2)
    before = fb.launch_count()
    for il, n in ((1, 1), (0, 3)):
        arr = (Vc1McRef * 3)(*[Vc1McRef(1 << 20, 1 << 20, 1 << 20, 64, 32, 0, 0, il, 0)] * 3)
        planes = (C.c_void_p * 3)(1 << 20, 1 << 20, 1 << 20)
        assert L.b200_vc1_mc_frame_device(None, n, C.cast(arr, C.c_void_p), planes, 64, 32, 2, 2, H, V, 1, 1 << 20) == (ENOSYS if il else EINVAL)
    assert fb.launch_count() == before


def smoke(dev):
    """smoke(): a small P picture (4MV, mspel, IC) and a B picture (hpel, range reduction) through both entries, bit-compared with
    the checker"""
    for k, (b, ms, rnd, rr, ic) in enumerate(((False, 1, 1, (0, 0), (1, 0)), (True, 0, 0, (1, 0), (0, 1)))):
        refs, ops, dst, H, V = v1.mc_case(31 + k, 5, 4, None, None, b, ms, rnd, rr, ic)
        mc = mc_on_device(dev, 5, 4, H, V, refs, ops, dst)
        exp = v1.orc_mc_frame(5, 4, H, V, refs, ops, dst)
        assert same(mc, exp), ("vc1 mc mismatch", k)
        rops, coef = v1.residual_case(33 + k, 5, 4, "extreme")
        assert same(residual_on_device(dev, 5, 4, rops, coef, mc), v1.orc_residual_frame(5, 4, rops, coef, exp)), ("vc1 residual mismatch", k)


def test_smoke(dev):
    smoke(dev)
