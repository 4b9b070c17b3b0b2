"""GPU tier for HEVC intra prediction (ffmpeg_b200/csrc/hevcpred.cu) on the H100: whole planes through the level wavefront
(b200_hevc_intra_pred_batch_device, then a BYPASS b200_hevc_transform_add_batch_device call for the same TUs, per level) against the
fixture hashes of the reference's planes and against the checker (oracle/hevcpred_oracle.c) on seeded pictures, for luma and 4:2:0 /
4:2:2 / 4:4:4 chroma with constrained intra prediction off and on; the strong-smoothing decision at its threshold; every member of
the context at every depth against the checker and the stored reference digests; out-of-range and out-of-plane ops; one call whose
ops lie beyond 2^31 bytes.  Only committed fixtures and the checker are read."""
import numpy as np
import pytest

import hevcpredlib as hl

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


def on_device(dev, p):
    """the component through the wavefront on the device (one prediction call and one residual-add call per level); returns the framed
    plane as numpy and the number of levels"""
    import torch
    from ffmpeg_b200 import hevcdsp
    buf = hl.framed(p.plane, p.depth)
    off = hl.MARGIN * buf.strides[0] + hl.MARGIN * buf.itemsize
    coef, base = hl.packed_residuals(p)
    nl = int(p.levels.max()) + 1
    st = torch.cuda.ExternalStream(dev.stream)
    with torch.cuda.stream(st):
        dbuf, dcoef = _t(buf), _t(coef)
        dmap = None if p.map is None else _t(p.map)
        pix = dbuf.data_ptr() + off
        for lv in range(nl):
            sel = np.nonzero(p.levels == lv)[0]
            dops = _t(np.ascontiguousarray(p.ops[sel]).view(np.uint8))
            hevcdsp.hevc_intra_pred_batch_device(dev, p.depth, pix, buf.strides[0], p.W, p.H, p.hs, p.vs, len(sel), dops, dmap,
                                                 0 if p.map is None else p.map.strides[0], p.log2_min_pu)
            dtu = _t(hl.tu_ops(p, sel, buf.strides[0], base).view(np.uint8))
            hevcdsp.hevc_transform_add_batch_device(dev, p.depth, len(sel), dtu, dcoef, pix, buf.strides[0])
        dev.sync()
        return dbuf.cpu().numpy().view(buf.dtype), nl


@pytest.mark.parametrize("depth", hl.DEPTHS)
def test_planes_vs_fixture(dev, depth):
    """luma and every chroma format, CIP off and on: the reference's plane bit for bit, guard samples included"""
    hs = hl.fixture_hashes()
    for name in hl.FIXTURE_CFMT:
        for cip in (False, True):
            got, nl = on_device(dev, hl.fixture_case(depth, name, cip))
            assert nl > 1 and hl.digest(got) == hs[(depth, hl.fixture_key(name, cip))], (name, cip)


@pytest.mark.parametrize("cip", (False, True), ids=("nocip", "cip"))
@pytest.mark.parametrize("name", ("luma", "420", "422", "444"))
def test_planes_vs_checker(dev, name, cip):
    """seeded pictures at every depth (CTB 16 / 32 / 64, slices, tiles, smoothing on and off, 4 seeds each), a 1920x1080 one at 8 and
    10 bit: the checker's plane bit for bit, guard samples included"""
    cfmt, comp = hl.FIXTURE_CFMT[name]
    shapes = [(200, 136, 4, dict(nslices=3)), (232, 120, 5, dict(tiles=(2, 2), nslices=2)), (200, 136, 6, dict(nslices=2, smoothing=False)),
              (136, 72, 5, dict(strong=False, tiles=(2, 1)))]
    for depth in hl.DEPTHS:
        for k, (W, H, l2, kw) in enumerate(shapes):
            p = hl.picture_case(20000 + 100 * depth + 10 * k + 2 * cfmt + int(cip), depth, W, H, l2, cfmt, comp, cip=cip, **kw)
            assert np.array_equal(on_device(dev, p)[0], hl.orc_plane(p)), (depth, k)
    for depth in (8, 10):
        p = hl.picture_case(31 + depth + cfmt, depth, 1920, 1080, 6, cfmt, comp, cip=cip, tiles=(3, 2), nslices=4)
        assert np.array_equal(on_device(dev, p)[0], hl.orc_plane(p)), depth


@pytest.mark.parametrize("depth", hl.DEPTHS)
def test_strong_threshold(dev, depth):
    """32x32 luma blocks whose strong-smoothing second differences lie at t - 1 and t on either side: the checker and the reference"""
    p = hl.strong_case(40 + depth, depth)
    got = on_device(dev, p)[0]
    assert np.array_equal(got, hl.orc_plane(p))
    assert hl.digest_like_refcheck([got]) == hl.stored_digest(f"test_hevc_pred.py::test_emu_strong_threshold[{depth}]#0")


@pytest.mark.parametrize("depth", hl.DEPTHS)
def test_members_vs_checker(dev, depth):
    """every prediction member at every size x mode x luma / chroma on other seeds, and both filters: the checker"""
    from ffmpeg_b200 import hevcdsp
    ctx = hevcdsp.ff_hevc_pred_init(depth)
    for c in hl.member_cases(1700 + depth, depth):
        assert np.array_equal(hl.ctx_member(ctx, depth, c), hl.orc_member(depth, c)), c[:4]
    for k, c in enumerate(hl.filter_cases(1800 + depth, depth)):
        assert all(np.array_equal(a, b) for a, b in zip(hl.ctx_filters(ctx, depth, c, k % 3), hl.orc_filters(depth, c))), c[0]


@pytest.mark.parametrize("depth", hl.DEPTHS)
def test_members_vs_reference(dev, depth):
    """every prediction member at every size x mode x luma / chroma, and both filters: the stored reference digests"""
    from ffmpeg_b200 import hevcdsp
    ctx = hevcdsp.ff_hevc_pred_init(depth)
    ours = [hl.ctx_member(ctx, depth, c) for c in hl.member_cases(700 + depth, depth)]
    assert hl.digest_like_refcheck(ours) == hl.stored_digest(f"test_hevc_pred.py::test_emu_every_member[{depth}]#0")
    ours = [a for k, c in enumerate(hl.filter_cases(800 + depth, depth)) for a in hl.ctx_filters(ctx, depth, c, k % 3)]
    assert hl.digest_like_refcheck(ours) == hl.stored_digest(f"test_hevc_pred.py::test_emu_every_member[{depth}]#1")


def test_out_of_range_ops_change_nothing(dev):
    import torch
    from ffmpeg_b200 import hevcdsp
    p = hl.picture_case(3, 10, 64, 64, 5, 0, 0)
    buf = hl.framed(p.plane, 10)
    bad = np.zeros(9, hl.INTRA_DTYPE)
    bad[:] = [(0, 0, 1, 0, 0, (0,) * 4), (0, 0, 6, 0, 0, (0,) * 4), (8, 8, 2, 35, 0, (0,) * 4), (-4, 0, 2, 0, 0, (0,) * 4),
              (0, -4, 2, 0, 0, (0,) * 4), (60, 0, 3, 0, 0, (0,) * 4), (0, 60, 3, 0, 0, (0,) * 4),
              (0, 8, 2, 0, hl.INTRA_CAND_L, (0,) * 4), (8, 0, 2, 0, hl.INTRA_CAND_U, (0,) * 4)]
    st = torch.cuda.ExternalStream(dev.stream)
    with torch.cuda.stream(st):
        d, o = _t(buf), _t(bad.view(np.uint8))
        off = hl.MARGIN * buf.strides[0] + hl.MARGIN * 2
        hevcdsp.hevc_intra_pred_batch_device(dev, 10, d.data_ptr() + off, buf.strides[0], 64, 64, 0, 0, len(bad), o)
        dev.sync()
        assert np.array_equal(d.cpu().numpy().view(np.uint16), buf)


def test_ops_beyond_2g(dev):
    """one call on an 8-bit plane of 65536-byte rows x 40000 rows (2.6 GB): 35 ops near the bottom (every mode, all neighbours,
    smoothing), equal to the same ops on a small copy of their neighbourhood"""
    import torch
    from ffmpeg_b200 import hevcdsp
    W, H, S = 4096, 40000, 65536
    rng = np.random.default_rng(5)
    small = rng.integers(0, 256, (80, W)).astype(np.uint8)
    ops = np.zeros(35, hl.INTRA_DTYPE)                      # 32x32 luma blocks 96 samples apart: independent
    for m in range(35):
        ops[m] = (8 + 96 * m, 8, 5, m, 0x7F, (0,) * 4)
    y0 = H - 80
    st = torch.cuda.ExternalStream(dev.stream)
    with torch.cuda.stream(st):
        big = torch.zeros(H * S, dtype=torch.uint8, device="cuda")
        big.view(H, S)[y0:, :W] = torch.from_numpy(small).cuda()
        o = ops.copy()
        o["y"] += y0
        hevcdsp.hevc_intra_pred_batch_device(dev, 8, big, S, W, H, 0, 0, len(o), _t(o.view(np.uint8)))
        ref = _t(small)
        hevcdsp.hevc_intra_pred_batch_device(dev, 8, ref, W, W, 80, 0, 0, len(ops), _t(ops.view(np.uint8)))
        dev.sync()
        got = big.view(H, S)[y0:, :W].cpu().numpy()
        assert not np.array_equal(got, small) and np.array_equal(got, ref.cpu().numpy())
        del big
        torch.cuda.empty_cache()


def smoke(dev):
    """smoke(): the fixture's luma plane and its 4:2:0 chroma plane with CIP at 8 and 10 bit through the wavefront, against the
    fixture hashes of the reference's planes and the checker"""
    hs = hl.fixture_hashes()
    for depth in (8, 10):
        for name, cip in (("luma", False), ("420", True)):
            p = hl.fixture_case(depth, name, cip)
            got, _ = on_device(dev, p)
            assert hl.digest(got) == hs[(depth, hl.fixture_key(name, cip))], ("hevc intra mismatch", depth, name)
            assert np.array_equal(got, hl.orc_plane(p)), ("hevc intra mismatch with the checker", depth, name)
