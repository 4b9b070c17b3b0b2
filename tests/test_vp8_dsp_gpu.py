"""GPU tier for VP8 / VP7 motion compensation and residual (ffmpeg_b200/csrc/vp8mc.cu, vp8idct.cu) on the H100: both frame entries
against the reference's fixture hashes and the checker, seeded 1920x1088 and 3840x2160 frames with epel and bilinear prediction and
the VP7 and VP8 residual, one call of more ops than one launch takes, every drop-in member through host pointers, and the refusals.
Only committed fixtures and the checker are read."""
import ctypes as C

import numpy as np
import pytest

import cpulibs as cl
import vp8dsplib as v8

pytestmark = pytest.mark.gpu
EINVAL = -22


@pytest.fixture(scope="module")
def dev():
    import ffmpeg_b200 as fb
    d = fb.Device(0)
    d.set_default()
    yield d


def _t(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def mc_on_device(dev, bilinear, mbw, mbh, refs, ops, dst):
    """one MC frame call on device copies; returns the three planes as numpy"""
    import torch
    from ffmpeg_b200 import vp8dsp
    with torch.cuda.stream(torch.cuda.ExternalStream(dev.stream)):
        drefs = [tuple(_t(p) for p in r) for r in refs]
        dd, do = [_t(p) for p in dst], _t(ops.view(np.uint8))
        vp8dsp.vp8_mc_frame_device(dev, bilinear, mbw, mbh, [(y, u, v, r[0].strides[0], r[1].strides[0]) for (y, u, v), r in zip(drefs, refs)],
                                   len(ops), do, dd, dst[0].strides[0], dst[1].strides[0])
        dev.sync()
        return [d.cpu().numpy() for d in dd]


def residual_on_device(dev, is_vp7, ops, coef, dst):
    import torch
    from ffmpeg_b200 import vp8dsp
    with torch.cuda.stream(torch.cuda.ExternalStream(dev.stream)):
        dd, do, dc = [_t(p) for p in dst], _t(ops.view(np.uint8)), _t(coef)
        vp8dsp.vp8_residual_frame_device(dev, is_vp7, len(ops), do, dc, dd, dst[0].strides[0], dst[1].strides[0])
        dev.sync()
        return [d.cpu().numpy() for d in dd]


def same(a, b):
    return all(np.array_equal(x, y) for x, y in zip(a, b))


@pytest.mark.parametrize("is_vp7,bilinear", v8.FIXTURE_CASES, ids=("vp8-epel", "vp8-bilinear", "vp7-epel", "vp7-bilinear"))
def test_fixture_frames(dev, is_vp7, bilinear):
    """MC then residual on the fixture frames: the reference's planes bit for bit, sentinels included"""
    refs, ops, dst, rops, coef = v8.fixture_case(is_vp7, bilinear)
    mc = mc_on_device(dev, bilinear, 12, 9, refs, ops, dst)
    assert same(mc, v8.orc_mc_frame(bilinear, 12, 9, refs, ops, dst))
    got = residual_on_device(dev, is_vp7, rops, coef, mc)
    assert v8.digest(got) == v8.fixture_hashes()[(is_vp7, bilinear)]


@pytest.mark.parametrize("size", ((120, 68), (240, 135)), ids=("1920x1088", "3840x2160"))
@pytest.mark.parametrize("is_vp7,bilinear", ((0, 0), (0, 1), (1, 0)), ids=("vp8-epel", "vp8-bilinear", "vp7-epel"))
def test_seeded_frames(dev, size, is_vp7, bilinear):
    """a whole inter frame (every partitioning, windows up to 80 samples outside) and its residual (decoder-shaped coefficients)"""
    mbw, mbh = size
    seed = 1000 + mbw + 2 * is_vp7 + bilinear
    refs, ops, dst = v8.mc_case(seed, mbw, mbh, intra=0.02)
    mc = mc_on_device(dev, bilinear, mbw, mbh, refs, ops, dst)
    exp = v8.orc_mc_frame(bilinear, mbw, mbh, refs, ops, dst)
    assert same(mc, exp)
    rops, coef = v8.residual_case(seed + 1, mbw, mbh, is_vp7)
    assert same(residual_on_device(dev, is_vp7, rops, coef, mc), v8.orc_residual_frame(is_vp7, rops, coef, exp))


@pytest.mark.parametrize("is_vp7", (0, 1), ids=("vp8", "vp7"))
@pytest.mark.parametrize("kind", ("dense", "extreme"))
def test_residual_arbitrary_coefficients(dev, is_vp7, kind):
    rng = np.random.default_rng(7 + is_vp7)
    ops, coef = v8.residual_case(20 + is_vp7 + len(kind), 40, 30, is_vp7, kind)
    dst = [rng.integers(0, 256, p.shape).astype(np.uint8) for p in v8.dst_planes(40, 30)]
    assert same(residual_on_device(dev, is_vp7, ops, coef, dst), v8.orc_residual_frame(is_vp7, ops, coef, dst))


def test_more_ops_than_one_launch(dev):
    """2^20 + 4099 ops in one call of each entry (more than one launch's 2^20): MC 4x4 luma blocks tiling a 4096 x 4128 plane; residual
    ops of which every 257th and the last 4099 have coefficients (the others write nothing), every block against the checker"""
    n = (1 << 20) + 4099
    rng = np.random.default_rng(5)
    mbw, mbh = 256, 258
    refs = v8.ref_frames(rng, mbw, mbh, 2)
    ops = np.zeros(n, v8.MC_DTYPE)
    i = np.arange(n)
    ops["dst_x"], ops["dst_y"] = (i % 1024) * 4, (i // 1024) * 4
    ops["plane"], ops["w"], ops["h"], ops["ref"] = 0, 4, 4, i % 2
    ops["src_x"], ops["src_y"] = ops["dst_x"] + rng.integers(-20, 21, n), ops["dst_y"] + rng.integers(-20, 21, n)
    ops["mx"], ops["my"] = rng.integers(0, 8, n), rng.integers(0, 8, n)
    dst = v8.dst_planes(mbw, mbh)
    got = mc_on_device(dev, 0, mbw, mbh, refs, ops, dst)
    assert same(got, v8.orc_mc_frame(0, mbw, mbh, refs, ops, dst))
    rops = np.zeros(n, v8.RES_DTYPE)
    active = np.flatnonzero((i % 257 == 0) | (i >= 1 << 20))
    rops["mb_x"][active], rops["mb_y"][active] = np.arange(len(active)) % 128, np.arange(len(active)) // 128
    rops["coef_off"] = (i % 64) * v8.MB_COEFS
    rops["nnz"][active] = rng.integers(0, 3, (len(active), 6, 4))
    rops["flags"], rops["y2_nnz"] = 1, i % 3
    coef = rng.integers(-600, 601, 64 * v8.MB_COEFS).astype(np.int16)
    rdst = [rng.integers(0, 256, p.shape).astype(np.uint8) for p in v8.dst_planes(128, 65)]
    assert same(residual_on_device(dev, 0, rops, coef, rdst), v8.orc_residual_frame(0, rops, coef, rdst))


def run_ctx_mc(ctx, call, pic, dst0):
    """one call through put_vp8_{epel,bilinear}_pixels_tab[size][v][h], HOST pointers, the reference's argument order"""
    bilinear, w, v, h, hh, mx, my = call
    d = dst0.copy()
    src = pic.ctypes.data + v8.MARGIN * pic.strides[0] + v8.MARGIN
    tab = ctx.put_vp8_bilinear_pixels_tab if bilinear else ctx.put_vp8_epel_pixels_tab
    tab[v8.WIDTHS.index(w)][v][h](d.ctypes.data, d.strides[0], src, pic.strides[0], hh, mx, my)
    return d


def check_mc_members(ctx, bilinear, seed, cls, stride=1):
    """every stride-th call of mc_calls through the context's members against the checker"""
    O = cl.oracle()
    pic, dst0 = v8.member_case(seed, cls)
    for call in list(v8.mc_calls(seed, bilinear))[::stride]:
        assert np.array_equal(run_ctx_mc(ctx, call, pic, dst0), v8.run_mc(O, "orc_vp8_mc", call, pic, dst0)), call


def check_residual_members(ctx, is_vp7, seed):
    """every residual member on decoder-shaped, dense and int16-extreme blocks against the checker, coefficients written back included"""
    O = cl.oracle()
    rng = np.random.default_rng(seed)
    for kind in ("decoder", "dense", "extreme"):
        for dc_only in (0, 1):
            for _ in range(6):
                dc = v8.coef_blocks(rng, 1, kind)[0]
                block = (np.arange(256, dtype=np.int64) * 37 % 2001 - 1000).astype(np.int16).reshape(4, 4, 16)
                d = dc.copy()
                (ctx.vp8_luma_dc_wht_dc if dc_only else ctx.vp8_luma_dc_wht)(block.ctypes.data, d.ctypes.data)
                eb, ed = v8.run_wht(O, "orc_vp8_wht", is_vp7, dc_only, dc)
                assert np.array_equal(block, eb) and np.array_equal(d, ed), (kind, dc_only)
        members = (ctx.vp8_idct_add, ctx.vp8_idct_dc_add, ctx.vp8_idct_dc_add4y, ctx.vp8_idct_dc_add4uv)
        for which, nb in ((0, 1), (1, 1), (2, 4), (3, 4)):
            for _ in range(6):
                blocks = v8.coef_blocks(rng, nb, kind)
                dst0 = rng.integers(0, 256, (8, 16)).astype(np.uint8)
                d, b = dst0.copy(), blocks.copy()
                members[which](d.ctypes.data, b.ctypes.data, d.strides[0])
                ed, eb = v8.run_idct(O, "orc_vp8_idct", is_vp7, which, blocks, dst0)
                assert np.array_equal(d, ed) and np.array_equal(b, eb), (kind, which)


@pytest.mark.parametrize("is_vp7", (0, 1), ids=("vp8", "vp7"))
def test_dropin_members(dev, is_vp7):
    """VP8DSPContext from ff_vp8dsp_init through the library: every MC entry of both tables at every phase (a third of the calls on the
    extremes picture), every residual member"""
    from ffmpeg_b200 import vp8dsp
    ctx = vp8dsp.ff_vp8dsp_init(is_vp7)
    for bil in (0, 1):
        check_mc_members(ctx, bil, 60 + is_vp7 + 2 * bil, 0)
        check_mc_members(ctx, bil, 64 + is_vp7 + 2 * bil, 1, stride=3)
    check_residual_members(ctx, is_vp7, 68 + is_vp7)


def test_member_out_of_domain_writes_nothing(dev):
    from ffmpeg_b200 import vp8dsp
    import ffmpeg_b200 as fb
    ctx = vp8dsp.ff_vp8dsp_init(0)
    pic, dst0 = v8.member_case(1, 0)
    for call in ((0, 8, 2, 2, 0, 3, 3), (0, 8, 2, 2, 17, 3, 3), (0, 8, 2, 0, 8, 3, 0), (0, 4, 1, 1, 4, 8, 3), (1, 4, 1, 1, 4, 8, 3),
                 (0, 8, 0, 2, 4, 0, 1)):
        assert np.array_equal(run_ctx_mc(ctx, call, pic, dst0), dst0), call
        assert b"vp8 mc member" in fb.lib().b200_last_error()


def test_refusals(dev):
    """the B200_EINVAL cases of both entries launch nothing; the init entry's EINVAL"""
    import torch
    import ffmpeg_b200 as fb
    from ffmpeg_b200._lib import VP8DSPContext, Vp8McRef
    L = fb.lib()
    buf = torch.zeros(1 << 16, dtype=torch.uint8, device="cuda")
    p = buf.data_ptr()
    ops = np.zeros(1, v8.MC_DTYPE)
    ops["w"] = ops["h"] = 4
    dops = _t(ops.view(np.uint8))
    before = fb.launch_count()

    def mc(nrefs=1, n=1, o=dops.data_ptr(), planes=(p + 1024, p + 4096, p + 8192), ls_y=64, mbw=2):
        arr = (Vp8McRef * 3)(*[Vp8McRef(p + 16384, p + 20480, p + 24576, 64, 32)] * 3)
        return L.b200_vp8_mc_frame_device(dev.handle, 0, mbw, 2, nrefs, C.cast(arr, C.c_void_p), n, o, (C.c_void_p * 3)(*planes), ls_y, 32)
    assert mc(n=0) == 0
    assert mc(n=-1) == EINVAL and mc(nrefs=0) == EINVAL and mc(nrefs=4) == EINVAL and mc(mbw=0) == EINVAL
    assert mc(o=None) == EINVAL and mc(o=dops.data_ptr() + 2) == EINVAL and mc(ls_y=66) == EINVAL
    assert mc(planes=(p + 1024, 0, p + 8192)) == EINVAL and mc(planes=(p + 1025, p + 4096, p + 8192)) == EINVAL

    def res(v7=0, n=1, coef=p + 32768, ls_y=64):
        return L.b200_vp8_residual_frame_device(dev.handle, v7, n, dops.data_ptr(), coef, (C.c_void_p * 3)(p + 1024, p + 4096, p + 8192), ls_y, 32)
    assert res(n=0) == 0
    assert res(n=-1) == EINVAL and res(v7=2) == EINVAL and res(coef=None) == EINVAL and res(coef=p + 32770) == EINVAL and res(ls_y=2) == EINVAL
    dev.sync()
    assert fb.launch_count() == before and not buf.any().item()
    ctx = VP8DSPContext()
    assert L.b200_vp8_dsp_init(C.byref(ctx), 2) == EINVAL and L.b200_vp8_dsp_init(None, 0) == EINVAL


def smoke(dev):
    """smoke(): one small VP8 epel and one VP7 bilinear frame through both entries, bit-compared with the checker"""
    for is_vp7, bil in ((0, 0), (1, 1)):
        refs, ops, dst = v8.mc_case(31 + is_vp7, 6, 4)
        mc = mc_on_device(dev, bil, 6, 4, refs, ops, dst)
        exp = v8.orc_mc_frame(bil, 6, 4, refs, ops, dst)
        assert same(mc, exp), ("vp8 mc mismatch", is_vp7, bil)
        rops, coef = v8.residual_case(33 + is_vp7, 6, 4, is_vp7)
        assert same(residual_on_device(dev, is_vp7, rops, coef, mc), v8.orc_residual_frame(is_vp7, rops, coef, exp)), ("vp8 residual mismatch", is_vp7)
