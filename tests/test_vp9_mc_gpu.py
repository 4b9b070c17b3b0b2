"""GPU tier for VP9 motion compensation (ffmpeg_b200/csrc/vp9mc.cu) on the H100: b200_vp9_mc_batch_device against the checker and the
reference's fixture hashes at every depth for a luma-shaped and a 4:2:0-chroma-shaped plane, unscaled and scaled references, one
3840x2160 call of mixed block sizes and kinds, one call of more ops than one launch takes, compound ops whose two references differ in
size and step, every drop-in member of the mc / smc tables through host pointers, and the refusals.  Only committed fixtures and the
checker are read."""
import ctypes as C

import numpy as np
import pytest

import cpulibs as cl
import vp9mclib as vm

pytestmark = pytest.mark.gpu
EINVAL, ENOSYS = -22, -38


@pytest.fixture(scope="module")
def dev():
    import ffmpeg_b200 as fb
    d = fb.Device(0)
    d.set_default()
    yield d


def on_device(dev, depth, planes, steps, dst, ops):
    """one batched call on device copies; returns dst as numpy"""
    import torch
    from ffmpeg_b200 import vp9dsp
    st = torch.cuda.ExternalStream(dev.stream)
    with torch.cuda.stream(st):
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.int16) if a.dtype == np.uint16 else np.ascontiguousarray(a)).cuda()
        dp, dd, do = [t(p) for p in planes], t(dst), t(ops.view(np.uint8))
        refs = [(d, p.strides[0], p.shape[1], p.shape[0], dx, dy) for d, p, (dx, dy) in zip(dp, planes, steps)]
        vp9dsp.vp9_mc_batch_device(dev, depth, refs, len(ops), do, dd, dst.strides[0])
        dev.sync()
        return dd.cpu().numpy().view(dst.dtype)


@pytest.mark.parametrize("depth", vm.DEPTHS)
@pytest.mark.parametrize("chroma", (0, 1), ids=("luma", "chroma"))
def test_batch_vs_fixture(dev, depth, chroma):
    """the fixture batch (both kinds, every width and bank, eight references of different sizes and steps, edges, corners, windows wholly
    outside): the reference's destination picture bit for bit, sentinels around every block included"""
    case = vm.fixture_case(depth, chroma)
    got = on_device(dev, depth, *case)
    assert vm.digest(got) == vm.fixture_hashes()[(depth, bool(chroma))]
    assert np.array_equal(got, vm.orc_batch(depth, *case))


@pytest.mark.parametrize("depth", vm.DEPTHS)
@pytest.mark.parametrize("scaled", (False, True), ids=("unscaled", "scaled"))
@pytest.mark.parametrize("cls", (0, 1, 2, 3), ids=("noise", "zero", "max", "extremes"))
def test_batch_vs_checker(dev, depth, scaled, cls):
    case = vm.batch_case(2000 + 37 * depth + 5 * scaled + cls, 512, depth, cls=cls, scaled=scaled)
    assert np.array_equal(on_device(dev, depth, *case), vm.orc_batch(depth, *case))


def frame_case(seed, depth, W, H):
    """a W x H plane tiled with 8x8, 16x16, 32x32 and 64x64 blocks (64 x 64 superblocks, each split at random), every block an op of a
    seeded kind, bank and phases from two same-size references, motion within +-64 samples (so some windows leave the picture)"""
    rng = np.random.default_rng(seed)
    planes = [vm.picture(rng, H, W, depth, 0) for _ in range(2)]
    dst = np.zeros((H, W), vm.sdtype(depth))
    units = []

    def split(x, y, s):
        if s > 8 and rng.random() < 0.6:
            for dy in (0, s // 2):
                for dx in (0, s // 2):
                    split(x + dx, y + dy, s // 2)
        elif x + s <= W and y < H:
            units.append((x, y, s, min(s, H - y)))
    for y in range(0, H, 64):
        for x in range(0, W, 64):
            split(x, y, 64)
    ops = np.zeros(len(units), vm.OP_DTYPE)
    u = np.array(units)
    ops["dst_off"] = u[:, 1] * dst.strides[0] + u[:, 0] * dst.itemsize
    ops["w"], ops["h"] = u[:, 2], u[:, 3]
    ops["kind"] = rng.integers(0, 2, len(u))
    ops["filter"] = rng.integers(0, 4, len(u))
    for r in (0, 1):
        ops["ref"][:, r] = rng.integers(0, 2, len(u))
        ops["x"][:, r] = u[:, 0] + rng.integers(-64, 65, len(u))
        ops["y"][:, r] = u[:, 1] + rng.integers(-64, 65, len(u))
        ops["mx"][:, r] = rng.integers(0, 16, len(u)) * (rng.random(len(u)) < 0.8)
        ops["my"][:, r] = rng.integers(0, 16, len(u)) * (rng.random(len(u)) < 0.8)
    return planes, [(16, 16), (16, 16)], dst, ops


@pytest.mark.parametrize("depth,chroma", [(8, 0), (10, 0), (8, 1), (12, 1)], ids=("8-luma", "10-luma", "8-chroma", "12-chroma"))
def test_frame_3840x2160(dev, depth, chroma):
    W, H = (3840, 2160) if not chroma else (1920, 1080)
    case = frame_case(77 + depth + chroma, depth, W, H)
    got = on_device(dev, depth, *case)
    assert np.array_equal(got, vm.orc_batch(depth, *case))
    assert (got != 0).mean() > 0.5


def test_more_ops_than_one_launch(dev):
    """2^20 + 4099 ops of 4x2 (more than one launch's 2^20), a scaled reference among them: every block against the checker"""
    n, cols = (1 << 20) + 4099, 1024
    rng = np.random.default_rng(3)
    planes = [vm.picture(rng, 64, 96, 8, 0), vm.picture(rng, 64, 96, 8, 0), vm.picture(rng, 40, 120, 8, 0)]
    steps = [(16, 16), (16, 16), (20, 10)]
    dst = np.zeros(((n + cols - 1) // cols * 2, cols * 4), np.uint8)
    ops = np.zeros(n, vm.OP_DTYPE)
    i = np.arange(n)
    ops["dst_off"] = (i // cols) * 2 * dst.strides[0] + (i % cols) * 4
    ops["w"], ops["h"], ops["kind"], ops["filter"] = 4, 2, i % 2, (i // 2) % 4
    for r in (0, 1):
        ops["ref"][:, r] = rng.integers(0, 3, n)
        ops["x"][:, r] = rng.integers(-8, 100, n)
        ops["y"][:, r] = rng.integers(-8, 70, n)
        ops["mx"][:, r] = rng.integers(0, 16, n)
        ops["my"][:, r] = rng.integers(0, 16, n)
    got = on_device(dev, 8, planes, steps, dst, ops)
    assert np.array_equal(got, vm.orc_batch(8, planes, steps, dst, ops))


@pytest.mark.parametrize("depth", (8, 10))
def test_compound_references_of_different_size(dev, depth):
    """every compound op predicts from two references of different size and scale step (all ordered pairs of the eight in turn)"""
    planes, steps, dst, ops = vm.batch_case(41 + depth, 448, depth)
    ops["kind"] = vm.COMPOUND
    pairs = [(a, b) for a in range(8) for b in range(8) if a != b and (a > 1 or b > 1)]
    for k in range(len(ops)):
        ops["ref"][k] = pairs[k % len(pairs)]
    got = on_device(dev, depth, planes, steps, dst, ops)
    assert np.array_equal(got, vm.orc_batch(depth, planes, steps, dst, ops))
    assert not np.array_equal(got, dst)


def run_ctx_mc(ctx, call, pic, dst0):
    """one call through mc[size][bank][avg][h][v], HOST pointers, the reference's argument order"""
    w, bank, avg, hdir, vdir, h, mx, my = call
    d = dst0.copy()
    src = pic.ctypes.data + vm.MARGIN * pic.strides[0] + vm.MARGIN * pic.itemsize
    ctx.mc[vm.WIDTHS.index(w)][bank][avg][hdir][vdir](d.ctypes.data, d.strides[0], src, pic.strides[0], h, mx, my)
    return d


def run_ctx_smc(ctx, call, pic, dst0):
    w, bank, avg, h, mx, my, dx, dy = call
    d = dst0.copy()
    src = pic.ctypes.data + vm.MARGIN * pic.strides[0] + vm.MARGIN * pic.itemsize
    ctx.smc[vm.WIDTHS.index(w)][bank][avg](d.ctypes.data, d.strides[0], src, pic.strides[0], h, mx, my, dx, dy)
    return d


def check_members(ctx, depth, seed, cls, stride=1):
    """every stride-th call of mc_calls / smc_calls through the context's members against the checker"""
    O = cl.oracle()
    pic, dst0 = vm.member_case(seed, depth, cls, False)
    for call in list(vm.mc_calls(seed))[::stride]:
        assert np.array_equal(run_ctx_mc(ctx, call, pic, dst0), vm.run_mc(O, "orc_vp9_mc", depth, call, pic, dst0)), (depth, call)
    pic, dst0 = vm.member_case(seed, depth, cls, True)
    for call in list(vm.smc_calls(seed))[::stride]:
        assert np.array_equal(run_ctx_smc(ctx, call, pic, dst0), vm.run_smc(O, "orc_vp9_smc", depth, call, pic, dst0)), (depth, call)


@pytest.mark.parametrize("depth", vm.DEPTHS)
def test_dropin_members(dev, depth):
    """VP9DSPContext from ff_vp9dsp_init through the library: every mc and smc entry called with host pointers against the checker
    (every phase of every entry on noise; a fifth of the calls on each of the other content classes)"""
    from ffmpeg_b200 import vp9dsp
    ctx = vp9dsp.ff_vp9dsp_init(depth)
    check_members(ctx, depth, 60 + depth, 0)
    for cls in (1, 2, 3):
        check_members(ctx, depth, 60 + depth + cls, cls, stride=5)


def test_member_out_of_domain_writes_nothing(dev):
    from ffmpeg_b200 import vp9dsp
    import ffmpeg_b200 as fb
    ctx = vp9dsp.ff_vp9dsp_init(8)
    pic, dst0 = vm.member_case(1, 8, 0, True)
    for call in ((16, 1, 0, 1, 1, 0, 3, 3), (16, 1, 0, 1, 1, 65, 3, 3), (16, 1, 1, 1, 1, 8, 16, 3), (16, 1, 0, 1, 1, 8, 3, -1)):
        assert np.array_equal(run_ctx_mc(ctx, call, pic, dst0), dst0), call
        assert b"vp9 mc member" in fb.lib().b200_last_error()
    for call in ((16, 1, 0, 8, 3, 3, 0, 16), (16, 1, 1, 8, 3, 3, 16, 33), (8, 3, 0, 8, 3, 16, 16, 16)):
        assert np.array_equal(run_ctx_smc(ctx, call, pic, dst0), dst0), call


def test_refusals(dev):
    """the B200_EINVAL cases of the batch entry launch nothing; the init entry's ENOSYS / EINVAL"""
    import torch
    import ffmpeg_b200 as fb
    from ffmpeg_b200._lib import VP9DSPContext, Vp9McRef
    L = fb.lib()
    buf = torch.zeros(8192, dtype=torch.uint8, device="cuda")
    p = buf.data_ptr()
    ops = np.zeros(1, vm.OP_DTYPE)
    ops["w"] = ops["h"] = 4
    dops = torch.from_numpy(ops.view(np.uint8)).cuda()
    before = fb.launch_count()

    def call(depth=8, nrefs=1, n=1, ops=dops.data_ptr(), dst=p + 64, ds=64, refs=True, data=p + 4096, rs=64, w=16, h=16, dx=16, dy=16):
        arr = (Vp9McRef * 8)(*[Vp9McRef(data, rs, w, h, dx, dy)] * 8)
        return L.b200_vp9_mc_batch_device(dev.handle, depth, nrefs, C.cast(arr, C.c_void_p) if refs else None, n, ops, dst, ds)
    assert call(n=0) == 0 and call(n=0, ops=None, dst=None, refs=False) == 0
    assert call(n=-1) == EINVAL and call(nrefs=0) == EINVAL and call(nrefs=9) == EINVAL
    for depth in (0, 7, 9, 11, 14, 16):
        assert call(depth=depth) == EINVAL, depth
    assert call(w=0) == EINVAL and call(h=0) == EINVAL and call(dx=0) == EINVAL and call(dy=33) == EINVAL and call(data=None) == EINVAL
    assert call(depth=10, ds=63) == EINVAL and call(depth=10, rs=65) == EINVAL and call(depth=10, data=p + 4097) == EINVAL
    assert call(ops=None) == EINVAL and call(dst=None) == EINVAL and call(refs=False) == EINVAL
    assert call(depth=10, dst=p + 65) == EINVAL and call(ops=dops.data_ptr() + 4) == EINVAL
    dev.sync()
    assert fb.launch_count() == before and not buf.any().item()
    ctx = VP9DSPContext()
    for depth in (0, 7, 9, 11, 14, 16):
        assert L.b200_vp9_dsp_init(C.byref(ctx), depth) == ENOSYS, depth
    assert L.b200_vp9_dsp_init(None, 8) == EINVAL


def smoke(dev):
    """smoke(): one small luma- and chroma-shaped batch at 8 and 10 bit, the luma one over scaled references, bit-compared with the
    checker"""
    for depth in (8, 10):
        for chroma in (0, 1):
            case = vm.batch_case(11 + depth + chroma, 64, depth, *((100, 60) if chroma else (200, 120)), scaled=not chroma)
            got = on_device(dev, depth, *case)
            assert np.array_equal(got, vm.orc_batch(depth, *case)), ("vp9 mc mismatch", depth, chroma)
