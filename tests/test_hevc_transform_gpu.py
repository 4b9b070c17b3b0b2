"""GPU tier for the HEVC residual (ffmpeg_b200/csrc/hevcidct.cu) on the H100: b200_hevc_transform_add_batch_device against the
reference's fixture hashes and the checker at every depth, a 3840x2160 luma plane and its 4:2:0 chroma planes tiled with mixed TU sizes
and kinds, a call of more ops than one launch takes, offsets beyond 2^31 bytes, and every drop-in member of the context through host
pointers.  Only committed fixtures and the checker are read."""
import numpy as np
import pytest

import cpulibs as cl
import hevcidctlib as hi

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


def on_device(dev, depth, coef, dst, ops):
    """one batched call on device copies; returns dst as numpy (and checks that coef was not written)"""
    import torch
    from ffmpeg_b200 import hevcdsp
    st = torch.cuda.ExternalStream(dev.stream)
    with torch.cuda.stream(st):
        dc, dd, do = _t(coef), _t(dst), _t(ops.view(np.uint8))
        hevcdsp.hevc_transform_add_batch_device(dev, depth, len(ops), do, dc, dd, dst.strides[0])
        dev.sync()
        assert np.array_equal(dc.cpu().numpy(), coef)
        return dd.cpu().numpy().view(dst.dtype)


@pytest.mark.parametrize("depth", hi.DEPTHS)
@pytest.mark.parametrize("chroma", (0, 1), ids=("luma", "chroma"))
def test_batch_vs_fixture(dev, depth, chroma):
    """the fixture batch (every size, kind and flag, every input class): the reference's destination bit for bit, sentinels included"""
    case = hi.fixture_case(depth, chroma)
    got = on_device(dev, depth, *case)
    assert hi.digest(got) == hi.fixture_hashes()[(depth, bool(chroma))]
    assert np.array_equal(got, hi.orc_batch(depth, *case))


@pytest.mark.parametrize("depth", hi.DEPTHS)
@pytest.mark.parametrize("cls", hi.CLASSES)
def test_batch_vs_checker(dev, depth, cls):
    for chroma in (False, True):
        case = hi.batch_case(2000 + 37 * depth + 5 * chroma + hi.CLASSES.index(cls), 700, depth, chroma, cls=cls)
        assert np.array_equal(on_device(dev, depth, *case), hi.orc_batch(depth, *case))


def plane_case(seed, depth, W, H, chroma):
    """a W x H plane tiled with TUs: 32 x 32 blocks (16 x 16 for chroma) split at random down to 4 x 4 (and wherever one crosses the
    plane's edge), every TU an op of a seeded kind
    with a parser-shaped or dense block; the coefficient buffer frame-wide, in op order"""
    rng = np.random.default_rng(seed)
    maxv = (1 << depth) - 1
    dst = rng.integers(0, maxv + 1, (H, W)).astype(hi.sdtype(depth))
    tus = []

    def split(x, y, s):
        if x >= W or y >= H:
            return
        if s > 4 and (rng.random() < 0.5 or x + s > W or y + s > H):
            for dy in (0, s // 2):
                for dx in (0, s // 2):
                    split(x + dx, y + dy, s // 2)
        else:
            tus.append((x, y, s))
    top = 16 if chroma else 32
    for y in range(0, H, top):
        for x in range(0, W, top):
            split(x, y, top)
    n = len(tus)
    ops = np.zeros(n, hi.TU_DTYPE)
    u = np.array(tus)
    log2 = np.log2(u[:, 2]).astype(np.uint8)
    ops["dst_off"] = u[:, 1] * dst.strides[0] + u[:, 0] * dst.itemsize
    ops["log2_size"] = log2
    sizes = u[:, 2].astype(np.int64) ** 2
    ops["coef_off"] = np.concatenate([[0], np.cumsum(sizes)[:-1]])
    coef = np.zeros(int(sizes.sum()) + 8, np.int16)
    for i in range(n):
        k, f = hi.op_kind(rng, int(log2[i]), chroma)
        c, lim = hi.block(rng, int(log2[i]), "decoder" if rng.random() < 0.8 else "dense")
        ops[i]["kind"], ops[i]["flags"], ops[i]["col_limit"] = k, f, lim
        coef[ops[i]["coef_off"]:ops[i]["coef_off"] + sizes[i]] = c.ravel()
    return coef, dst, ops


@pytest.mark.parametrize("depth", (8, 10))
def test_planes_3840x2160_420(dev, depth):
    """one luma plane and both 4:2:0 chroma planes, one call each"""
    for seed, (W, H, chroma) in enumerate(((3840, 2160, False), (1920, 1080, True), (1920, 1080, True))):
        case = plane_case(77 + depth + seed, depth, W, H, chroma)
        got = on_device(dev, depth, *case)
        assert np.array_equal(got, hi.orc_batch(depth, *case))
        assert (got != case[1]).mean() > 0.3


def test_more_ops_than_one_launch(dev):
    """2^20 + 4099 4x4 ops (more than one launch's 2^20) of every kind: every block against the checker"""
    n, cols = (1 << 20) + 4099, 1024
    rng = np.random.default_rng(3)
    dst = rng.integers(0, 256, ((n + cols - 1) // cols * 4, cols * 4)).astype(np.uint8)
    i = np.arange(n)
    ops = np.zeros(n, hi.TU_DTYPE)
    ops["dst_off"] = (i // cols) * 4 * dst.strides[0] + (i % cols) * 4
    ops["coef_off"] = i * 16
    ops["log2_size"] = 2
    ops["kind"] = i % 5
    ops["flags"] = rng.integers(0, 8, n)
    ops["col_limit"] = rng.integers(-8, 40, n)
    coef = rng.integers(-4096, 4096, n * 16 + 8).astype(np.int16)
    assert np.array_equal(on_device(dev, 8, coef, dst, ops), hi.orc_batch(8, coef, dst, ops))


def test_offsets_beyond_2gb(dev):
    """dst_off beyond 2^31 bytes and coef_off beyond 2^31 elements: the blocks land where the 64-bit offsets say"""
    import torch
    from ffmpeg_b200 import hevcdsp
    coef, dst, ops = hi.batch_case(9, 64, 10)
    big_d, big_c = (1 << 31) + (1 << 20), (1 << 31) + 4096           # bytes of dst, elements of coef in front of the case
    st = torch.cuda.ExternalStream(dev.stream)
    with torch.cuda.stream(st):
        dd = torch.zeros(big_d + dst.nbytes, dtype=torch.uint8, device="cuda")
        dc = torch.zeros(big_c + coef.size, dtype=torch.int16, device="cuda")
        dd[big_d:] = torch.from_numpy(dst.view(np.uint8).ravel()).cuda()
        dc[big_c:] = torch.from_numpy(coef).cuda()
        far = ops.copy()
        far["dst_off"] += big_d
        far["coef_off"] += big_c
        do = _t(far.view(np.uint8))
        hevcdsp.hevc_transform_add_batch_device(dev, 10, len(far), do, dc, dd, dst.strides[0])
        dev.sync()
        got = dd[big_d:].cpu().numpy().view(np.uint16).reshape(dst.shape)
        assert int(dd[:big_d].count_nonzero()) == 0
        del dd, dc
        torch.cuda.empty_cache()
    assert np.array_equal(got, hi.orc_batch(10, coef, dst, ops))


@pytest.mark.parametrize("depth", hi.DEPTHS)
def test_dropin_members(dev, depth):
    """HEVCDSPContext from ff_hevc_dsp_init + ff_hevc_dsp_init_transform: all 15 residual member pointers called with host pointers
    against the checker, on every input class; the MC tables the first init filled are still there"""
    from ffmpeg_b200 import hevcdsp
    ctx = hevcdsp.ff_hevc_dsp_init(depth)
    mc = bytes(ctx.put_hevc_qpel)
    hevcdsp.ff_hevc_dsp_init_transform(ctx, depth)
    assert bytes(ctx.put_hevc_qpel) == mc
    for cls in hi.CLASSES:
        for call in hi.member_calls(60 + depth + hi.CLASSES.index(cls), depth, cls):
            assert np.array_equal(hi.ctx_tx(ctx, call), hi.run_tx(cl.oracle(), "orc_hevc_tx", depth, call)), (call[0], call[1], call[3])
    for call in hi.residual_calls(30 + depth, depth):
        assert np.array_equal(hi.ctx_add(ctx, call), hi.run_add(cl.oracle(), "orc_hevc_add_residual", depth, call))


def smoke(dev):
    """smoke(): one small mixed batch at 8 and 10 bit, bit-compared with the checker"""
    for depth in (8, 10):
        case = hi.batch_case(11 + depth, 96, depth)
        got = on_device(dev, depth, *case)
        assert np.array_equal(got, hi.orc_batch(depth, *case)), ("hevc transform mismatch", depth)
