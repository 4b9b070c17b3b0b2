"""GPU tier for VP9 inverse transforms (ffmpeg_b200/csrc/vp9itxfm.cu) on the H100: b200_vp9_itxfm_add_batch_device against the
reference's fixture hashes and the checker at every depth and coefficient class, a 3840x2160 luma and a 1920x1080 4:2:0 chroma plane
tiled with mixed sizes and types, a call of more ops than one launch takes, offsets beyond 2^31 bytes, every drop-in member through host
pointers (coefficient write-back included), and the refusals.  Only committed fixtures and the checker are read."""
import ctypes as C

import numpy as np
import pytest

import cpulibs as cl  # noqa: F401
import vp9itxfmlib as vt

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
    a = np.ascontiguousarray(a)
    return torch.from_numpy(a.view(np.int16) if a.dtype == np.uint16 else a).cuda()


def on_device(dev, depth, dst, coef, ops):
    """one batched call on device copies; returns dst as numpy (and checks that coef is unchanged)"""
    import torch
    from ffmpeg_b200 import vp9dsp
    st = torch.cuda.ExternalStream(dev.stream)
    with torch.cuda.stream(st):
        dd, dc, do = _t(dst), _t(coef), _t(ops.view(np.uint8))
        vp9dsp.vp9_itxfm_add_batch_device(dev, depth, len(ops), do, dc, dd, dst.strides[0])
        dev.sync()
        assert np.array_equal(dc.cpu().numpy(), coef)
        return dd.cpu().numpy().view(dst.dtype)


@pytest.mark.parametrize("depth", vt.DEPTHS)
@pytest.mark.parametrize("cls", vt.FIXTURE_CLASSES)
def test_batch_vs_fixture(dev, depth, cls):
    """the fixture batch (every member, sentinels around every block): the reference's destination picture bit for bit"""
    case = vt.fixture_case(depth, cls)
    got = on_device(dev, depth, *case)
    assert vt.digest(got) == vt.fixture_hashes()[(depth, cls)]
    assert np.array_equal(got, vt.orc_batch(depth, *case))


@pytest.mark.parametrize("depth", vt.DEPTHS)
@pytest.mark.parametrize("cls", vt.CLASSES)
def test_batch_vs_checker(dev, depth, cls):
    case = vt.batch_case(2000 + 37 * depth + vt.CLASSES.index(cls), 2000, depth, cls, cols=40)
    assert np.array_equal(on_device(dev, depth, *case), vt.orc_batch(depth, *case))


def plane_case(seed, depth, W, H, sb=64):
    """a W x H plane tiled with transform blocks of every size (sb x sb superblocks split at random down to 4x4), each of a seeded type,
    lossless blocks among the 4x4 ones, decoder-shaped coefficients (a quarter of them DC-only with eob 1)"""
    rng = np.random.default_rng(seed)
    dst = rng.integers(0, 1 << depth, (H, W)).astype(vt.sdtype(depth))
    units = []

    def split(x, y, s):
        if s > 4 and (s > 32 or rng.random() < 0.55):
            for dy in (0, s // 2):
                for dx in (0, s // 2):
                    split(x + dx, y + dy, s // 2)
        elif x + s <= W and y + s <= H:
            units.append((x, y, s))
    for y in range(0, H, sb):
        for x in range(0, W, sb):
            split(x, y, sb)
    n = len(units)
    ops = np.zeros(n, vt.TX_DTYPE)
    u = np.array(units)
    ops["dst_off"] = u[:, 1] * dst.strides[0] + u[:, 0] * dst.itemsize
    tx = np.log2(u[:, 2]).astype(int) - 2
    tx[(tx == 0) & (rng.random(n) < 0.1)] = 4
    ops["tx"] = tx
    ops["type"] = rng.integers(0, 4, n)
    sizes = u[:, 2] ** 2
    ops["coef_off"] = np.concatenate([[0], np.cumsum(sizes)[:-1]])
    coef = np.zeros(int(sizes.sum()), vt.cdtype(depth))
    amp = 1 << (depth + 3)
    k = rng.integers(1, 5, n)
    dc = rng.random(n) < 0.25
    for i in range(n):
        s = int(u[i, 2])
        kk = 1 if dc[i] else min(int(k[i]), s)
        blk = np.zeros((s, s), np.int64)
        blk[:kk, :kk] = rng.integers(-amp, amp + 1, (kk, kk))
        coef[int(ops["coef_off"][i]):int(ops["coef_off"][i]) + s * s] = blk.ravel()
        ops["eob"][i] = 1 if dc[i] else kk * kk + int(rng.integers(0, 2))
    return dst, coef, ops


@pytest.mark.parametrize("depth,chroma", [(8, 0), (10, 0), (12, 0), (8, 1), (10, 1)],
                         ids=("8-luma", "10-luma", "12-luma", "8-chroma", "10-chroma"))
def test_plane(dev, depth, chroma):
    """3840x2160 luma / 1920x1080 4:2:0 chroma, mixed sizes and types"""
    W, H = (3840, 2160) if not chroma else (1920, 1080)
    case = plane_case(77 + depth + chroma, depth, W, H)
    got = on_device(dev, depth, *case)
    assert np.array_equal(got, vt.orc_batch(depth, *case))


def test_more_ops_than_one_launch(dev):
    """2^20 + 4099 ops of 4x4 (every type, lossless among them) in one call: more than one launch's 2^20"""
    n, cols = (1 << 20) + 4099, 1024
    rng = np.random.default_rng(3)
    dst = rng.integers(0, 256, ((n + cols - 1) // cols * 4, cols * 4)).astype(np.uint8)
    ops = np.zeros(n, vt.TX_DTYPE)
    i = np.arange(n)
    ops["dst_off"] = (i // cols) * 4 * dst.strides[0] + (i % cols) * 4
    ops["tx"] = np.where(i % 7 == 0, 4, 0)
    ops["type"] = i % 4
    ops["eob"] = rng.integers(0, 3, n)
    ops["coef_off"] = rng.integers(0, 4096, n) * 16
    coef = rng.integers(-2048, 2048, 4096 * 16 + 16).astype(np.int16)
    got = on_device(dev, 8, dst, coef, ops)
    assert np.array_equal(got, vt.orc_batch(8, dst, coef, ops))


@pytest.mark.parametrize("depth", (8, 10))
def test_offsets_beyond_2_31_bytes(dev, depth):
    """dst_off and coef_off * sizeof(coefficient) above 2^31 bytes: blocks near the end of a 2.2 GB plane from coefficients near the end
    of a 2.2 GB buffer; only the touched windows are copied and compared"""
    import torch
    from ffmpeg_b200 import vp9dsp
    bps, cs = (1, 2) if depth == 8 else (2, 4)
    stride = 4096
    rows = (2 ** 31 + 2 ** 27) // stride
    base_row = rows - 64
    small_dst, small_coef, ops = vt.batch_case(9 + depth, 40, depth, classes=vt.CLASSES, cols=stride // bps // vt.CELL)
    small_dst = np.ascontiguousarray(np.pad(small_dst, ((0, 0), (0, stride // bps - small_dst.shape[1])), constant_values=7))
    assert small_dst.shape[0] <= 64
    coef_base = (2 ** 31 + 2 ** 26) // cs // 16 * 16
    big_ops = ops.copy()
    big_ops["dst_off"] += base_row * stride
    big_ops["coef_off"] += coef_base
    assert big_ops["dst_off"].min() > 2 ** 31 and big_ops["coef_off"].min() * cs > 2 ** 31
    st = torch.cuda.ExternalStream(dev.stream)
    with torch.cuda.stream(st):
        d = torch.zeros(rows * stride, dtype=torch.uint8, device="cuda")
        c = torch.zeros((coef_base + small_coef.size + 16) * cs, dtype=torch.uint8, device="cuda")
        d[base_row * stride:base_row * stride + small_dst.nbytes] = torch.from_numpy(small_dst.view(np.uint8).ravel()).cuda()
        c[coef_base * cs:(coef_base + small_coef.size) * cs] = torch.from_numpy(small_coef.view(np.uint8)).cuda()
        vp9dsp.vp9_itxfm_add_batch_device(dev, depth, len(ops), _t(big_ops.view(np.uint8)), c, d, stride)
        dev.sync()
        got = d[base_row * stride:base_row * stride + small_dst.nbytes].cpu().numpy().view(small_dst.dtype).reshape(small_dst.shape)
        assert not d[:base_row * stride].any().item()
        del d, c
        torch.cuda.empty_cache()
    assert np.array_equal(got, vt.orc_batch(depth, small_dst, small_coef, ops))


@pytest.mark.parametrize("depth", vt.DEPTHS)
def test_dropin_members(dev, depth):
    """VP9DSPContext from ff_vp9dsp_init + ff_vp9dsp_init_itxfm through the library: every itxfm_add member called with host pointers
    against the checker, the destination (sentinels included) and the coefficients the member leaves behind; the mc tables untouched"""
    from ffmpeg_b200 import vp9dsp
    from test_vp9_itxfm import check_members
    ctx = vp9dsp.ff_vp9dsp_init(depth)
    mc = bytes(ctx.mc)
    vp9dsp.ff_vp9dsp_init_itxfm(ctx, depth)
    assert bytes(ctx.mc) == mc and all(ctx.itxfm_add[t][y] for t in range(5) for y in range(4))
    for cls in vt.CLASSES:
        check_members(ctx, depth, 60 + depth, cls, per=2)


def test_refusals(dev):
    """the B200_EINVAL cases of the batch entry launch nothing; the init entry's ENOSYS / EINVAL"""
    import torch
    import ffmpeg_b200 as fb
    from ffmpeg_b200._lib import VP9DSPContext
    L = fb.lib()
    buf = torch.zeros(8192, dtype=torch.uint8, device="cuda")
    p = buf.data_ptr()
    ops = np.zeros(1, vt.TX_DTYPE)
    dops = _t(ops.view(np.uint8))
    o = dops.data_ptr()
    before = fb.launch_count()

    def call(depth=8, n=1, ops=o, coef=p + 1024, dst=p + 4096, ds=64):
        return L.b200_vp9_itxfm_add_batch_device(dev.handle, depth, n, ops, coef, dst, ds)
    assert call(n=0) == 0 and call(n=0, ops=None, coef=None, dst=None) == 0
    assert call(n=-1) == EINVAL
    for depth in (0, 7, 9, 11, 14, 16):
        assert call(depth=depth) == EINVAL, depth
    assert call(ops=None) == EINVAL and call(coef=None) == EINVAL and call(dst=None) == EINVAL
    assert call(ops=o + 4) == EINVAL and call(coef=p + 1032) == EINVAL and call(dst=p + 4098) == EINVAL
    assert call(depth=10, dst=p + 4100) == EINVAL and call(ds=62) == EINVAL and call(depth=12, ds=68) == EINVAL
    dev.sync()
    assert fb.launch_count() == before and not buf.any().item()
    ctx = VP9DSPContext()
    for depth in (0, 7, 9, 11, 14, 16):
        assert L.b200_vp9_dsp_init_itxfm(C.byref(ctx), depth) == ENOSYS, depth
    assert L.b200_vp9_dsp_init_itxfm(None, 8) == EINVAL


def smoke(dev):
    """smoke(): one small batch of every member at 8 and 10 bit, decoder-shaped and extreme coefficients, bit-compared with the
    checker"""
    for depth in (8, 10):
        for cls in ("decoder", "extremes"):
            case = vt.batch_case(11 + depth, 100, depth, cls)
            got = on_device(dev, depth, *case)
            assert np.array_equal(got, vt.orc_batch(depth, *case)), ("vp9 itxfm mismatch", depth, cls)
