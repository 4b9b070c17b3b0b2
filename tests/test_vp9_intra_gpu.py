"""GPU tier for VP9 intra reconstruction (ffmpeg_b200/csrc/vp9intra.cu) on the H100: b200_vp9_intra_recon_frame_device against the
reference's fixture hashes and the checker, seeded frames at 8, 10 and 12 bit in every chroma format up to 3840x2160, one call of more
than 2^20 ops, every drop-in member through host pointers, a whole inter frame with intra blocks rebuilt on the device by motion
compensation, the inter residual, intra reconstruction and the loop filter against the chain of the four checkers, and the refusals.
After every test the intra entry's wait-timeout counter is still 0.  Only committed fixtures and the checkers are read."""
import copy
import ctypes as C

import numpy as np
import pytest

import cpulibs as cl
import vp9intralib as vi

pytestmark = pytest.mark.gpu
EINVAL, ENOSYS = -22, -38


@pytest.fixture(scope="module")
def dev():
    import ffmpeg_b200 as fb
    d = fb.Device(0)
    d.set_default()
    yield d


@pytest.fixture(autouse=True)
def no_timeouts(dev):
    yield
    from ffmpeg_b200 import vp9dsp
    assert vp9dsp.vp9_intra_timeouts(dev) == 0


def _t(a):
    import torch
    a = np.ascontiguousarray(a)
    return torch.from_numpy(a.view(np.int16) if a.dtype == np.uint16 else a).cuda()


def _back(t, like):
    return t.cpu().numpy().view(like.dtype)


def _ptrs(ts, arrs, margin):
    return [t.data_ptr() + margin * a.strides[0] + margin * a.itemsize for t, a in zip(ts, arrs)]


def on_device(dev, f):
    """one frame entry call on device copies of the full arrays (sentinels included); returns the three arrays"""
    import torch
    from ffmpeg_b200 import vp9dsp
    st = torch.cuda.ExternalStream(dev.stream)
    with torch.cuda.stream(st):
        ts = [_t(p) for p in f.planes]
        ops = _t(np.ascontiguousarray(f.ops).view(np.uint8))
        coef = _t(f.coef)
        ls_y, ls_uv = f.strides()
        vp9dsp.vp9_intra_recon_frame_device(dev, f.depth, f.ss_h, f.ss_v, f.width, f.height, _ptrs(ts, f.planes, vi.MARGIN), ls_y, ls_uv,
                                            len(f.ops), ops, coef)
        dev.sync()
        return [_back(t, p) for t, p in zip(ts, f.planes)]


def same(a, b):
    return all(np.array_equal(x, y) for x, y in zip(a, b))


@pytest.mark.parametrize("name", vi.FIXTURE_NAMES)
def test_frame_vs_fixture(dev, name):
    """the fixture frame: the reference's three planes bit for bit (sentinels around every plane unchanged), and the checker's"""
    f = vi.frame_case(name)
    got = on_device(dev, f)
    assert vi.digest(got) == vi.fixture_hashes()[name]
    assert same(got, vi.orc_frame(f))


LARGE = [(d, fmt, size, kw) for d in vi.DEPTHS for fmt in vi.FORMATS for size, kw in (((1920, 1080), {}), ((3840, 2160), {"sizes": "4x4"}))
         if fmt == "420" or size[0] == 1920 or d == 10]


@pytest.mark.parametrize("depth,fmt,size,kw", LARGE, ids=[f"{d}-{fmt}-{s[1]}p" for d, fmt, s, _ in LARGE])
def test_large_frames(dev, depth, fmt, size, kw):
    """seeded decoder-shaped frames (mixed block sizes at 1080p, all 4x4 at 2160p, where the dependency chains are longest)"""
    f = vi.Frame(900 + depth + size[1] + len(fmt), depth, fmt, *size, **kw)
    assert same(on_device(dev, f), vi.orc_frame(f))


def test_inter_frame_with_intra_blocks(dev):
    """a 1080p 10-bit inter frame with about 10% intra blocks and tile columns, lossless off: intra blocks among samples already in the plane"""
    f = vi.Frame(31, 10, "420", 1920, 1080, kind="inter", p_intra=0.1, tiles=4)
    assert same(on_device(dev, f), vi.orc_frame(f))


def test_more_than_2_20_ops(dev):
    """one call of more than 2^20 ops: an 8-bit 4:4:4 3840x2160 frame of 4x4 blocks"""
    f = vi.Frame(77, 8, "444", 3840, 2160, sizes="4x4", p_skip=0.5)
    assert len(f.ops) > 1 << 20
    assert same(on_device(dev, f), vi.orc_frame(f))


def test_lossless_repeats(dev):
    """a lossless 1080p frame four times: every run equal to the checker (the warps' interleaving differs from run to run)"""
    f = vi.Frame(12, 12, "420", 1920, 1080, lossless=True)
    want = vi.orc_frame(f)
    for _ in range(4):
        assert same(on_device(dev, f), want)


@pytest.mark.parametrize("depth", vi.DEPTHS)
def test_dropin_members(dev, depth):
    """VP9DSPContext from ff_vp9dsp_init + ff_vp9dsp_init_intrapred through the library: every intra_pred member called with host
    pointers against the checker on random edges and edges at both clip bounds; the mc tables untouched"""
    from ffmpeg_b200 import vp9dsp
    ctx = vp9dsp.ff_vp9dsp_init(depth)
    mc = bytes(ctx.mc)
    vp9dsp.ff_vp9dsp_init_intrapred(ctx, depth)
    assert bytes(ctx.mc) == mc
    for edges in ("random", "low", "high"):
        for call in vi.member_calls(60 + depth, depth, per=2, edges=edges):
            tx, mode = call[0], call[1]
            got = vi.run_member(vp9dsp.VP9_INTRA_FUNC(ctx.intra_pred[tx][mode]), depth, call)
            assert np.array_equal(got, vi.run_member(vi.orc_member(depth, tx, mode), depth, call)), (depth, tx, mode, edges)


# ---------------------------------------------------------------- a whole frame on the device: MC -> residual -> intra -> loop filter
def chain_case(seed, depth):
    """a 4:2:0 inter frame (1280x720: cols even, so the chroma areas of the intra and loop-filter entries coincide) with about 20% intra
    blocks: per plane, the MC ops and the inter residual ops of the inter blocks that lie inside the picture, one reference picture per
    plane, the intra frame, and decoder-shaped loop-filter records"""
    import vp9itxfmlib as vt
    import vp9lflib as vl
    from ffmpeg_b200 import vp9dsp
    f = vi.Frame(seed, depth, "420", 1280, 720, kind="inter", p_intra=0.2)
    rng = np.random.default_rng(seed)
    refs = [rng.integers(0, 1 << depth, (f.H[p] + 64, f.W[p] + 64)).astype(vi.sdtype(depth)) for p in range(3)]
    mc, tx, coefs = [[], [], []], [[], [], []], [[], [], []]
    coff = [0, 0, 0]
    for r in f.blocks:
        if r[12]:
            continue
        row, col, bs, t = int(r[0]), int(r[1]), int(r[2]), int(r[3])
        bw, bh = vi.BWH4[bs][0] * 4, vi.BWH4[bs][1] * 4
        for p in range(3):
            sh, sv = (f.ss_h, f.ss_v) if p else (0, 0)
            x0, y0, w, h = col * 8 >> sh, row * 8 >> sv, bw >> sh, bh >> sv
            if w < 4 or x0 + w > f.W[p] or y0 + h > f.H[p]:
                continue
            op = np.zeros(1, vp9dsp.OP_DTYPE)
            op["dst_off"] = (vi.MARGIN + y0) * f.planes[p].strides[0] + (vi.MARGIN + x0) * f.planes[p].itemsize
            op["x"][0, 0], op["y"][0, 0] = x0 + int(rng.integers(-8, 9)), y0 + int(rng.integers(-8, 9))
            op["mx"][0, 0], op["my"][0, 0] = rng.integers(0, 16, 2)
            op["w"], op["h"], op["filter"], op["kind"] = w, h, int(rng.integers(0, 4)), vp9dsp.SINGLE
            mc[p].append(op)
            n = min(4 << (t if p == 0 else max(t - 1, 0)), w, h)
            if n < 4:
                continue
            ts = {4: 0, 8: 1, 16: 2, 32: 3}[n]
            for yy in range(0, h, n):
                for xx in range(0, w, n):
                    if r[5]:
                        continue
                    b, eob = vt.coefs(rng, depth, ts, "decoder")
                    o = np.zeros(1, vp9dsp.TX_DTYPE)
                    o["dst_off"] = (vi.MARGIN + y0 + yy) * f.planes[p].strides[0] + (vi.MARGIN + x0 + xx) * f.planes[p].itemsize
                    o["coef_off"], o["tx"], o["type"], o["eob"] = coff[p], ts, int(rng.integers(0, 4)), eob
                    tx[p].append(o)
                    coefs[p].append(b.ravel())
                    coff[p] += b.size
    mc = [np.concatenate(m) for m in mc]
    tx = [np.concatenate(t) for t in tx]
    coefs = [np.concatenate(c).astype(vi.cdtype(depth)) for c in coefs]
    lf = vl.Frame(seed, depth, "420", 1280, 720)
    assert all(a.shape == b.shape for a, b in zip(lf.planes, f.planes))
    return f, refs, mc, tx, coefs, lf


def chain_checkers(f, refs, mc, tx, coefs, lf):
    import vp9itxfmlib as vt
    import vp9lflib as vl
    import vp9mclib as vm
    planes = [vm.orc_batch(f.depth, [refs[p]], [(16, 16)], f.planes[p], mc[p]) for p in range(3)]
    planes = [vt.orc_batch(f.depth, planes[p], coefs[p], tx[p]) for p in range(3)]
    g = copy.copy(f)
    g.planes = planes
    planes = vi.orc_frame(g)
    return vl._frame(cl.oracle(), "orc_vp9_lf_frame", lf, 0, planes)


def chain_device(dev, f, refs, mc, tx, coefs, lf):
    import torch
    from ffmpeg_b200 import vp9dsp
    st = torch.cuda.ExternalStream(dev.stream)
    with torch.cuda.stream(st):
        ts = [_t(p) for p in f.planes]
        rts = [_t(r) for r in refs]
        for p in range(3):
            vp9dsp.vp9_mc_batch_device(dev, f.depth, [(rts[p], refs[p].strides[0], refs[p].shape[1], refs[p].shape[0], 16, 16)], len(mc[p]),
                                       _t(np.ascontiguousarray(mc[p]).view(np.uint8)), ts[p], f.planes[p].strides[0])
            vp9dsp.vp9_itxfm_add_batch_device(dev, f.depth, len(tx[p]), _t(np.ascontiguousarray(tx[p]).view(np.uint8)), _t(coefs[p]), ts[p],
                                              f.planes[p].strides[0])
        ptrs = _ptrs(ts, f.planes, vi.MARGIN)
        ls_y, ls_uv = f.strides()
        vp9dsp.vp9_intra_recon_frame_device(dev, f.depth, f.ss_h, f.ss_v, f.width, f.height, ptrs, ls_y, ls_uv, len(f.ops),
                                            _t(np.ascontiguousarray(f.ops).view(np.uint8)), _t(f.coef))
        vp9dsp.vp9_loopfilter_frame_device(dev, f.depth, f.ss_h, f.ss_v, f.width, f.height, ptrs, ls_y, ls_uv,
                                           _t(np.ascontiguousarray(lf.lflvl).view(np.uint8)), lf.lstride, lf.lim, lf.mblim)
        dev.sync()
        return [_back(t, p) for t, p in zip(ts, f.planes)]


@pytest.mark.parametrize("depth", (8, 10))
def test_whole_frame_on_device(dev, depth):
    """MC batch per plane, residual batch per plane for the inter blocks, one intra frame call, the loop filter: all on one stream,
    nothing on the host in between, equal to the four checkers run in the same order"""
    from ffmpeg_b200 import vp9dsp
    case = chain_case(40 + depth, depth)
    assert all(len(m) for m in case[2]) and len(case[0].ops)
    assert same(chain_device(dev, *case), chain_checkers(*case))
    assert vp9dsp.vp9_loopfilter_timeouts(dev) == 0


def test_refusals(dev):
    """the B200_EINVAL cases of the frame entry launch nothing and write nothing"""
    import torch
    import ffmpeg_b200 as fb
    from ffmpeg_b200._lib import VP9DSPContext
    L = fb.lib()
    buf = torch.zeros(1 << 16, dtype=torch.uint8, device="cuda")
    p = buf.data_ptr()
    before = fb.launch_count()

    def call(depth=8, ss_h=1, ss_v=1, w=64, h=64, planes=(p, p + 8192, p + 12288), ls_y=64, ls_uv=32, nops=1, ops=p + 16384, coef=p + 32768):
        arr = (C.c_void_p * 3)(*planes)
        return L.b200_vp9_intra_recon_frame_device(dev.handle, depth, ss_h, ss_v, w, h, arr, ls_y, ls_uv, nops, ops, coef)
    for depth in (0, 7, 9, 11, 16):
        assert call(depth=depth) == EINVAL, depth
    assert call(ss_h=2) == EINVAL and call(w=0) == EINVAL and call(h=-1) == EINVAL and call(ops=None) == EINVAL
    assert call(planes=(p, None, p)) == EINVAL and call(ls_y=63) == EINVAL and call(ls_uv=31) == EINVAL and call(coef=p + 8) == EINVAL
    assert call(depth=10, ls_y=128, ls_uv=64, planes=(p + 1, p + 8192, p + 12288)) == EINVAL and call(depth=10, ls_y=129, ls_uv=64) == EINVAL
    assert call(nops=-1) == EINVAL and call(nops=0, ops=None, coef=None) == 0
    dev.sync()
    assert fb.launch_count() == before and not buf.any().item()
    ctx = VP9DSPContext()
    for depth in (0, 7, 9, 11, 16):
        assert L.b200_vp9_dsp_init_intrapred(C.byref(ctx), depth) == ENOSYS, depth
    assert L.b200_vp9_dsp_init_intrapred(None, 8) == EINVAL


def smoke(dev):
    """smoke(): a small 4:2:0 intra frame at 8 and 10 bit (mixed block sizes, tile columns), bit-compared with the checker, and no wait
    ran out"""
    from ffmpeg_b200 import vp9dsp
    for depth in (8, 10):
        f = vi.Frame(5 + depth, depth, "420", 200, 140, tiles=2)
        assert same(on_device(dev, f), vi.orc_frame(f)), ("vp9 intra mismatch", depth)
    assert vp9dsp.vp9_intra_timeouts(dev) == 0
