"""GPU tier: the 8-bit H.264 motion-compensation kernels (csrc/pel.cu: qpel_kernel, hpel_kernel, chroma_kernel, edge_kernel;
csrc/h264weight.cu: h264_weight_kernel) bit for bit against the checker, in the plane layouts of tests/cases.py (aligned, odd strides
with misaligned bases, bottom-up), on random and extreme pictures, at the batch lengths the kernels' loops branch on.

Every call checks the whole destination allocation, slack included, against the checker applied to a copy of it, and checks that
the source allocation is unchanged."""
import ctypes as C

import numpy as np
import pytest

import cpulibs as cl
from cases import HPEL_DEFINED, HPEL_UNDEFINED, PEL_LAYOUTS, PEL_SLACK, edge_windows, pel_layout_case, pel_picture

pytestmark = pytest.mark.gpu
B200_EINVAL = -22
KINDS = ("random", "extremes")


def on_stream(device):
    import torch
    return torch.cuda.stream(torch.cuda.ExternalStream(device.stream))


def run_gpu(device, case, call):
    """Copies the case's source and destination allocations to the device, runs call(src, dst, t) with src / dst the device
    addresses of the planes' sample (0, 0) and t(array) -> device tensor, and returns (destination, source) allocations after it."""
    import torch
    src, dst = case["src"], case["dst"]
    with on_stream(device):
        ds, dd = torch.from_numpy(src.buf).cuda(), torch.from_numpy(dst.buf).cuda()
        assert ds.data_ptr() % 64 == 0 and dd.data_ptr() % 64 == 0           # the layouts' alignments are offsets from here
        keep = []

        def t(a):
            keep.append(torch.from_numpy(np.ascontiguousarray(a)).cuda())
            return keep[-1]
        call(ds.data_ptr() + src.base, dd.data_ptr() + dst.base, t)
        device.sync()
        return dd.cpu().numpy(), ds.cpu().numpy()


def assert_same(case, got, exp, what):
    got_dst, got_src = got
    assert np.array_equal(got_src, case["src"].buf), ("source changed", what)
    if not np.array_equal(got_dst, exp):
        bad = np.flatnonzero(got_dst != exp)
        raise AssertionError(f"{what}: {bad.size} bytes differ, the first at offset {int(bad[0]) - case['dst'].base} from sample (0, 0)")


def u8at(a, off):
    return C.cast(a.ctypes.data + int(off), cl.u8p)


# ---------------------------------------------------------------------------------------------- qpel
def qpel_expected(case, ops):
    """orc_h264qpel_batch over the ops that name a table of the reference (size index 3 writes nothing)"""
    src, dst = case["src"], case["dst"]
    exp = dst.buf.copy()
    ok = ((ops >> 1) & 3) != 3
    o, do, so = ops[ok].copy(), case["doff"][ok].copy(), case["soff"][ok].copy()
    cl.oracle().orc_h264qpel_batch(len(o), cl.ptr(o), u8at(exp, dst.base), cl.ptr(do, cl.i64p), u8at(src.buf, src.base),
                                   cl.ptr(so, cl.i64p), src.stride)
    return exp


def qpel_gpu(device, case, ops, n=None):
    from ffmpeg_b200 import pel
    n = len(ops) if n is None else n
    return run_gpu(device, case, lambda s, d, t: pel.h264qpel_batch_device(device, n, t(ops), d, t(case["doff"]), s, t(case["soff"]),
                                                                           case["src"].stride))


def qpel_size(op):
    return 16 >> ((op >> 1) & 3)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("layout", PEL_LAYOUTS)
def test_qpel_every_op_at_every_phase(device, layout, kind):
    """All 96 op codes (put / avg x 16x16, 8x8, 4x4 x 16 positions), each at all 16 source address phases, in one call in a shuffled
    order (so that one warp's 32 ops mix sizes and the look-ahead windows differ in size from the op being computed)."""
    from ffmpeg_b200 import pel
    rng = np.random.default_rng(100 + PEL_LAYOUTS.index(layout))
    codes = [pel.qpel_op(a, s, p) for a in (0, 1) for s in range(3) for p in range(16)]
    order = rng.permutation(len(codes) * 16)
    ops = np.array([codes[i // 16] for i in order], np.uint8)
    phases = order % 16
    case = pel_layout_case(layout, kind, [(qpel_size(o),) * 2 for o in ops], 200, margin=(2, 3), cell=(32, 16), phases=phases)
    assert_same(case, qpel_gpu(device, case, ops), qpel_expected(case, ops), (layout, kind))


def test_qpel_batch_lengths(device):
    """Layout B at batch lengths below, at and above the look-ahead ring (QD = 4), one warp's share (QK = 32) and one CTA's (128):
    the first n ops of one list."""
    from ffmpeg_b200 import pel
    rng = np.random.default_rng(7)
    N = 4097
    ops = np.array([pel.qpel_op(int(a), int(s), int(p)) for a, s, p in zip(rng.integers(0, 2, N), rng.integers(0, 3, N),
                                                                             rng.integers(0, 16, N))], np.uint8)
    case = pel_layout_case("B", "random", [(qpel_size(o),) * 2 for o in ops], 300, margin=(2, 3), cell=(32, 16),
                           phases=rng.integers(0, 16, N))
    for n in (1, 2, 3, 4, 31, 32, 33, 127, 128, 129, 4097):
        sub = dict(case, soff=case["soff"][:n], doff=case["doff"][:n])
        assert_same(sub, qpel_gpu(device, sub, ops[:n]), qpel_expected(sub, ops[:n]), n)


def test_qpel_1080p_plane_of_4x4(device):
    """Every 4x4 block of a 1920x1088 destination, random op codes and vectors, odd stride: 130,560 ops, 4,080 CTAs."""
    from ffmpeg_b200 import pel
    rng = np.random.default_rng(8)
    n = 480 * 272
    ops = (rng.integers(0, 2, n) | 2 << 1 | rng.integers(0, 16, n) << 3).astype(np.uint8)
    case = pel_layout_case("B", "random", [(4, 4)] * n, 400, src_h=1088, margin=(2, 3), cell=(4, 4), cols=480)
    assert case["dst"].w == 1920 and case["dst"].h == 1088
    assert_same(case, qpel_gpu(device, case, ops), qpel_expected(case, ops), "1080p")


# ---------------------------------------------------------------------------------------------- chroma
def chroma_expected(case, op, h, xy, n=None):
    src, dst = case["src"], case["dst"]
    exp = dst.buf.copy()
    n = len(op) if n is None else n
    cl.oracle().orc_h264chroma_batch(n, op.ctypes.data, h.ctypes.data, xy.ctypes.data, exp.ctypes.data + dst.base, case["doff"].ctypes.data,
                                     src.buf.ctypes.data + src.base, case["soff"].ctypes.data, src.stride)
    return exp


def chroma_gpu(device, case, op, h, xy, n=None):
    from ffmpeg_b200 import pel
    n = len(op) if n is None else n
    return run_gpu(device, case, lambda s, d, t: pel.h264chroma_batch_device(device, n, t(op), t(h), t(xy), d, t(case["doff"]), s,
                                                                             t(case["soff"]), case["src"].stride))


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("layout", PEL_LAYOUTS)
def test_chroma_every_phase_width_height(device, layout, kind):
    """Widths 8, 4, 2 x put / avg x all 64 eighth-pel phases x heights 1, 2, 3, 4, 7, 8, 9, 15, 16 (3456 ops, one call)."""
    from ffmpeg_b200 import pel
    rng = np.random.default_rng(20 + PEL_LAYOUTS.index(layout))
    combos = [(pel.chroma_op(a, i), hh, p) for a in (0, 1) for i in range(3) for p in range(64) for hh in (1, 2, 3, 4, 7, 8, 9, 15, 16)]
    combos = [combos[k] for k in rng.permutation(len(combos))]
    op, h, xy = (np.array([c[k] for c in combos], np.uint8) for k in range(3))
    case = pel_layout_case(layout, kind, [(8 >> (o >> 1), hh) for o, hh in zip(op, h)], 500, margin=(0, 1), cell=(16, 16),
                           phases=rng.integers(0, 16, len(op)))
    assert_same(case, chroma_gpu(device, case, op, h, xy), chroma_expected(case, op, h, xy), (layout, kind))


def test_chroma_batch_lengths(device):
    """The persistent grid covers P = sm_count x CK_MINB (8 CTAs per SM) x WARPS (4) x 4 * CK (8 ops per warp trip) = sm_count x 256 ops
    per pass: lengths around one 8-op trip and around one and three passes, so that warps take second and fourth trips and use the
    descriptors they prefetched.  Layout B, the first n ops of one list."""
    from ffmpeg_b200 import pel
    P = device.sm_count * 8 * 4 * 8
    N = 3 * P + 5
    rng = np.random.default_rng(9)
    op = (rng.integers(0, 2, N) | rng.integers(0, 3, N) << 1).astype(np.uint8)
    h = rng.choice(np.array([1, 2, 3, 4, 7, 8], np.uint8), N)
    xy = rng.integers(0, 64, N).astype(np.uint8)
    case = pel_layout_case("B", "random", [(8 >> (o >> 1), hh) for o, hh in zip(op, h)], 600, margin=(0, 1), cell=(16, 8), cols=256)
    for n in (1, 7, 8, 9, P - 1, P, P + 1, N):
        assert_same(case, chroma_gpu(device, case, op, h, xy, n), chroma_expected(case, op, h, xy, n), n)


# ---------------------------------------------------------------------------------------------- hpel
def hpel_expected(case, op, h):
    src, dst = case["src"], case["dst"]
    exp = dst.buf.copy()
    for o, hh, do, so in zip(op.tolist(), h.tolist(), case["doff"].tolist(), case["soff"].tolist()):
        cl.oracle().orc_hpel(o & 3, (o >> 2) & 3, (o >> 4) & 3, u8at(exp, dst.base + do), u8at(src.buf, src.base + so), src.stride, hh)
    return exp


def hpel_gpu(device, case, op, h):
    from ffmpeg_b200 import pel
    return run_gpu(device, case, lambda s, d, t: pel.hpel_batch_device(device, len(op), t(op), t(h), d, t(case["doff"]), s,
                                                                       t(case["soff"]), case["src"].stride))


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("layout", PEL_LAYOUTS)
def test_hpel_every_defined_op(device, layout, kind):
    """Every (table, width, xy) the reference defines x heights 1, 2, 3, 4, 8, 9, 16, each at four source phases (1232 ops, one
    call); avg_pixels2_xy2 stores without averaging, like the reference."""
    from ffmpeg_b200 import pel
    rng = np.random.default_rng(30 + PEL_LAYOUTS.index(layout))
    combos = [(pel.hpel_op(tb, s, q), hh) for tb, s in HPEL_DEFINED for q in range(4) for hh in (1, 2, 3, 4, 8, 9, 16)] * 4
    combos = [combos[k] for k in rng.permutation(len(combos))]
    op, h = (np.array([c[k] for c in combos], np.uint8) for k in range(2))
    case = pel_layout_case(layout, kind, [(16 >> ((o >> 2) & 3), hh) for o, hh in zip(op, h)], 700, margin=(0, 1), cell=(32, 16),
                           phases=rng.integers(0, 16, len(op)))
    assert_same(case, hpel_gpu(device, case, op, h), hpel_expected(case, op, h), (layout, kind))


# ---------------------------------------------------------------------------------------------- weight / biweight
WEIGHTS, OFFSETS = (-128, -1, 0, 1, 127), (-128, 0, 127)


def weight_run(device, layout, bi, seed):
    from ffmpeg_b200 import pel
    geo = [(idx, hh, ld, off) for idx in range(4) for hh in (1, 2, 3, 4, 8, 16) for ld in range(8) for off in OFFSETS]
    wts = [(wd, ws) for wd in WEIGHTS for ws in WEIGHTS] if bi else [(wd, 0) for wd in WEIGHTS]
    params = np.array([pel.weight_params(idx, hh, ld, wd, ws, off) for idx, hh, ld, off in geo for wd, ws in wts], np.int32)
    params = params[np.random.default_rng(seed).permutation(len(params))]
    case = pel_layout_case(layout, "extremes", [(16 >> (p & 3), (p >> 8) & 255) for p in params[:, 0]], seed, cell=(32, 16),
                           phases=np.random.default_rng(seed + 1).integers(0, 16, len(params)))
    dst = case["dst"]
    dst.fill(pel_picture("extremes", dst.h, dst.w, seed + 5))           # both operands at the clip limits
    src, exp, O = case["src"], dst.buf.copy(), cl.oracle()
    for (p0, wd, ws, off), do, so in zip(params.tolist(), case["doff"].tolist(), case["soff"].tolist()):
        idx, hh, ld = p0 & 3, (p0 >> 8) & 255, (p0 >> 16) & 31
        if bi:
            O.orc_h264_biweight(idx, u8at(exp, dst.base + do), u8at(src.buf, src.base + so), dst.stride, hh, ld, wd, ws, off)
        else:
            O.orc_h264_weight(idx, u8at(exp, dst.base + do), dst.stride, hh, ld, wd, off)
    got = run_gpu(device, case, lambda s, d, t: pel.h264_weight_batch_device(device, len(params), t(params), d, t(case["doff"]),
                                                                             s if bi else None, t(case["soff"]) if bi else None, dst.stride))
    assert_same(case, got, exp, (layout, "biweight" if bi else "weight"))


@pytest.mark.parametrize("layout", PEL_LAYOUTS)
def test_weight_every_parameter(device, layout):
    """Every width index x heights 1, 2, 3, 4, 8, 16 x log2_denom 0..7 x weights {-128, -1, 0, 1, 127} x offsets {-128, 0, 127}
    on the extremes (2880 blocks, one call)."""
    weight_run(device, layout, False, 800)


@pytest.mark.parametrize("layout", PEL_LAYOUTS)
def test_biweight_every_parameter(device, layout):
    """The same with every pair of destination and source weights (14,400 blocks, one call); in layout B the source and the
    destination planes have different alignments."""
    weight_run(device, layout, True, 900)


# ---------------------------------------------------------------------------------------------- emulated_edge_mc
@pytest.mark.parametrize("pic", [(1, 1), (1, 37), (37, 1), (100, 60)])
def test_emulated_edge_mc_windows(device, pic):
    """Windows up to 80x80 (so that the 32-lane column loop takes three trips) from three pictures in one call, the pictures at an
    odd source line size and misaligned bases, the windows written at an odd buffer line size."""
    import torch
    from ffmpeg_b200 import pel
    W, H = pic
    NF, LS, BLS = 3, W + 13, 83
    geom = np.array(edge_windows(W, H), np.int32)
    n = len(geom)
    rng = np.random.default_rng(W * 100 + H)
    fbytes = LS * H + 5
    pics = rng.integers(0, 256, PEL_SLACK + NF * fbytes + PEL_SLACK, dtype=np.uint8)
    fr = rng.integers(0, NF, n)
    origin = (PEL_SLACK + 3 + fr * fbytes).astype(np.int64)
    boff = (PEL_SLACK + np.arange(n) * 80 * BLS).astype(np.int64)
    buf0 = rng.integers(0, 256, PEL_SLACK + n * 80 * BLS + PEL_SLACK, dtype=np.uint8)
    exp = buf0.copy()
    for (bw, bh, sx, sy), o, b in zip(geom.tolist(), origin.tolist(), boff.tolist()):
        cl.oracle().orc_emulated_edge_mc(u8at(exp, b), pics.ctypes.data + o + sy * LS + sx, BLS, LS, bw, bh, sx, sy, W, H)
    with on_stream(device):
        d_buf, d_pics = torch.from_numpy(buf0).cuda(), torch.from_numpy(pics).cuda()
        d_geom = torch.from_numpy(geom).cuda()
        pel.emulated_edge_mc_batch_device(device, n, d_buf, torch.from_numpy(boff).cuda(), BLS, d_pics, torch.from_numpy(origin).cuda(), LS,
                                          d_geom, W, H)
        device.sync()
        got = d_buf.cpu().numpy()
        assert np.array_equal(d_pics.cpu().numpy(), pics)
    assert np.array_equal(got, exp), int((got != exp).sum())


# ---------------------------------------------------------------------------------------------- refusals and undefined op codes
def test_refusals_launch_nothing(device):
    """NULL pointers and n < 0 return B200_EINVAL before anything is launched; n == 0 returns 0 and writes nothing; so do an
    emulated_edge_mc call with w == 0 or h == 0; a geom that is not 16-byte aligned is refused."""
    import torch
    import ffmpeg_b200 as fb
    from ffmpeg_b200._lib import lib
    L, dv = lib(), device.handle
    with on_stream(device):
        dst0 = torch.randint(0, 256, (4096,), dtype=torch.uint8, device="cuda")
        dst = dst0.clone()
        src = torch.randint(0, 256, (4096,), dtype=torch.uint8, device="cuda")
        off = torch.full((8,), 1024, dtype=torch.int64, device="cuda")
        u8 = torch.zeros(16, dtype=torch.uint8, device="cuda")
        geom = torch.tensor([[8, 8, 0, 0]] * 2, dtype=torch.int32, device="cuda")
        params = torch.tensor([[0 | 16 << 8, 1, 1, 0]] * 2, dtype=torch.int32, device="cuda")
        device.sync()
    p = lambda x: x.data_ptr()
    entries = {
        "qpel": (L.b200_h264qpel_batch_device, [p(u8), p(dst), p(off), p(src), p(off), 64]),
        "hpel": (L.b200_hpel_batch_device, [p(u8), p(u8), p(dst), p(off), p(src), p(off), 64]),
        "chroma": (L.b200_h264chroma_batch_device, [p(u8), p(u8), p(u8), p(dst), p(off), p(src), p(off), 64]),
        "weight": (L.b200_h264_weight_batch_device, [p(params), p(dst), p(off), p(src), p(off), 64]),
        "edge": (L.b200_emulated_edge_mc_batch_device, [p(dst), p(off), 64, p(src), p(off), 64, p(geom), 16, 16]),
    }
    for name, (fn, args) in entries.items():
        ptrs = [k for k, a in enumerate(args) if isinstance(a, int) and a > 4096]
        for k in ptrs:
            if name == "weight" and k == 3:
                continue                                                     # src NULL selects weight (not biweight)
            bad = list(args)
            bad[k] = None
            before = fb.launch_count()
            assert fn(dv, 2, *bad) == B200_EINVAL and fb.launch_count() == before, (name, k)
        before = fb.launch_count()
        assert fn(None, 2, *args) == B200_EINVAL and fn(dv, -1, *args) == B200_EINVAL and fb.launch_count() == before, name
        assert fn(dv, 0, *args) == 0 and fb.launch_count() == before, name
    before = fb.launch_count()
    edge, eargs = entries["edge"]
    assert edge(dv, 2, *eargs[:6], p(geom) + 4, 16, 16) == B200_EINVAL                       # geom not 16-byte aligned
    assert edge(dv, 2, *eargs[:7], 0, 16) == 0 and edge(dv, 2, *eargs[:7], 16, 0) == 0       # w == 0 / h == 0
    wfn, wargs = entries["weight"]
    assert wfn(dv, 2, p(params) + 4, *wargs[1:]) == B200_EINVAL                                # params not 16-byte aligned
    assert wfn(dv, 2, *wargs[:4], None, 64) == B200_EINVAL                                     # src without src_off
    assert fb.launch_count() == before
    device.sync()
    assert torch.equal(dst, dst0)


def test_undefined_op_codes_write_nothing(device):
    """Op codes naming a table entry the reference leaves NULL (qpel size index 3, hpel put_no_rnd at 4 and 2 wide and avg_no_rnd
    below 16 wide, chroma width index 3), interleaved with valid ops in one call: their blocks keep the sentinel, the valid ops
    around them match the checker."""
    from ffmpeg_b200 import pel
    rng = np.random.default_rng(11)
    # qpel: every third op undefined (all 32 of its codes), the rest drawn from the 96 valid ones
    n = 192
    ops = np.array([pel.qpel_op(int(rng.integers(0, 2)), 3 if i % 3 == 1 else int(rng.integers(0, 3)), int(rng.integers(0, 16)))
                    for i in range(n)], np.uint8)
    case = pel_layout_case("B", "random", [(16, 16)] * n, 1000, margin=(2, 3), cell=(32, 16), phases=rng.integers(0, 16, n))
    case["dst"].buf[:] = 0x5A
    exp = qpel_expected(case, ops)
    got = qpel_gpu(device, case, ops)
    assert_same(case, got, exp, "qpel")
    for o, do in zip(ops, case["doff"]):
        if (o >> 1) & 3 == 3:
            d = case["dst"]
            assert all((got[0][d.base + do + y * d.stride:][:2] == 0x5A).all() for y in range(2))
    # hpel: the undefined (table, size) pairs at every xy between defined ops
    und = [pel.hpel_op(tb, s, q) for tb, s in HPEL_UNDEFINED for q in range(4)]
    dfn = [pel.hpel_op(tb, s, q) for tb, s in HPEL_DEFINED for q in range(4)]
    op = np.array([x for pair in zip(und, dfn[:len(und)]) for x in pair], np.uint8)
    h = rng.choice(np.array([2, 4, 8, 9], np.uint8), len(op))
    case = pel_layout_case("C", "random", [(16 >> ((o >> 2) & 3), hh) for o, hh in zip(op, h)], 1100, margin=(0, 1), cell=(32, 16))
    case["dst"].buf[:] = 0x5A
    assert_same(case, hpel_gpu(device, case, op, h), hpel_expected(case, op, h), "hpel")
    # chroma: width index 3 (1 wide) between the defined widths, put and avg, every phase
    m = 256
    op = np.array([pel.chroma_op(i & 1, 3 if i % 4 == 2 else (i >> 2) % 3) for i in range(m)], np.uint8)
    h = rng.choice(np.array([2, 4, 8, 16], np.uint8), m)
    xy = (np.arange(m) % 64).astype(np.uint8)
    case = pel_layout_case("B", "random", [(max(1, 8 >> (o >> 1)), hh) for o, hh in zip(op, h)], 1200, margin=(0, 1), cell=(16, 16))
    case["dst"].buf[:] = 0x5A
    assert_same(case, chroma_gpu(device, case, op, h, xy), chroma_expected(case, op, h, xy), "chroma")
