"""GPU tier: the 9- to 14-bit H.264 kernels (csrc/pel_hbd.cu: qpel_hbd_kernel, chroma_hbd_kernel; csrc/h264weight.cu and
csrc/h264idct.cu: the uint16_t instances; csrc/videodsp.cu: edge_kernel<uint16_t>) and both instances of the deblocking kernel
(csrc/h264lf.cu) bit for bit against the checkers, in the plane layouts of tests/cases.py (aligned, odd sample strides with misaligned
bases, bottom-up), on random and extreme pictures, at the alignments, thresholds and batch lengths the kernels branch on, at depths 9, 10,
12 and 14 (and 8 for deblocking).  The last test deblocks a 1080p 4:2:0 frame with the schedule INTEGRATION.md gives the decoder.

Every call checks the whole destination allocation, slack included, against the checker applied to a copy of it, and checks that
the source allocation is unchanged."""
import ctypes as C

import numpy as np
import pytest

import cpulibs as cl
from cases import PEL_LAYOUTS, PelPlane, edge_windows, pel_layout_case, pel_picture
from test_oracle_hbd_layouts import idct_blocks, idct_layout, lib
from test_pel_paths_gpu import assert_same, on_stream, run_gpu

pytestmark = pytest.mark.gpu
B200_EINVAL, B200_ENOSYS = -22, -38
DEPTHS = (9, 10, 12, 14)
KINDS = ("random", "extremes")
GRID_PASS = 132 * 32 * 8           # qpel_hbd_kernel / chroma_hbd_kernel: 132 x 32 CTAs of 8 warps, one op per warp per trip


def orc():
    O, _ = lib("orc")
    O.orc_h264qpel_hbd_batch.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_ssize_t]
    return O


# ---------------------------------------------------------------------------------------------- qpel
def qpel_size(op):
    return 16 >> ((op >> 1) & 3)


def qpel_expected(case, ops, depth):
    """orc_h264qpel_hbd_batch over the ops that name a table of the reference (size index 3 writes nothing)"""
    src, dst = case["src"], case["dst"]
    exp = dst.buf.copy()
    ok = ((ops >> 1) & 3) != 3
    o, do, so = ops[ok].copy(), case["doff"][ok].copy(), case["soff"][ok].copy()
    orc().orc_h264qpel_hbd_batch(depth, len(o), o.ctypes.data, exp.ctypes.data + dst.base, do.ctypes.data, src.buf.ctypes.data + src.base,
                                 so.ctypes.data, src.stride)
    return exp


def qpel_gpu(device, case, ops, depth):
    from ffmpeg_b200 import pel
    return run_gpu(device, case, lambda s, d, t: pel.h264qpel_hbd_batch_device(device, depth, len(ops), t(ops), d, t(case["doff"]), s,
                                                                               t(case["soff"]), case["src"].stride))


@pytest.mark.parametrize("depth", DEPTHS)
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("layout", PEL_LAYOUTS)
def test_qpel_hbd_every_op_at_every_phase(device, layout, kind, depth):
    """All 128 op codes (the 32 at size index 3 included, which write nothing), each at the 8 even source byte phases mod 16, in one
    call in a shuffled order"""
    rng = np.random.default_rng(100 + 10 * PEL_LAYOUTS.index(layout) + depth)
    order = rng.permutation(128 * 8)
    ops = (order // 8).astype(np.uint8)                                 # op code = avg | size index << 1 | position << 3
    case = pel_layout_case(layout, kind, [(qpel_size(o),) * 2 for o in ops], 200 + depth, margin=(2, 3), cell=(32, 16),
                           phases=order % 8 * 2, depth=depth)
    assert_same(case, qpel_gpu(device, case, ops, depth), qpel_expected(case, ops, depth), (layout, kind, depth))


@pytest.mark.parametrize("depth", DEPTHS)
def test_qpel_hbd_batch_lengths(device, depth):
    """Layout B at batch lengths around a warp's op, a CTA's 8 and one pass of the capped grid (33,792 ops): the first n ops of one list"""
    rng = np.random.default_rng(7 + depth)
    N = GRID_PASS + 1
    ops = (rng.integers(0, 2, N) | rng.integers(0, 3, N) << 1 | rng.integers(0, 16, N) << 3).astype(np.uint8)
    case = pel_layout_case("B", "random", [(qpel_size(o),) * 2 for o in ops], 300 + depth, margin=(2, 3), cell=(32, 16),
                           phases=rng.integers(0, 8, N) * 2, depth=depth)
    for n in (1, 7, 8, 9, GRID_PASS - 1, GRID_PASS, GRID_PASS + 1):
        sub = dict(case, soff=case["soff"][:n], doff=case["doff"][:n])
        assert_same(sub, qpel_gpu(device, sub, ops[:n], depth), qpel_expected(sub, ops[:n], depth), (depth, n))


@pytest.mark.parametrize("depth", DEPTHS)
def test_qpel_hbd_1080p_plane_of_4x4(device, depth):
    """Every 4x4 block of a 1920x1088 destination, random op codes and vectors, odd sample stride: 130,560 ops, almost four passes"""
    rng = np.random.default_rng(8 + depth)
    n = 480 * 272
    ops = (rng.integers(0, 2, n) | 2 << 1 | rng.integers(0, 16, n) << 3).astype(np.uint8)
    case = pel_layout_case("B", "random", [(4, 4)] * n, 400 + depth, src_h=1088, margin=(2, 3), cell=(4, 4), cols=480, depth=depth)
    assert case["dst"].w == 1920 and case["dst"].h == 1088
    assert_same(case, qpel_gpu(device, case, ops, depth), qpel_expected(case, ops, depth), ("1080p", depth))


# ---------------------------------------------------------------------------------------------- chroma
def chroma_expected(case, op, h, xy, n=None):
    src, dst = case["src"], case["dst"]
    exp, O = dst.buf.copy(), orc()
    n = len(op) if n is None else n
    for o, hh, p, do, so in zip(op[:n].tolist(), h[:n].tolist(), xy[:n].tolist(), case["doff"][:n].tolist(), case["soff"][:n].tolist()):
        if (o >> 1) & 3 != 3:
            O.orc_h264chroma_hbd(o & 1, o >> 1, exp.ctypes.data + dst.base + do, src.buf.ctypes.data + src.base + so, src.stride, hh, p & 7, p >> 3)
    return exp


def chroma_gpu(device, case, op, h, xy, n=None):
    from ffmpeg_b200 import pel
    n = len(op) if n is None else n
    return run_gpu(device, case, lambda s, d, t: pel.h264chroma_hbd_batch_device(device, n, t(op), t(h), t(xy), d, t(case["doff"]), s,
                                                                                 t(case["soff"]), case["src"].stride))


@pytest.mark.parametrize("depth", DEPTHS)
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("layout", PEL_LAYOUTS)
def test_chroma_hbd_every_width_phase_height(device, layout, kind, depth):
    """Width indices 0 to 3 (3 writes nothing) x put / avg x all 64 eighth-pel positions x heights 1 to 16 (8192 ops, one call), on
    random and extreme pictures"""
    from ffmpeg_b200 import pel
    rng = np.random.default_rng(20 + 10 * PEL_LAYOUTS.index(layout) + depth)
    combos = [(pel.chroma_op(a, i), hh, p) for a in (0, 1) for i in range(4) for p in range(64) for hh in range(1, 17)]
    combos = [combos[k] for k in rng.permutation(len(combos))]
    op, h, xy = (np.array([c[k] for c in combos], np.uint8) for k in range(3))
    case = pel_layout_case(layout, kind, [(max(1, 8 >> (o >> 1)), hh) for o, hh in zip(op, h)], 500 + depth, margin=(0, 2),
                           cell=(16, 16), phases=rng.integers(0, 8, len(op)) * 2, depth=depth)
    assert_same(case, chroma_gpu(device, case, op, h, xy), chroma_expected(case, op, h, xy), (layout, kind, depth))


@pytest.mark.parametrize("depth", DEPTHS)
def test_chroma_hbd_batch_lengths(device, depth):
    """Layout B around a CTA's 8 ops and one pass of the capped grid (33,792 ops): the first n ops of one list"""
    from ffmpeg_b200 import pel
    N = GRID_PASS + 1
    rng = np.random.default_rng(9 + depth)
    op = (rng.integers(0, 2, N) | rng.integers(0, 3, N) << 1).astype(np.uint8)
    h = rng.choice(np.array([1, 2, 3, 4, 7, 8], np.uint8), N)
    xy = rng.integers(0, 64, N).astype(np.uint8)
    case = pel_layout_case("B", "random", [(8 >> (o >> 1), hh) for o, hh in zip(op, h)], 600 + depth, margin=(0, 2), cell=(16, 8), cols=256,
                           depth=depth)
    for n in (1, 7, 8, 9, GRID_PASS - 1, GRID_PASS, GRID_PASS + 1):
        assert_same(case, chroma_gpu(device, case, op, h, xy, n), chroma_expected(case, op, h, xy, n), (depth, n))


# ---------------------------------------------------------------------------------------------- weight / biweight
WEIGHTS = (-128, -1, 0, 1, 127)


def weight_expected(case, params, bi, depth, n=None):
    src, dst = case["src"], case["dst"]
    exp, O = dst.buf.copy(), orc()
    n = len(params) if n is None else n
    for (p0, wd, ws, off), do, so in zip(params[:n].tolist(), case["doff"][:n].tolist(), case["soff"][:n].tolist()):
        idx, hh, ld = p0 & 3, (p0 >> 8) & 255, (p0 >> 16) & 31
        if bi:
            O.orc_h264_biweight_hbd(depth, idx, exp.ctypes.data + dst.base + do, src.buf.ctypes.data + src.base + so, dst.stride, hh, ld, wd, ws, off)
        else:
            O.orc_h264_weight_hbd(depth, idx, exp.ctypes.data + dst.base + do, dst.stride, hh, ld, wd, off)
    return exp


def weight_gpu(device, case, params, bi, depth, n=None):
    from ffmpeg_b200 import pel
    n = len(params) if n is None else n
    return run_gpu(device, case, lambda s, d, t: pel.h264_weight_hbd_batch_device(device, depth, n, t(params), d, t(case["doff"]),
                                                                                  s if bi else None, t(case["soff"]) if bi else None,
                                                                                  case["dst"].stride))


def weight_params(bi, seed):
    from ffmpeg_b200 import pel
    geo = [(idx, hh, ld, off) for idx in range(4) for hh in (1, 2, 3, 4, 8, 16) for ld in range(8) for off in WEIGHTS]
    wts = [(wd, ws) for wd in WEIGHTS for ws in WEIGHTS] if bi else [(wd, 0) for wd in WEIGHTS]
    params = np.array([pel.weight_params(idx, hh, ld, wd, ws, off) for idx, hh, ld, off in geo for wd, ws in wts], np.int32)
    return params[np.random.default_rng(seed).permutation(len(params))]


def extremes_case(layout, params, seed, depth, **kw):
    case = pel_layout_case(layout, "extremes", [(16 >> (p & 3), (p >> 8) & 255) for p in params[:, 0]], seed, cell=(32, 16), depth=depth,
                           phases=np.random.default_rng(seed + 1).integers(0, 8, len(params)) * 2, **kw)
    dst = case["dst"]
    dst.fill(pel_picture("extremes", dst.h, dst.w, seed + 5, depth))        # both operands at the clip limits
    return case


@pytest.mark.parametrize("depth", DEPTHS)
@pytest.mark.parametrize("bi", [False, True], ids=["weight", "biweight"])
@pytest.mark.parametrize("layout", PEL_LAYOUTS)
def test_weight_hbd_every_parameter(device, layout, bi, depth):
    """Every width index x heights 1, 2, 3, 4, 8, 16 x log2_denom 0..7 x weights and offsets in {-128, -1, 0, 1, 127} (biweight: every
    pair of weights) on the extremes, one call: 4,800 / 24,000 blocks"""
    params = weight_params(bi, 800 + depth)
    case = extremes_case(layout, params, 810 + depth, depth)
    assert_same(case, weight_gpu(device, case, params, bi, depth), weight_expected(case, params, bi, depth), (layout, bi, depth))


@pytest.mark.parametrize("depth", DEPTHS)
def test_weight_hbd_word_alignment(device, depth):
    """Strides = 2, 4 and 6 mod 8 bytes (the 8-byte word path turns on and off from row to row), and biweight with the destination and
    the source at every pair of byte offsets mod 8 (destination aligned and source not, and the other way round).  Weights and offsets
    come from {-128, -1, 0, 1, 127} in odd ops and from the whole range -128..127 in even ones."""
    from ffmpeg_b200 import pel
    rng = np.random.default_rng(850 + depth)
    n = 4 * 6 * 16
    w8 = lambda i: int(rng.choice(WEIGHTS)) if i % 2 else int(rng.integers(-128, 128))
    params = np.array([pel.weight_params(i % 4, (1, 2, 3, 4, 8, 16)[i // 4 % 6], int(rng.integers(0, 8)), w8(i), w8(i), w8(i))
                       for i in range(n)], np.int32)
    i = np.arange(n)
    for extra in (2, 4, 6):
        w, h = 65 * 16, (n + 63) // 64 * 16 + 1                      # 64 cells of 16 samples per row, shifted by up to 3
        pitch = w * 2 + extra
        src = PelPlane("A", w, h, "src", 860 + depth, 2, pitch=pitch, mis=0).fill(pel_picture("extremes", h, w, 861, depth))
        dst = PelPlane("A", w, h, "dst", 862 + depth, 2, pitch=pitch, mis=0).fill(pel_picture("random", h, w, 863, depth))
        cx, cy = (i % 64) * 16, (i // 64) * 16
        case = dict(src=src, dst=dst, doff=dst.off(cx + i % 4, cy).astype(np.int64), soff=src.off(cx + i // 4 % 4, cy).astype(np.int64))
        for bi in (False, True):
            assert_same(case, weight_gpu(device, case, params, bi, depth), weight_expected(case, params, bi, depth), (extra, bi, depth))


@pytest.mark.parametrize("depth", DEPTHS)
def test_weight_hbd_batch_lengths(device, depth):
    """Layout B at batch lengths around one CTA's 4 blocks: the first n ops of one list"""
    params = weight_params(True, 870 + depth)[:5]
    case = extremes_case("B", params, 880 + depth, depth)
    for bi in (False, True):
        for n in (1, 3, 4, 5):
            assert_same(case, weight_gpu(device, case, params, bi, depth, n), weight_expected(case, params, bi, depth, n), (bi, n))


# ---------------------------------------------------------------------------------------------- residual add
@pytest.mark.parametrize("depth", DEPTHS)
def test_h264_idct_hbd_strides_shifts_and_extremes(device, depth):
    """All 4 kinds on coefficients at the int32 limits and the depth's transform range; strides = 0 and 8 mod 16 bytes, an odd sample
    count and a negative stride; destinations shifted by 0, 2 and 8 bytes; coefficient blocks 4-byte but not 16-byte aligned; batch
    lengths 127, 128 and 129 (one CTA of 128 threads and one more).  The destination and the cleared coefficients are compared."""
    import torch
    from ffmpeg_b200._lib import check, lib as blib, vp
    for kind in range(4):
        N, n = (64 if kind & 1 else 16), 129
        blocks = idct_blocks(depth, kind, n, 1000 * depth + kind)
        coef = np.random.default_rng(kind).integers(-50, 50, n * (N + 1) + 8).astype(np.int32)
        boff = (np.arange(n) * (N + 1) + 1).astype(np.int64)                 # block k at 4 + 4 (N + 1) k bytes
        for k in range(n):
            coef[boff[k]:boff[k] + N] = blocks[k]
        for si, stride in enumerate((256, 264, 258, -256)):
            buf, base, doff0 = idct_layout(depth, kind, stride, n, 2000 * depth + 10 * kind + si)
            for shift in (0, 2, 8):
                doff = doff0 + shift
                for m in (127, 128, 129):
                    exp, eb = buf.copy(), coef.copy()
                    for k in range(m):
                        orc().orc_h264_idct_hbd(depth, kind, exp.ctypes.data + base + int(doff[k]), eb.ctypes.data + 4 * int(boff[k]), stride)
                    with on_stream(device):
                        d_p, d_b = torch.from_numpy(buf).cuda(), torch.from_numpy(coef).cuda()
                        d_bo, d_do = torch.from_numpy(boff).cuda(), torch.from_numpy(doff).cuda()
                        check(blib().b200_h264_idct_hbd_batch_device(device.handle, depth, kind, m, vp(d_b.data_ptr()), vp(d_bo.data_ptr()),
                                                                     vp(d_p.data_ptr() + base), vp(d_do.data_ptr()), stride), "h264_idct_hbd")
                        device.sync()
                        got, gb = d_p.cpu().numpy(), d_b.cpu().numpy()
                    assert np.array_equal(got, exp), (kind, stride, shift, m, int((got != exp).sum()))
                    assert np.array_equal(gb, eb), (kind, stride, shift, m, "coefficients")


# ---------------------------------------------------------------------------------------------- emulated_edge_mc
@pytest.mark.parametrize("sign", [1, -1], ids=["top_down", "bottom_up"])
@pytest.mark.parametrize("pic", [(1, 1), (1, 37), (37, 1), (100, 60)])
def test_emulated_edge_mc_hbd_windows(device, pic, sign):
    """Windows up to 80x80 (so that the 32-lane column loop takes three trips) from three pictures in one call, at an odd sample line
    size and misaligned bases, written at an odd sample buffer line size; bottom_up: both line sizes negative.  Samples below
    1 << depth for each depth (the kernel itself has no depth)."""
    import torch
    from ffmpeg_b200 import pel
    W, H = pic
    NF, LS, BLS = 3, ((W + 13) | 1) * 2, 83 * 2
    geom = np.array(edge_windows(W, H), np.int32)
    n = len(geom)
    for depth in DEPTHS:
        rng = np.random.default_rng(W * 100 + H + depth)
        fbytes = LS * H + 6
        pics = rng.integers(0, 1 << depth, (64 + NF * fbytes + 64) // 2).astype(np.uint16).view(np.uint8)
        fr = rng.integers(0, NF, n)
        origin = (64 + 2 + fr * fbytes + (0 if sign > 0 else (H - 1) * LS)).astype(np.int64)   # sample (0, 0) of the window's picture
        slot = 80 * BLS
        boff = (64 + np.arange(n) * slot + (0 if sign > 0 else 79 * BLS)).astype(np.int64)     # row 0 of window i
        buf0 = rng.integers(0, 256, 64 + n * slot + 64, dtype=np.uint8)
        exp = buf0.copy()
        for (bw, bh, sx, sy), o, b in zip(geom.tolist(), origin.tolist(), boff.tolist()):
            orc().orc_emulated_edge_mc_hbd(exp.ctypes.data + b, pics.ctypes.data + o + sy * sign * LS + sx * 2, sign * BLS, sign * LS, bw, bh,
                                           sx, sy, W, H)
        with on_stream(device):
            d_buf, d_pics = torch.from_numpy(buf0).cuda(), torch.from_numpy(pics).cuda()
            pel.emulated_edge_mc_hbd_batch_device(device, n, d_buf, torch.from_numpy(boff).cuda(), sign * BLS, d_pics,
                                                  torch.from_numpy(origin).cuda(), sign * LS, torch.from_numpy(geom).cuda(), W, H)
            device.sync()
            got = d_buf.cpu().numpy()
            assert np.array_equal(d_pics.cpu().numpy(), pics)
        assert np.array_equal(got, exp), (depth, int((got != exp).sum()))


# ---------------------------------------------------------------------------------------------- deblocking
def lf_gpu(device, depth, n, kinds, buf, off, stride, alpha, beta, tc0, base=0):
    """the batched entry of the depth on a copy of the allocation `buf` (pix = its address + base); returns the allocation after it"""
    import torch
    from ffmpeg_b200._lib import check, lib as blib, vp
    with on_stream(device):
        dp = torch.from_numpy(buf).cuda()
        d = [torch.from_numpy(np.ascontiguousarray(v)).cuda() for v in (kinds, off, alpha, beta, tc0)]
        p = [vp(x.data_ptr()) for x in d]
        if depth == 8:
            r = blib().b200_h264_loop_filter_batch_device(device.handle, n, p[0], vp(dp.data_ptr() + base), p[1], stride, p[2], p[3], p[4])
        else:
            r = blib().b200_h264_loop_filter_hbd_batch_device(device.handle, depth, n, p[0], vp(dp.data_ptr() + base), p[1], stride, p[2], p[3], p[4])
        check(r, "h264_loop_filter_batch")
        device.sync()
        return dp.cpu().numpy()


def lf_orc(depth, buf, base, stride, kinds, off, alpha, beta, tc0):
    """the checker edge by edge, in list order, on a copy of the allocation"""
    out = buf.copy()
    f = cl.oracle().orc_h264_loop_filter if depth == 8 else cl.oracle().orc_h264_loop_filter_hbd
    f.argtypes = ([] if depth == 8 else [C.c_int]) + [C.c_int, C.c_void_p, C.c_ssize_t, C.c_int, C.c_int, C.c_void_p]
    d = () if depth == 8 else (depth,)
    for e in range(len(kinds)):
        t = np.ascontiguousarray(tc0[e])
        assert f(*d, int(kinds[e]), out.ctypes.data + base + int(off[e]), stride, int(alpha[e]), int(beta[e]), t.ctypes.data) == 0
    return out


def relayout(pic, off, seed):
    """the case picture in a noise allocation at an odd stride (bytes at depth 8, samples above) and an odd base (+2 bytes above):
    (allocation, base, stride, offsets)"""
    h, w = pic.shape
    bps = pic.itemsize
    stride = (w + 7) * bps
    base = 64 + (3 if bps == 1 else 2)
    buf = np.random.default_rng(seed).integers(0, 256, base + h * stride + 64, dtype=np.uint8)
    for y in range(h):
        buf[base + y * stride:][:w * bps] = pic[y].view(np.uint8)
    row, col = off // pic.strides[0], off % pic.strides[0] // bps
    return buf, base, stride, (row * stride + col * bps).astype(np.int64)


@pytest.mark.parametrize("depth", (8,) + DEPTHS)
def test_loop_filter_at_thresholds(device, depth):
    """1024 edges of all 16 kinds whose lines sit on both sides of every threshold after the depth scaling (cpulibs.h264lf_threshold_case),
    at an odd stride and an odd base, through the 8-bit entry at depth 8 and the 16-bit one above"""
    pic, kinds, off, alpha, beta, tc0 = cl.h264lf_threshold_case(300 + depth, 1024, depth)
    buf, base, stride, off = relayout(pic, off, depth)
    exp = lf_orc(depth, buf, base, stride, kinds, off, alpha, beta, tc0)
    got = lf_gpu(device, depth, len(kinds), kinds, buf, off, stride, alpha, beta, tc0, base)
    assert not np.array_equal(exp, buf)
    assert np.array_equal(got, exp), int((got != exp).sum())


@pytest.mark.parametrize("depth", (8,) + DEPTHS)
def test_loop_filter_batch_lengths(device, depth):
    """Batch lengths around one CTA's 8 edges (1, 7, 8, 9) and 65,537 edges (4,097 CTAs), random content"""
    for n, cols in ((9, 16), (65537, 256)):
        pic, kinds, off, alpha, beta, tc0 = (cl.h264lf_case(500, n, cols) if depth == 8 else cl.h264lf_hbd_case(500, n, depth, cols))
        buf = pic.view(np.uint8).reshape(-1)
        stride = pic.strides[0]
        for m in ((1, 7, 8, 9) if n == 9 else (n,)):
            exp = lf_orc(depth, buf, 0, stride, kinds[:m], off[:m], alpha[:m], beta[:m], tc0[:m])
            got = lf_gpu(device, depth, m, kinds[:m], buf, off[:m], stride, alpha[:m], beta[:m], tc0[:m])
            assert np.array_equal(got, exp), (depth, m, int((got != exp).sum()))


def frame_edges(depth, seed, W=1920, H=1088):
    """A 4:2:0 frame (three uint8 / uint16 planes with blocky content) and the edges a decoder filters: per macroblock, luma vertical
    edges 0-3 then horizontal edges 0-3 (edge 0 intra in intra macroblocks, the picture's left and top borders not filtered, one edge in
    five with bS 0 left out), and the same at chroma edges 0 and 2.  Returns (planes, strides, edges) with edges a list of
    (plane, mb_x, mb_y, dir, pos, kind, offset in bytes, alpha, beta, tc0[4]) in the decoder's order."""
    rng = np.random.default_rng(seed)
    sh, mx = depth - 8, (1 << depth) - 1
    dt, bps = (np.uint8, 1) if depth == 8 else (np.uint16, 2)
    planes, strides = [], []
    for p, (w, h, bs) in enumerate(((W, H, 4), (W // 2, H // 2, 2), (W // 2, H // 2, 2))):
        lvl = np.cumsum(rng.integers(-6, 7, (h // bs, w // bs)), axis=1) + int(rng.integers(60, 196))
        pic = (np.kron(lvl, np.ones((bs, bs), np.int64)) << sh) + rng.integers(-(2 << sh), (2 << sh) + 1, (h, w))
        stride = (w + 32) * bps
        full = np.zeros((h, w + 32), dt)
        full[:, :w] = pic.clip(0, mx)
        planes.append(full)
        strides.append(stride)
    edges = []
    for my in range(H // 16):
        for mx_ in range(W // 16):
            intra = rng.random() < 0.3
            a, b = int(rng.integers(16, 256)), int(rng.integers(2, 19))
            for p in range(3):
                size, step = (16, 4) if p == 0 else (8, 2)
                x0, y0 = mx_ * size, my * size
                for dr in (0, 1):                                     # 0: vertical edges (filtered across x), 1: horizontal edges
                    for pos in ((0, 1, 2, 3) if p == 0 else (0, 2)):
                        if pos == 0 and (mx_ if dr == 0 else my) == 0:
                            continue
                        if pos and rng.random() < 0.2:
                            continue
                        e0 = pos == 0 and intra
                        if p == 0:
                            kind = (4 if e0 else 1) if dr == 0 else (3 if e0 else 0)
                        else:
                            kind = (10 if e0 else 7) if dr == 0 else (9 if e0 else 6)
                        x, y = (x0 + pos * step, y0) if dr == 0 else (x0, y0 + pos * step)
                        tc = rng.integers(-1, 26, 4).astype(np.int8)
                        edges.append((p, mx_, my, dr, pos, kind, y * strides[p] + x * bps, a, b, tc))
    return planes, strides, edges


@pytest.mark.parametrize("depth", (8, 10))
def test_loop_filter_frame_schedule(device, depth):
    """A 1920x1088 4:2:0 frame deblocked the way INTEGRATION.md tells the decoder to: one batch call per plane and key (macroblock
    anti-diagonal mb_x + 2 mb_y, vertical edges 0-3 before horizontal edges 0-3) in key order, against the checker applied edge by edge
    in the decoder's order (macroblocks in raster order, each one's vertical edges and then its horizontal edges)"""
    planes, strides, edges = frame_edges(depth, 1200 + depth)
    exp = []
    for p in range(3):
        es = [e for e in edges if e[0] == p]
        cols = list(zip(*es))
        exp.append(lf_orc(depth, planes[p].view(np.uint8).reshape(-1), 0, strides[p], np.array(cols[5], np.uint8), np.array(cols[6], np.int64),
                          np.array(cols[7], np.uint8), np.array(cols[8], np.uint8), np.stack(cols[9])))
    import torch
    from ffmpeg_b200._lib import check, lib as blib, vp
    got = []
    for p in range(3):
        es = sorted((e for e in edges if e[0] == p), key=lambda e: (e[1] + 2 * e[2], e[3], e[4]))
        keys = np.array([(e[1] + 2 * e[2]) * 8 + e[3] * 4 + e[4] for e in es])
        starts = np.flatnonzero(np.r_[True, keys[1:] != keys[:-1]])
        ends = np.r_[starts[1:], len(es)]
        cols = list(zip(*es))
        arrs = [np.array(cols[5], np.uint8), np.array(cols[6], np.int64), np.array(cols[7], np.uint8), np.array(cols[8], np.uint8),
                np.stack(cols[9])]
        with on_stream(device):
            dp = torch.from_numpy(planes[p].view(np.uint8).reshape(-1).copy()).cuda()
            dk, do, da, db, dt = (torch.from_numpy(a).cuda() for a in arrs)
            for s, e in zip(starts.tolist(), ends.tolist()):
                args = (e - s, vp(dk.data_ptr() + s), vp(dp.data_ptr()), vp(do.data_ptr() + 8 * s), strides[p], vp(da.data_ptr() + s),
                        vp(db.data_ptr() + s), vp(dt.data_ptr() + 4 * s))
                check(blib().b200_h264_loop_filter_batch_device(device.handle, *args) if depth == 8 else
                      blib().b200_h264_loop_filter_hbd_batch_device(device.handle, depth, *args), "h264_loop_filter_batch")
            device.sync()
            got.append(dp.cpu().numpy())
    for p in range(3):
        assert not np.array_equal(exp[p], planes[p].view(np.uint8).reshape(-1)), p
        assert np.array_equal(got[p], exp[p]), (p, int((got[p] != exp[p]).sum()))


# ---------------------------------------------------------------------------------------------- refusals
def test_hbd_refusals_launch_nothing(device):
    """Odd strides, odd bases, unsupported depths, n < 0 and negative deblocking strides are refused before anything is launched;
    n == 0 returns 0 and launches nothing"""
    import torch
    import ffmpeg_b200 as fb
    from ffmpeg_b200._lib import lib as blib
    L, dv = blib(), device.handle
    with on_stream(device):
        dst0 = torch.randint(0, 1024, (4096,), dtype=torch.int16, device="cuda")
        dst = dst0.clone()
        src = torch.randint(0, 1024, (4096,), dtype=torch.int16, device="cuda")
        off = torch.full((8,), 1024, dtype=torch.int64, device="cuda")
        u8 = torch.zeros(16, dtype=torch.uint8, device="cuda")
        i32 = torch.tensor([[0 | 16 << 8, 1, 1, 0]] * 2, dtype=torch.int32, device="cuda")
        coef = torch.zeros(256, dtype=torch.int32, device="cuda")
        device.sync()
    p = lambda x: x.data_ptr()
    D, S = p(dst), p(src)
    # (entry, args before n, args after n, index of the stride / base in the full argument list, depth index or None)
    entries = {
        "qpel": (L.b200_h264qpel_hbd_batch_device, [10], [p(u8), D, p(off), S, p(off), 64]),
        "chroma": (L.b200_h264chroma_hbd_batch_device, [], [p(u8), p(u8), p(u8), D, p(off), S, p(off), 64]),
        "weight": (L.b200_h264_weight_hbd_batch_device, [10], [p(i32), D, p(off), S, p(off), 64]),
        "idct": (L.b200_h264_idct_hbd_batch_device, [10, 0], [p(coef), p(off), D, p(off), 64]),
        "edge": (L.b200_emulated_edge_mc_hbd_batch_device, [], [D, p(off), 64, S, p(off), 64, p(i32), 16, 16]),
        "deblock": (L.b200_h264_loop_filter_hbd_batch_device, [10], [p(u8), D, p(off), 64, p(u8), p(u8), p(u8)]),
    }
    bad_stride = {"qpel": [5], "chroma": [7], "weight": [5], "idct": [4], "edge": [2, 5], "deblock": [3]}
    bad_base = {"qpel": [1, 3], "chroma": [3, 5], "weight": [1, 3], "idct": [2], "edge": [0, 3], "deblock": [1]}
    before = fb.launch_count()
    for name, (fn, pre, args) in entries.items():
        for k in bad_stride[name]:
            a = list(args)
            a[k] += 1
            assert fn(dv, *pre, 2, *a) == B200_EINVAL, (name, "odd stride", k)
        for k in bad_base[name]:
            a = list(args)
            a[k] += 1
            assert fn(dv, *pre, 2, *a) == B200_EINVAL, (name, "odd base", k)
        if pre:
            for dep in (8, 11, 16):
                assert fn(dv, *([dep] + pre[1:]), 2, *args) == B200_ENOSYS, (name, dep)
        assert fn(dv, *pre, -1, *args) == B200_EINVAL, (name, "n < 0")
        assert fn(dv, *pre, 0, *args) == 0, (name, "n == 0")
    fn, pre, args = entries["deblock"]
    a = list(args)
    a[3] = -64
    assert fn(dv, *pre, 2, *a) == B200_EINVAL
    assert L.b200_h264_loop_filter_batch_device(dv, 2, p(u8), D, p(off), -64, p(u8), p(u8), p(u8)) == B200_EINVAL
    assert L.b200_h264_loop_filter_batch_device(dv, -1, p(u8), D, p(off), 64, p(u8), p(u8), p(u8)) == B200_EINVAL
    assert L.b200_h264_loop_filter_batch_device(dv, 0, p(u8), D, p(off), 64, p(u8), p(u8), p(u8)) == 0
    assert fb.launch_count() == before
    device.sync()
    assert torch.equal(dst, dst0)
