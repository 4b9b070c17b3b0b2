"""CPU tier: pin the 9- to 14-bit H.264 checkers (orc_h264qpel_hbd, orc_h264chroma_hbd, orc_h264_weight_hbd / orc_h264_biweight_hbd,
orc_h264_idct_hbd, orc_emulated_edge_mc_hbd) and both deblocking checkers (orc_h264_loop_filter, orc_h264_loop_filter_hbd) to the
compiled reference on the domain tests/test_h264_hbd_paths_gpu.py uses: uint16 planes with odd sample strides and misaligned bases
(layout B), bottom-up planes (layout C), extreme pictures, coefficients at the int32 limits, and deblocking lines on both sides of every
threshold.  Where oracle/_ref is built every comparison runs live; elsewhere the results are checked against the reference's digests in
tests/golden/hbd_layout_ref_digests.json (written by scripts/gen_hbd_layout_digests.py)."""
import ctypes as C
import os

import numpy as np
import pytest

import cpulibs as cl
from cases import edge_windows, pel_layout_case

DIGESTS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "hbd_layout_ref_digests.json")
DEPTHS = (9, 10, 12, 14)
CASES = [(layout, kind) for layout in ("B", "C") for kind in ("random", "extremes")]
WEIGHTS = (-128, -1, 0, 1, 127)
VP, SS, I = C.c_void_p, C.c_ssize_t, C.c_int


def lib(which):
    """the checker (cl.oracle(), "orc") or the reference (cl.ref(), "ffref") with the argument types of its 16-bit functions set"""
    L, pre = (cl.oracle(), "orc") if which == "orc" else (cl.ref(), "ffref")
    d = [I] if pre == "ffref" else []                                  # the reference's chroma and its weights take the depth first
    getattr(L, pre + "_h264qpel_hbd").argtypes = [I, I, I, I, VP, VP, SS]
    getattr(L, pre + "_h264chroma_hbd").argtypes = d + [I, I, VP, VP, SS, I, I, I]
    getattr(L, pre + "_h264_weight_hbd").argtypes = [I, I, VP, SS, I, I, I, I]
    getattr(L, pre + "_h264_biweight_hbd").argtypes = [I, I, VP, VP, SS, I, I, I, I, I]
    getattr(L, pre + "_h264_idct_hbd").argtypes = [I, I, VP, VP, SS]
    getattr(L, pre + "_emulated_edge_mc_hbd").argtypes = [VP, VP, SS, SS] + [I] * 6
    getattr(L, pre + "_emulated_edge_mc_hbd").restype = None
    return L, pre


def both(buf, fn):
    """fn(lib, prefix, copy) applied to two copies of an allocation: (the checker's result, thunk for the reference's)"""
    ours = buf.copy()
    fn(*lib("orc"), ours)

    def theirs():
        b = buf.copy()
        fn(*lib("ffref"), b)
        return b
    return ours, theirs


@pytest.mark.parametrize("depth", DEPTHS)
@pytest.mark.parametrize("layout,kind", CASES)
def test_qpel_hbd_oracle_vs_ref_on_layouts(layout, kind, depth):
    """All 96 op codes the reference defines, each at the 8 even source byte phases mod 16"""
    ops = [(a, s, p) for a in (0, 1) for s in range(3) for p in range(16)]
    ops = [o for o in ops for _ in range(8)]
    phases = np.tile(np.arange(8) * 2, 96)
    case = pel_layout_case(layout, kind, [(16 >> s,) * 2 for _, s, _ in ops], 51 + depth, margin=(2, 3), cell=(32, 16), phases=phases,
                           depth=depth)
    src, dst = case["src"], case["dst"]

    def run(L, pre, buf):
        f = getattr(L, pre + "_h264qpel_hbd")
        for (a, s, p), do, so in zip(ops, case["doff"].tolist(), case["soff"].tolist()):
            f(depth, a, s, p, buf.ctypes.data + dst.base + do, src.buf.ctypes.data + src.base + so, src.stride)
    with cl.RefCheck(DIGESTS) as rc:
        ours, theirs = both(dst.buf, run)
        assert rc.same(ours, theirs), (layout, kind, depth)


@pytest.mark.parametrize("layout,kind", CASES)
def test_chroma_hbd_oracle_vs_ref_on_layouts(layout, kind):
    """Widths 8, 4, 2 x put / avg x all 64 eighth-pel positions, heights 1 to 16 in rotation, at depths 9, 10, 12 and 14"""
    rng = np.random.default_rng(60)
    ops = [(a, i, xy, 1 + (xy + 5 * i + a) % 16) for a in (0, 1) for i in range(3) for xy in range(64)]
    with cl.RefCheck(DIGESTS) as rc:
        for depth in DEPTHS:
            case = pel_layout_case(layout, kind, [(8 >> i, h) for _, i, _, h in ops], 61 + depth, margin=(0, 1), depth=depth,
                                   phases=rng.integers(0, 8, len(ops)) * 2)
            src, dst = case["src"], case["dst"]

            def run(L, pre, buf):
                f = getattr(L, pre + "_h264chroma_hbd")
                d = (depth,) if pre == "ffref" else ()
                for (a, i, xy, h), do, so in zip(ops, case["doff"].tolist(), case["soff"].tolist()):
                    assert f(*d, a, i, buf.ctypes.data + dst.base + do, src.buf.ctypes.data + src.base + so, src.stride, h, xy & 7, xy >> 3) == 0
            ours, theirs = both(dst.buf, run)
            assert rc.same(ours, theirs), depth


@pytest.mark.parametrize("depth", DEPTHS)
@pytest.mark.parametrize("layout", ["B", "C"])
def test_weight_hbd_oracle_vs_ref_on_layouts(layout, depth):
    """Every width index x heights 1, 2, 3, 4, 8, 16 x log2_denom 0..7 x weights and offsets in {-128, -1, 0, 1, 127} on extreme
    pictures; biweight takes the source weights in rotation.  The source phase is drawn apart from the destination's jittered one."""
    from cases import pel_picture
    prm = [(idx, h, ld, wd, WEIGHTS[(idx + h + ld + k) % 5], off) for idx in range(4) for h in (1, 2, 3, 4, 8, 16) for ld in range(8)
           for k, wd in enumerate(WEIGHTS) for off in WEIGHTS]
    rng = np.random.default_rng(70 + depth)
    case = pel_layout_case(layout, "extremes", [(16 >> p[0], p[1]) for p in prm], 71 + depth, cell=(32, 16), depth=depth,
                           phases=rng.integers(0, 8, len(prm)) * 2)
    src, dst = case["src"], case["dst"]
    dst.fill(pel_picture("extremes", dst.h, dst.w, 72 + depth, depth))

    def run(bi):
        def go(L, pre, buf):
            for (idx, h, ld, wd, ws, off), do, so in zip(prm, case["doff"].tolist(), case["soff"].tolist()):
                if bi:
                    getattr(L, pre + "_h264_biweight_hbd")(depth, idx, buf.ctypes.data + dst.base + do, src.buf.ctypes.data + src.base + so,
                                                            dst.stride, h, ld, wd, ws, off)
                else:
                    getattr(L, pre + "_h264_weight_hbd")(depth, idx, buf.ctypes.data + dst.base + do, dst.stride, h, ld, wd, off)
        return go
    with cl.RefCheck(DIGESTS) as rc:
        for bi in (False, True):
            ours, theirs = both(dst.buf, run(bi))
            assert rc.same(ours, theirs), bi


IDCT_STRIDES = (256, 264, 258, -256)           # bytes: = 0, 8 and 2 mod 16, and the first one bottom-up


def idct_blocks(depth, kind, n, seed):
    """n int32 coefficient blocks: every coefficient drawn from INT32_MIN, INT32_MAX, +-2^(depth + 6), 0 and random values of three
    magnitudes; one block in seven DC only, like the decoder's"""
    rng = np.random.default_rng(seed)
    N = 64 if kind & 1 else 16
    lim = 1 << (depth + 6)
    special = np.array([-(1 << 31), (1 << 31) - 1, lim, -lim, 0], np.int64)
    pick = rng.integers(0, 8, (n, N))
    rand = [rng.integers(-m, m, (n, N)) for m in (300, lim, 1 << 30)]
    b = np.select([pick < 5, pick == 5, pick == 6], [special[np.minimum(pick, 4)], rand[0], rand[1]], rand[2]).astype(np.int32)
    b[::7, 1:] = 0
    return b


def idct_layout(depth, kind, stride, n, seed):
    """(noise allocation, base, pixel offsets): n blocks on a grid of 10 x 8-sample cells, each at an x jitter of 0..2 samples, in a
    plane of `stride` bytes (bottom-up when negative) filled with random samples"""
    rng = np.random.default_rng(seed)
    B, cols = (8 if kind & 1 else 4), 12
    rows = (n + cols - 1) // cols
    h, pitch = rows * B, abs(stride)
    base = 64 + ((h - 1) * pitch if stride < 0 else 0)
    buf = rng.integers(0, 256, 128 + h * pitch, dtype=np.uint8)
    for y in range(h):
        buf[base + y * stride:][:pitch - 2].view(np.uint16)[:] = rng.integers(0, 1 << depth, (pitch - 2) // 2)
    i = np.arange(n)
    doff = (i // cols) * B * stride + ((i % cols) * (B + 2) + rng.integers(0, 3, n)) * 2
    return buf, base, doff.astype(np.int64)


@pytest.mark.parametrize("depth", DEPTHS)
def test_h264_idct_hbd_oracle_vs_ref_extremes(depth):
    """All 4 kinds on coefficients at the int32 limits and the depth's transform range, at strides = 0, 8 and 2 mod 16 bytes and a
    negative one; the destination and the cleared coefficients both compared"""
    with cl.RefCheck(DIGESTS) as rc:
        for kind in range(4):
            for si, stride in enumerate(IDCT_STRIDES):
                n = 96
                blocks = idct_blocks(depth, kind, n, 100 * depth + 10 * kind + si)
                buf, base, doff = idct_layout(depth, kind, stride, n, 200 * depth + 10 * kind + si)
                N = blocks.shape[1]

                def run(L, pre, which):
                    b, p = blocks.copy(), buf.copy()
                    f = getattr(L, pre + "_h264_idct_hbd")
                    for k in range(n):
                        assert f(depth, kind, p.ctypes.data + base + int(doff[k]), b.ctypes.data + 4 * N * k, stride) == 0
                    return [p, b]
                ours = run(*lib("orc"), None)
                assert rc.same(ours, lambda: run(*lib("ffref"), None)), (kind, stride)


def test_emulated_edge_mc_hbd_oracle_vs_ref_on_new_pictures():
    """cases.edge_windows on 1x1, 1x37, 37x1 and 100x60 pictures at an odd sample line size, written at an odd sample buffer line size;
    then the same with both line sizes negative (pictures and windows stored bottom-up), as tests/test_h264_hbd_paths_gpu.py runs them"""
    with cl.RefCheck(DIGESTS) as rc:
        for sign in (1, -1):
            for W, H in ((1, 1), (1, 37), (37, 1), (100, 60)):
                LS, BLS = ((W + 13) | 1) * 2, 83 * 2
                pic = np.random.default_rng(W * 100 + H).integers(0, 1 << 14, (H, LS // 2)).astype(np.uint16)
                row0 = pic.ctypes.data + (0 if sign > 0 else (H - 1) * LS)                  # picture row 0
                for bw, bh, sx, sy in edge_windows(W, H):
                    src = row0 + sy * sign * LS + sx * 2

                    def run(L, pre, _):
                        b = np.full((80, BLS // 2), 7, np.uint16)
                        out = b.ctypes.data + (0 if sign > 0 else 79 * BLS)                 # window row 0
                        getattr(L, pre + "_emulated_edge_mc_hbd")(out, src, sign * BLS, sign * LS, bw, bh, sx, sy, W, H)
                        return b
                    assert rc.same(run(*lib("orc"), None), lambda: run(*lib("ffref"), None)), (sign, W, H, bw, bh, sx, sy)


@pytest.mark.parametrize("depth", (8, 9, 10, 12, 14))
def test_loop_filter_oracle_vs_ref_at_thresholds(depth):
    """1024 edges of all 16 kinds whose lines sit on both sides of every threshold (cpulibs.h264lf_threshold_case), through the
    8-bit checker at depth 8 and the 16-bit one above"""
    case = cl.h264lf_threshold_case(300 + depth, 1024, depth)
    orc, ref = (cl.orc_h264lf, cl.ref_h264lf) if depth == 8 else (lambda *a: cl.orc_h264lf_hbd(depth, *a), lambda *a: cl.ref_h264lf_hbd(depth, *a))
    with cl.RefCheck(DIGESTS) as rc:
        ours = orc(*case)
        assert not np.array_equal(ours, case[0])
        assert rc.same(ours, lambda: ref(*case))
