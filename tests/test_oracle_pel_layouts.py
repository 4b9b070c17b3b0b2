"""CPU tier: pin the 8-bit motion-compensation checker (orc_h264qpel, orc_hpel, orc_h264chroma, orc_emulated_edge_mc,
orc_h264_weight / orc_h264_biweight) to the compiled reference on the domain tests/test_pel_paths_gpu.py uses: odd strides with
misaligned bases (layout B), bottom-up planes (layout C), the heights outside the decoders' usual set and the extreme pictures.
Where oracle/_ref is built every comparison runs live; elsewhere the results are checked against the reference's digests in
tests/golden/pel_layout_ref_digests.json (written by scripts/gen_pel_layout_digests.py)."""
import ctypes as C
import os

import numpy as np
import pytest

import cpulibs as cl
from cases import HPEL_DEFINED, edge_windows, pel_layout_case

DIGESTS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "pel_layout_ref_digests.json")
ODD_H = (1, 3, 7, 9, 15)
CASES = [(layout, kind) for layout in ("B", "C") for kind in ("random", "extremes")]


def u8at(a, off):
    return C.cast(a.ctypes.data + int(off), cl.u8p)


def both(case, fn):
    """fn(lib, prefix, dst_buf) applied to two copies of the destination allocation: (checker's, reference's thunk)"""
    ours = case["dst"].buf.copy()
    fn(cl.oracle(), "orc", ours)

    def theirs():
        b = case["dst"].buf.copy()
        fn(cl.ref(), "ffref", b)
        return b
    return ours, theirs


@pytest.mark.parametrize("layout,kind", CASES)
def test_qpel_oracle_vs_ref_on_layouts(layout, kind):
    rng = np.random.default_rng(40)
    ops = [(a, s, p) for a in (0, 1) for s in range(3) for p in range(16)] * 2
    case = pel_layout_case(layout, kind, [(16 >> s,) * 2 for _, s, _ in ops], 41, margin=(2, 3), cell=(32, 16),
                           phases=rng.integers(0, 16, len(ops)))
    src, dst = case["src"], case["dst"]

    def run(L, pre, buf):
        f = getattr(L, pre + "_h264qpel")
        for (a, s, p), do, so in zip(ops, case["doff"].tolist(), case["soff"].tolist()):
            f(a, s, p, u8at(buf, dst.base + do), u8at(src.buf, src.base + so), src.stride)
    with cl.RefCheck(DIGESTS) as rc:
        ours, theirs = both(case, run)
        assert rc.same(ours, theirs)


@pytest.mark.parametrize("layout,kind", CASES)
def test_chroma_oracle_vs_ref_on_layouts(layout, kind):
    rng = np.random.default_rng(42)
    ops = [(a, i, xy, ODD_H[(xy + i) % len(ODD_H)]) for a in (0, 1) for i in range(3) for xy in range(64)]
    case = pel_layout_case(layout, kind, [(8 >> i, h) for _, i, _, h in ops], 43, margin=(0, 1), phases=rng.integers(0, 16, len(ops)))
    src, dst = case["src"], case["dst"]

    def run(L, pre, buf):
        f = getattr(L, pre + "_h264chroma")
        for (a, i, xy, h), do, so in zip(ops, case["doff"].tolist(), case["soff"].tolist()):
            assert f(a, i, u8at(buf, dst.base + do), u8at(src.buf, src.base + so), src.stride, h, xy & 7, xy >> 3) == 0
    with cl.RefCheck(DIGESTS) as rc:
        ours, theirs = both(case, run)
        assert rc.same(ours, theirs)


@pytest.mark.parametrize("layout,kind", CASES)
def test_hpel_oracle_vs_ref_on_layouts(layout, kind):
    """The xy2 functions (xy = 3) of the reference compute two rows per step (hpeldsp.c:134-330): an odd h is outside their domain
    (hpeldsp.h:34-38) and they write h + 1 rows.  The checker and the kernel write h rows; the pin covers odd heights for the other
    positions and even heights for xy2."""
    rng = np.random.default_rng(44)
    ops = [(tb, s, q, h) for tb, s in HPEL_DEFINED for q in range(4) for h in ((2, 4, 8, 16) if q == 3 else ODD_H + (16,))]
    case = pel_layout_case(layout, kind, [(16 >> s, h) for _, s, _, h in ops], 45, margin=(0, 1), cell=(32, 16),
                           phases=rng.integers(0, 16, len(ops)))
    src, dst = case["src"], case["dst"]

    def run(L, pre, buf):
        f = getattr(L, pre + "_hpel")
        for (tb, s, q, h), do, so in zip(ops, case["doff"].tolist(), case["soff"].tolist()):
            assert f(tb, s, q, u8at(buf, dst.base + do), u8at(src.buf, src.base + so), src.stride, h) == 0
    with cl.RefCheck(DIGESTS) as rc:
        ours, theirs = both(case, run)
        assert rc.same(ours, theirs)


@pytest.mark.parametrize("layout", ["B", "C"])
def test_weight_oracle_vs_ref_on_layouts(layout):
    rng = np.random.default_rng(46)
    n = 600
    prm = [(int(rng.integers(0, 4)), int(rng.choice([1, 2, 3, 4, 8, 16])), int(rng.integers(0, 8)), int(rng.choice([-128, -1, 0, 1, 127])),
            int(rng.choice([-128, -1, 0, 1, 127])), int(rng.choice([-128, 0, 127]))) for _ in range(n)]
    case = pel_layout_case(layout, "extremes", [(16 >> p[0], p[1]) for p in prm], 47, cell=(32, 16), phases=rng.integers(0, 16, n))
    src, dst = case["src"], case["dst"]

    def run(bi):
        def go(L, pre, buf):
            for (idx, h, ld, wd, ws, off), do, so in zip(prm, case["doff"].tolist(), case["soff"].tolist()):
                if bi:
                    getattr(L, pre + "_h264_biweight")(idx, u8at(buf, dst.base + do), u8at(src.buf, src.base + so), dst.stride, h, ld, wd, ws, off)
                else:
                    getattr(L, pre + "_h264_weight")(idx, u8at(buf, dst.base + do), dst.stride, h, ld, wd, off)
        return go
    with cl.RefCheck(DIGESTS) as rc:
        for bi in (False, True):
            ours, theirs = both(case, run(bi))
            assert rc.same(ours, theirs), bi


def test_emulated_edge_mc_oracle_vs_ref_on_new_pictures():
    with cl.RefCheck(DIGESTS) as rc:
        for W, H in ((1, 1), (1, 37), (37, 1), (100, 60)):
            LS, BLS = W + 13, 83
            pic = np.random.default_rng(W * 100 + H).integers(0, 256, (H, LS), dtype=np.uint8)
            for bw, bh, sx, sy in edge_windows(W, H)[::3]:
                src = pic.ctypes.data + sy * LS + sx
                ours = np.full((80, BLS), 7, np.uint8)
                cl.oracle().orc_emulated_edge_mc(cl.ptr(ours), src, BLS, LS, bw, bh, sx, sy, W, H)

                def theirs():
                    b = np.full((80, BLS), 7, np.uint8)
                    cl.ref().ffref_emulated_edge_mc(cl.ptr(b), src, BLS, LS, bw, bh, sx, sy, W, H)
                    return b
                assert rc.same(ours, theirs), (W, H, bw, bh, sx, sy)
