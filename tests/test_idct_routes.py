"""CPU tier of the simple-IDCT / inverse-quantiser route tests (tests/test_idct_routes_gpu.py).

This file owns what those tests are built from, so that it can be checked without a GPU:
  - the coefficient classes: the six of tests/cases.py:idct_blocks plus
      dcrows    every row on its own either DC-only, row[0] over the whole int16 range, or dense: the row DC shortcut (and its
                (row[0] << 3) & 0xffff wrap) inside blocks whose other rows take the full row pass
      zero      all-zero blocks
      saturate  a full-range DC with strong low-frequency ramps: put and add clip at 0 and at 255 inside one block
      maxabs    +32767 / -32767 / -32768 sign patterns: every row and column sum wraps modulo 2^32
  - the inverse-quantiser "extreme" case: levels over the full int16 range, qscale 1 and 31, matrices up to 255, DC scales whose
    product wraps int16, last_index 0 / 63 (and -1 for the MPEG variants), both scans;
  - a mirror of the CTA width choice of launch_mb420 / launch_mb420_fused (csrc/idct.cu:649-655, 680-685) and the table of
    macroblock-row widths, which must reach every (width, idle segments, partial last segment) cell on both tiled routes.
Its tests pin the checker (oracle/) to the compiled reference on the new classes, negative and odd line sizes and the extreme
quantiser case.  Without oracle/_ref the reference's results come from tests/golden/idct_routes_ref_digests.json."""
import ctypes as C
import os

import numpy as np
import pytest

import cpulibs as cl
from cases import idct_blocks

DIGESTS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "idct_routes_ref_digests.json")
OLD_CLASSES = ("dense", "wide", "extreme", "sparse", "dc63", "dconly")
CLASSES = OLD_CLASSES + ("dcrows", "zero", "saturate", "maxabs")


# ---------------------------------------------------------------------------------------------- coefficient classes
def class_blocks(kind, n, seed):
    """n int16[64] blocks of one class"""
    if kind in OLD_CLASSES:
        return idct_blocks(kind, n, seed)
    rng = np.random.default_rng([seed, CLASSES.index(kind)])
    if kind == "zero":
        return np.zeros((n, 64), np.int16)
    if kind == "dcrows":
        b = rng.integers(-256, 257, (n, 8, 8))
        dc = rng.random((n, 8)) < 0.5
        keep = rng.random(n) < 0.9                                      # most blocks keep at least one dense row
        dc[np.nonzero(keep)[0], rng.integers(0, 8, int(keep.sum()))] = False
        b[dc] = 0
        r0 = rng.integers(-32768, 32768, (n, 8))
        r0.flat[:12] = [-32768, 32767, 4096, -4096, 4095, -4097, 8192, -8192, 8191, 16384, -16385, 1]    # around the wrap points
        b[..., 0] = np.where(dc, r0, b[..., 0])
        return b.reshape(n, 64).astype(np.int16)
    if kind == "saturate":
        b = np.zeros((n, 64), np.int64)
        b[:, 0] = rng.integers(-2048, 2048, n)
        for j in (1, 8):
            b[:, j] = rng.choice([-1, 1], n) * rng.integers(1000, 2048, n)
        for j in (2, 9, 16):
            b[:, j] = rng.integers(-300, 301, n)
        return b.astype(np.int16)
    if kind == "maxabs":
        i, j = np.divmod(np.arange(64), 8)
        pats = np.stack([np.full(64, 32767), np.full(64, -32768), np.where((i + j) & 1, -32768, 32767),
                         np.where(i & 1, -32768, 32767), np.where(j & 1, 32767, -32768), np.where(i < 4, 32767, -32767)])
        b = pats[rng.integers(0, len(pats), n)]
        rnd = rng.integers(0, 4, n) == 0                                 # and a random mix of the three values
        b[rnd] = rng.choice([32767, -32767, -32768], (int(rnd.sum()), 64))
        return b.astype(np.int16)
    raise ValueError(kind)


def mixed_blocks(n, seed):
    """n blocks with every class in about equal numbers, in a seeded random order: (blocks [n, 64] int16, class index [n])"""
    rng = np.random.default_rng(seed)
    cls = np.arange(n) % len(CLASSES)
    rng.shuffle(cls)
    out = np.zeros((n, 64), np.int16)
    for c, kind in enumerate(CLASSES):
        sel = cls == c
        out[sel] = class_blocks(kind, int(sel.sum()), seed * 16 + c)
    return out, cls


# ---------------------------------------------------------------------------------------------- inverse-quantiser cases
H263 = (5, 6)


def extreme_unquant_case(seed, variant, nblocks, q_scale_type, h263_aic, ac_pred):
    """(cfg, blocks, blk_n, qscale, last_index) at the edges of the quantisers' arithmetic; the blocks are all ten classes used as
    levels, every coefficient set, so those past last_index must come through unchanged"""
    rng = np.random.default_rng([seed, variant, q_scale_type, h263_aic, ac_pred])
    im, nm = rng.integers(1, 256, 64).astype(np.uint16), rng.integers(1, 256, 64).astype(np.uint16)
    im[rng.integers(0, 64, 12)] = 255
    nm[rng.integers(0, 64, 12)] = 255
    cfg = dict(intra_matrix=im, inter_matrix=nm, alternate_scan=int(rng.integers(0, 2)), y_dc_scale=int(rng.integers(100, 256)),
               c_dc_scale=int(rng.integers(2, 64)), q_scale_type=q_scale_type, h263_aic=h263_aic, ac_pred=ac_pred)
    blocks, _ = mixed_blocks(nblocks, seed + 7 * variant)
    qscale = rng.integers(1, 32, nblocks).astype(np.uint8)
    qscale[rng.random(nblocks) < 0.25] = 1
    qscale[::4] = 31
    # last_index: 0 and 63 often, -1 (no coded coefficient) only where it is in the quantiser's domain (the MPEG variants: the H.263
    # ones index raster_end[last_index])
    last = rng.integers(0 if variant in H263 else -1, 64, nblocks).astype(np.int8)
    last[::3] = 63
    last[1::5] = 0
    if variant not in H263:
        last[2::7] = -1
    blk_n = rng.integers(0, 6, nblocks).astype(np.uint8)
    return cfg, blocks, blk_n, qscale, last


def extreme_configs():
    """(q_scale_type, h263_aic, ac_pred): all eight"""
    return [(q, a, p) for q in (0, 1) for a in (0, 1) for p in (0, 1)]


# ---------------------------------------------------------------------------------------------- tiled kernel geometry
MAX_SEGS = 6


def mb420_segs(mb_w):
    """(segments per CTA, idle segments in the last CTA of a row) as launch_mb420 picks them (csrc/idct.cu:649-655): a segment
    is 8 macroblocks of one row; the CTA width wasting the fewest segments wins, the wider one on a tie"""
    segs_row = (mb_w + 7) // 8
    best, waste = 4, 1 << 30
    for s in range(3, MAX_SEGS + 1):
        wst = -(-segs_row // s) * s - segs_row
        if wst < waste or (wst == waste and s > best):
            best, waste = s, wst
    return best, waste


def width_cell(mb_w):
    best, waste = mb420_segs(mb_w)
    return best, waste > 0, mb_w % 8 != 0


def width_id(mb_w):
    best, idle, partial = width_cell(mb_w)
    return f"s{best}-{'idle' if idle else 'noidle'}-{'partial' if partial else 'whole'}-w{mb_w}"


# macroblock-row widths of the tiled and fused cases: every CTA width with and without idle segments, with and without a partial
# last segment (e.g. 85: 11 segments -> 2 CTAs of 6, one idle; 110: 14 -> 3 CTAs of 5, one idle)
MB420_WIDTHS = (1, 8, 9, 17, 24, 25, 32, 33, 40, 41, 48, 55, 56, 85, 88, 104, 110, 120)
WIDTH_CASES = {"tiled": MB420_WIDTHS, "fused": MB420_WIDTHS}


def mb420_height(mb_w):
    """frames of at least 64 macroblocks, at least two macroblock rows"""
    return max(2, -(-64 // mb_w))


# ---------------------------------------------------------------------------------------------- 8x8 destinations
def private_rows(line_sizes, shifts, head=256, tail=256, width=8, elem=1):
    """Block i gets a region of its own holding 8 rows of `width` samples `line_sizes[i]` bytes apart (negative: bottom-up, the
    block starts at the region's last row), starting `shifts[i]` bytes into the region.  Returns (byte offsets, buffer size)."""
    ls = np.asarray(line_sizes, np.int64)
    span = 7 * int(np.abs(ls).max()) + width * elem + int(np.max(shifts)) + 16
    span = -(-span // 16) * 16
    base = head + np.arange(len(ls), dtype=np.int64) * span
    off = base + np.asarray(shifts, np.int64) + np.where(ls < 0, -7 * ls, 0)
    return off, head + len(ls) * span + tail


def footprint(off, line_sizes, width=8, elem=1):
    """byte positions of every sample of the 8-row destinations (off [n], line_sizes [n] or scalar)"""
    ls = np.broadcast_to(np.asarray(line_sizes, np.int64), off.shape)
    r = np.arange(8, dtype=np.int64)[None, :, None]
    c = np.arange(width * elem, dtype=np.int64)[None, None, :]
    return (off[:, None, None] + r * ls[:, None, None] + c).ravel()


def orc_idct8(kind, blocks, dest, off, line_sizes):
    """the checker over blocks with per-block destinations and line sizes: (blocks after, dest after)"""
    O = cl.oracle()
    b, d = blocks.copy(), None if dest is None else dest.copy()
    ls = np.broadcast_to(np.asarray(line_sizes, np.int64), (b.shape[0],))
    for v in np.unique(ls):
        sel = np.nonzero(ls == v)[0]
        bs = np.ascontiguousarray(b[sel])
        o = np.ascontiguousarray(off[sel], np.int64) if kind else None
        O.orc_idct_batch(kind, cl.ptr(bs, cl.i16p), len(sel), cl.ptr(d) if kind else None, int(v), cl.ptr(o, cl.i64p) if kind else None)
        b[sel] = bs
    return b, d


def ref_idct8(kind, blocks, dest, off, line_sizes):
    b, d = blocks.copy(), dest.copy()
    ls = np.broadcast_to(np.asarray(line_sizes, np.int64), (b.shape[0],))
    for i in range(b.shape[0]):
        o = np.array([off[i]], np.int64)
        cl.ref().ffref_idct_batch(kind, cl.ptr(b[i], cl.i16p), 1, cl.ptr(d) if kind else None, int(ls[i]), cl.ptr(o, cl.i64p) if kind else None)
    return b, d


def _hbd_run(fn, depth, kind, blocks, dest, off, line_sizes):
    f = fn
    f.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_ssize_t, C.c_void_p]
    b, d = blocks.copy(), dest.copy()
    ls = np.broadcast_to(np.asarray(line_sizes, np.int64), (b.shape[0],))
    for i in range(b.shape[0]):
        assert f(depth, kind, d.ctypes.data + int(off[i]), int(ls[i]), b[i].ctypes.data) == 0
    return b, d


def orc_hbd(depth, kind, blocks, dest, off, line_sizes):
    """10 / 12 bit checker, per-block byte offsets and line sizes into a uint8 buffer (depth 9 runs the 10-bit functions)"""
    return _hbd_run(cl.oracle().orc_idct_hbd, 10 if depth == 9 else depth, kind, blocks, dest, off, line_sizes)


def ref_hbd(depth, kind, blocks, dest, off, line_sizes):
    return _hbd_run(cl.ref().ffref_idct_hbd, depth, kind, blocks, dest, off, line_sizes)


def _prores_run(fn, bits, blocks, qmat, dest, off, line_sizes):
    fn.argtypes = [C.c_int, C.c_void_p, C.c_ssize_t, C.c_void_p, C.c_void_p]
    b, d = blocks.copy(), dest.copy()
    ls = np.broadcast_to(np.asarray(line_sizes, np.int64), (b.shape[0],))
    for i in range(b.shape[0]):
        assert fn(bits, d.ctypes.data + int(off[i]), int(ls[i]), b[i].ctypes.data, qmat.ctypes.data) == 0
    return b, d


def orc_prores(bits, blocks, qmat, dest, off, line_sizes):
    return _prores_run(cl.oracle().orc_prores_idct_put, bits, blocks, qmat, dest, off, line_sizes)


def ref_prores(bits, blocks, qmat, dest, off, line_sizes):
    return _prores_run(cl.ref().ffref_prores_idct_put, bits, blocks, qmat, dest, off, line_sizes)


def prores_qmat(seed):
    """quantiser matrices whose products with full-range levels wrap int16 (values up to 255, at least one 255)"""
    q = np.random.default_rng(seed).integers(1, 256, 64).astype(np.int16)
    q[seed % 64] = 255
    return q


# mixed line sizes for the per-block destinations (bytes): positive, negative, odd; 8-bit and high bit depth (even only)
LS8 = (8, 16, 24, 40, 64, 1024, 9, 13, 37, 257, -8, -16, -40, -1024, -9, -13, -257)
LS16 = (16, 32, 48, 96, 2048, 18, 22, 50, 34, -16, -32, -96, -2048, -18, -22, -50)


# ---------------------------------------------------------------------------------------------- tests
def test_case_table_fills_every_width_cell():
    """the tiled and fused cases reach every segments-per-CTA choice with and without idle segments, with and without a partial
    last segment; and the mirror of the choice gives the widths the table's comment names"""
    grid = {(s, idle, part) for s in range(3, MAX_SEGS + 1) for idle in (False, True) for part in (False, True)}
    for route, widths in WIDTH_CASES.items():
        missing = grid - {width_cell(w) for w in widths}
        assert not missing, (route, sorted(missing))
    assert mb420_segs(85) == (6, 1) and mb420_segs(110) == (5, 1) and mb420_segs(240) == (6, 0) and mb420_segs(1) == (3, 2)
    assert [mb420_segs(w)[0] for w in (17, 25, 33, 41)] == [3, 4, 5, 6]
    assert 6 * (48 * 128 + 3072) > 48 * 1024                            # six segments need the dynamic shared-memory opt-in


def test_classes_reach_their_edges():
    """each new class holds what it is there for"""
    b = class_blocks("dcrows", 4000, 1).reshape(-1, 8, 8)
    dc_row = (b[:, :, 1:] == 0).all(axis=2)
    wraps = dc_row & (np.abs(b[:, :, 0].astype(np.int64)) >= 4096)
    assert (wraps & ~dc_row.all(axis=1)[:, None]).sum() > 1000           # wrapping DC-only rows inside blocks with a dense row
    assert not class_blocks("zero", 10, 1).any()
    m = class_blocks("maxabs", 600, 1)
    assert set(np.unique(m)) <= {-32768, -32767, 32767}
    s = class_blocks("saturate", 600, 1)
    out, _ = orc_idct8(0, s, None, None, 0)
    assert ((out < 0).any(axis=1) & (out > 255).any(axis=1)).sum() > 100  # blocks that clip on both sides under put
    blocks, cls = mixed_blocks(1000, 3)
    assert np.bincount(cls, minlength=len(CLASSES)).min() == 100
    for v in range(7):
        cfg, blocks, _, q, last = extreme_unquant_case(1, v, 300, 1, 1, 1)
        assert {0, 63} <= set(last.tolist()) and ((-1 in last) == (v not in H263)) and {1, 31} <= set(q.tolist())
        assert cfg["intra_matrix"].max() == 255 and np.abs(blocks.astype(np.int64)[:, 0] * cfg["y_dc_scale"]).max() > 32767


@pytest.mark.parametrize("kind", CLASSES)
def test_idct8_oracle_vs_reference_classes(kind):
    """8-bit simple IDCT, in place / put / add, uniform line size, then per-block positive, negative and odd line sizes"""
    n = 600
    blocks = class_blocks(kind, n, 11)
    rng = np.random.default_rng(12)
    with cl.RefCheck(DIGESTS) as rc:
        off = (rng.permutation(n) * 8).astype(np.int64)
        dest = rng.integers(0, 256, 8 * (n * 8 + 8), dtype=np.uint8)
        for op in (0, 1, 2):
            ours = orc_idct8(op, blocks, dest, off, n * 8 + 8)
            assert rc.same(list(ours), lambda: list(ref_idct8(op, blocks, dest, off, n * 8 + 8))), (kind, op)
        ls = np.array(LS8)[rng.integers(0, len(LS8), n)]
        off, size = private_rows(ls, rng.integers(0, 8, n))
        dest = rng.integers(0, 256, size, dtype=np.uint8)
        for op in (1, 2):
            ours = orc_idct8(op, blocks, dest, off, ls)
            assert rc.same(list(ours[1:]), lambda: [ref_idct8(op, blocks, dest, off, ls)[1]]), (kind, op, "per-block line sizes")


def test_unquant_oracle_vs_reference_extreme():
    with cl.RefCheck(DIGESTS) as rc:
        for variant in range(7):
            for (qt, aic, acp) in extreme_configs():
                cfg, blocks, blk_n, q, last = extreme_unquant_case(20, variant, 400, qt, aic, acp)
                ours = cl.orc_unquant(variant, cfg, blocks, blk_n, q, last)
                assert rc.same(ours, lambda: cl.ref_unquant(variant, cfg, blocks, blk_n, q, last)), (cl.UNQUANT_VARIANTS[variant], qt, aic, acp)


@pytest.mark.parametrize("depth", [9, 10, 12])
def test_idct_hbd_oracle_vs_reference_classes(depth):
    """10 / 12 bit (and 9 bit, which gets the 10-bit functions) on every class, per-block positive and negative line sizes"""
    n = 300
    blocks, _ = mixed_blocks(n, 40 + depth)
    rng = np.random.default_rng(depth)
    ls = np.array(LS16)[rng.integers(0, len(LS16), n)]
    off, size = private_rows(ls, 2 * rng.integers(0, 8, n), elem=2)
    dest = np.frombuffer(rng.integers(0, 1 << (12 if depth == 12 else 10), size // 2, dtype=np.uint16).tobytes(), np.uint8).copy()
    with cl.RefCheck(DIGESTS) as rc:
        for kind in (0, 1, 2):
            ours = orc_hbd(depth, kind, blocks, dest, off, ls)
            assert rc.same(list(ours), lambda: list(ref_hbd(depth, kind, blocks, dest, off, ls))), (depth, kind)


@pytest.mark.parametrize("bits", [10, 12])
def test_prores_oracle_vs_reference_wrapping_qmat(bits):
    """ProRes idct_put on every class with quantiser matrices whose products wrap int16, per-block and negative line sizes"""
    n = 300
    blocks, _ = mixed_blocks(n, 60 + bits)
    rng = np.random.default_rng(bits)
    ls = np.array(LS16)[rng.integers(0, len(LS16), n)]
    off, size = private_rows(ls, 2 * rng.integers(0, 8, n), elem=2)
    dest = rng.integers(0, 256, size, dtype=np.uint8)
    with cl.RefCheck(DIGESTS) as rc:
        for seed in (1, 2, 3):
            qmat = prores_qmat(seed)
            ours = orc_prores(bits, blocks, qmat, dest, off, ls)[1]
            assert rc.same(ours, lambda: ref_prores(bits, blocks, qmat, dest, off, ls)[1]), (bits, seed)
