"""Test infrastructure for the HEVC residual (the transform members of HEVCDSPContext and b200_hevc_transform_add_batch_device): the
seeded case generators, runners of the checker (oracle/liboracle.so: orc_hevc_tx, orc_hevc_add_residual, orc_hevc_tu_batch) and of the
compiled reference (oracle/_ref/libffref_hevcidct.so, built by oracle/ref/Makefile), and RefCheck, which keeps the reference's
results as digests in tests/golden/hevcidct_ref_digests.json for machines without the reference."""
import ctypes as C
import hashlib
import os

import numpy as np

import cpulibs as cl
from ffmpeg_b200.hevcdsp import TU_DTYPE, IDCT, IDCT_DC, DST4, SKIP, BYPASS, RDPCM, RDPCM_VER, ROTATE

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_LIB = "libffref_hevcidct"
REF_DIGESTS = os.path.join(ROOT, "tests", "golden", "hevcidct_ref_digests.json")
FIXTURE = os.path.join(ROOT, "tests", "golden", "hevcidct_hashes.txt")
DEPTHS = (8, 9, 10, 12)
FNS = ("idct", "idct_dc", "transform_4x4_luma", "dequant", "transform_rdpcm")     # orc_hevc_tx / ffref_hevc_tx fn 0..4
CLASSES = ("decoder", "dense", "extreme", "small_limit", "odd_limit")


def have_ref():
    return cl.have_ref(REF_LIB)


def ref():
    return cl.ref_lib(REF_LIB)


def RefCheck():
    return cl.RefCheck(REF_DIGESTS, REF_LIB)


def sdtype(depth):
    return np.uint8 if depth == 8 else np.uint16


# ---------------------------------------------------------------- coefficient blocks
def scan_order(n, scan):
    """(x, y) positions of an n x n block in HEVC coefficient scan order: 4x4 sub-blocks in diagonal (up-right), horizontal or
    vertical order, the positions of each sub-block in the same order"""
    def order(m):
        if scan == "diag":
            return [(x, s - x) for s in range(2 * m - 1) for x in range(m) if 0 <= s - x < m]
        if scan == "horiz":
            return [(x, y) for y in range(m) for x in range(m)]
        return [(x, y) for x in range(m) for y in range(m)]
    return [(sx * 4 + x, sy * 4 + y) for sx, sy in order(n // 4) for x, y in order(4)]


def col_limit_of(lx, ly):
    """hevc/cabac.c:1258-1265"""
    cl_, mxy = lx + ly + 4, max(lx, ly)
    if mxy < 4:
        cl_ = min(4, cl_)
    elif mxy < 8:
        cl_ = min(8, cl_)
    elif mxy < 12:
        cl_ = min(24, cl_)
    return cl_


def decoder_block(rng, log2):
    """a parser-shaped block: a last significant position in a seeded scan, values only at positions before it in that scan, and
    the col_limit the decoder computes for it"""
    n = 1 << log2
    order = scan_order(n, ("diag", "horiz", "vert")[int(rng.integers(0, 3))])
    last = int(rng.integers(0, len(order))) if rng.random() < 0.8 else int(rng.integers(0, min(len(order), 12)))
    c = np.zeros((n, n), np.int16)
    big = int(rng.choice([64, 512, 4096, 32767]))
    for x, y in order[:last]:
        if rng.random() < 0.5:
            c[y, x] = int(rng.integers(-big, big + 1))
    lx, ly = order[last]
    c[ly, lx] = int(rng.choice([-1, 1])) * int(rng.integers(1, big + 1))
    return c, col_limit_of(lx, ly)


def block(rng, log2, cls):
    """(coefficients, col_limit) of one input class: decoder-shaped; dense over the whole int16 range with an in-range limit;
    extreme (only -32768 / 32767 / 0); dense with a small limit; dense with a negative or oversized limit"""
    n = 1 << log2
    if cls == "decoder":
        return decoder_block(rng, log2)
    if cls == "extreme":
        c = rng.choice(np.array([-32768, 32767, 0, -32768], np.int16), (n, n))
    else:
        c = rng.integers(-32768, 32768, (n, n)).astype(np.int16)
    if cls == "small_limit":
        return c, int(rng.integers(0, 8))
    if cls == "odd_limit":
        return c, int(rng.choice([-1, -4, -5, -100, -(1 << 20), n + 1, 37, 100, 1 << 20, int(rng.integers(-40, 40))]))
    return c, int(rng.integers(1, n + 5)) if cls == "extreme" else int(rng.integers(0, n + 1))


# ---------------------------------------------------------------- single members
def member_calls(seed, depth, cls):
    """every (fn, log2) member of the depth (4x4 luma at log2 2 only) with 6 seeded blocks of the class each; rdpcm with modes 0, 1
    and other non-zero ints; yields (fn, log2, coefficients, arg)"""
    rng = np.random.default_rng(seed)
    for fn in range(5):
        for log2 in ((2,) if fn == 2 else (2, 3, 4, 5)):
            for k in range(6):
                c, lim = block(rng, log2, cls)
                arg = lim if fn == 0 else (k % 2, 1, -3, 1 << 30, 0, 2)[k] if fn == 4 else 0
                yield fn, log2, c, arg


def run_tx(L, name, depth, call):
    fn, log2, c, arg = call
    f = getattr(L, name)
    f.argtypes = [C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int]
    d = c.copy()
    assert f(depth, fn, log2, d.ctypes.data, arg) == 0
    return d


def run_members(L, name, seed, depth, cls):
    return [run_tx(L, name, depth, call) for call in member_calls(seed, depth, cls)]


def residual_calls(seed, depth):
    """add_residual at every size: residuals over the int16 range and near the sample range's ends, pixels at 0, at the maximum and
    in between; yields (log2, dst, res)"""
    rng = np.random.default_rng(seed)
    maxv = (1 << depth) - 1
    for log2 in (2, 3, 4, 5):
        n = 1 << log2
        for k in range(4):
            dst = rng.choice(np.array([0, maxv, maxv // 2, 1, maxv - 1]), (n, n + 8)).astype(sdtype(depth)) if k % 2 else \
                rng.integers(0, maxv + 1, (n, n + 8)).astype(sdtype(depth))
            res = rng.integers(-32768, 32768, (n, n)).astype(np.int16) if k < 2 else rng.integers(-maxv - 2, maxv + 3, (n, n)).astype(np.int16)
            yield log2, dst, res


def run_add(L, name, depth, call):
    log2, dst, res = call
    f = getattr(L, name)
    f.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_ssize_t]
    d = dst.copy()
    assert f(depth, log2, d.ctypes.data, res.ctypes.data, d.strides[0]) == 0
    return d


# ---------------------------------------------------------------- batches (b200_hevc_transform_add_batch_device)
CELL = 40          # dst: one op per 40 x 40 cell, block at (4, 4): sentinels all around every block


def op_kind(rng, log2, chroma):
    """a kind and flags the decoder can produce for a TU of that size"""
    k = int(rng.choice([IDCT, IDCT, IDCT, IDCT_DC, SKIP, BYPASS] + ([DST4, DST4] if log2 == 2 and not chroma else [])))
    f = 0
    if k in (SKIP, BYPASS) and rng.random() < 0.6:
        f |= RDPCM | (RDPCM_VER if rng.random() < 0.5 else 0)
    if k == SKIP and rng.random() < 0.5:
        f |= ROTATE                                    # only acts on 4x4 blocks
    return k, f


def batch_case(seed, n, depth, chroma=False, cols=16, cls=None):
    """(coef [int16], dst [rows*CELL, cols*CELL] of sentinels, ops TU_DTYPE [n]): n ops of seeded sizes (4x4..32x32, 4x4..16x16 for
    chroma) and kinds, blocks of every input class (or only `cls`), coefficient blocks at offsets that are multiples of 8 with gaps
    between them; destination samples over the whole range with runs at 0 and at the maximum"""
    rng = np.random.default_rng(seed)
    maxv = (1 << depth) - 1
    rows = (n + cols - 1) // cols
    dst = np.full((rows * CELL, cols * CELL), 0x5A5A if depth > 8 else 0x5A, sdtype(depth))
    ops = np.zeros(n, TU_DTYPE)
    chunks, off = [], 0
    bps = dst.itemsize
    for i in range(n):
        log2 = int(rng.integers(2, 5 if chroma else 6))
        sz = 1 << log2
        k, f = op_kind(rng, log2, chroma)
        c, lim = block(rng, log2, cls or CLASSES[i % len(CLASSES)])
        if k in (SKIP, BYPASS) and rng.random() < 0.5:  # rdpcm sums that wrap
            c = rng.integers(-32768, 32768, (sz, sz)).astype(np.int16)
        y0, x0 = (i // cols) * CELL + 4, (i % cols) * CELL + 4
        sel = rng.integers(0, 3)
        dst[y0:y0 + sz, x0:x0 + sz] = 0 if sel == 0 else maxv if sel == 1 else rng.integers(0, maxv + 1, (sz, sz))
        ops[i]["dst_off"] = y0 * dst.strides[0] + x0 * bps
        ops[i]["coef_off"] = off
        ops[i]["log2_size"], ops[i]["kind"], ops[i]["flags"], ops[i]["col_limit"] = log2, k, f, lim
        chunks.append(c.ravel())
        gap = 8 * int(rng.integers(0, 3))
        chunks.append(np.full(gap, 0x7777, np.int16))
        off += sz * sz + gap
    coef = np.concatenate(chunks + [np.zeros(8, np.int16)])
    return coef, dst, ops


def _batch(L, name, depth, coef, dst, ops):
    f = getattr(L, name)
    f.restype = C.c_int64
    f.argtypes = [C.c_int, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_ssize_t]
    d = dst.copy()
    c = coef.copy()
    assert f(depth, len(ops), ops.ctypes.data, c.ctypes.data, d.ctypes.data, d.strides[0]) >= 0
    assert np.array_equal(c, coef)
    return d


def orc_batch(depth, coef, dst, ops):
    return _batch(cl.oracle(), "orc_hevc_tu_batch", depth, coef, dst, ops)


def ref_batch(depth, coef, dst, ops):
    return _batch(globals()["ref"](), "ffref_hevc_tu_batch", depth, coef, dst, ops)


def fixture_case(depth, chroma):
    """the seeded batch behind each line of tests/golden/hevcidct_hashes.txt: 1200 ops, luma (4x4..32x32, DST4 included) or chroma
    sized (4x4..16x16)"""
    return batch_case(700 + 10 * depth + chroma, 1200, depth, bool(chroma))


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def fixture_hashes():
    out = {}
    for line in open(FIXTURE):
        d, what, h = line.split()
        out[(int(d), what == "chroma")] = h
    return out


# ---------------------------------------------------------------- members through a filled HEVCDSPContext (host pointers)
def ctx_tx(ctx, call):
    """one orc_hevc_tx-style call through the context's member; returns the coefficients it leaves"""
    from ffmpeg_b200 import hevcdsp as hd
    fn, log2, c, arg = call
    d = c.copy()
    p = d.ctypes.data
    if fn == 0:
        hd.IDCT_FN(ctx.idct[log2 - 2])(p, arg)
    elif fn == 1:
        hd.IDCT_DC_FN(ctx.idct_dc[log2 - 2])(p)
    elif fn == 2:
        hd.TRANSFORM_4X4_LUMA(ctx.transform_4x4_luma)(p)
    elif fn == 3:
        hd.DEQUANT(ctx.dequant)(p, log2)
    else:
        hd.TRANSFORM_RDPCM(ctx.transform_rdpcm)(p, log2, arg)
    return d


def ctx_add(ctx, call):
    from ffmpeg_b200 import hevcdsp as hd
    log2, dst, res = call
    d, r = dst.copy(), res.copy()
    hd.ADD_RESIDUAL(ctx.add_residual[log2 - 2])(d.ctypes.data, r.ctypes.data, d.strides[0])
    assert np.array_equal(r, res)
    return d
