"""Test infrastructure for VP9 motion compensation (the mc / smc tables of VP9DSPContext and b200_vp9_mc_batch_device): the seeded case
generators, runners of the checker (oracle/liboracle.so: orc_vp9_mc, orc_vp9_smc, orc_vp9_mc_batch) and of the compiled reference
(oracle/_ref/libffref_vp9dsp.so, built by oracle/ref/vp9dsp.mk).  The reference's results are kept as digests in
tests/golden/vp9mc_ref_digests.json (cpulibs.RefCheck) for machines without the reference."""
import ctypes as C
import hashlib
import os

import numpy as np

import cpulibs as cl
from ffmpeg_b200._lib import Vp9McRef
from ffmpeg_b200.vp9dsp import OP_DTYPE, SINGLE, COMPOUND

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_SO = os.path.join(ROOT, "oracle", "_ref", "libffref_vp9dsp.so")
REF_DIGESTS = os.path.join(ROOT, "tests", "golden", "vp9mc_ref_digests.json")
FIXTURE = os.path.join(ROOT, "tests", "golden", "vp9mc_hashes.txt")
DEPTHS = (8, 10, 12)
WIDTHS = (64, 32, 16, 8, 4)                             # table index 0..4
BANKS = ("smooth", "regular", "sharp", "bilinear")      # FilterMode order
STEPS = (1, 5, 8, 15, 16, 17, 20, 31, 32)
_ref = None


def have_ref():
    return os.path.exists(REF_SO) and cl.have_ref()


def ref():
    global _ref
    if _ref is None:
        _ref = C.CDLL(REF_SO)
    return _ref


def RefCheck():
    return cl.RefCheck(REF_DIGESTS)


def sdtype(depth):
    return np.uint8 if depth == 8 else np.uint16


def picture(rng, h, w, depth, cls):
    """cls 0: uniform noise, 1: all 0, 2: all 2^depth - 1, 3: only the two extremes, alternating in runs of seeded lengths 1..4 along
    rows and columns (drives every filter's overshoot to both clip bounds)"""
    maxv = (1 << depth) - 1
    if cls == 1:
        return np.zeros((h, w), sdtype(depth))
    if cls == 2:
        return np.full((h, w), maxv, sdtype(depth))
    if cls == 3:
        cols = np.repeat(np.arange(w) % 2, rng.integers(1, 5, w))[:w]
        rows = np.repeat(np.arange(h) % 2, rng.integers(1, 5, h))[:h]
        return ((cols[None, :] ^ rows[:, None]) * maxv).astype(sdtype(depth))
    return rng.integers(0, maxv + 1, (h, w)).astype(sdtype(depth))


# ---------------------------------------------------------------- single members (mc[size][bank][avg][h][v], smc[size][bank][avg])
MARGIN = 8           # samples around the block in a member's source picture


def member_case(seed, depth, cls, scaled):
    """(source picture with MARGIN samples before the block and room for the largest window after it, dst0 [64, 72])"""
    rng = np.random.default_rng(seed)
    side = MARGIN + (134 if scaled else 64 + 7) + MARGIN
    return picture(rng, side, side, depth, cls), rng.integers(0, 1 << depth, (64, 72)).astype(sdtype(depth))


def mc_calls(seed):
    """every mc entry: (w, bank, avg, hdir, vdir, h, mx, my), each entry that filters with all 16 phases in its filtered directions
    (each also handed a non-zero phase for a direction it does not filter, which it must ignore), heights 1..64 incl. odd ones"""
    rng = np.random.default_rng(seed)
    for w in WIDTHS:
        for bank in range(4):
            for avg in (0, 1):
                for hdir in (0, 1):
                    for vdir in (0, 1):
                        for p in range(16 if hdir or vdir else 2):
                            h = int(rng.choice([1, 2, 3, 4, 7, 8, 16, 17, 32, 64, int(rng.integers(1, 65))]))
                            yield (w, bank, avg, hdir, vdir, h, p, (p * 7 + 3 + bank) % 16)


def smc_calls(seed):
    """every smc entry: (w, bank, avg, h, mx, my, dx, dy), 16 calls each: all start phases, the step pairs of STEPS x STEPS in turn (all
    81 within any two sizes)"""
    rng = np.random.default_rng(seed)
    pairs = [(a, b) for a in STEPS for b in STEPS]
    e = 0
    for w in WIDTHS:
        for bank in range(4):
            for avg in (0, 1):
                for j in range(16):
                    dx, dy = pairs[(e * 16 + j * 13 + seed) % len(pairs)]
                    h = int(rng.choice([1, 2, 3, 8, 16, 33, 64, int(rng.integers(1, 65))]))
                    yield (w, bank, avg, h, j, (j * 5 + e) % 16, dx, dy)
                e += 1


def run_mc(L, name, depth, call, pic, dst0):
    """one call of orc_vp9_mc / ffref_vp9_mc on the block at (MARGIN, MARGIN) of pic; returns dst"""
    w, bank, avg, hdir, vdir, h, mx, my = call
    f = getattr(L, name)
    f.argtypes = [C.c_int] * 5 + [C.c_void_p, C.c_ssize_t, C.c_void_p, C.c_ssize_t] + [C.c_int] * 4
    d = dst0.copy()
    src = pic.ctypes.data + MARGIN * pic.strides[0] + MARGIN * pic.itemsize
    assert f(depth, bank, avg, hdir, vdir, d.ctypes.data, d.strides[0], src, pic.strides[0], w, h, mx, my) == 0
    return d


def run_smc(L, name, depth, call, pic, dst0):
    w, bank, avg, h, mx, my, dx, dy = call
    f = getattr(L, name)
    f.argtypes = [C.c_int] * 3 + [C.c_void_p, C.c_ssize_t, C.c_void_p, C.c_ssize_t] + [C.c_int] * 6
    d = dst0.copy()
    src = pic.ctypes.data + MARGIN * pic.strides[0] + MARGIN * pic.itemsize
    assert f(depth, bank, avg, d.ctypes.data, d.strides[0], src, pic.strides[0], w, h, mx, my, dx, dy) == 0
    return d


def run_members(L, prefix, seed, depth, cls, scaled):
    pic, dst0 = member_case(seed, depth, cls, scaled)
    if scaled:
        return [run_smc(L, prefix + "_vp9_smc", depth, c, pic, dst0) for c in smc_calls(seed)]
    return [run_mc(L, prefix + "_vp9_mc", depth, c, pic, dst0) for c in mc_calls(seed)]


def subpel_filters(L, name):
    f = getattr(L, name)
    f.restype = C.POINTER(C.c_int16)
    return np.ctypeslib.as_array(f(), (3, 16, 8)).copy()


# ---------------------------------------------------------------- batches (b200_vp9_mc_batch_device)
CELL = 72          # dst: one op per 72 x 72 cell, block at (4, 4): sentinels all around every block
# reference planes of a batch case: (width, height as sixteenths of the base size, dx, dy); the first two have the current picture's size
REF_SHAPES = ((16, 16, 16, 16), (16, 16, 16, 16), (32, 32, 32, 32), (8, 8, 8, 8), (20, 5, 20, 5), (17, 31, 17, 31), (3, 15, 1, 15), (16, 24, 16, 24))


def batch_case(seed, n, depth, pic_w=200, pic_h=120, cols=16, cls=0, far=80, scaled=True):
    """(planes, steps, dst [rows*CELL, cols*CELL] of sentinels, ops OP_DTYPE [n]): eight reference planes of different sizes and steps
    (REF_SHAPES; only the two same-size ones with scaled=False), n ops of both kinds, every width and bank, heights 1..64, positions
    anywhere from `far` samples before to `far` after the reference (every edge and corner, whole windows outside), every phase with 0
    weighted up, compound ops whose slots name different references, and compound ops with one full-pel and one fractional slot"""
    rng = np.random.default_rng(seed)
    shapes = REF_SHAPES if scaled else REF_SHAPES[:2]
    planes = [picture(rng, max(1, pic_h * sh // 16), max(1, pic_w * sw // 16), depth, cls if k != 1 else (0 if cls else 3))
              for k, (sw, sh, _, _) in enumerate(shapes)]
    steps = [(dx, dy) for (_, _, dx, dy) in shapes]
    rows = (n + cols - 1) // cols
    dst = np.full((rows * CELL, cols * CELL), 0x5A5A if depth > 8 else 0x5A, sdtype(depth))
    ops = np.zeros(n, OP_DTYPE)
    i = np.arange(n)
    ops["dst_off"] = ((i // cols) * CELL + 4) * dst.strides[0] + ((i % cols) * CELL + 4) * dst.itemsize
    for k in range(n):
        o = ops[k]
        o["kind"] = k % 2
        o["w"] = WIDTHS[(k // 2) % 5]
        o["filter"] = (k // 10) % 4
        o["h"] = int(rng.choice([int(rng.integers(1, 65)), 1, 4, 8, 16, 64]))
        for r in (0, 1):
            ri = int(rng.integers(0, len(planes)))
            o["ref"][r] = ri
            ph, pw = planes[ri].shape
            bw, bh = int(o["w"]) * steps[ri][0] // 16, int(o["h"]) * steps[ri][1] // 16
            sel = rng.integers(0, 6)
            if sel == 0:        # hugging a corner
                o["x"][r] = int(rng.choice([-3, 0, 3, pw - bw - 5, pw - bw - 4, pw - bw, pw - bw + 3]))
                o["y"][r] = int(rng.choice([-3, 0, 3, ph - bh - 6, ph - bh - 5, ph - bh, ph - bh + 3]))
            elif sel == 1:      # whole window outside
                o["x"][r] = int(rng.choice([-far - bw, pw + far, int(rng.integers(-far, pw + far))]))
                o["y"][r] = int(rng.choice([-far - bh, ph + far, int(rng.integers(-far, ph + far))]))
            else:
                o["x"][r] = int(rng.integers(-far, pw + far))
                o["y"][r] = int(rng.integers(-far, ph + far))
            o["mx"][r] = 0 if rng.random() < 0.25 else int(rng.integers(0, 16))
            o["my"][r] = 0 if rng.random() < 0.25 else int(rng.integers(0, 16))
        if k % 8 == 1:          # one full-pel slot, one fractional, on the same-size references
            z = int(rng.integers(0, 2))
            o["ref"][0], o["ref"][1] = k % 4 // 2, 1 - k % 4 // 2
            o["mx"][z] = o["my"][z] = 0
            o["mx"][1 - z] = int(rng.integers(1, 16))
            o["my"][1 - z] = int(rng.integers(1, 16))
    return planes, steps, dst, ops


def ref_array(planes, steps, ptrs=None):
    """the B200Vp9McRef array of a case; ptrs = device addresses of the planes (default: the numpy arrays themselves)"""
    arr = (Vp9McRef * len(planes))()
    for k, (p, (dx, dy)) in enumerate(zip(planes, steps)):
        arr[k] = Vp9McRef(p.ctypes.data if ptrs is None else ptrs[k], p.strides[0], p.shape[1], p.shape[0], dx, dy)
    return arr


def _batch(L, name, depth, planes, steps, dst, ops):
    f = getattr(L, name)
    f.restype = C.c_int64
    f.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_ssize_t]
    d = dst.copy()
    ops = np.ascontiguousarray(ops)
    r = f(depth, len(planes), C.cast(ref_array(planes, steps), C.c_void_p), len(ops), ops.ctypes.data, d.ctypes.data, d.strides[0])
    assert r >= 0
    return d


def orc_batch(depth, planes, steps, dst, ops):
    return _batch(cl.oracle(), "orc_vp9_mc_batch", depth, planes, steps, dst, ops)


def ref_batch(depth, planes, steps, dst, ops):
    return _batch(ref(), "ffref_vp9_mc_batch", depth, planes, steps, dst, ops)


def fixture_case(depth, chroma):
    """the seeded batch behind each line of tests/golden/vp9mc_hashes.txt: 1536 ops over the eight references of a 200 x 120 (luma) /
    100 x 60 (4:2:0 chroma) picture"""
    return batch_case(700 + 10 * depth + chroma, 1536, depth, *((100, 60) if chroma else (200, 120)))


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def fixture_hashes():
    out = {}
    for line in open(FIXTURE):
        d, what, h = line.split()
        out[(int(d), what == "chroma")] = h
    return out
