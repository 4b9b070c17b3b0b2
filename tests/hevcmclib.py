"""Test infrastructure for HEVC motion compensation (the put_hevc_{q,e}pel tables of HEVCDSPContext and b200_hevc_mc_batch_device):
the seeded case generators, runners of the checker (oracle/liboracle.so: orc_hevc_mc, orc_hevc_mc_batch) and of the compiled reference
(oracle/_ref/libffref_hevcdsp.so, built by oracle/ref/Makefile), and RefCheck, which keeps the reference's results as digests in
tests/golden/hevcmc_ref_digests.json for machines without the reference."""
import ctypes as C
import hashlib
import os

import numpy as np

import cpulibs as cl
from ffmpeg_b200.hevcdsp import OP_DTYPE

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_LIB = "libffref_hevcdsp"
REF_DIGESTS = os.path.join(ROOT, "tests", "golden", "hevcmc_ref_digests.json")
FIXTURE = os.path.join(ROOT, "tests", "golden", "hevcmc_hashes.txt")
DEPTHS = (8, 9, 10, 12)
WIDTHS = (2, 4, 6, 8, 12, 16, 24, 32, 48, 64)
WEIGHTS = (-128, 0, 1, 128, 255)
FORMS = ("", "_uni", "_uni_w", "_bi", "_bi_w")          # orc_hevc_mc / ffref_hevc_mc form 0..4


def have_ref():
    return cl.have_ref(REF_LIB)


def ref():
    return cl.ref_lib(REF_LIB)


def RefCheck():
    return cl.RefCheck(REF_DIGESTS, REF_LIB)


def sdtype(depth):
    return np.uint8 if depth == 8 else np.uint16


def picture(rng, h, w, depth, cls):
    """cls 0: uniform noise, 1: all 0, 2: all 2^depth - 1, 3: noise of only the extremes (drives every filter to its bounds)"""
    maxv = (1 << depth) - 1
    if cls == 1:
        return np.zeros((h, w), sdtype(depth))
    if cls == 2:
        return np.full((h, w), maxv, sdtype(depth))
    if cls == 3:
        return (rng.integers(0, 2, (h, w)) * maxv).astype(sdtype(depth))
    return rng.integers(0, maxv + 1, (h, w)).astype(sdtype(depth))


# ---------------------------------------------------------------- single members (put_hevc_?pel*[idx][v][h])
def member_calls(seed, depth, epel):
    """every (form, table position [v][h], width) with a seeded height in 2..64, the phases cycling through every (mx, my) including 0
    (a filtered direction at phase 0 uses the reference's all-zero row), src2 over the whole int16 range, denom 0..7, wx / wx0 / wx1 from
    WEIGHTS and ox at both ends of its range (-128..127 uni, -256..254 bi) or in between; yields (form, v, h, width, height, mx, my, denom,
    wx0, wx1, ox)"""
    rng = np.random.default_rng(seed)
    P = 8 if epel else 4
    phases = [(a, b) for a in range(P) for b in range(P)]
    k = 0
    for form in range(5):
        for v in (0, 1):
            for h in (0, 1):
                for width in WIDTHS:
                    mx, my = phases[(k * 7 + seed) % len(phases)]
                    k += 1
                    height = int(rng.choice([2, 4, 8, 16, 32, 64, int(rng.integers(1, 65))]))
                    lo, hi = (-128, 127) if form < 3 else (-256, 254)
                    ox = int(rng.choice([lo, hi, int(rng.integers(lo, hi + 1))]))
                    yield (form, v, h, width, height, mx, my, int(rng.integers(0, 8)), int(rng.choice(WEIGHTS)), int(rng.choice(WEIGHTS)), ox)


def run_member(L, name, depth, epel, call, src_pic, src2, dst0):
    """one call of orc_hevc_mc / ffref_hevc_mc; src_pic: a picture with >= 8 samples around the block at (8, 8); returns dst"""
    form, v, h, width, height, mx, my, denom, wx0, wx1, ox = call
    f = getattr(L, name)
    f.argtypes = [C.c_int] * 5 + [C.c_void_p, C.c_ssize_t, C.c_void_p, C.c_ssize_t, C.c_void_p] + [C.c_int] * 8
    bps = src_pic.itemsize
    src = src_pic.ctypes.data + 8 * src_pic.strides[0] + 8 * bps
    if form == 0:
        d = np.zeros((64, 64), np.int16)
        stride = 128
    else:
        d = dst0.copy()
        stride = d.strides[0]
    r = f(depth, epel, form, v, h, d.ctypes.data, stride, src, src_pic.strides[0], src2.ctypes.data, height, denom, wx0, wx1, ox, mx, my, width)
    assert r == 0
    return d


def member_case(seed, depth, epel, cls):
    rng = np.random.default_rng(seed)
    pic = picture(rng, 64 + 16, 64 + 16, depth, cls)
    src2 = rng.integers(-32768, 32768, (64, 64)).astype(np.int16)
    dst0 = rng.integers(0, 1 << depth, (64, 72)).astype(sdtype(depth))
    return pic, src2, dst0


def run_members(L, name, seed, depth, epel, cls):
    pic, src2, dst0 = member_case(seed, depth, epel, cls)
    return [run_member(L, name, depth, epel, c, pic, src2, dst0) for c in member_calls(seed, depth, epel)]


# ---------------------------------------------------------------- batches (b200_hevc_mc_batch_device)
CELL = 72          # dst: one op per 72 x 72 cell, block at (4, 4): sentinels all around every block


def batch_case(seed, n, depth, epel, pic_w=200, pic_h=120, cols=16, cls=0, far=80):
    """(ref [2, pic_h, pic_w], dst [rows*CELL, cols*CELL] of sentinels, ops OP_DTYPE [n]): n ops cycling through the four kinds, every
    width in WIDTHS, heights 1..64, both pictures (reference r of op i is picture (i + r) % 2, reached through a negative ref_off for
    picture 0 from a `ref` pointer at picture 1), positions anywhere from `far` samples before to `far` after the picture (every edge and
    corner, whole windows outside), every phase with 0 weighted up, bi ops with one integer and one fractional reference"""
    rng = np.random.default_rng(seed)
    ref = np.stack([picture(rng, pic_h, pic_w, depth, cls), picture(rng, pic_h, pic_w, depth, 0 if cls else 3)])
    rows = (n + cols - 1) // cols
    bps = ref.itemsize
    dst = np.full((rows * CELL, cols * CELL), 0x5A5A if depth > 8 else 0x5A, sdtype(depth))
    ops = np.zeros(n, OP_DTYPE)
    P = 8 if epel else 4
    i = np.arange(n)
    ops["dst_off"] = ((i // cols) * CELL + 4) * dst.strides[0] + ((i % cols) * CELL + 4) * bps
    pic_bytes = ref.strides[0]
    for k in range(n):
        o = ops[k]
        o["kind"] = k % 4
        o["w"] = WIDTHS[(k // 4) % len(WIDTHS)]
        o["h"] = int(rng.choice([int(rng.integers(1, 65)), 2, 4, 8, 16, 64]))
        for r in (0, 1):
            o["ref_off"][r] = -pic_bytes if (k + r) % 2 == 0 else 0
            sel = rng.integers(0, 6)
            if sel == 0:        # hugging a corner
                o["x"][r] = int(rng.choice([-3, 0, pic_w - int(o["w"]), pic_w - int(o["w"]) + 3]))
                o["y"][r] = int(rng.choice([-3, 0, pic_h - int(o["h"]), pic_h - int(o["h"]) + 3]))
            elif sel == 1:      # whole window outside
                o["x"][r] = int(rng.choice([-far, pic_w + far - 64, int(rng.integers(-far, pic_w + far))]))
                o["y"][r] = int(rng.choice([-far, pic_h + far - 64, int(rng.integers(-far, pic_h + far))]))
            else:
                o["x"][r] = int(rng.integers(-far, pic_w + far))
                o["y"][r] = int(rng.integers(-far, pic_h + far))
            o["mx"][r] = 0 if rng.random() < 0.25 else int(rng.integers(0, P))
            o["my"][r] = 0 if rng.random() < 0.25 else int(rng.integers(0, P))
        if k % 8 in (2, 3):     # one integer reference, one fractional
            z = int(rng.integers(0, 2))
            o["mx"][z] = o["my"][z] = 0
            o["mx"][1 - z] = int(rng.integers(1, P))
            o["my"][1 - z] = int(rng.integers(1, P))
        o["denom"] = int(rng.integers(0, 8))
        o["wx0"] = int(rng.choice(WEIGHTS))
        o["wx1"] = int(rng.choice(WEIGHTS))
        lo, hi = (-256, 254) if o["kind"] >= 2 else (-128, 127)
        o["ox"] = int(rng.choice([lo, hi, int(rng.integers(lo, hi + 1))]))
    return ref, dst, ops


def _batch(L, name, depth, epel, ref, dst, ops):
    f = getattr(L, name)
    f.restype = C.c_int64
    f.argtypes = [C.c_int, C.c_int, C.c_int64, C.c_void_p, C.c_void_p, C.c_ssize_t, C.c_void_p, C.c_ssize_t, C.c_int, C.c_int]
    d = dst.copy()
    r = f(depth, epel, len(ops), ops.ctypes.data, d.ctypes.data, d.strides[0], ref.ctypes.data + ref.strides[0], ref.strides[1],
          ref.shape[2], ref.shape[1])
    assert r >= 0
    return d


def orc_batch(depth, epel, ref, dst, ops):
    """the checker's batch; `ref` = pointer to picture 1 of the [2, h, w] reference array"""
    return _batch(cl.oracle(), "orc_hevc_mc_batch", depth, epel, ref, dst, ops)


def ref_batch(depth, epel, ref, dst, ops):
    return _batch(globals()["ref"](), "ffref_hevc_mc_batch", depth, epel, ref, dst, ops)


def fixture_case(depth, epel):
    """the seeded batch behind each line of tests/golden/hevcmc_hashes.txt: 2048 ops on a 200 x 120 (luma) / 100 x 60 (chroma) picture"""
    return batch_case(900 + 10 * depth + epel, 2048, depth, epel, *((100, 60) if epel else (200, 120)))


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def fixture_hashes():
    out = {}
    for line in open(FIXTURE):
        d, what, h = line.split()
        out[(int(d), what == "chroma")] = h
    return out
