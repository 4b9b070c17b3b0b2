"""Test infrastructure for VP9 inverse transforms (the itxfm_add members of VP9DSPContext and b200_vp9_itxfm_add_batch_device): the
seeded case generators, runners of the checker (oracle/liboracle.so: orc_vp9_itxfm, orc_vp9_itxfm_batch) and of the compiled reference
(oracle/_ref/libffref_vp9itxfm.so, built by oracle/ref/vp9itxfm.mk).  The reference's results are kept as digests in
tests/golden/vp9itxfm_ref_digests.json (cpulibs.RefCheck) for machines without the reference."""
import ctypes as C
import hashlib
import os

import numpy as np

import cpulibs as cl
from ffmpeg_b200.vp9dsp import TX_DTYPE

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_SO = os.path.join(ROOT, "oracle", "_ref", "libffref_vp9itxfm.so")
REF_DIGESTS = os.path.join(ROOT, "tests", "golden", "vp9itxfm_ref_digests.json")
FIXTURE = os.path.join(ROOT, "tests", "golden", "vp9itxfm_hashes.txt")
DEPTHS = (8, 10, 12)
CLASSES = ("decoder", "noise", "extremes", "dcmix")
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


def size(tx):
    return 4 if tx == 4 else 4 << tx


def sdtype(depth):
    return np.uint8 if depth == 8 else np.uint16


def cdtype(depth):
    return np.int16 if depth == 8 else np.int32


def coefs(rng, depth, tx, cls):
    """one block's sz * sz coefficients (row-major as the decoder stores them) and its eob.
    decoder: a low-frequency corner of values of the size a dequantiser gives (larger above 8 bit), eob of the corner;
    noise: dense, |c| < 2^(depth + 6); extremes: only the storage type's extremes and neighbours, or full-range values, dense;
    dcmix: eob 1 with the other coefficients non-zero (the DC-only path must ignore them)"""
    n = size(tx)
    ct = cdtype(depth)
    info = np.iinfo(ct)
    if cls == "decoder":
        b = np.zeros((n, n), np.int64)
        k = int(rng.integers(1, n + 1))
        amp = 1 << (depth + 3)
        b[:k, :k] = rng.integers(-amp, amp + 1, (k, k)) // (1 + np.add.outer(np.arange(k), np.arange(k)))
        eob = int(rng.choice([1, k * k, n * n])) if k > 1 else 1
        if tx == 4:
            b = b >> 2 << 2
    elif cls == "noise":
        b = rng.integers(-(1 << (depth + 6)), 1 << (depth + 6), (n, n))
        eob = int(rng.choice([0, 2, n * n, int(rng.integers(1, n * n + 1))]))
    elif cls == "extremes":
        pool = np.array([info.max, info.min, info.min + 1, info.max - 1, 0, -1, 1], np.int64)
        b = pool[rng.integers(0, len(pool), (n, n))]
        full = rng.integers(info.min, info.max + 1, (n, n), dtype=np.int64)
        b = np.where(rng.random((n, n)) < 0.3, full, b)
        eob = int(rng.choice([0, 1, n * n]))
    else:
        b = rng.integers(-(1 << (depth + 4)), 1 << (depth + 4), (n, n))
        b[0, 0] = int(rng.choice([info.max, info.min, int(rng.integers(-4096, 4096))]))
        eob = 1
    return b.astype(ct), eob


# ---------------------------------------------------------------- single members (itxfm_add[tx][type])
MARGIN = 4           # sentinel samples around a member's destination block


def member_calls(seed, depth, cls, per=4):
    """(tx, type, eob, block [sz, sz], dst0 [sz + 2 MARGIN, sz + 2 MARGIN]) for every one of the 20 members, `per` calls each"""
    rng = np.random.default_rng(seed)
    for tx in range(5):
        for typ in range(4):
            for _ in range(per):
                n = size(tx)
                b, eob = coefs(rng, depth, tx, cls)
                dst0 = rng.integers(0, 1 << depth, (n + 2 * MARGIN, n + 2 * MARGIN)).astype(sdtype(depth))
                yield tx, typ, eob, b, dst0


def run_member(L, name, depth, call):
    """one call of orc_vp9_itxfm / ffref_vp9_itxfm on copies; returns (dst, coefficients after)"""
    tx, typ, eob, b, dst0 = call
    f = getattr(L, name)
    f.argtypes = [C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_ssize_t, C.c_void_p, C.c_int]
    d, blk = dst0.copy(), np.ascontiguousarray(b.copy())
    p = d.ctypes.data + MARGIN * d.strides[0] + MARGIN * d.itemsize
    assert f(depth, tx, typ, p, d.strides[0], blk.ctypes.data, eob) == 0
    return d, blk


def run_members(L, prefix, seed, depth, cls):
    out = []
    for call in member_calls(seed, depth, cls):
        out.extend(run_member(L, prefix + "_vp9_itxfm", depth, call))
    return out


# ---------------------------------------------------------------- batches (b200_vp9_itxfm_add_batch_device)
CELL = 40            # dst: one op per 40 x 40 cell, block at (4, 4): sentinels all around every block


def batch_case(seed, n, depth, cls="decoder", cols=16, classes=None):
    """(dst [rows * CELL, cols * CELL] of sentinels, coef, ops TX_DTYPE [n]): every tx and type in turn, the blocks' coefficients packed
    in a shuffled order with gaps of 16 elements between some of them; `classes` cycles coefficient classes per op"""
    rng = np.random.default_rng(seed)
    rows = (n + cols - 1) // cols
    dst = np.full((rows * CELL, cols * CELL), 0x5A5A & ((1 << depth) - 1) if depth > 8 else 0x5A, sdtype(depth))
    ops = np.zeros(n, TX_DTYPE)
    i = np.arange(n)
    ops["dst_off"] = ((i // cols) * CELL + 4) * dst.strides[0] + ((i % cols) * CELL + 4) * dst.itemsize
    ops["tx"] = i % 5
    ops["type"] = rng.integers(0, 4, n)
    blocks = []
    for k in range(n):
        c = cls if classes is None else classes[k % len(classes)]
        b, eob = coefs(rng, depth, int(ops["tx"][k]), c)
        ops["eob"][k] = eob
        blocks.append(b.ravel())
    order = rng.permutation(n)
    off, parts = 0, []
    for k in order:
        if rng.random() < 0.2:
            parts.append(np.zeros(16, cdtype(depth)))
            off += 16
        ops["coef_off"][k] = off
        parts.append(blocks[k])
        off += blocks[k].size
    coef = np.concatenate(parts) if parts else np.zeros(16, cdtype(depth))
    return dst, coef, ops


def _batch(L, name, depth, dst, coef, ops):
    f = getattr(L, name)
    f.restype = C.c_int64
    f.argtypes = [C.c_int, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_ssize_t]
    d, c = dst.copy(), np.ascontiguousarray(coef)
    ops = np.ascontiguousarray(ops)
    before = c.copy()
    assert f(depth, len(ops), ops.ctypes.data, c.ctypes.data, d.ctypes.data, d.strides[0]) >= 0
    assert np.array_equal(c, before)
    return d


def orc_batch(depth, dst, coef, ops):
    return _batch(cl.oracle(), "orc_vp9_itxfm_batch", depth, dst, coef, ops)


def ref_batch(depth, dst, coef, ops):
    return _batch(ref(), "ffref_vp9_itxfm_batch", depth, dst, coef, ops)


def fixture_case(depth, cls):
    """the seeded batch behind each line of tests/golden/vp9itxfm_hashes.txt: 1000 ops, every member, 40 x 40 cells"""
    return batch_case(900 + 10 * depth + CLASSES.index(cls), 1000, depth, cls, cols=25)


FIXTURE_CLASSES = ("decoder", "extremes")


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def fixture_hashes():
    out = {}
    for line in open(FIXTURE):
        d, what, h = line.split()
        out[(int(d), what)] = h
    return out
