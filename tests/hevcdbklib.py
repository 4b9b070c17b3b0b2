"""Test infrastructure for HEVC deblocking (the loop-filter members of HEVCDSPContext and b200_hevc_deblock_plane_device): the seeded
case generators, runners of the checker (oracle/liboracle.so: orc_hevc_dbk_member, orc_hevc_dbk_plane) and of the compiled reference
(oracle/_ref/libffref_hevcdbk.so, built by oracle/ref/Makefile: single members and the plane in the decoder's CTB order), and
RefCheck, which keeps the reference's results as digests in tests/golden/hevcdbk_ref_digests.json for machines without the reference."""
import ctypes as C
import hashlib
import os

import numpy as np

import cpulibs as cl
from ffmpeg_b200.hevcdsp import DBK_DTYPE, NO_P, NO_Q

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_LIB = "libffref_hevcdbk"
REF_DIGESTS = os.path.join(ROOT, "tests", "golden", "hevcdbk_ref_digests.json")
FIXTURE = os.path.join(ROOT, "tests", "golden", "hevcdbk_hashes.txt")
DEPTHS = (8, 9, 10, 12)
FNS = ("h_luma", "v_luma", "h_chroma", "v_chroma")     # ffref_hevc_dbk_member fn 0..3 (4..7: the _c twins)
CLASSES = ("decoder", "dense", "extreme")
BRANCHES = ("skip_d_ge_beta", "strong", "weak_ndp1", "weak_ndp2", "weak_ndq1", "weak_ndq2", "weak_line_skipped", "tc_le_0",
            "chroma_filtered")                          # orc_hevc_dbk_* cnt[0..8]
MARGIN = 8         # rows and columns of sentinels around a plane
SENT8, SENT16 = 0xA5, 0xA5A5

# H.265 Table 8-12 (beta' by Q = 0..51, tc' by Q = 0..53)
BETATABLE = [0] * 16 + [6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 17, 18, 20, 22, 24, 26, 28, 30, 32, 34, 36, 38, 40, 42, 44, 46, 48, 50,
                        52, 54, 56, 58, 60, 62, 64]
TCTABLE = [0] * 18 + [1, 1, 1, 1, 1, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 5, 5, 6, 6, 7, 8, 9, 10, 11, 13, 14, 16, 18, 20, 22, 24]
assert len(BETATABLE) == 52 and len(TCTABLE) == 54


def have_ref():
    return cl.have_ref(REF_LIB)


def ref():
    return cl.ref_lib(REF_LIB)


def RefCheck():
    return cl.RefCheck(REF_DIGESTS, REF_LIB)


def sdtype(depth):
    return np.uint8 if depth == 8 else np.uint16


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


# ---------------------------------------------------------------- content
def blocky(rng, depth, h, w, block=8):
    """blocks of a flat level each, some with a smooth ramp and some with texture, clipped to the sample range"""
    maxv = (1 << depth) - 1
    out = np.zeros((h, w), np.int64)
    s = 1 << (depth - 8)
    for by in range(0, h, block):
        for bx in range(0, w, block):
            kind = rng.integers(0, 4)
            hh, ww = min(block, h - by), min(block, w - bx)
            base = int(rng.integers(0, maxv + 1))
            if kind == 0:                                    # flat
                v = np.full((hh, ww), base)
            elif kind == 1:                                  # ramp
                gy, gx = rng.integers(-3, 4, 2) * s
                v = base + gy * np.arange(hh)[:, None] + gx * np.arange(ww)[None, :]
            elif kind == 2:                                  # slight texture
                v = base + rng.integers(-2 * s, 2 * s + 1, (hh, ww))
            else:                                            # strong texture
                v = base + rng.integers(-40 * s, 40 * s + 1, (hh, ww))
            out[by:by + hh, bx:bx + ww] = v
    return np.clip(out, 0, maxv).astype(sdtype(depth))


# ---------------------------------------------------------------- single members
EDGE = 8           # member buffers: 16 x 16 samples, Q0 of line 0 at (EDGE, EDGE)


def member_calls(seed, depth, cls):
    """8 seeded calls of every member kind (FNS index 0..3) of the class, on a 16 x 16 buffer: yields (fn, buf, beta, tc[2], no_p[2],
    no_q[2]).  decoder: blocky content across the edge with table beta / tc; dense: random samples, beta 0..255, tc -255..255 and
    random no_p / no_q bytes; extreme: samples at 0 and the maximum, beta and tc 255 (a few tc 0 or negative)"""
    rng = np.random.default_rng(seed)
    maxv = (1 << depth) - 1
    for fn in range(4):
        for k in range(8):
            if cls == "decoder":
                buf = blocky(rng, depth, 16, 16, int(rng.choice([4, 8])))
                qp = int(rng.integers(15, 52))
                beta = BETATABLE[min(max(qp + int(rng.integers(-6, 7)) * 2, 0), 51)]
                tc = [TCTABLE[min(max(qp + 2 * int(b) - 2, 0), 53)] if b else 0 for b in rng.integers(0, 3, 2)]
                no = rng.random(4) < 0.15
                no_p, no_q = [int(no[0]), int(no[1])], [int(no[2]), int(no[3])]
            elif cls == "dense":
                buf = rng.integers(0, maxv + 1, (16, 16)).astype(sdtype(depth))
                beta = int(rng.integers(0, 256))
                tc = [int(x) for x in rng.integers(-255, 256, 2)]
                no_p = [int(x) for x in rng.choice([0, 0, 1, 0x80, 0xFE], 2)]
                no_q = [int(x) for x in rng.choice([0, 0, 1, 0x40, 0xFF], 2)]
            else:
                buf = rng.choice(np.array([0, maxv]), (16, 16)).astype(sdtype(depth))
                if k % 2:                                       # a step across the edge
                    buf[:, :EDGE] = 0 if k % 4 == 1 else maxv
                    buf[:, EDGE:] = maxv - buf[0, 0]
                    if fn % 2 == 0:
                        buf = np.ascontiguousarray(buf.T)
                beta = 255
                tc = [255 if k < 6 else int(rng.choice([0, -1, -255])), 255]
                no_p, no_q = [0, int(k == 3)], [int(k == 5), 0]
            yield fn, buf, beta, tc, no_p, no_q


def _member_args(call):
    fn, buf, beta, tc, no_p, no_q = call
    d = buf.copy()
    return d, d.ctypes.data + EDGE * d.strides[0] + EDGE * d.itemsize, d.strides[0], beta, (C.c_int32 * 2)(*tc), \
        (C.c_uint8 * 2)(*no_p), (C.c_uint8 * 2)(*no_q)


def orc_member(depth, call, cnt=None):
    fn = call[0]
    L = cl.oracle()
    L.orc_hevc_dbk_member.argtypes = [C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_ssize_t, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.c_void_p]
    d, p, st, beta, tc, no_p, no_q = _member_args(call)
    L.orc_hevc_dbk_member(depth, fn >= 2, fn % 2 == 0, p, st, beta, tc, no_p, no_q, None if cnt is None else cnt.ctypes.data)
    return d


def ref_member(depth, call, twin=False):
    f = ref().ffref_hevc_dbk_member
    f.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_ssize_t, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    d, p, st, beta, tc, no_p, no_q = _member_args(call)
    assert f(depth, call[0] + (4 if twin else 0), p, st, beta, tc, no_p, no_q) == 0
    return d


def ctx_member(ctx, call, twin=False):
    """one call through the context's member (the plain or the _c pointer)"""
    from ffmpeg_b200 import hevcdsp as hd
    fn = call[0]
    d, p, st, beta, tc, no_p, no_q = _member_args(call)
    name = "hevc_" + ("h" if fn % 2 == 0 else "v") + "_loop_filter_" + ("chroma" if fn >= 2 else "luma") + ("_c" if twin else "")
    ptr = getattr(ctx, name)
    if fn >= 2:
        hd.LOOP_FILTER_CHROMA(ptr)(p, st, tc, no_p, no_q)
    else:
        hd.LOOP_FILTER_LUMA(ptr)(p, st, beta, tc, no_p, no_q)
    return d


# ---------------------------------------------------------------- planes
def grids(width, height):
    """empty vertical and horizontal segment grids of a plane, each with 3 records of padding per row"""
    return np.zeros(((height + 3) // 4, (width + 7) // 8 + 3), DBK_DTYPE), np.zeros(((height + 7) // 8, width // 4 + 3), DBK_DTYPE)


def decoder_grids(rng, W, H, chroma, hs=1, vs=1, ctb=32):
    """grids shaped like deblocking_filter_CTB's calls for a plane (luma, or a chroma plane subsampled by hs / vs): a quadtree of CUs
    (8..ctb luma samples) with an intra flag, a QP, a pcm / bypass flag and a per-CTB beta / tc offset; boundary strength 2 where
    either side is intra, 0 or 1 between inter CUs, 0 inside a CU; beta and tc from the tables (tc by bs), chroma tc only where bs is
    2; no_p / no_q on pcm / bypass sides.  Returns (vseg, hseg) on the plane's grid."""
    sx, sy = (1 << hs) if chroma else 1, (1 << vs) if chroma else 1
    LW, LH = W * sx, H * sy                                  # the luma picture
    n4w, n4h = (LW + 3) // 4, (LH + 3) // 4
    cu = np.zeros((n4h, n4w), np.int64)
    ncu = [0]
    attrs = []

    def split(x, y, s):
        if x >= LW or y >= LH:
            return
        if s > 8 and (rng.random() < 0.55 or x + s > LW or y + s > LH):
            for dy in (0, s // 2):
                for dx in (0, s // 2):
                    split(x + dx, y + dy, s // 2)
            return
        cu[y // 4:(y + s) // 4, x // 4:(x + s) // 4] = ncu[0]
        attrs.append((rng.random() < 0.3, int(rng.integers(20, 52)), rng.random() < 0.08))
        ncu[0] += 1
    offs = {}
    for y in range(0, LH, ctb):
        for x in range(0, LW, ctb):
            split(x, y, ctb)
            offs[(y // ctb, x // ctb)] = (int(rng.integers(-6, 7)) * 2, int(rng.integers(-6, 7)) * 2)
    intra = np.array([a[0] for a in attrs])
    qp = np.array([a[1] for a in attrs])
    pcm = np.array([a[2] for a in attrs])

    def seg(px, py, qx, qy):
        """the segment between luma 4x4 blocks P and Q (luma sample coordinates of each), with Q's CTB offsets"""
        a, b = cu[py // 4, px // 4], cu[qy // 4, qx // 4]
        if a == b:
            bs = 0
        elif intra[a] or intra[b]:
            bs = 2
        else:
            bs = int(rng.choice([0, 1, 1]))
        q = (qp[a] + qp[b] + 1) >> 1
        bo, to = offs[(qy // ctb, qx // ctb)]
        if chroma:
            q = min(max(q + int(rng.integers(-2, 3)), 0), 51)
            beta, tc = 0, TCTABLE[min(max(q + 2 + (to & -2), 0), 53)] if bs == 2 else 0
        else:
            beta = BETATABLE[min(max(q + bo, 0), 51)]
            tc = TCTABLE[min(max(q + 2 * (bs - 1) + (to & -2), 0), 53)] if bs else 0
        return beta, tc, (NO_P if pcm[a] else 0) | (NO_Q if pcm[b] else 0), 0
    vg, hg = grids(W, H)
    for y in range(0, H, 4):
        for x in range(8, W, 8):
            vg[y // 4, x // 8] = seg(x * sx - 1, y * sy, x * sx, y * sy)
    for y in range(8, H, 8):
        for x in range(0, W, 4):
            hg[y // 8, x // 4] = seg(x * sx, y * sy - 1, x * sx, y * sy)
    return vg, hg


def plane_case(seed, depth, W, H, chroma, cls="decoder", hs=1, vs=1, ctb=32):
    """(buf, vseg, hseg): buf = the W x H plane at [MARGIN:MARGIN + H, MARGIN:MARGIN + W] of a sentinel-filled array with MARGIN
    samples on every side; grids with garbage in their padding and at x = 0 / y = 0"""
    rng = np.random.default_rng(seed)
    maxv = (1 << depth) - 1
    buf = np.full((H + 2 * MARGIN, W + 2 * MARGIN), SENT8 if depth == 8 else SENT16, sdtype(depth))
    if cls == "decoder":
        plane = blocky(rng, depth, H, W, 8 if chroma else int(rng.choice([8, 16])))
        vg, hg = decoder_grids(rng, W, H, chroma, hs, vs, ctb)
    else:
        vg, hg = grids(W, H)
        if cls == "dense":
            plane = rng.integers(0, maxv + 1, (H, W)).astype(sdtype(depth))
            for g in (vg, hg):
                g["beta"] = rng.integers(0, 256, g.shape)
                g["tc"] = rng.integers(0, 256, g.shape)
                g["flags"] = rng.integers(0, 256, g.shape)
        else:
            plane = rng.choice(np.array([0, maxv]), (H, W)).astype(sdtype(depth))
            for g in (vg, hg):
                g["beta"], g["tc"] = 255, 255
                g["flags"] = rng.choice([0, 0, 0, 1, 2, 3], g.shape)
    buf[MARGIN:MARGIN + H, MARGIN:MARGIN + W] = plane
    # ignored entries: the picture edges and the grid padding
    rg = np.random.default_rng(seed + 1)
    for g in (vg, hg):
        g["reserved"] = rg.integers(0, 256, g.shape)
    for g, first in ((vg, vg[:, 0]), (hg, hg[0, :])):
        first["beta"], first["tc"], first["flags"] = 200, 200, 0xFC
    vg[:, (W + 7) // 8:] = np.frombuffer(rg.integers(1, 256, vg[:, (W + 7) // 8:].size * 4, dtype=np.uint8).tobytes(), DBK_DTYPE).reshape(vg[:, (W + 7) // 8:].shape)
    hg[:, W // 4:] = np.frombuffer(rg.integers(1, 256, hg[:, W // 4:].size * 4, dtype=np.uint8).tobytes(), DBK_DTYPE).reshape(hg[:, W // 4:].shape)
    return buf, vg, hg


def _plane_ptr(buf):
    return buf.ctypes.data + MARGIN * buf.strides[0] + MARGIN * buf.itemsize


def orc_plane(depth, chroma, buf, vg, hg, W, H, cnt=None):
    L = cl.oracle()
    f = L.orc_hevc_dbk_plane
    f.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_ssize_t, C.c_int, C.c_int, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p]
    d = buf.copy()
    assert f(depth, chroma, _plane_ptr(d), d.strides[0], W, H, vg.ctypes.data, vg.shape[1], hg.ctypes.data, hg.shape[1],
             None if cnt is None else cnt.ctypes.data) == 0
    return d


def ref_plane_ctb(depth, chroma, buf, vg, hg, W, H, log2_w, log2_h):
    f = ref().ffref_hevc_dbk_plane_ctb
    f.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_ssize_t, C.c_int, C.c_int, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int,
                  C.c_int]
    d = buf.copy()
    assert f(depth, chroma, _plane_ptr(d), d.strides[0], W, H, vg.ctypes.data, vg.shape[1], hg.ctypes.data, hg.shape[1], log2_w, log2_h) == 0
    return d


def branch_counts(depth, chroma, buf, vg, hg, W, H):
    cnt = np.zeros(9, np.int64)
    orc_plane(depth, chroma, buf, vg, hg, W, H, cnt)
    return dict(zip(BRANCHES, cnt.tolist()))


def fixture_case(depth, chroma):
    """the seeded plane behind each line of tests/golden/hevcdbk_hashes.txt: a 204x140 luma plane or a 100x68 4:2:0 chroma plane
    (sizes = 4 mod 8, not multiples of a kernel tile), decoder-shaped"""
    W, H = (100, 68) if chroma else (204, 140)
    return plane_case(900 + 10 * depth + chroma, depth, W, H, bool(chroma)), W, H


def fixture_hashes():
    out = {}
    for line in open(FIXTURE):
        d, what, h = line.split()
        out[(int(d), what == "chroma")] = h
    return out
