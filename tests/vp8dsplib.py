"""Test infrastructure for VP8 / VP7 motion compensation and residual (VP8DSPContext's MC tables and residual members,
b200_vp8_mc_frame_device, b200_vp8_residual_frame_device): the seeded case generators, runners of the checker (oracle/liboracle.so:
orc_vp8_*) and of the compiled reference (oracle/_ref/libffref_vp8dsp.so, built by oracle/ref/vp8dsp.mk).  The reference's results are
kept as digests in tests/golden/vp8dsp_ref_digests.json (cpulibs.RefCheck) for machines without the reference."""
import ctypes as C
import hashlib
import os

import numpy as np

import cpulibs as cl
from ffmpeg_b200._lib import Vp8McRef
from ffmpeg_b200.vp8dsp import MC_DTYPE, RES_DTYPE, LUMA, CHROMA, RESIDUAL_LUMA, MB_COEFS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_LIB = "libffref_vp8dsp"
REF_DIGESTS = os.path.join(ROOT, "tests", "golden", "vp8dsp_ref_digests.json")
FIXTURE = os.path.join(ROOT, "tests", "golden", "vp8dsp_hashes.txt")
WIDTHS = (16, 8, 4)                                  # table index 0..2
SENTINEL = 0x5A
ZIGZAG = (0, 1, 4, 8, 5, 2, 3, 6, 9, 12, 13, 10, 7, 11, 14, 15)   # ff_zigzag_scan


def have_ref():
    return cl.have_ref(REF_LIB)


def ref():
    return cl.ref_lib(REF_LIB)


def RefCheck():
    return cl.RefCheck(REF_DIGESTS, REF_LIB)


def picture(rng, h, w, cls):
    """cls 0: uniform noise, 1: only 0 and 255 alternating in runs of seeded lengths 1..3 along rows and columns (drives the 6-tap sums
    past both clip bounds in both passes)"""
    if cls == 1:
        cols = np.repeat(np.arange(w) % 2, rng.integers(1, 4, w))[:w]
        rows = np.repeat(np.arange(h) % 2, rng.integers(1, 4, h))[:h]
        return ((cols[None, :] ^ rows[:, None]) * 255).astype(np.uint8)
    return rng.integers(0, 256, (h, w)).astype(np.uint8)


# ---------------------------------------------------------------- MC members: put_vp8_{epel,bilinear}_pixels_tab[size][v][h]
MARGIN = 8


def member_case(seed, cls):
    """(source picture with MARGIN samples before the block and room after it, dst0 [32, 24])"""
    rng = np.random.default_rng(seed)
    return picture(rng, MARGIN + 32 + 8, MARGIN + 16 + 8, cls), rng.integers(0, 256, (32, 24)).astype(np.uint8)


def positions(bilinear):
    """the non-NULL table positions (size index, v, h)"""
    for i, w in enumerate(WIDTHS):
        for v in range(3):
            for h in range(3):
                if not bilinear and w == 16 and (v == 1 or h == 1):
                    continue
                yield i, v, h


def mc_calls(seed, bilinear):
    """every non-NULL entry with every phase it takes in its filtered directions (epel 1..7, bilinear 0..7; both directions jointly
    for 2-D entries), a seeded out-of-range phase in a direction it does not filter (which it must ignore), heights 1..2w"""
    rng = np.random.default_rng(seed)
    lo = 0 if bilinear else 1
    for i, v, h in positions(bilinear):
        w = WIDTHS[i]
        px = range(lo, 8) if h else [int(rng.integers(0, 200))]
        py = range(lo, 8) if v else [int(rng.integers(0, 200))]
        for mx in px:
            for my in py:
                hh = int(rng.choice([1, 2, 3, w, 2 * w, int(rng.integers(1, 2 * w + 1))]))
                yield (bilinear, w, v, h, hh, mx, my)


def run_mc(L, name, call, pic, dst0):
    bilinear, w, v, h, hh, mx, my = call
    f = getattr(L, name)
    f.argtypes = [C.c_int] * 4 + [C.c_void_p, C.c_ssize_t, C.c_void_p, C.c_ssize_t] + [C.c_int] * 3
    d = dst0.copy()
    src = pic.ctypes.data + MARGIN * pic.strides[0] + MARGIN
    assert f(bilinear, w, v, h, d.ctypes.data, d.strides[0], src, pic.strides[0], hh, mx, my) == 0
    return d


def run_members(L, prefix, seed, bilinear, cls):
    pic, dst0 = member_case(seed, cls)
    return [run_mc(L, prefix + "_vp8_mc", c, pic, dst0) for c in mc_calls(seed, bilinear)]


def subpel_filters(L, name):
    f = getattr(L, name)
    f.restype = C.POINTER(C.c_uint8)
    return np.ctypeslib.as_array(f(), (7, 6)).copy()


# ---------------------------------------------------------------- residual members
def coef_blocks(rng, n, kind):
    """n x 16 int16: 'decoder' (a few low-frequency coefficients in zigzag order, many blocks DC only), 'dense' (uniform over
    +-2048), 'extreme' (int16 -32768 / 32767 and values near them)"""
    if kind == "dense":
        return rng.integers(-2048, 2049, (n, 16)).astype(np.int16)
    if kind == "extreme":
        v = rng.choice(np.array([-32768, -32767, -32766, 32767, 32766, 32765, 0, -1, 1], np.int64), (n, 16))
        return v.astype(np.int16)
    b = np.zeros((n, 16), np.int16)
    last = rng.integers(0, 17, n)
    for k in range(n):
        for j in range(last[k]):
            b[k, ZIGZAG[j]] = rng.integers(-300, 301) >> int(rng.integers(0, 4))
    return b


def run_wht(L, name, is_vp7, dc_only, dc):
    """(block[4][4][16] after the member, dc after the member); block starts as a seeded pattern whose coefficient 0s must change"""
    f = getattr(L, name)
    f.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    f.restype = None
    block = (np.arange(256, dtype=np.int64) * 37 % 2001 - 1000).astype(np.int16).reshape(4, 4, 16)
    d = dc.astype(np.int16).copy()
    f(is_vp7, dc_only, block.ctypes.data, d.ctypes.data)
    return block, d


def run_idct(L, name, is_vp7, which, blocks, dst0):
    """which 0 idct_add (1 block), 1 dc_add (1), 2 dc_add4y (4), 3 dc_add4uv (4) on dst0 [8, 16]; returns (dst, blocks after)"""
    f = getattr(L, name)
    f.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_ssize_t]
    f.restype = None
    d, b = dst0.copy(), np.ascontiguousarray(blocks.astype(np.int16)).copy()
    f(is_vp7, which, d.ctypes.data, b.ctypes.data, d.strides[0])
    return d, b


def residual_member_runs(L, prefix, seed, is_vp7, kind):
    """every residual member on seeded blocks of one kind; returns the list of all outputs"""
    rng = np.random.default_rng(seed)
    out = []
    for dc_only in (0, 1):
        for _ in range(24):
            out += list(run_wht(L, prefix + "_vp8_wht", is_vp7, dc_only, coef_blocks(rng, 1, kind)[0]))
    for which, nb in ((0, 1), (1, 1), (2, 4), (3, 4)):
        for _ in range(24):
            out += list(run_idct(L, prefix + "_vp8_idct", is_vp7, which, coef_blocks(rng, nb, kind), rng.integers(0, 256, (8, 16)).astype(np.uint8)))
    return out


# ---------------------------------------------------------------- frames
PAD = 24            # sentinel samples right of and below every dst plane


def mb_partitions(rng, mbw, mbh, nrefs=3, far=80, intra=0.1):
    """per inter MB (mb_x, mb_y, ref, partitioning, mvs): partitioning 0 none, 1 16x8, 2 8x16, 3 8x8, 4 4x4 split, with quarter-sample
    MVs whose source windows reach up to `far` samples outside the plane; a fraction `intra` of the MBs is left out (sentinels)"""
    W, H = 16 * mbw, 16 * mbh
    mbs = []
    for y in range(mbh):
        for x in range(mbw):
            if rng.random() < intra:
                continue
            part = int(rng.choice(5, p=[0.6, 0.1, 0.1, 0.1, 0.1]))
            nmv = (1, 2, 2, 4, 16)[part]
            mvs = []
            for _ in range(nmv):
                sel = rng.random()
                if sel < 0.15:
                    mvs.append((0, 0))
                elif sel < 0.45:                           # anywhere, up to `far` samples outside the plane
                    tx, ty = int(rng.integers(-far - 16, W + far)), int(rng.integers(-far - 16, H + far))
                    mvs.append((4 * (tx - 16 * x) + int(rng.integers(0, 4)), 4 * (ty - 16 * y) + int(rng.integers(0, 4))))
                else:
                    mvs.append((int(rng.integers(-64, 65)), int(rng.integers(-64, 65))))
            mbs.append((x, y, int(rng.integers(0, nrefs)), part, mvs))
    return mbs


def mc_ops(mbs):
    """the ops of inter_predict (vp8.c:2001-2083): luma (x_off + (mv >> 2), (mv * 2) & 7), chroma (x_off + (mv >> 3), mv & 7), the
    split-MV chroma average of the 4x4 partitioning (no profile-3 rounding)"""
    ops = []

    def add(plane, dx, dy, w, h, ref, sx, sy, mx, my):
        ops.append((sx, sy, dx, dy, plane, w, h, ref, mx, my, (0, 0)))

    for (x, y, ref, part, mvs) in mbs:
        xo, yo = 16 * x, 16 * y
        if part == 4:
            for k, (mvx, mvy) in enumerate(mvs):
                bx, by = 4 * (k % 4), 4 * (k // 4)
                add(LUMA, xo + bx, yo + by, 4, 4, ref, xo + bx + (mvx >> 2), yo + by + (mvy >> 2), (mvx * 2) & 7, (mvy * 2) & 7)
            for cy in range(2):
                for cx in range(2):
                    idx = [2 * cy * 4 + 2 * cx, 2 * cy * 4 + 2 * cx + 1, (2 * cy + 1) * 4 + 2 * cx, (2 * cy + 1) * 4 + 2 * cx + 1]
                    sx, sy = sum(mvs[i][0] for i in idx), sum(mvs[i][1] for i in idx)
                    ux, uy = (sx + 2 + (-1 if sx < 0 else 0)) >> 2, (sy + 2 + (-1 if sy < 0 else 0)) >> 2
                    cxo, cyo = xo // 2 + 4 * cx, yo // 2 + 4 * cy
                    add(CHROMA, cxo, cyo, 4, 4, ref, cxo + (ux >> 3), cyo + (uy >> 3), ux & 7, uy & 7)
            continue
        parts = {0: [(0, 0, 16, 16)], 1: [(0, 0, 16, 8), (0, 8, 16, 8)], 2: [(0, 0, 8, 16), (8, 0, 8, 16)],
                 3: [(0, 0, 8, 8), (8, 0, 8, 8), (0, 8, 8, 8), (8, 8, 8, 8)]}[part]
        for (bx, by, bw, bh), (mvx, mvy) in zip(parts, mvs):
            add(LUMA, xo + bx, yo + by, bw, bh, ref, xo + bx + (mvx >> 2), yo + by + (mvy >> 2), (mvx * 2) & 7, (mvy * 2) & 7)
            cxo, cyo = (xo + bx) // 2, (yo + by) // 2
            add(CHROMA, cxo, cyo, bw // 2, bh // 2, ref, cxo + (mvx >> 3), cyo + (mvy >> 3), mvx & 7, mvy & 7)
    return np.array(ops, MC_DTYPE) if ops else np.zeros(0, MC_DTYPE)


def ref_frames(rng, mbw, mbh, nrefs=3, cls=0, pad=16):
    """nrefs frames (y, u, v) with `pad` columns of other samples right of each plane (never read: reads clamp to the plane)"""
    out = []
    for _ in range(nrefs):
        out.append(tuple(picture(rng, s * mbh, s * mbw + pad, cls) for s in (16, 8, 8)))
    return out


def dst_planes(mbw, mbh, fill=SENTINEL):
    return [np.full((16 * mbh + PAD, 16 * mbw + PAD), fill, np.uint8)] + [np.full((8 * mbh + PAD, 8 * mbw + PAD), fill, np.uint8) for _ in range(2)]


def mc_case(seed, mbw, mbh, cls=0, far=80, intra=0.1):
    """(refs, ops, dst planes of sentinels) of a decoder-shaped inter frame"""
    rng = np.random.default_rng(seed)
    refs = ref_frames(rng, mbw, mbh, 3, cls)
    ops = mc_ops(mb_partitions(rng, mbw, mbh, 3, far, intra))
    return refs, ops, dst_planes(mbw, mbh)


def ref_array(refs, ptrs=None):
    arr = (Vp8McRef * len(refs))()
    for k, (y, u, v) in enumerate(refs):
        p = (y.ctypes.data, u.ctypes.data, v.ctypes.data) if ptrs is None else ptrs[k]
        arr[k] = Vp8McRef(p[0], p[1], p[2], y.strides[0], u.strides[0])
    return arr


def _mc_frame(L, name, bilinear, mbw, mbh, refs, ops, dst):
    f = getattr(L, name)
    f.restype = C.c_int64
    f.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_ssize_t, C.c_ssize_t]
    d = [p.copy() for p in dst]
    ops = np.ascontiguousarray(ops)
    planes = (C.c_void_p * 3)(*[p.ctypes.data for p in d])
    r = f(bilinear, mbw, mbh, len(refs), C.cast(ref_array(refs), C.c_void_p), len(ops), ops.ctypes.data, planes, d[0].strides[0], d[1].strides[0])
    assert r >= 0
    return d


def orc_mc_frame(bilinear, mbw, mbh, refs, ops, dst):
    return _mc_frame(cl.oracle(), "orc_vp8_mc_frame", bilinear, mbw, mbh, refs, ops, dst)


def ref_mc_frame(bilinear, mbw, mbh, refs, ops, dst):
    return _mc_frame(ref(), "ffref_vp8_mc_frame", bilinear, mbw, mbh, refs, ops, dst)


def residual_case(seed, mbw, mbh, is_vp7, kind="decoder", skip=0.1):
    """(ops RES_DTYPE, coef int16 [n * 400]) of one frame: per MB a mode (I4x4: no luma; VP8 split: no Y2; otherwise Y2), the nnz
    cache and Y2 nnz as decode_mb_coeffs sets them (luma blocks with Y2 count nnz + block_dc), coefficients within each block's nnz in
    zigzag order ('decoder'); 'dense' / 'extreme' put arbitrary values in all 400 coefficients (non-zero DCs in nnz-0 blocks included)
    under a random nnz cache"""
    rng = np.random.default_rng(seed)
    mbs = [(x, y) for y in range(mbh) for x in range(mbw) if rng.random() >= skip]
    n = len(mbs)
    ops = np.zeros(n, RES_DTYPE)
    coef = np.zeros(n * MB_COEFS, np.int16)
    for k, (x, y) in enumerate(mbs):
        o = ops[k]
        o["coef_off"], o["mb_x"], o["mb_y"] = k * MB_COEFS, x, y
        mode = int(rng.choice(3, p=[0.1, 0.0, 0.9] if is_vp7 else [0.1, 0.1, 0.8]))    # 0 I4x4, 1 split, 2 Y2
        o["flags"] = 0 if mode == 0 else RESIDUAL_LUMA
        c = coef[k * MB_COEFS:(k + 1) * MB_COEFS]
        if kind != "decoder":
            c[:] = coef_blocks(rng, 25, kind).reshape(-1)
            o["nnz"] = rng.choice(np.array([0, 0, 1, 1, 2, 5, 16]), (6, 4))
            o["y2_nnz"] = int(rng.choice([0, 1, 2, 16])) if mode == 2 else 0
            continue
        y2 = 0
        if mode == 2:
            y2 = int(rng.choice([0, 1, 1, 2, 5, 16]))
            if y2:
                d = np.zeros(16, np.int16)
                for j in range(y2):
                    d[ZIGZAG[j]] = rng.integers(-2000, 2001) if j == 0 or rng.random() < 0.5 else 0
                c[384:400] = d
        o["y2_nnz"] = y2
        for b in range(24):
            luma = b < 16
            start = 1 if (luma and mode == 2) else 0
            nz = int(rng.choice([0, 0, 1, 1, 2, 3, 6, 16]))
            nz = 0 if nz <= start and start else nz
            blk = np.zeros(16, np.int16)
            for j in range(start, nz):
                blk[ZIGZAG[j]] = rng.integers(-400, 401) if j == nz - 1 or rng.random() < 0.6 else 0
            if nz and not blk.any():
                blk[ZIGZAG[nz - 1]] = 7
            c[16 * b:16 * b + 16] = blk
            o["nnz"][b // 4, b % 4] = nz + (1 if (luma and mode == 2 and y2) else 0)
    return ops, coef


def _res_frame(L, name, is_vp7, ops, coef, dst):
    f = getattr(L, name)
    f.restype = C.c_int64
    f.argtypes = [C.c_int, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_ssize_t, C.c_ssize_t]
    d = [p.copy() for p in dst]
    ops = np.ascontiguousarray(ops)
    planes = (C.c_void_p * 3)(*[p.ctypes.data for p in d])
    assert f(is_vp7, len(ops), ops.ctypes.data, coef.ctypes.data, planes, d[0].strides[0], d[1].strides[0]) >= 0
    return d


def orc_residual_frame(is_vp7, ops, coef, dst):
    return _res_frame(cl.oracle(), "orc_vp8_residual_frame", is_vp7, ops, coef, dst)


def ref_residual_frame(is_vp7, ops, coef, dst):
    return _res_frame(ref(), "ffref_vp8_residual_frame", is_vp7, ops, coef, dst)


# ---------------------------------------------------------------- fixture: MC then residual on one decoder-shaped frame
FIXTURE_CASES = ((0, 0), (0, 1), (1, 0), (1, 1))       # (is_vp7, bilinear)


def fixture_case(is_vp7, bilinear):
    """the seeded frame behind each line of tests/golden/vp8dsp_hashes.txt: 12 x 9 macroblocks, every partitioning, windows up to 80
    samples outside the plane, then the residual of every MB (decoder-shaped nnz and coefficients)"""
    seed = 900 + 2 * is_vp7 + bilinear
    refs, ops, dst = mc_case(seed, 12, 9)
    rops, coef = residual_case(seed + 50, 12, 9, is_vp7)
    return refs, ops, dst, rops, coef


def digest(planes):
    h = hashlib.sha256()
    for p in planes:
        h.update(np.ascontiguousarray(p).tobytes())
    return h.hexdigest()


def fixture_hashes():
    out = {}
    for line in open(FIXTURE):
        v7, bil, h = line.split()
        out[(int(v7), int(bil))] = h
    return out
