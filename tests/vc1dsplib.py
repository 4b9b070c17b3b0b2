"""Test infrastructure for VC-1 motion compensation and inverse transforms (VC1DSPContext's MC tables and transforms,
b200_vc1_mc_frame_device, b200_vc1_residual_frame_device): the seeded case generators, runners of the checker (oracle/liboracle.so:
orc_vc1_*) and of the compiled reference (oracle/_ref/libffref_vc1dsp.so, built by oracle/ref/vc1dsp.mk).  The reference's results are
kept as digests in tests/golden/vc1dsp_ref_digests.json (cpulibs.RefCheck) for machines without the reference.

Reference pictures are held with PAD samples of poison around the h_edge_pos x v_edge_pos picture (values unrelated to the edge
samples), so that a read past the decoder's window, or a clamp where the decoder reads the plane, changes the result."""
import ctypes as C
import hashlib
import os

import numpy as np

import cpulibs as cl
from ffmpeg_b200.vc1dsp import MC_DTYPE, RES_DTYPE, VC1RefDesc, ref_array, MC_1MV, MC_LUMA8, MC_CHROMA8, MSPEL, RND, AVG  # noqa: F401

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_LIB = "libffref_vc1dsp"
REF_DIGESTS = os.path.join(ROOT, "tests", "golden", "vc1dsp_ref_digests.json")
FIXTURE = os.path.join(ROOT, "tests", "golden", "vc1dsp_hashes.txt")
SENTINEL = 0x5A
PAD = 32                                                # poisoned samples around each reference plane
I16 = (-32768, -32767, -1, 0, 1, 32766, 32767)


def have_ref():
    return cl.have_ref(REF_LIB)


def ref():
    return cl.ref_lib(REF_LIB)


def RefCheck():
    return cl.RefCheck(REF_DIGESTS, REF_LIB)


# ---------------------------------------------------------------- members
MARGIN = 4


def member_case(seed):
    """(source picture with MARGIN samples before the block and room after it, dst0) — extremes and noise mixed, so the 2-D mspel
    sums leave 0..255"""
    rng = np.random.default_rng(seed)
    pic = rng.integers(0, 256, (MARGIN + 24, MARGIN + 24)).astype(np.uint8)
    pic[rng.random(pic.shape) < 0.3] = 0
    pic[rng.random(pic.shape) < 0.3] = 255
    return pic, rng.integers(0, 256, (20, 20)).astype(np.uint8)


def _mspel_fn(L, name):
    f = getattr(L, name)
    f.restype = C.c_int
    f.argtypes = [C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_ssize_t, C.c_int]
    return f


def _chroma_fn(L, name):
    f = getattr(L, name)
    f.restype = C.c_int
    f.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_ssize_t, C.c_int, C.c_int, C.c_int]
    return f


def _itx_fn(L, name):
    f = getattr(L, name)
    f.restype = C.c_int
    f.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_ssize_t, C.c_void_p]
    return f


def mspel_calls():
    """(avg, size, dxy, rnd) of every mspel entry with both rnd values"""
    return [(avg, size, dxy, rnd) for avg in (0, 1) for size in (0, 1) for dxy in range(16) for rnd in (0, 1)]


def chroma_calls():
    """(avg, idx, h, x, y): both widths, every eighth-sample position, heights 1, 4, 8 and 16"""
    return [(avg, idx, h, x, y) for avg in (0, 1) for idx in (0, 1) for h in (1, 4, 8, 16) for x in range(8) for y in range(8)
            if (x + 3 * y + h + idx) % 3 == 0 or h == 8]


def run_members(L, prefix, seed):
    """every mspel and chroma member call on one picture; src and dst share the stride as in the reference's signature"""
    pic, dst0 = member_case(seed)
    stride = 40
    P = np.zeros((MARGIN + 24, stride), np.uint8)
    P[:, :pic.shape[1]] = pic
    D0 = np.zeros((20, stride), np.uint8)
    D0[:, :20] = dst0
    mspel, chroma = _mspel_fn(L, prefix + "_vc1_mspel"), _chroma_fn(L, prefix + "_vc1_chroma")
    out = []
    for avg, size, dxy, rnd in mspel_calls():
        d = D0.copy()
        assert mspel(avg, size, dxy, d.ctypes.data, P[MARGIN:, MARGIN:].ctypes.data, stride, rnd) == 0
        out.append(d)
    for avg, idx, h, x, y in chroma_calls():
        d = D0.copy()
        assert chroma(avg, idx, d.ctypes.data, P[MARGIN:, MARGIN:].ctypes.data, stride, h, x, y) == 0
        out.append(d)
    return out


def coef_blocks(rng, n, kind):
    """n blocks of 64 int16: "decoder" (sparse dequantised values), "dense" (uniform int16) or "extreme" (int16 limits)"""
    if kind == "extreme":
        return rng.choice(np.array(I16, np.int16), (n, 64))
    if kind == "dense":
        return rng.integers(-32768, 32768, (n, 64)).astype(np.int16)
    b = np.zeros((n, 64), np.int16)
    for k in range(n):
        m = rng.integers(1, 12)
        pos = rng.choice(64, m, replace=False)
        q = int(rng.integers(1, 32))
        b[k, pos] = (rng.integers(-40, 41, m) * 2 * q + np.sign(rng.integers(-1, 2, m)) * q).astype(np.int16)
    return b


def run_itx(L, prefix, seed, kind):
    """every transform member (tt x dc) on n blocks: the dest and block each leaves"""
    rng = np.random.default_rng(seed)
    f = _itx_fn(L, prefix + "_vc1_itx")
    blocks = coef_blocks(rng, 12, kind)
    out = []
    for tt in range(4):
        for dc in (0, 1):
            for b in blocks:
                blk = b.copy()
                dest = rng.integers(0, 256, (8, 16)).astype(np.uint8)
                assert f(tt, dc, dest.ctypes.data, dest.strides[0], blk.ctypes.data) == 0
                out += [blk, dest]
    return out


# ---------------------------------------------------------------- frames
class RefPic:
    """a reference picture: three planes with PAD samples of poison around h_edge_pos x v_edge_pos (chroma: halves), and the
    decoder's per-reference state"""

    def __init__(self, rng, H, V, rangered=0, use_ic=0, interlaced=0):
        self.planes, self.offs = [], []
        for c, (w, h) in enumerate(((H, V), (H >> 1, V >> 1), (H >> 1, V >> 1))):
            ls = (w + 2 * PAD + 63) // 64 * 64
            buf = rng.integers(0, 256, (h + 2 * PAD, ls)).astype(np.uint8)        # poison everywhere, then the picture
            buf[PAD:PAD + h, PAD:PAD + w] = rng.integers(0, 256, (h, w)).astype(np.uint8)
            self.planes.append(buf)
            self.offs.append(PAD * ls + PAD)
        self.rangered, self.use_ic, self.interlaced = rangered, use_ic, interlaced
        self.luty = rng.integers(0, 256, (2, 256)).astype(np.uint8) if use_ic else None
        self.lutuv = rng.integers(0, 256, (2, 256)).astype(np.uint8) if use_ic else None

    def desc(self, bases=None):
        """VC1RefDesc with host addresses, or with `bases` (the planes' buffer addresses elsewhere, e.g. on the device)"""
        bases = bases or [p.ctypes.data for p in self.planes]
        a = [b + o for b, o in zip(bases, self.offs)]
        return VC1RefDesc(a[0], a[1], a[2], self.planes[0].strides[0], self.planes[1].strides[0], self.rangered, self.use_ic, self.luty,
                          self.lutuv, self.interlaced)


def dst_planes(mbw, mbh, fill=SENTINEL):
    return [np.full((16 * mbh + 8, 16 * mbw + 16), fill, np.uint8)] + [np.full((8 * mbh + 8, 8 * mbw + 16), fill, np.uint8) for _ in range(2)]


def _uv(mv, fast):
    """chroma vector of a luma vector (vc1_mc.c:204-219)"""
    uv = (mv + ((mv & 3) == 3)) >> 1
    if fast:
        uv = uv + ((uv & 1) if uv < 0 else -(uv & 1))
    return uv


def _src(op_src, ref, mbx, mby, mx, my, fast, mbw, mbh, n_off=(0, 0)):
    """the decoder's positions of a 1MV (or 4MV block n_off) source, simple / main profile clip (vc1_mc.c:258-263)"""
    op_src["ref"] = ref
    op_src["x"] = np.clip(mbx * 16 + n_off[0] + (mx >> 2), -16, mbw * 16)
    op_src["y"] = np.clip(mby * 16 + n_off[1] + (my >> 2), -16, mbh * 16)
    op_src["mx"], op_src["my"] = mx & 3, my & 3
    uvmx, uvmy = _uv(mx, fast), _uv(my, fast)
    op_src["uvx"] = np.clip(mbx * 8 + (uvmx >> 2), -8, mbw * 8)
    op_src["uvy"] = np.clip(mby * 8 + (uvmy >> 2), -8, mbh * 8)
    op_src["uvmx"], op_src["uvmy"] = uvmx & 3, uvmy & 3


def _mv(rng, far):
    """a quarter-sample vector: mostly small, sometimes far enough to leave the picture"""
    r = far if rng.random() < 0.25 else 24
    return int(rng.integers(-4 * r, 4 * r + 1)), int(rng.integers(-4 * r, 4 * r + 1))


def mc_ops(rng, mbw, mbh, b_frame, mspel, rnd, fast=0, far=48, intra=0.08):
    """decoder-shaped ops of a progressive picture: P (random 1MV / 4MV macroblocks, some intra) or B (forward, backward and
    interpolated 1MV macroblocks); flags per op, vectors near every edge"""
    ops = []
    flags = (MSPEL if mspel else 0) | (RND if rnd else 0)
    for mby in range(mbh):
        for mbx in range(mbw):
            if rng.random() < intra:
                continue
            edge = mbx in (0, mbw - 1) or mby in (0, mbh - 1)
            if b_frame or rng.random() < 0.6:
                o = np.zeros((), MC_DTYPE)
                o["dst_x"], o["dst_y"], o["kind"], o["flags"] = 16 * mbx, 16 * mby, MC_1MV, flags
                mode = rng.integers(0, 3) if b_frame else 0                     # 0 forward, 1 backward, 2 interpolated
                first = 1 if mode == 1 else 0
                mx, my = _mv(rng, far if edge else 24)
                _src(o["src"][0], first, mbx, mby, mx, my, fast, mbw, mbh)
                if mode == 2:
                    o["flags"] |= AVG
                    mx, my = _mv(rng, far if edge else 24)
                    _src(o["src"][1], 1, mbx, mby, mx, my, fast, mbw, mbh)
                ops.append(o)
                continue
            for n in range(4):                                                  # 4MV: four luma blocks, then the chroma op
                o = np.zeros((), MC_DTYPE)
                o["dst_x"], o["dst_y"], o["kind"], o["flags"] = 16 * mbx + (n & 1) * 8, 16 * mby + (n & 2) * 4, MC_LUMA8, flags
                mx, my = _mv(rng, far if edge else 24)
                _src(o["src"][0], 0, mbx, mby, mx, my, fast, mbw, mbh, ((n & 1) * 8, (n & 2) * 4))
                ops.append(o)
            o = np.zeros((), MC_DTYPE)
            o["dst_x"], o["dst_y"], o["kind"], o["flags"] = 8 * mbx, 8 * mby, MC_CHROMA8, flags
            mx, my = _mv(rng, far if edge else 24)
            _src(o["src"][0], 0, mbx, mby, mx, my, fast, mbw, mbh)
            ops.append(o)
    return np.array(ops, MC_DTYPE)


def mc_case(seed, mbw, mbh, H=None, V=None, b_frame=False, mspel=1, rnd=0, rangered=(0, 0), use_ic=(0, 0), far=48):
    """(refs, ops, dst planes of sentinels, H, V) of a decoder-shaped progressive picture; H / V default to the MB grid minus a few
    samples, so the poison lies inside the grid"""
    rng = np.random.default_rng(seed)
    H = 16 * mbw - 6 if H is None else H
    V = 16 * mbh - 10 if V is None else V
    refs = [RefPic(rng, H, V, rangered[k], use_ic[k]) for k in range(2 if b_frame else 1)]
    ops = mc_ops(rng, mbw, mbh, b_frame, mspel, rnd, fast=seed & 1, far=far)
    return refs, ops, dst_planes(mbw, mbh), H, V


def _mc_frame(L, name, mbw, mbh, H, V, refs, ops, dst):
    f = getattr(L, name)
    f.restype = C.c_int64
    f.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_ssize_t, C.c_ssize_t, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int64, C.c_void_p]
    d = [p.copy() for p in dst]
    ops = np.ascontiguousarray(ops)
    planes = (C.c_void_p * 3)(*[p.ctypes.data for p in d])
    arr = ref_array([r.desc() for r in refs])
    r = f(len(refs), C.cast(arr, C.c_void_p), planes, d[0].strides[0], d[1].strides[0], mbw, mbh, H, V, len(ops), ops.ctypes.data)
    assert r >= 0
    return d


def orc_mc_frame(mbw, mbh, H, V, refs, ops, dst):
    return _mc_frame(cl.oracle(), "orc_vc1_mc_frame", mbw, mbh, H, V, refs, ops, dst)


def ref_mc_frame(mbw, mbh, H, V, refs, ops, dst):
    return _mc_frame(ref(), "ffref_vc1_mc_frame", mbw, mbh, H, V, refs, ops, dst)


def residual_case(seed, mbw, mbh, kind="decoder", skip=0.1):
    """(ops, coef): the six blocks of every inter macroblock (4 luma in raster order, U, V), each with a random transform type, a
    random sub-block pattern that leaves at least one sub-block (as the decoder's cbp does) and DC-only bits"""
    rng = np.random.default_rng(seed)
    ops = []
    for mby in range(mbh):
        for mbx in range(mbw):
            if rng.random() < skip:
                continue
            for b in range(6):
                o = np.zeros((), RES_DTYPE)
                o["plane"] = 0 if b < 4 else b - 3
                o["x"] = 16 * mbx + (b & 1) * 8 if b < 4 else 8 * mbx
                o["y"] = 16 * mby + (b & 2) * 4 if b < 4 else 8 * mby
                tt = int(rng.integers(0, 4))
                o["ttblk"] = tt
                nsub = 1 if tt == 0 else 4 if tt == 3 else 2
                pat = int(rng.integers(0, (1 << nsub) - 1)) if tt else 0
                o["subblkpat"] = pat
                o["dc"] = int(rng.integers(0, 1 << nsub))
                o["coef_off"] = 64 * len(ops)
                ops.append(o)
    ops = np.array(ops, RES_DTYPE)
    coef = coef_blocks(rng, max(1, len(ops)), kind).reshape(-1)
    return ops, np.ascontiguousarray(coef)


def _res_frame(L, name, mbw, mbh, ops, coef, dst):
    f = getattr(L, name)
    f.restype = C.c_int64
    f.argtypes = [C.c_void_p, C.c_ssize_t, C.c_ssize_t, C.c_int, C.c_int, C.c_void_p, C.c_int64, C.c_void_p]
    d = [p.copy() for p in dst]
    ops = np.ascontiguousarray(ops)
    planes = (C.c_void_p * 3)(*[p.ctypes.data for p in d])
    assert f(planes, d[0].strides[0], d[1].strides[0], mbw, mbh, coef.ctypes.data, len(ops), ops.ctypes.data) >= 0
    return d


def orc_residual_frame(mbw, mbh, ops, coef, dst):
    return _res_frame(cl.oracle(), "orc_vc1_residual_frame", mbw, mbh, ops, coef, dst)


def ref_residual_frame(mbw, mbh, ops, coef, dst):
    return _res_frame(ref(), "ffref_vc1_residual_frame", mbw, mbh, ops, coef, dst)


# ---------------------------------------------------------------- fixture: MC then residual on decoder-shaped pictures
# (name, mbw, mbh, H, V, b_frame, mspel, rnd, rangered, use_ic): P and B, mspel and hpel, rnd 0 / 1, with and without range reduction
# and IC (different LUTs per parity and per reference), and one picture whose edge positions are below 22
FIXTURE_CASES = (
    ("p-mspel-rnd0", 9, 7, None, None, False, 1, 0, (0, 0), (0, 0)),
    ("p-mspel-rnd1-ic", 9, 7, None, None, False, 1, 1, (0, 0), (1, 0)),
    ("p-hpel-rnd0-rangered", 9, 7, None, None, False, 0, 0, (1, 0), (0, 0)),
    ("p-hpel-rnd1", 9, 7, 141, 99, False, 0, 1, (0, 0), (0, 0)),
    ("b-mspel-rnd0-ic-next", 9, 7, None, None, True, 1, 0, (0, 0), (0, 1)),
    ("b-hpel-rnd1-rangered-ic", 9, 7, None, None, True, 0, 1, (1, 1), (1, 0)),
    ("p-small-edges", 2, 2, 18, 20, False, 1, 1, (0, 0), (0, 0)),
    ("b-small-edges", 2, 2, 21, 17, True, 0, 0, (0, 0), (0, 0)),
)


def fixture_case(name):
    k = [c[0] for c in FIXTURE_CASES].index(name)
    _, mbw, mbh, H, V, b, ms, rnd, rr, ic = FIXTURE_CASES[k]
    refs, ops, dst, H, V = mc_case(700 + k, mbw, mbh, H, V, b, ms, rnd, rr, ic)
    rops, coef = residual_case(750 + k, mbw, mbh, "decoder" if k % 2 == 0 else "extreme")
    return mbw, mbh, H, V, refs, ops, dst, rops, coef


def digest(planes):
    h = hashlib.sha256()
    for p in planes:
        h.update(np.ascontiguousarray(p).tobytes())
    return h.hexdigest()


def fixture_hashes():
    out = {}
    for line in open(FIXTURE):
        name, h = line.split()
        out[name] = h
    return out
