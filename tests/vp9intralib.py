"""Test infrastructure for VP9 intra reconstruction (the intra_pred members of VP9DSPContext and b200_vp9_intra_recon_frame_device):
a decoder-shaped frame generator (random partition trees per 64x64 superblock in decode_sb's order, intra and inter blocks, per-4x4
modes, skip, lossless frames, tile columns, every chroma format, odd sizes) with the op list built the way intra_recon's loops clip it,
runners of the checker (oracle/liboracle.so: orc_vp9_intra_pred, orc_vp9_intra_frame) and of the compiled reference
(oracle/_ref/libffref_vp9intra.so, built by oracle/ref/vp9intra.mk).  The reference's results are kept as digests in
tests/golden/vp9intra_ref_digests.json (cpulibs.RefCheck) for machines without the reference."""
import ctypes as C
import hashlib
import os

import numpy as np

import cpulibs as cl
from ffmpeg_b200.vp9dsp import INTRA_DTYPE, INTRA_HAVE_LEFT, INTRA_HAVE_RIGHT, INTRA_LOSSLESS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_SO = os.path.join(ROOT, "oracle", "_ref", "libffref_vp9intra.so")
REF_DIGESTS = os.path.join(ROOT, "tests", "golden", "vp9intra_ref_digests.json")
FIXTURE = os.path.join(ROOT, "tests", "golden", "vp9intra_hashes.txt")
DEPTHS = (8, 10, 12)
FORMATS = {"420": (1, 1), "422": (1, 0), "440": (0, 1), "444": (0, 0)}
MARGIN = 8           # sentinel samples around every plane's area
# ff_vp9_bwh_tab[1] (vp9data.c): block size in 8x8 units, and [0] in 4x4 units, by BlockSize
BWH8 = ((8, 8), (8, 4), (4, 8), (4, 4), (4, 2), (2, 4), (2, 2), (2, 1), (1, 2), (1, 1), (1, 1), (1, 1), (1, 1))
BWH4 = ((16, 16), (16, 8), (8, 16), (8, 8), (8, 4), (4, 8), (4, 4), (4, 2), (2, 4), (2, 2), (2, 1), (1, 2), (1, 1))
_ref = None


def have_ref():
    return os.path.exists(REF_SO) and cl.have_ref()


def ref():
    global _ref
    if _ref is None:
        _ref = C.CDLL(REF_SO)
        _ref.ffref_vp9_intra_pred.argtypes = [C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_ssize_t, C.c_void_p, C.c_void_p]
        _ref.ffref_vp9_intra_frame.argtypes = [C.c_int] * 5 + [C.c_void_p, C.c_ssize_t, C.c_ssize_t, C.c_int, C.c_int, C.c_void_p,
                                                               C.c_void_p, C.c_void_p]
    return _ref


def RefCheck():
    return cl.RefCheck(REF_DIGESTS)


def sdtype(depth):
    return np.uint8 if depth == 8 else np.uint16


def cdtype(depth):
    return np.int16 if depth == 8 else np.int32


class Frame:
    """One frame's intra work on planes that already hold an inter reconstruction (random samples).
    kind: "intra" (every block intra) or "inter" (intra blocks with probability p_intra among inter blocks); sizes: "mixed" (random
    partition trees) or "4x4" (every 8x8 split into 4x4 blocks with 4x4 transforms).  tiles: tile columns (split evenly over the
    superblock columns).  Planes are the 8-aligned area with MARGIN sentinel samples all around; ops / coef / blocks / eobs feed the
    entry, the checker and the reference."""

    def __init__(self, seed, depth, fmt, width, height, kind="intra", sizes="mixed", tiles=1, lossless=False, p_skip=0.2, p_intra=0.1):
        rng = np.random.default_rng(seed)
        self.depth, self.fmt, self.width, self.height, self.lossless = depth, fmt, width, height, lossless
        self.ss_h, self.ss_v = FORMATS[fmt]
        self.cols, self.rows = (width + 7) >> 3, (height + 7) >> 3
        self.W = [self.cols * 8, self.cols * 8 >> self.ss_h, self.cols * 8 >> self.ss_h]
        self.H = [self.rows * 8, self.rows * 8 >> self.ss_v, self.rows * 8 >> self.ss_v]
        st = sdtype(depth)
        sent = 0x5A5A & ((1 << depth) - 1) if depth > 8 else 0x5A
        self.planes = []
        for p in range(3):
            a = np.full((self.H[p] + 2 * MARGIN, self.W[p] + 2 * MARGIN), sent, st)
            a[MARGIN:-MARGIN, MARGIN:-MARGIN] = rng.integers(0, 1 << depth, (self.H[p], self.W[p]))
            self.planes.append(a)
        sb_cols = (self.cols + 7) >> 3
        starts = sorted({(sb_cols * t // tiles) * 8 for t in range(tiles)})
        blocks, ops = [], []
        self._coef_n = 0

        def tile_start(col):
            return max(s for s in starts if s <= col)

        def block(row, col, bl, bp):
            bs = bl * 3 + bp
            intra = kind == "intra" or rng.random() < p_intra
            if bs > 9:
                tx = 0
            else:
                mx = min(int(np.log2(min(BWH4[bs]))), 3)
                tx = 0 if sizes == "4x4" else int(rng.integers(0, mx + 1))
            if lossless:
                tx = 0
            w8, h8 = BWH8[bs]
            uvtx = tx - int((self.ss_h and w8 * 2 == 1 << tx) or (self.ss_v and h8 * 2 == 1 << tx))
            m = [int(v) for v in rng.integers(0, 10, 4)]
            if bs == 10:
                m[1], m[3] = m[0], m[2]
            elif bs == 11:
                m[2], m[3] = m[0], m[1]
            elif bs < 10:
                m = [m[0]] * 4
            rec = [row, col, bs, tx, uvtx, int(rng.random() < p_skip), *m, int(rng.integers(0, 10)), tile_start(col), int(intra), 0, 0, 0]
            eob = np.zeros(768, np.uint8)
            if intra:
                self._ops(rng, rec, eob, ops)
            blocks.append(rec)
            self.eob_rows.append(eob)

        def sb(row, col, bl):
            hbs = 4 >> bl
            if bl == 3:
                block(row, col, bl, 3 if sizes == "4x4" else int(rng.integers(0, 4)))
                return
            if col + hbs < self.cols and row + hbs < self.rows:
                bp = 3 if sizes == "4x4" else int(rng.choice(4, p=(0.15, 0.15, 0.15, 0.55)))
            elif col + hbs < self.cols:
                bp = 3 if sizes == "4x4" else int(rng.choice([1, 3]))
            elif row + hbs < self.rows:
                bp = 3 if sizes == "4x4" else int(rng.choice([2, 3]))
            else:
                bp = 3
            inside_r, inside_c = row + hbs < self.rows, col + hbs < self.cols
            if bp == 0:
                block(row, col, bl, 0)
            elif bp == 1:
                block(row, col, bl, 1)
                if inside_r:
                    block(row + hbs, col, bl, 1)
            elif bp == 2:
                block(row, col, bl, 2)
                if inside_c:
                    block(row, col + hbs, bl, 2)
            else:
                sb(row, col, bl + 1)
                if inside_c:
                    sb(row, col + hbs, bl + 1)
                if inside_r:
                    sb(row + hbs, col, bl + 1)
                    if inside_c:
                        sb(row + hbs, col + hbs, bl + 1)

        self.eob_rows = []
        for r in range(0, self.rows, 8):
            for c in range(0, self.cols, 8):
                sb(r, c, 0)
        self.blocks = np.array(blocks, np.int32).reshape(-1, 16)
        self.eobs = np.concatenate(self.eob_rows) if self.eob_rows else np.zeros(768, np.uint8)
        del self.eob_rows
        self.ops = np.zeros(len(ops), INTRA_DTYPE)
        if ops:
            o = np.array(ops, np.int64)
            for k, name in enumerate(("coef_off", "x", "y", "eob", "plane", "tx", "mode", "flags")):
                self.ops[name] = o[:, k]
        self.coef = self._coefs(rng)

    def _ops(self, rng, rec, eob, ops):
        """intra_recon's loops (vp9recon.c:225-286) for one block: ops in its order, eob[] and coefficient offsets as the decoder has them"""
        row, col, bs, tx, uvtx, skip = rec[:6]
        w4, h4 = BWH8[bs][0] << 1, BWH8[bs][1] << 1
        end_x, end_y = min(2 * (self.cols - col), w4), min(2 * (self.rows - row), h4)
        lossless = INTRA_LOSSLESS if self.lossless else 0
        tcs = rec[11]

        def one(p, bx, by, x, y, t, mode, n, w, base, ebase):
            N = 4 << t
            e = 0
            if not skip:
                e = int(rng.choice([0, 1, 1, int(rng.integers(1, N * N + 1))]))
            if t > 1:
                eob[ebase + n:ebase + n + 2] = np.array([e], "<u2").view(np.uint8)
            else:
                eob[ebase + n] = e
            flags = lossless | (INTRA_HAVE_LEFT if (col > tcs or x > 0) else 0) | (INTRA_HAVE_RIGHT if x < w - 1 else 0)
            ops.append((base + 16 * n, bx + 4 * x, by + 4 * y, e, p, t, mode, flags))

        base = self._coef_n
        rec[13] = base
        step1d, step, n = 1 << tx, 1 << (2 * tx), 0
        for y in range(0, end_y, step1d):
            for x in range(0, end_x, step1d):
                mode = rec[6 + (y * 2 + x if bs > 9 and tx == 0 else 0)]
                one(0, col * 8, row * 8, x, y, tx, mode, n, w4, base, 0)
                n += step
        self._coef_n += 16 * max(n, 1)
        w4, end_x, end_y = w4 >> self.ss_h, end_x >> self.ss_h, end_y >> self.ss_v
        step1d, step = 1 << uvtx, 1 << (2 * uvtx)
        for p in range(2):
            base = self._coef_n
            rec[14 + p] = base
            n = 0
            for y in range(0, end_y, step1d):
                for x in range(0, end_x, step1d):
                    one(1 + p, col * (8 >> self.ss_h), row * (8 >> self.ss_v), x, y, uvtx, rec[10], n, w4, base, 256 * (1 + p))
                    n += step
            self._coef_n += 16 * max(n, 1)

    def _coefs(self, rng):
        """decoder-shaped coefficients for every op with an eob: a decaying low-frequency corner (Walsh-Hadamard-sized in lossless frames)"""
        coef = np.zeros(self._coef_n + 16, cdtype(self.depth))
        amp = 1 << (self.depth + 3)
        for t in range(4):
            sel = np.nonzero((self.ops["tx"] == t) & (self.ops["eob"] > 0))[0]
            if not len(sel):
                continue
            n = 4 << t
            decay = 1 + np.add.outer(np.arange(n), np.arange(n))
            vals = rng.integers(-amp, amp + 1, (len(sel), n, n)) // decay
            k = rng.integers(1, n + 1, len(sel))
            vals = np.where((np.arange(n)[None, :, None] < k[:, None, None]) & (np.arange(n)[None, None, :] < k[:, None, None]), vals, 0)
            if self.lossless:
                vals = vals >> 2 << 2
            idx = self.ops["coef_off"][sel][:, None] + np.arange(n * n)[None, :]
            coef[idx] = vals.reshape(len(sel), -1)
        return coef

    def strides(self):
        return self.planes[0].strides[0], self.planes[1].strides[0]

    def ptrs(self, arrs):
        return [a.ctypes.data + MARGIN * a.strides[0] + MARGIN * a.itemsize for a in arrs]

    def area(self, arrs):
        return [a[MARGIN:a.shape[0] - MARGIN, MARGIN:a.shape[1] - MARGIN] for a in arrs]


def orc_frame(f, order=0):
    """the checker on copies of the planes (sentinels included)"""
    L = cl.oracle()
    L.orc_vp9_intra_frame.restype = C.c_int64
    L.orc_vp9_intra_frame.argtypes = [C.c_int] * 5 + [C.c_void_p, C.c_ssize_t, C.c_ssize_t, C.c_int64, C.c_void_p, C.c_void_p, C.c_int]
    out = [p.copy() for p in f.planes]
    arr = (C.c_void_p * 3)(*f.ptrs(out))
    ls_y, ls_uv = f.strides()
    ops = np.ascontiguousarray(f.ops)
    assert L.orc_vp9_intra_frame(f.depth, f.ss_h, f.ss_v, f.width, f.height, arr, ls_y, ls_uv, len(ops), ops.ctypes.data, f.coef.ctypes.data,
                                 order) >= 0
    return out


def ref_frame(f, tight=False):
    """the reference's intra_recon block by block on the planes' areas: with tight line sizes (8-aligned width, the emu path whenever
    a block passes it) or with the margin arrays' line sizes; returns the three areas"""
    if tight:
        arrs = [np.ascontiguousarray(a) for a in f.area([p.copy() for p in f.planes])]
        ptrs = [a.ctypes.data for a in arrs]
    else:
        big = []
        for a in f.planes:                                   # room on the right for the blocks that pass the area without emu
            b = np.zeros((a.shape[0], a.shape[1] + 64), a.dtype)
            b[:, :a.shape[1]] = a
            big.append(b)
        arrs = big
        ptrs = f.ptrs(big)
    ls_y, ls_uv = arrs[0].strides[0], arrs[1].strides[0]
    arr = (C.c_void_p * 3)(*ptrs)
    coef, eobs, blocks = f.coef.copy(), f.eobs.copy(), np.ascontiguousarray(f.blocks)
    assert ref().ffref_vp9_intra_frame(f.depth, f.ss_h, f.ss_v, f.width, f.height, arr, ls_y, ls_uv, int(f.lossless), len(blocks),
                                       blocks.ctypes.data, coef.ctypes.data, eobs.ctypes.data) == 0
    if tight:
        return arrs
    return [b[MARGIN:MARGIN + f.H[p], MARGIN:MARGIN + f.W[p]] for p, b in enumerate(big)]


# ---------------------------------------------------------------- fixtures
FIXTURES = {
    "420-8-intra": (1, 8, "420", 200, 136, {}),
    "420-10-mixed-inter": (2, 10, "420", 250, 130, {"kind": "inter", "p_intra": 0.4}),
    "422-12-tiles": (3, 12, "422", 300, 100, {"tiles": 2}),
    "440-8-lossless": (4, 8, "440", 131, 77, {"lossless": True}),
    "444-10-4x4": (5, 10, "444", 96, 72, {"sizes": "4x4"}),
    "420-12-odd-skip": (6, 12, "420", 137, 59, {"p_skip": 0.6}),
    "444-8-inter-tiles": (7, 8, "444", 270, 140, {"kind": "inter", "p_intra": 0.3, "tiles": 3}),
    "422-10-4x4-odd": (8, 10, "422", 75, 41, {"sizes": "4x4"}),
}
FIXTURE_NAMES = tuple(FIXTURES)


def frame_case(name):
    seed, depth, fmt, w, h, kw = FIXTURES[name]
    return Frame(700 + seed, depth, fmt, w, h, **kw)


def digest(arrs):
    h = hashlib.sha256()
    for a in arrs:
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


def fixture_hashes():
    out = {}
    for line in open(FIXTURE):
        name, h = line.split()
        out[name] = h
    return out


# ---------------------------------------------------------------- single members (intra_pred[tx][mode])
def member_calls(seed, depth, per=3, edges="random"):
    """(tx, mode, left [n], top [-1 .. 2n - 1] as an array of 2n + 1, dst0 [n, n]) for all 60 members; edges "random", "low" (0 and
    near it) or "high" (the depth's maximum and near it)"""
    rng = np.random.default_rng(seed)
    mx = (1 << depth) - 1
    for tx in range(4):
        n = 4 << tx
        for mode in range(15):
            for _ in range(per):
                if edges == "random":
                    e = rng.integers(0, mx + 1, 3 * n + 1)
                elif edges == "low":
                    e = rng.integers(0, 3, 3 * n + 1)
                else:
                    e = mx - rng.integers(0, 3, 3 * n + 1)
                st = sdtype(depth)
                yield tx, mode, e[:n].astype(st), e[n:].astype(st), rng.integers(0, mx + 1, (n, n)).astype(st)


def run_member(fn, depth, call):
    """one member call (fn(dst, stride, left, top) with host pointers) on copies; returns dst"""
    tx, mode, left, top, dst0 = call
    d, lb, tb = dst0.copy(), np.ascontiguousarray(left), np.ascontiguousarray(top)
    fn(d.ctypes.data, d.strides[0], lb.ctypes.data, tb.ctypes.data + tb.itemsize)
    return d


def orc_member(depth, tx, mode):
    L = cl.oracle()
    L.orc_vp9_intra_pred.argtypes = [C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_ssize_t, C.c_void_p, C.c_void_p]
    return lambda d, s, lp, tp: L.orc_vp9_intra_pred(depth, tx, mode, d, s, lp, tp)


def ref_member(depth, tx, mode):
    return lambda d, s, lp, tp: ref().ffref_vp9_intra_pred(depth, tx, mode, d, s, lp, tp)
