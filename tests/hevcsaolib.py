"""Test infrastructure for HEVC sample adaptive offset (the SAO members of HEVCDSPContext and b200_hevc_sao_plane_device): seeded
picture descriptions (slice and tile maps, loop_filter_across_slices / _tiles, PCM / bypass maps, per-CTB SAO syntax), the
B200HevcSaoCtb grids derived from them by the recipe INTEGRATION.md documents, runners of the checker (oracle/liboracle.so:
orc_hevc_sao_*) and of the compiled reference (oracle/_ref/libffref_hevcsao.so, built by oracle/ref/hevcsao.mk: the members, and
whole pictures through the decoder's own hevc/filter.c), and RefCheck, which keeps the reference's results as digests in
tests/golden/hevcsao_ref_digests.json for machines without the reference."""
import ctypes as C
import hashlib
import json
import os

import numpy as np

import cpulibs as cl
from ffmpeg_b200._lib import SAOParams
from ffmpeg_b200.hevcdsp import (SAO_DTYPE, SAO_NONE, SAO_BAND, SAO_EDGE, SAO_RESTORE, SAO_VERT_L, SAO_VERT_R, SAO_HORIZ_T, SAO_HORIZ_B,
                                 SAO_DIAG_TL, SAO_DIAG_TR, SAO_DIAG_BR, SAO_DIAG_BL)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_SO = os.path.join(ROOT, "oracle", "_ref", "libffref_hevcsao.so")
REF_DIGESTS = os.path.join(ROOT, "tests", "golden", "hevcsao_ref_digests.json")
FIXTURE = os.path.join(ROOT, "tests", "golden", "hevcsao_hashes.txt")
DEPTHS = (8, 9, 10, 12)
OUTCOMES = ("band", "edge_h", "edge_v", "edge_135", "edge_45", "border", "vert_l", "vert_r", "horiz_t", "horiz_b", "diag_tl", "diag_tr",
            "diag_br", "diag_bl", "save_ul", "save_ur", "save_lr", "save_ll", "keep", "keep_quirk", "clip_0", "clip_max")   # cnt[0..21]
SHIFTS = {0: (0, 0), 1: (1, 1), 2: (1, 0), 3: (0, 0)}  # chroma_format_idc -> chroma (hshift, vshift)
MARGIN = 4         # samples of sentinel around a plane
SENT8, SENT16 = 0xA5, 0xA5A5
EDGE_STRIDE = 192  # the edge member's implicit source stride in bytes

_ref = None


def have_ref():
    return os.path.exists(REF_SO)


def ref():
    global _ref
    if _ref is None:
        _ref = C.CDLL(REF_SO)
        _ref.ffref_hevc_sao_restore_fn.restype = C.c_void_p
    return _ref


def orc():
    L = cl.oracle()
    if not getattr(L, "_sao_types", False):
        vp = C.c_void_p
        L.orc_hevc_sao_band.argtypes = [C.c_int, vp, vp, C.c_ssize_t, C.c_ssize_t, vp, C.c_int, C.c_int, C.c_int, vp]
        L.orc_hevc_sao_edge.argtypes = [C.c_int, vp, vp, C.c_ssize_t, vp, C.c_int, C.c_int, C.c_int, vp]
        L.orc_hevc_sao_restore.argtypes = [C.c_int, C.c_int, vp, vp, C.c_ssize_t, C.c_ssize_t, vp, vp, C.c_int, C.c_int, C.c_int, vp, vp, vp, vp]
        L.orc_hevc_sao_restore_sweep.argtypes = [C.c_int, C.c_int, vp, C.c_int, C.c_int, C.c_uint32]
        L.orc_hevc_sao_restore_sweep.restype = C.c_uint64
        L.orc_hevc_sao_plane.argtypes = [C.c_int, vp, C.c_ssize_t, vp, C.c_ssize_t, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, vp, C.c_int64,
                                         vp, C.c_int64, C.c_int, C.c_int, vp]
        L._sao_types = True
    return L


_digests = None
_blocks = {}


def _write_digests():
    with open(REF_DIGESTS, "w") as f:
        json.dump(_digests, f, indent=0, sort_keys=True)
        f.write("\n")


class RefCheck:
    """with RefCheck() as rc: assert rc.same(ours, lambda: theirs) -- hevcdbklib.RefCheck's scheme with this path's own digest file:
    live comparison (and a check of the stored digest) where libffref_hevcsao.so is built, the stored digest of `ours` elsewhere;
    FFDSP_RECORD_REF=1 with the reference built rewrites the digests at exit."""

    def __enter__(self):
        global _digests
        nodeid = os.environ.get("PYTEST_CURRENT_TEST", "?").rsplit(" (", 1)[0]
        path, _, name = nodeid.partition("::")
        test = f"{os.path.basename(path)}::{name}"
        k = _blocks[test] = _blocks.get(test, -1) + 1
        self.key, self.h = f"{test}#{k}", hashlib.sha256()
        self.live, self.record = have_ref(), have_ref() and os.environ.get("FFDSP_RECORD_REF") == "1"
        if _digests is None:
            _digests = json.load(open(REF_DIGESTS)) if os.path.exists(REF_DIGESTS) else {}
            if self.record:
                import atexit
                atexit.register(_write_digests)
        assert self.live or self.key in _digests, f"no stored reference result for {self.key} ({REF_DIGESTS})"
        return self

    def _add(self, v):
        for x in (v if isinstance(v, (list, tuple)) else [v]):
            x = np.asarray(x)
            self.h.update(f"{x.dtype.str}{x.shape}".encode())
            self.h.update(np.ascontiguousarray(x).tobytes())

    def same(self, ours, ref_fn):
        if not self.live:
            self._add(ours)
            return True
        theirs = ref_fn()
        self._add(theirs)
        if isinstance(ours, (list, tuple)):
            return len(ours) == len(theirs) and all(np.array_equal(a, b) for a, b in zip(ours, theirs))
        return bool(np.array_equal(ours, theirs))

    def __exit__(self, typ, *_):
        if typ is not None:
            return False
        if self.record:
            _digests[self.key] = self.h.hexdigest()[:32]
        else:
            assert self.key in _digests, f"no stored reference result for {self.key} ({REF_DIGESTS})"
            assert self.h.hexdigest()[:32] == _digests[self.key], f"differs from the stored reference results ({self.key})"
        return False


def sdtype(depth):
    return np.uint8 if depth == 8 else np.uint16


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def sentinel(depth):
    return SENT8 if depth == 8 else SENT16


def content(rng, depth, h, w):
    """blocky content: flat, ramp and textured 8x8 blocks, some at 0 or the maximum, so that every edge category and both clips occur"""
    maxv = (1 << depth) - 1
    s = 1 << (depth - 8)
    out = np.zeros((h, w), np.int64)
    for by in range(0, h, 8):
        for bx in range(0, w, 8):
            hh, ww = min(8, h - by), min(8, w - bx)
            kind = rng.integers(0, 5)
            base = int(rng.integers(0, maxv + 1))
            if kind == 0:
                v = np.full((hh, ww), base)
            elif kind == 1:
                v = base + rng.integers(-3, 4) * s * np.arange(hh)[:, None] + rng.integers(-3, 4) * s * np.arange(ww)[None, :]
            elif kind == 2:
                v = base + rng.integers(-3 * s, 3 * s + 1, (hh, ww))
            elif kind == 3:
                v = rng.choice(np.array([0, 1, maxv - 1, maxv]), (hh, ww))
            else:
                v = rng.integers(0, maxv + 1, (hh, ww))
            out[by:by + hh, bx:bx + ww] = v
    return np.clip(out, 0, maxv).astype(sdtype(depth))


# ---------------------------------------------------------------- picture descriptions
class Picture:
    """A picture as the decoder sees it at the loop filter: luma W x H, chroma_format_idc, the CTB grid, tiles (col_bd / row_bd in CTBs)
    and the tile scan, slices (contiguous in tile scan; slice_addr per CTB, lf_across per CTB), the PCM / bypass map (is_pcm per luma
    min PU, used when `pcm`), per-CTB SAOParams as hls_sao_param leaves them, and the deblocked planes."""


def picture_case(seed, depth, W, H, log2_ctb, cfmt, nslices=3, lf_slices=None, tiles=(1, 1), lf_tiles=True, pcm=True, log2_pu=2,
                 sao_mix=(0.2, 0.3, 0.5), scatter=0.0):
    """scatter: the fraction of CTBs whose slice address is replaced by another slice's.  Contiguous slices never give a CTB the
    same slice as its upper-left (lower-right) neighbour but not its left or upper (right or lower) one, which is what makes
    sao_edge_restore_1's save_upper_left (save_lower_right) matter; sao_filter_CTB computes its flags from any map."""
    rng = np.random.default_rng(seed)
    p = Picture()
    p.depth, p.W, p.H, p.log2_ctb, p.cfmt, p.log2_pu = depth, W, H, log2_ctb, cfmt, log2_pu
    ctb = 1 << log2_ctb
    cw, ch = -(-W // ctb), -(-H // ctb)
    p.cw, p.ch, n = cw, ch, cw * ch
    ncols, nrows = tiles
    p.col_bd = [cw * k // ncols for k in range(ncols + 1)]
    p.row_bd = [ch * k // nrows for k in range(nrows + 1)]
    p.tiles_enabled, p.lf_tiles = ncols > 1 or nrows > 1, bool(lf_tiles)
    ts_to_rs, tile_of_ts = [], []
    for tr in range(nrows):
        for tc in range(ncols):
            for y in range(p.row_bd[tr], p.row_bd[tr + 1]):
                for x in range(p.col_bd[tc], p.col_bd[tc + 1]):
                    ts_to_rs.append(y * cw + x)
                    tile_of_ts.append(tr * ncols + tc)
    p.ts_to_rs = np.array(ts_to_rs)
    p.rs_to_ts = np.argsort(p.ts_to_rs)
    p.tile_id = np.array(tile_of_ts)                    # by ts
    starts = sorted(set([0] + [int(v) for v in rng.choice(np.arange(1, n), min(nslices - 1, n - 1), replace=False)])) if n > 1 else [0]
    p.slice_addr = np.zeros(n, np.int32)
    p.lf_across = np.zeros(n, np.uint8)
    for k, s0 in enumerate(starts):
        s1 = starts[k + 1] if k + 1 < len(starts) else n
        lf = bool(rng.integers(0, 2)) if lf_slices is None else bool(lf_slices[k % len(lf_slices)])
        for ts in range(s0, s1):
            p.slice_addr[ts_to_rs[ts]] = ts_to_rs[s0]
            p.lf_across[ts_to_rs[ts]] = lf
    if scatter:
        addrs = np.unique(p.slice_addr)
        sel = rng.random(n) < scatter
        p.slice_addr[sel] = rng.choice(addrs, int(sel.sum()))
    p.pcm = bool(pcm)
    npw, nph = W >> log2_pu, H >> log2_pu
    p.is_pcm = (rng.random((nph, npw)) < 0.12).astype(np.uint8) if pcm else np.zeros((nph, npw), np.uint8)
    # SAO syntax per CTB and component (hevcdec.c:1232-1285): Cr shares Cb's type and class
    p.sao = (SAOParams * n)()
    ncomp = 3 if cfmt else 1
    scale = int(rng.integers(0, depth - 9)) if depth > 10 else 0        # log2_sao_offset_scale (range extensions)
    amax = (1 << (min(depth, 10) - 5)) - 1
    for rs in range(n):
        s = p.sao[rs]
        for c in range(ncomp):
            if c == 2:
                s.type_idx[2], s.eo_class[2] = s.type_idx[1], s.eo_class[1]
            else:
                s.type_idx[c] = int(rng.choice(3, p=list(sao_mix)))
                s.eo_class[c] = int(rng.integers(0, 4))
            if s.type_idx[c] == SAO_NONE:
                continue
            for i in range(4):
                s.offset_abs[c][i] = int(rng.integers(0, amax + 1)) if rng.random() < 0.8 else amax
                s.offset_sign[c][i] = int(rng.integers(0, 2)) if s.type_idx[c] == SAO_BAND and s.offset_abs[c][i] else 0
            s.band_position[c] = int(rng.integers(0, 32))
            s.offset_val[c][0] = 0
            for i in range(4):
                v = s.offset_abs[c][i]
                if (s.type_idx[c] == SAO_EDGE and i > 1) or (s.type_idx[c] == SAO_BAND and s.offset_sign[c][i]):
                    v = -v
                s.offset_val[c][i + 1] = v * (1 << scale)
    p.planes = []
    for c in range(ncomp):
        hs, vs = SHIFTS[cfmt] if c else (0, 0)
        p.planes.append(content(rng, depth, H >> vs, W >> hs))
    return p


def ctb_flags(p, x, y):
    """B200HevcSaoCtb.flags of CTB (x, y): sao_filter_CTB's restore / vert_edge / horiz_edge / diag_edge (hevc/filter.c:283-329)"""
    cw = p.cw
    rs = y * cw + x
    ts = p.rs_to_ts[rs]
    lfase = bool(p.lf_across[rs])
    no_tile = p.tiles_enabled and not p.lf_tiles
    if not (no_tile or not lfase):
        return 0
    e = (x == 0, y == 0, x == cw - 1, y == p.ch - 1)

    def tile_edge(nrs):
        return no_tile and p.tile_id[ts] != p.tile_id[p.rs_to_ts[nrs]]

    def slice_edge(nx, ny):
        return (not lfase) and p.slice_addr[rs] != p.slice_addr[ny * cw + nx]
    f = SAO_RESTORE
    lt = rt = ut = bt = False
    if not e[0]:
        lt = tile_edge(rs - 1)
        f |= SAO_VERT_L if slice_edge(x - 1, y) or lt else 0
    if not e[2]:
        rt = tile_edge(rs + 1)
        f |= SAO_VERT_R if slice_edge(x + 1, y) or rt else 0
    if not e[1]:
        ut = tile_edge(rs - cw)
        f |= SAO_HORIZ_T if slice_edge(x, y - 1) or ut else 0
    if not e[3]:
        bt = tile_edge(rs + cw)
        f |= SAO_HORIZ_B if slice_edge(x, y + 1) or bt else 0
    if not e[0] and not e[1]:
        f |= SAO_DIAG_TL if slice_edge(x - 1, y - 1) or lt or ut else 0
    if not e[1] and not e[2]:
        f |= SAO_DIAG_TR if slice_edge(x + 1, y - 1) or rt or ut else 0
    if not e[2] and not e[3]:
        f |= SAO_DIAG_BR if slice_edge(x + 1, y + 1) or rt or bt else 0
    if not e[0] and not e[3]:
        f |= SAO_DIAG_BL if slice_edge(x - 1, y + 1) or lt or bt else 0
    return f


def records(p, c, pad=2, garbage_seed=None):
    """the component's B200HevcSaoCtb grid (INTEGRATION.md's recipe), `pad` records of padding per row (garbage when a seed is given,
    with garbage in `reserved` and in unknown flag bits too)"""
    g = np.zeros((p.ch, p.cw + pad), SAO_DTYPE)
    for y in range(p.ch):
        for x in range(p.cw):
            s = p.sao[y * p.cw + x]
            t = s.type_idx[c]
            g[y, x]["offset_val"] = list(s.offset_val[c])
            g[y, x]["type"] = t
            g[y, x]["cls"] = s.band_position[c] if t == SAO_BAND else s.eo_class[c] if t == SAO_EDGE else 0
            g[y, x]["flags"] = ctb_flags(p, x, y)
    if garbage_seed is not None:
        rg = np.random.default_rng(garbage_seed)
        g["reserved"] = rg.integers(0, 1 << 16, g.shape)
        g["flags"] |= (rg.integers(0, 1 << 7, g.shape) << 9).astype(np.uint16)
        if pad:
            g[:, p.cw:] = np.frombuffer(rg.integers(0, 256, g[:, p.cw:].size * 16, dtype=np.uint8).tobytes(), SAO_DTYPE).reshape(g[:, p.cw:].shape)
    return g


def comp_geometry(p, c):
    """(width, height, hshift, vshift) of component c"""
    hs, vs = SHIFTS[p.cfmt] if c else (0, 0)
    return p.W >> hs, p.H >> vs, hs, vs


def keep_map(p, pad=3):
    """is_pcm with `pad` columns of padding, or None when the decoder's condition is false"""
    if not p.pcm:
        return None
    k = np.zeros((p.is_pcm.shape[0], p.is_pcm.shape[1] + pad), np.uint8)
    k[:, :p.is_pcm.shape[1]] = p.is_pcm
    return k


def framed(plane, depth, margin=MARGIN):
    buf = np.full((plane.shape[0] + 2 * margin, plane.shape[1] + 2 * margin), sentinel(depth), plane.dtype)
    buf[margin:margin + plane.shape[0], margin:margin + plane.shape[1]] = plane
    return buf


def _ptr(buf, margin=MARGIN):
    return buf.ctypes.data + margin * buf.strides[0] + margin * buf.itemsize


def orc_plane(p, c, reverse=False, cnt=None, rec=None, keep="auto"):
    """the checker's SAO of component c: the whole sentinel-framed dst buffer"""
    W, H, hs, vs = comp_geometry(p, c)
    g = records(p, c) if rec is None else rec
    k = keep_map(p) if keep == "auto" else keep
    src = framed(p.planes[c], p.depth)
    dst = np.full_like(src, sentinel(p.depth))
    assert orc().orc_hevc_sao_plane(p.depth, _ptr(dst), dst.strides[0], _ptr(src), src.strides[0], W, H, p.log2_ctb, hs, vs, g.ctypes.data,
                                    g.shape[1], None if k is None else k.ctypes.data, 0 if k is None else k.shape[1], p.log2_pu,
                                    int(reverse), None if cnt is None else cnt.ctypes.data) == 0
    return dst


def ref_picture(p):
    """the decoder's loop filter over the whole picture: every component plane after SAO"""
    planes = [np.ascontiguousarray(x.copy()) for x in p.planes]
    ptrs = (C.c_void_p * 3)(*[x.ctypes.data for x in planes] + [None] * (3 - len(planes)))
    ls = (C.c_int * 3)(*[x.strides[0] for x in planes] + [0] * (3 - len(planes)))
    col = (C.c_int * len(p.col_bd))(*p.col_bd)
    row = (C.c_int * len(p.row_bd))(*p.row_bd)
    f = ref().ffref_hevc_sao_picture
    sa = np.ascontiguousarray(p.slice_addr, np.int32)
    lf = np.ascontiguousarray(p.lf_across, np.uint8)
    pcm = np.ascontiguousarray(p.is_pcm, np.uint8)
    assert f(p.depth, p.cfmt, p.W, p.H, p.log2_ctb, ptrs, ls, C.byref(p.sao), C.c_void_p(sa.ctypes.data), C.c_void_p(lf.ctypes.data),
             len(p.col_bd) - 1, col, len(p.row_bd) - 1, row, int(p.lf_tiles), C.c_void_p(pcm.ctypes.data), p.log2_pu, int(p.pcm)) == 0
    return planes


def inner(buf, H, W, margin=MARGIN):
    return buf[margin:margin + H, margin:margin + W]


def outcome_counts(p, comps=None):
    cnt = np.zeros(len(OUTCOMES), np.int64)
    for c in (range(len(p.planes)) if comps is None else comps):
        orc_plane(p, c, cnt=cnt)
    return dict(zip(OUTCOMES, cnt.tolist()))


# ---------------------------------------------------------------- single members
def band_cases(seed, depth):
    """yields (off[5], left_class, w, h, src): every left_class 0..31 and negative / large ones, int16 offsets up to the extremes,
    samples at 0 and the maximum among random ones"""
    rng = np.random.default_rng(seed)
    maxv = (1 << depth) - 1
    classes = list(range(32)) + [-1, -5, -32, -33, 32, 37, 1000, 2 ** 31 - 1, -2 ** 31]
    for k, lc in enumerate(classes):
        w, h = int(rng.integers(1, 65)), int(rng.integers(1, 65))
        if k % 4 == 0:
            off = rng.choice(np.array([-32768, 32767, -124, 124, 0]), 5)
        else:
            off = rng.integers(-(1 << (depth - 3)), 1 << (depth - 3), 5)
        src = rng.integers(0, maxv + 1, (h, w))
        src[rng.random((h, w)) < 0.2] = 0
        src[rng.random((h, w)) < 0.2] = maxv
        yield np.array(off, np.int16), lc, w, h, src.astype(sdtype(depth))


def edge_cases(seed, depth):
    """yields (off[5], eo, w, h, src (h + 2) x 96 samples at the 192-byte stride with the block at (1, 1)): every class at every width
    1..64 and every height 1..64"""
    rng = np.random.default_rng(seed)
    maxv = (1 << depth) - 1
    per = EDGE_STRIDE // np.dtype(sdtype(depth)).itemsize
    for k in range(64):
        for eo in range(4):
            w, h = (k + 1, int(rng.integers(1, 65))) if eo % 2 == 0 else (int(rng.integers(1, 65)), k + 1)
            off = rng.integers(-(1 << (depth - 4)), 1 << (depth - 4), 5) if k % 3 else rng.choice(np.array([-32768, 32767, 0, 124]), 5)
            src = rng.integers(0, maxv + 1, (h + 2, per))
            flat = rng.random((h + 2, per)) < 0.4               # equal neighbours
            src[flat] = maxv // 2
            src[rng.random((h + 2, per)) < 0.1] = maxv
            yield np.array(off, np.int16), eo, w, h, src.astype(sdtype(depth))


def orc_band(depth, case, dst=None, in_place=False):
    off, lc, w, h, src = case
    s = framed(src, depth)
    d = s if in_place else (framed(np.zeros_like(src), depth) if dst is None else dst.copy())
    orc().orc_hevc_sao_band(depth, _ptr(d), _ptr(s), d.strides[0], s.strides[0], off.ctypes.data, lc, w, h, None)
    return d


def ref_band(depth, case, in_place=False, idx=0):
    off, lc, w, h, src = case
    s = framed(src, depth)
    d = s if in_place else framed(np.zeros_like(src), depth)
    assert ref().ffref_hevc_sao_band(depth, idx, C.c_void_p(_ptr(d)), C.c_void_p(_ptr(s)), C.c_ssize_t(d.strides[0]), C.c_ssize_t(s.strides[0]),
                                     C.c_void_p(off.ctypes.data), lc, w, h) == 0
    return d


def ctx_band(ctx, depth, case, in_place=False, idx=0):
    from ffmpeg_b200 import hevcdsp as hd
    off, lc, w, h, src = case
    s = framed(src, depth)
    d = s if in_place else framed(np.zeros_like(src), depth)
    hd.SAO_BAND_FILTER(ctx.sao_band_filter[idx])(_ptr(d), _ptr(s), d.strides[0], s.strides[0], off.ctypes.data, lc, w, h)
    return d


def _edge_dst(depth, w, h):
    return np.full((h + 2 * MARGIN, w + 2 * MARGIN), sentinel(depth), sdtype(depth))


def _edge_src_ptr(src):
    return src.ctypes.data + EDGE_STRIDE + src.itemsize


def orc_edge(depth, case):
    off, eo, w, h, src = case
    d = _edge_dst(depth, w, h)
    orc().orc_hevc_sao_edge(depth, _ptr(d), _edge_src_ptr(src), d.strides[0], off.ctypes.data, eo, w, h, None)
    return d


def ref_edge(depth, case, idx=0):
    off, eo, w, h, src = case
    d = _edge_dst(depth, w, h)
    assert ref().ffref_hevc_sao_edge(depth, idx, C.c_void_p(_ptr(d)), C.c_void_p(_edge_src_ptr(src)), C.c_ssize_t(d.strides[0]),
                                     C.c_void_p(off.ctypes.data), eo, w, h) == 0
    return d


def ctx_edge(ctx, depth, case, idx=0):
    from ffmpeg_b200 import hevcdsp as hd
    off, eo, w, h, src = case
    d = _edge_dst(depth, w, h)
    hd.SAO_EDGE_FILTER(ctx.sao_edge_filter[idx])(_ptr(d), _edge_src_ptr(src), d.strides[0], off.ctypes.data, eo, w, h)
    return d


RESTORE_SIZES = ((2, 2), (5, 3), (16, 9), (64, 64))


def sweep(depth, which, fn=None, w=8, h=8, seed=1):
    """orc_hevc_sao_restore_sweep: every eo_class x borders x (for [1]) edge flags x c_idx through fn (a member address) or the checker"""
    return int(orc().orc_hevc_sao_restore_sweep(depth, which, fn, w, h, seed))


# ---------------------------------------------------------------- fixture
FIXTURE_SEEDS = {8: 4008, 9: 4009, 10: 4070, 12: 4032}   # seeds whose pictures reach every outcome


def fixture_case(depth):
    """the picture behind tests/golden/hevcsao_hashes.txt at each depth: 4:2:0, luma 328x200 (not a multiple of the 32-sample CTB), 2 x 2
    tiles not filtered across, nine slices alternating loop_filter_across_slices with 30 % of the CTBs' slice addresses scattered,
    a PCM / bypass map, mostly edge CTBs"""
    return picture_case(FIXTURE_SEEDS[depth], depth, 328, 200, 5, 1, nslices=9, lf_slices=(0, 1), tiles=(2, 2), lf_tiles=False, pcm=True,
                        sao_mix=(0.15, 0.25, 0.6), scatter=0.3)


def fixture_hashes():
    out = {}
    for line in open(FIXTURE):
        d, what, h = line.split()
        out[(int(d), what)] = h
    return out


def fixture_plane_hashes(depth):
    """{"luma": hash, "chroma420": hash} of the checker's Y and Cb planes (sentinel frame included)"""
    p = fixture_case(depth)
    return {"luma": digest(orc_plane(p, 0)), "chroma420": digest(orc_plane(p, 1))}
