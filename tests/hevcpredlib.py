"""Test infrastructure for HEVC intra prediction (HEVCPredContext and b200_hevc_intra_pred_batch_device): seeded pictures (CTBs of
16 / 32 / 64 split into transform quadtrees, slices and tiles, picture sizes that are not CTB multiples, luma and 4:2:0 / 4:2:2 / 4:4:4
chroma, constrained intra prediction with mixed intra / inter maps, smoothing and strong smoothing on and off), the decoder's call
sequence restated (ff_hevc_set_neighbour_available for the na bits, intra_pred's z-scan checks for the op flags, the chroma TU
placement of hls_transform_unit), the dependency-level scheduler INTEGRATION.md describes (the bench imports it too), runners of the
compiled reference (oracle/_ref/libffref_hevcpred.so, built by oracle/ref/hevcpred.mk: the members, and whole planes through the
reference's own intra_pred), runners of the checker (oracle/liboracle.so: orc_hevc_pred_* / orc_hevc_filter_* / orc_hevc_intra_plane),
seeded pictures whose 32x32 luma blocks put the strong-smoothing second differences on both sides of the threshold, and RefCheck, which keeps the reference's results as digests in tests/golden/hevcpred_ref_digests.json
for machines without the reference."""
import ctypes as C
import hashlib
import json
import os

import numpy as np

from ffmpeg_b200.hevcdsp import (INTRA_DTYPE, INTRA_CAND_BL, INTRA_CAND_L, INTRA_CAND_UL, INTRA_CAND_U, INTRA_CAND_UR, INTRA_LUMA,
                                 INTRA_SMOOTH, INTRA_STRONG)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_SO = os.path.join(ROOT, "oracle", "_ref", "libffref_hevcpred.so")
REF_DIGESTS = os.path.join(ROOT, "tests", "golden", "hevcpred_ref_digests.json")
FIXTURE = os.path.join(ROOT, "tests", "golden", "hevcpred_hashes.txt")
DEPTHS = (8, 9, 10, 12)
SHIFTS = {0: (0, 0), 1: (1, 1), 2: (1, 0), 3: (0, 0)}  # chroma_format_idc -> chroma (hshift, vshift)
MARGIN = 8                                             # guard samples around a plane
SENT8, SENT16 = 0xA5, 0xA5A5

_ref = None


def have_ref():
    return os.path.exists(REF_SO)


def ref():
    global _ref
    if _ref is None:
        _ref = C.CDLL(REF_SO)
    return _ref


def orc():
    import cpulibs as cl
    L = cl.oracle()
    if not getattr(L, "_ipred_types", False):
        vp = C.c_void_p
        L.orc_hevc_pred_planar.argtypes = [C.c_int, C.c_int, vp, vp, vp, C.c_ssize_t]
        L.orc_hevc_pred_dc.argtypes = [C.c_int, vp, vp, vp, C.c_ssize_t, C.c_int, C.c_int]
        L.orc_hevc_pred_angular.argtypes = [C.c_int, C.c_int, vp, vp, vp, C.c_ssize_t, C.c_int, C.c_int]
        L.orc_hevc_filter_3tap.argtypes = [C.c_int, vp, vp, vp, vp, C.c_int]
        L.orc_hevc_filter_strong.argtypes = [C.c_int, vp, vp, vp]
        L.orc_hevc_intra_plane.argtypes = [C.c_int, vp, C.c_ssize_t, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int64, vp, vp, C.c_ssize_t,
                                           C.c_int]
        L._ipred_types = True
    return L


def sdtype(depth):
    return np.uint8 if depth == 8 else np.uint16


def sentinel(depth):
    return SENT8 if depth == 8 else SENT16


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


_digests = None
_blocks = {}


def _write_digests():
    with open(REF_DIGESTS, "w") as f:
        json.dump(_digests, f, indent=0, sort_keys=True)
        f.write("\n")


class RefCheck:
    """with RefCheck() as rc: assert rc.same(ours, lambda: theirs) -- hevcsaolib.RefCheck's scheme with this path's own digest file:
    live comparison (and a check of the stored digest) where libffref_hevcpred.so is built, the stored digest of `ours` elsewhere;
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


def stored_digest(key):
    """the stored reference digest `key` of tests/golden/hevcpred_ref_digests.json"""
    return json.load(open(REF_DIGESTS))[key]


def digest_like_refcheck(values):
    """RefCheck's digest of a list of arrays, to compare a result with a digest stored by another test"""
    h = hashlib.sha256()
    for x in values:
        x = np.asarray(x)
        h.update(f"{x.dtype.str}{x.shape}".encode())
        h.update(np.ascontiguousarray(x).tobytes())
    return h.hexdigest()[:32]


# ---------------------------------------------------------------- pictures
def content(rng, depth, h, w):
    """blocky content: flat, ramp, textured and extreme 8x8 blocks, so that both filter decisions and both clips occur"""
    maxv = (1 << depth) - 1
    out = np.zeros((h, w), np.int64)
    for by in range(0, h, 8):
        for bx in range(0, w, 8):
            kind = rng.integers(0, 4)
            base = int(rng.integers(0, maxv + 1))
            hh, ww = min(8, h - by), min(8, w - bx)
            if kind == 0:
                v = np.full((hh, ww), base)
            elif kind == 1:
                v = base + rng.integers(-2, 3) * np.arange(hh)[:, None] + rng.integers(-2, 3) * np.arange(ww)[None, :]
            elif kind == 2:
                v = rng.choice(np.array([0, maxv]), (hh, ww))
            else:
                v = rng.integers(0, maxv + 1, (hh, ww))
            out[by:by + hh, bx:bx + ww] = v
    return np.clip(out, 0, maxv).astype(sdtype(depth))


class Picture:
    """One component of a picture as the decoder reconstructs it: the luma size W x H, the SPS sizes, the plane's initial content, the
    intra map (None without constrained intra prediction) and the TUs of that component in decode order, each
    (x0, y0, log2_size, mode, na, flags) with x0 / y0 in luma samples, na the five na.cand_* bits and flags the op's B200HevcIntraOp
    flags; res[k] the residual added after TU k."""


def zs_table(log2_ctb, log2_min_tb):
    """min_tb_addr_zs with its -1 row and column (hevc/ps.c): zs(x, y) = tab[(y + 1) * tw + x + 1]"""
    n = 1 << (log2_ctb - log2_min_tb)
    tw = n + 1
    tab = np.full((tw, tw), -1, np.int64)
    for y in range(n):
        for x in range(n):
            v = 0
            for i in range(log2_ctb - log2_min_tb):
                m = 1 << i
                v += (m * m if x & m else 0) + (2 * m * m if y & m else 0)
            tab[y + 1, x + 1] = v
    return tab


def picture_case(seed, depth, W, H, log2_ctb, cfmt, comp, cip=False, smoothing=True, strong=True, tiles=(1, 1), nslices=1, split=0.55,
                 log2_min_tb=2, log2_min_pu=2, inter_frac=0.4):
    rng = np.random.default_rng(seed)
    p = Picture()
    p.depth, p.W, p.H, p.log2_ctb, p.cfmt, p.comp = depth, W, H, log2_ctb, cfmt, comp
    p.log2_min_tb, p.log2_min_pu = log2_min_tb, log2_min_pu
    p.hs, p.vs = SHIFTS[cfmt] if comp else (0, 0)
    p.smoothing, p.strong = smoothing, strong
    ctb = 1 << log2_ctb
    cw, ch = -(-W // ctb), -(-H // ctb)
    ncols, nrows = tiles
    col_bd = [cw * k // ncols for k in range(ncols + 1)]
    row_bd = [ch * k // nrows for k in range(nrows + 1)]
    tiles_enabled = ncols > 1 or nrows > 1
    ts_to_rs, tile_of_ts = [], []
    for tr in range(nrows):
        for tc in range(ncols):
            for y in range(row_bd[tr], row_bd[tr + 1]):
                for x in range(col_bd[tc], col_bd[tc + 1]):
                    ts_to_rs.append(y * cw + x)
                    tile_of_ts.append((tr, tc))
    n = cw * ch
    rs_to_ts = np.argsort(ts_to_rs)
    tile_id = [tr * ncols + tc for tr, tc in tile_of_ts]
    starts = sorted(set([0] + [int(v) for v in rng.choice(np.arange(1, n), min(nslices - 1, n - 1), replace=False)])) if n > 1 else [0]
    slice_addr = np.zeros(n, np.int64)
    for k, s0 in enumerate(starts):
        s1 = starts[k + 1] if k + 1 < len(starts) else n
        for ts in range(s0, s1):
            slice_addr[ts_to_rs[ts]] = ts_to_rs[s0]
    p.map = (rng.random((H >> log2_min_pu, W >> log2_min_pu)) >= inter_frac).astype(np.uint8) if cip else None
    tab = zs_table(log2_ctb, log2_min_tb)
    tb_mask = (1 << (log2_ctb - log2_min_tb)) - 1

    def zs(x, y):
        return int(tab[y + 1, x + 1])

    tus = []
    end_x = W
    for ts in range(n):                                     # hls_decode_neighbour (hevcdec.c:2705-2754)
        rs = ts_to_rs[ts]
        xc, yc = (rs % cw) << log2_ctb, (rs // cw) << log2_ctb
        in_slice = rs - slice_addr[rs]
        if tiles_enabled:
            if ts == 0 or tile_id[ts] != tile_id[ts - 1]:
                tc = tile_of_ts[ts][1]
                end_x = xc + ((col_bd[tc + 1] - col_bd[tc]) << log2_ctb)
        end_y = min(yc + ctb, H)
        left_tile = tiles_enabled and xc > 0 and tile_id[ts] != tile_id[rs_to_ts[rs - 1]]
        up_tile = tiles_enabled and yc > 0 and tile_id[ts] != tile_id[rs_to_ts[rs - cw]]
        ctb_left = xc > 0 and in_slice > 0 and not left_tile
        ctb_up = yc > 0 and in_slice >= cw and not up_tile
        ctb_ur = yc > 0 and in_slice + 1 >= cw and rs + 1 - cw < n and tile_id[ts] == tile_id[rs_to_ts[rs + 1 - cw]]
        ctb_ul = xc > 0 and yc > 0 and in_slice - 1 >= cw and tile_id[ts] == tile_id[rs_to_ts[rs - 1 - cw]]

        def na(x0, y0, w, h):                               # ff_hevc_set_neighbour_available (mvs.c:43-59)
            xb, yb = x0 & (ctb - 1), y0 & (ctb - 1)
            up = bool(ctb_up or yb)
            left = bool(ctb_left or xb)
            ul = (left and up) if (xb or yb) else ctb_ul
            ur = (ctb_ur and not yb) if xb + w == ctb else up
            ur = ur and (x0 + w) < end_x
            bl = False if (y0 + h) >= end_y else left
            return int(bl) | int(left) << 1 | int(ul) << 2 | int(up) << 3 | int(ur) << 4

        def add(x0, y0, log2c, w, h):
            mode = int(rng.integers(0, 35)) if rng.random() < 0.8 else int(rng.choice([0, 1, 10, 26, 2, 18, 34]))
            tus.append((x0, y0, log2c, mode, na(x0, y0, w, h)))

        def quad(x0, y0, log2, blk, xb, yb):
            if x0 >= W or y0 >= H:
                return
            must = log2 > 5 or x0 + (1 << log2) > W or y0 + (1 << log2) > H
            if log2 > 2 and (must or rng.random() < split * (1.2 if log2 > 3 else 0.8)):
                h = 1 << (log2 - 1)
                for k, (dx, dy) in enumerate(((0, 0), (h, 0), (0, h), (h, h))):
                    quad(x0 + dx, y0 + dy, log2 - 1, k, x0, y0)
                return
            if comp == 0:
                add(x0, y0, log2, 1 << log2, 1 << log2)
            elif cfmt == 3:
                add(x0, y0, log2, 1 << log2, 1 << log2)
            elif log2 > 2:                                  # hevcdec.c:1395-1410 / 1485-1498
                lc = log2 - 1
                th, tv = 1 << (lc + p.hs), 1 << (lc + p.vs)
                for i in range(2 if cfmt == 2 else 1):
                    add(x0, y0 + (i << lc), lc, th, tv)
            elif blk == 3:                                  # hevcdec.c:1461-1468 / 1499-1510
                th, tv = 1 << (log2 + 1), 1 << (log2 + p.vs)
                for i in range(2 if cfmt == 2 else 1):
                    add(xb, yb + (i << log2), log2, th, tv)

        quad(xc, yc, log2_ctb, 0, xc, yc)

    ops = np.zeros(len(tus), INTRA_DTYPE)
    for k, (x0, y0, log2, mode, nab) in enumerate(tus):    # intra_pred's z-scan checks (pred_template.c:120-158)
        size = 1 << log2
        slh, slv = size << p.hs, size << p.vs
        sth, stv = slh >> log2_min_tb, slv >> log2_min_tb
        x_tb, y_tb = (x0 >> log2_min_tb) & tb_mask, (y0 >> log2_min_tb) & tb_mask
        spin = int(comp != 0 and not stv and bool((2 * y0) & (1 << log2_min_tb)))
        cur = zs(x_tb, y_tb)
        bl = bool(nab & 1) and cur > zs(x_tb - 1, (y_tb + stv + spin) & tb_mask)
        ur = bool(nab & 16) and not spin and cur > zs((x_tb + sth) & tb_mask, y_tb - 1)
        f = (INTRA_CAND_BL if bl else 0) | (nab & (INTRA_CAND_L | INTRA_CAND_UL | INTRA_CAND_U)) | (INTRA_CAND_UR if ur else 0)
        f |= INTRA_LUMA if comp == 0 else 0
        f |= INTRA_SMOOTH if smoothing and (comp == 0 or cfmt == 3) else 0
        f |= INTRA_STRONG if strong else 0
        ops[k] = (x0 >> p.hs, y0 >> p.vs, log2, mode, f, (0, 0, 0, 0))
    p.tus, p.ops = tus, ops
    p.pw, p.ph = W >> p.hs, H >> p.vs
    p.plane = content(rng, depth, p.ph, p.pw)
    amp = 6 << (depth - 8)
    p.res = [rng.integers(-amp, amp + 1, (1 << t[2], 1 << t[2])).astype(np.int16) for t in tus]
    p.levels = schedule(ops, p.pw, p.ph)
    return p


def schedule(ops, pw, ph):
    """dependency levels: an op's level is one above the highest level of the earlier ops (in decode order) whose written block
    intersects its read footprint (the row above from x - 1 to x + 2 * size - 1 and the column to the left from y - 1 to
    y + 2 * size - 1, clipped to the plane); returns the level of each op"""
    lev_map = np.full((ph + 1, pw + 1), -1, np.int32)        # +1: index -1 wraps onto the spare row / column, which stays -1
    out = np.zeros(len(ops), np.int32)
    for k, o in enumerate(ops):
        x, y, s = int(o["x"]), int(o["y"]), 1 << int(o["log2_size"])
        lv = -1
        if y > 0:
            lv = max(lv, int(lev_map[y - 1, max(x - 1, 0):min(x + 2 * s, pw)].max()))
        if x > 0:
            lv = max(lv, int(lev_map[max(y - 1, 0):min(y + 2 * s, ph), x - 1].max()))
        out[k] = lv + 1
        lev_map[y:y + s, x:x + s] = lv + 1
    return out


def framed(plane, depth, margin=MARGIN):
    buf = np.full((plane.shape[0] + 2 * margin, plane.shape[1] + 2 * margin), sentinel(depth), plane.dtype)
    buf[margin:margin + plane.shape[0], margin:margin + plane.shape[1]] = plane
    return buf


def inner(buf, p, margin=MARGIN):
    return buf[margin:margin + p.ph, margin:margin + p.pw]


def _ptr(buf, margin=MARGIN):
    return buf.ctypes.data + margin * buf.strides[0] + margin * buf.itemsize


class RefTu(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("x0", "y0", "log2_size", "c_idx", "mode", "na")]


def ref_plane(p):
    """the reference's intra_pred over the component, TU by TU in decode order with each residual added: the framed buffer"""
    buf = framed(p.plane, p.depth)
    tus = (RefTu * len(p.tus))(*[RefTu(x0, y0, l2, p.comp, m, nab) for x0, y0, l2, m, nab in p.tus])
    res = np.ascontiguousarray(np.concatenate([r.ravel() for r in p.res]) if p.res else np.zeros(1, np.int16))
    m = None if p.map is None else np.ascontiguousarray(p.map)
    assert ref().ffref_hevc_intra_plane(p.depth, p.cfmt, p.W, p.H, p.log2_ctb, p.log2_min_tb, p.log2_min_pu, C.c_void_p(_ptr(buf)),
                                        buf.strides[0], p.comp, len(p.tus), tus, C.c_void_p(res.ctypes.data),
                                        None if m is None else C.c_void_p(m.ctypes.data), int(not p.smoothing), int(p.strong)) == 0
    return buf


def orc_plane(p):
    """the checker's level wavefront over the component (one orc_hevc_intra_plane call per level, then the residual): the framed buffer"""
    m = None if p.map is None else np.ascontiguousarray(p.map)

    def call(buf, ops):
        assert orc().orc_hevc_intra_plane(p.depth, _ptr(buf), buf.strides[0], p.W, p.H, p.hs, p.vs, len(ops), ops.ctypes.data,
                                          None if m is None else m.ctypes.data, 0 if m is None else m.strides[0], p.log2_min_pu) == 0
    return run_levels(p, call)[0]


def strong_case(seed, depth):
    """the strong-smoothing decision at its threshold t = 1 << (depth - 5): a 256x128 luma picture of CTB 64 with one 32x32 TU at
    (32, 32) in each CTB (left, up-left and up available, bottom-left and up-right not: their runs repeat left[31] / top[31], so
    the second differences are corner - top[31] and corner - left[31]).  The eight TUs put these at t - 1, t, -(t - 1), -t on either
    side (smooth ramps elsewhere); modes that filter a 32x32 block."""
    rng = np.random.default_rng(seed)
    t = 1 << (depth - 5)
    p = Picture()
    p.depth, p.W, p.H, p.log2_ctb, p.cfmt, p.comp, p.log2_min_tb, p.log2_min_pu = depth, 256, 128, 6, 0, 0, 2, 2
    p.hs = p.vs = 0
    p.pw, p.ph, p.smoothing, p.strong, p.map = 256, 128, True, True, None
    plane = rng.integers(0, 1 << depth, (128, 256)).astype(np.int64)
    diffs = [(t - 1, t - 1), (t, t - 1), (t - 1, t), (-(t - 1), -(t - 1)), (-t, -(t - 1)), (-(t - 1), -t), (t, t), (1 - t, t - 1)]
    tus = []
    for k, (d_top, d_left) in enumerate(diffs):
        cx, cy = 64 * (k % 4) + 32, 64 * (k // 4) + 32
        c = int(rng.integers(t + 4, (1 << depth) - t - 4))
        ramp = np.arange(1, 33)
        plane[cy - 1, cx - 1] = c
        plane[cy - 1, cx:cx + 32] = c - (d_top * ramp) // 32        # top[31] = c - d_top
        plane[cy:cy + 32, cx - 1] = c - (d_left * ramp) // 32       # left[31] = c - d_left
        tus.append((cx, cy, 5, int(rng.choice([0, 2, 18, 34, 6, 30])), INTRA_CAND_L | INTRA_CAND_UL | INTRA_CAND_U))
    ops = np.zeros(len(tus), INTRA_DTYPE)
    for k, (x0, y0, l2, mode, nab) in enumerate(tus):
        ops[k] = (x0, y0, l2, mode, nab | INTRA_LUMA | INTRA_SMOOTH | INTRA_STRONG, (0, 0, 0, 0))
    p.tus, p.ops = tus, ops
    p.plane = plane.astype(sdtype(depth))
    p.res = [np.zeros((32, 32), np.int16) for _ in tus]
    p.levels = schedule(ops, p.pw, p.ph)
    return p


def tu_ops(p, sel, stride, coef_base):
    """BYPASS B200HevcTuOp records (b200_hevc_transform_add_batch_device) for the ops `sel` on the framed plane of `stride` bytes, the
    residual of op k at coef_base[k] (int16 elements)"""
    from ffmpeg_b200.hevcdsp import TU_DTYPE, BYPASS
    t = np.zeros(len(sel), TU_DTYPE)
    isz = 1 if p.depth == 8 else 2
    for i, k in enumerate(sel):
        o = p.ops[k]
        t[i]["dst_off"] = int(o["y"]) * stride + int(o["x"]) * isz
        t[i]["coef_off"] = coef_base[k]
        t[i]["log2_size"] = o["log2_size"]
        t[i]["kind"] = BYPASS
    return t


def packed_residuals(p):
    """(int16 array of every TU's residual padded to 8 elements, the element offset of each)"""
    base, parts, pos = [], [], 0
    for r in p.res:
        base.append(pos)
        parts.append(np.pad(r.ravel(), (0, (-r.size) % 8)))
        pos += parts[-1].size
    return (np.concatenate(parts) if parts else np.zeros(8, np.int16)), base


def add_residual(buf, p, sel):
    """the residual of the ops `sel` added and clipped on the host (what a BYPASS residual-add call does)"""
    maxv = (1 << p.depth) - 1
    for k in sel:
        o = p.ops[k]
        x, y, s = int(o["x"]) + MARGIN, int(o["y"]) + MARGIN, 1 << int(o["log2_size"])
        blk = buf[y:y + s, x:x + s].astype(np.int64) + p.res[k]
        buf[y:y + s, x:x + s] = np.clip(blk, 0, maxv).astype(buf.dtype)


def run_levels(p, predict_call, buf=None):
    """the level wavefront on the host plane `buf` (framed): per level, predict_call(buf, ops of the level), then the residual added;
    returns (buf, number of levels)"""
    buf = framed(p.plane, p.depth) if buf is None else buf
    nl = int(p.levels.max()) + 1 if len(p.levels) else 0
    for lv in range(nl):
        sel = np.nonzero(p.levels == lv)[0]
        predict_call(buf, np.ascontiguousarray(p.ops[sel]))
        add_residual(buf, p, sel)
    return buf, nl


# ---------------------------------------------------------------- single members
def edge_arrays(rng, depth, kind):
    """(top, left) int arrays of 2 * 64 + 1 + 16 samples, index -1 at position 0: random, flat, smooth ramps (strong filter taken) or
    extremes"""
    maxv = (1 << depth) - 1
    n = 2 * 64 + 1 + 16
    if kind == 0:
        return rng.integers(0, maxv + 1, n), rng.integers(0, maxv + 1, n)
    if kind == 1:
        v = int(rng.integers(0, maxv + 1))
        return np.full(n, v), np.full(n, v + (1 if v < maxv else -1))
    if kind == 2:
        a, b, c = (int(v) for v in rng.integers(0, maxv + 1, 3))
        t = np.clip(a + (b - a) * np.arange(-1, n - 1) // 64, 0, maxv)
        l_ = np.clip(a + (c - a) * np.arange(-1, n - 1) // 64, 0, maxv)
        return t, l_
    return rng.choice(np.array([0, maxv]), n), rng.choice(np.array([0, maxv]), n)


def member_cases(seed, depth):
    """yields (which, log2_size, mode, c_idx, top, left): every size x every mode (planar, DC, 2..34) x luma / chroma"""
    rng = np.random.default_rng(seed)
    for log2 in (2, 3, 4, 5):
        for mode in range(35):
            for c_idx in (0, 1):
                t, l_ = edge_arrays(rng, depth, int(rng.integers(0, 4)))
                yield (0 if mode == 0 else 1 if mode == 1 else 2), log2, mode, c_idx, t.astype(sdtype(depth)), l_.astype(sdtype(depth))


def _dst(depth, size):
    return np.full((size + 2 * MARGIN, size + 2 * MARGIN), sentinel(depth), sdtype(depth))


def ref_member(depth, case):
    which, log2, mode, c_idx, t, l_ = case
    t, l_ = t.copy(), l_.copy()
    d = _dst(depth, 1 << log2)
    assert ref().ffref_hevc_pred(depth, which, log2, C.c_void_p(_ptr(d)), C.c_void_p(t.ctypes.data + t.itemsize),
                                 C.c_void_p(l_.ctypes.data + l_.itemsize), C.c_ssize_t(d.strides[0] // d.itemsize), c_idx, mode) == 0
    return d


def orc_member(depth, case):
    which, log2, mode, c_idx, t, l_ = case
    t, l_ = t.copy(), l_.copy()
    d = _dst(depth, 1 << log2)
    tp, lp, st = t.ctypes.data + t.itemsize, l_.ctypes.data + l_.itemsize, d.strides[0] // d.itemsize
    if which == 0:
        orc().orc_hevc_pred_planar(depth, log2, _ptr(d), tp, lp, st)
    elif which == 1:
        orc().orc_hevc_pred_dc(depth, _ptr(d), tp, lp, st, log2, c_idx)
    else:
        orc().orc_hevc_pred_angular(depth, log2, _ptr(d), tp, lp, st, c_idx, mode)
    return d


def ctx_member(ctx, depth, case):
    from ffmpeg_b200 import hevcdsp as hd
    which, log2, mode, c_idx, t, l_ = case
    t, l_ = t.copy(), l_.copy()
    d = _dst(depth, 1 << log2)
    tp, lp, st = t.ctypes.data + t.itemsize, l_.ctypes.data + l_.itemsize, d.strides[0] // d.itemsize   # members: stride in samples
    if which == 0:
        hd.PRED_PLANAR(ctx.pred_planar[log2 - 2])(_ptr(d), tp, lp, st)
    elif which == 1:
        hd.PRED_DC(ctx.pred_dc)(_ptr(d), tp, lp, st, log2, c_idx)
    else:
        hd.PRED_ANGULAR(ctx.pred_angular[log2 - 2])(_ptr(d), tp, lp, st, c_idx, mode)
    return d


def filter_cases(seed, depth):
    rng = np.random.default_rng(seed)
    for size in (8, 16, 32):
        for kind in range(4):
            t, l_ = edge_arrays(rng, depth, kind)
            yield size, t.astype(sdtype(depth)), l_.astype(sdtype(depth))


def run_filters(depth, case, f3, fs):
    """f3(fl, ft, l, t, size), fs(ft, l, t) on copies with sentinel-filled outputs: (filtered left, filtered top, left after the strong
    filter, filtered top of the strong filter)"""
    size, t, l_ = case
    t, l_ = t.copy(), l_.copy()
    fl, ft = np.full_like(t, sentinel(depth)), np.full_like(t, sentinel(depth))
    f3(fl.ctypes.data + fl.itemsize, ft.ctypes.data + ft.itemsize, l_.ctypes.data + l_.itemsize, t.ctypes.data + t.itemsize, size)
    ft2 = np.full_like(t, sentinel(depth))
    fs(ft2.ctypes.data + ft2.itemsize, l_.ctypes.data + l_.itemsize, t.ctypes.data + t.itemsize)
    return fl, ft, l_, ft2


def ref_filters(depth, case, idx=0):
    r = ref()
    return run_filters(depth, case, lambda *a: r.ffref_hevc_filter_3tap(depth, idx, *[C.c_void_p(v) for v in a[:4]], a[4]),
                       lambda *a: r.ffref_hevc_filter_strong(depth, *[C.c_void_p(v) for v in a]))


def orc_filters(depth, case):
    L = orc()
    return run_filters(depth, case, lambda *a: L.orc_hevc_filter_3tap(depth, *a), lambda *a: L.orc_hevc_filter_strong(depth, *a))


def ctx_filters(ctx, depth, case, idx=0):
    from ffmpeg_b200 import hevcdsp as hd
    return run_filters(depth, case, hd.REF_FILTER_3TAP(ctx.ref_filter_3tap[idx]), hd.REF_FILTER_STRONG(ctx.ref_filter_strong))


# ---------------------------------------------------------------- fixture
FIXTURE_CFMT = {"luma": (0, 0), "420": (1, 1), "422": (2, 1), "444": (3, 1)}   # name -> (chroma_format_idc, component)


def fixture_case(depth, name, cip):
    cfmt, comp = FIXTURE_CFMT[name]
    return picture_case(9000 + 10 * depth + 2 * cfmt + int(cip), depth, 200, 136, 5, cfmt, comp, cip=cip, tiles=(2, 2), nslices=3)


def fixture_hashes():
    out = {}
    for line in open(FIXTURE):
        d, what, h = line.split()
        out[(int(d), what)] = h
    return out


def fixture_key(name, cip):
    return f"{name}_{'cip' if cip else 'nocip'}"
