"""Test infrastructure for HEVC intra reconstruction of a whole picture (b200_hevc_intra_recon_picture_device): seeded pictures (one
transform quadtree per CTB of 16 / 32 / 64, slices and tiles, sizes that are not CTB multiples, luma only or 4:2:0 / 4:2:2 / 4:4:4
chroma, constrained intra prediction, smoothing and strong smoothing on and off, every residual kind and flag and TUs without residual,
optionally sparse intra TUs among prefilled inter samples) whose TUs of all components come out interleaved as hls_transform_unit
(hevc/hevcdec.c:1306-1513) calls intra_pred: luma, then with a residual each Cb block then each Cr block, predicted and added one after
the other, without one Cb, Cr and the second 4:2:2 pair; chroma of 4x4 luma at blk_idx 3.  The neighbour flags, z-scan checks, content
and intra maps are hevcpredlib's; coefficients and TU kinds are hevcidctlib's.  Runners of the checker (orc_hevc_intra_picture, in decode
order or with no dependencies), of the compiled reference (oracle/_ref/libffref_hevcintra.so, built by oracle/ref/Makefile), of the
per-level path (one prediction and one residual batch per dependency level and plane), and RefCheck with its own digest file
tests/golden/hevcintra_ref_digests.json."""
import ctypes as C
import hashlib
import json
import os

import numpy as np

import cpulibs as cl
import hevcidctlib as hi
import hevcpredlib as hp
from ffmpeg_b200.hevcdsp import (RECON_DTYPE, TU_NONE, INTRA_DTYPE, TU_DTYPE, INTRA_CAND_BL, INTRA_CAND_L, INTRA_CAND_UL, INTRA_CAND_U,
                                 INTRA_CAND_UR, INTRA_LUMA, INTRA_SMOOTH, INTRA_STRONG)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_LIB = "libffref_hevcintra"
REF_DIGESTS = os.path.join(ROOT, "tests", "golden", "hevcintra_ref_digests.json")
FIXTURE = os.path.join(ROOT, "tests", "golden", "hevcintra_hashes.txt")
DEPTHS = (8, 9, 10, 12)
MARGIN = 8                                             # guard samples around a plane (and up to 15 more on the right: rows of 16 samples)


def have_ref():
    return cl.have_ref(REF_LIB)


def ref():
    return cl.ref_lib(REF_LIB)


def RefCheck():
    return cl.RefCheck(REF_DIGESTS, REF_LIB)


def orc():
    L = cl.oracle()
    if not getattr(L, "_hintra_types", False):
        vp = C.c_void_p
        L.orc_hevc_intra_picture.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, vp, C.c_ssize_t, C.c_ssize_t, C.c_int64, vp, vp, vp,
                                             C.c_ssize_t, C.c_int, C.c_int]
        L._hintra_types = True
    return L


def digest(planes):
    h = hashlib.sha256()
    for a in planes:
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


# ---------------------------------------------------------------- pictures
class Picture:
    """A picture as the decoder reconstructs its intra TUs: the luma size W x H, the SPS sizes, the planes' initial content (framed:
    MARGIN sentinel samples around, rows padded to 16 samples), the intra map (None without constrained intra prediction), and per TU
    in decode order tus[k] = (x0, y0, log2_size, c_idx, mode, na) as the decoder calls intra_pred, with ops[k] its RECON_DTYPE record;
    coef the int16 coefficients."""

    def shifts(self, c):
        return hp.SHIFTS[self.cfmt] if c else (0, 0)

    def dims(self, c):
        hs, vs = self.shifts(c)
        return self.W >> hs, self.H >> vs

    @property
    def nplanes(self):
        return 3 if self.cfmt else 1

    def framed(self):
        """fresh copies of the initial framed planes"""
        return [f.copy() for f in self.frames]

    def inner(self, bufs):
        return [b[MARGIN:MARGIN + self.dims(c)[1], MARGIN:MARGIN + self.dims(c)[0]] for c, b in enumerate(bufs)]

    def ptrs(self, bufs):
        return [b.ctypes.data + MARGIN * b.strides[0] + MARGIN * b.itemsize for b in bufs] + [0] * (3 - len(bufs))

    def strides(self, bufs):
        return bufs[0].strides[0], (bufs[1].strides[0] if len(bufs) > 1 else 0)


def _frame(plane, depth):
    h, w = plane.shape
    buf = np.full((h + 2 * MARGIN, -(-(w + 2 * MARGIN) // 16) * 16), hp.sentinel(depth), plane.dtype)
    buf[MARGIN:MARGIN + h, MARGIN:MARGIN + w] = plane
    return buf


def picture(seed, depth, cfmt, W, H, log2_ctb, cip=False, smoothing=True, strong=True, tiles=(1, 1), nslices=1, split=0.55,
            p_cbf=0.7, p_intra=1.0, log2_min_tb=2, log2_min_pu=2):
    rng = np.random.default_rng(seed)
    p = Picture()
    p.depth, p.cfmt, p.W, p.H, p.log2_ctb, p.log2_min_tb, p.log2_min_pu = depth, cfmt, W, H, log2_ctb, log2_min_tb, log2_min_pu
    p.smoothing, p.strong = smoothing, strong
    chs, cvs = hp.SHIFTS[cfmt]
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
    p.map = (rng.random((H >> log2_min_pu, W >> log2_min_pu)) >= 0.4).astype(np.uint8) if cip else None
    tab = hp.zs_table(log2_ctb, log2_min_tb)
    tb_mask = (1 << (log2_ctb - log2_min_tb)) - 1
    tus, res = [], []                                        # res[k]: None or (kind, flags, coefficients, col_limit)

    def zs(x, y):
        return int(tab[y + 1, x + 1])

    end_x = W
    for ts in range(n):                                      # hls_decode_neighbour (hevcdec.c:2705-2754), as hevcpredlib.picture_case
        rs = ts_to_rs[ts]
        xc, yc = (rs % cw) << log2_ctb, (rs // cw) << log2_ctb
        in_slice = rs - slice_addr[rs]
        if tiles_enabled and (ts == 0 or tile_id[ts] != tile_id[ts - 1]):
            tc = tile_of_ts[ts][1]
            end_x = xc + ((col_bd[tc + 1] - col_bd[tc]) << log2_ctb)
        end_y = min(yc + ctb, H)
        left_tile = tiles_enabled and xc > 0 and tile_id[ts] != tile_id[rs_to_ts[rs - 1]]
        up_tile = tiles_enabled and yc > 0 and tile_id[ts] != tile_id[rs_to_ts[rs - cw]]
        ctb_left = xc > 0 and in_slice > 0 and not left_tile
        ctb_up = yc > 0 and in_slice >= cw and not up_tile
        ctb_ur = yc > 0 and in_slice + 1 >= cw and rs + 1 - cw < n and tile_id[ts] == tile_id[rs_to_ts[rs + 1 - cw]]
        ctb_ul = xc > 0 and yc > 0 and in_slice - 1 >= cw and tile_id[ts] == tile_id[rs_to_ts[rs - 1 - cw]]

        def na(x0, y0, w, h):                                # ff_hevc_set_neighbour_available (mvs.c:43-59)
            xb, yb = x0 & (ctb - 1), y0 & (ctb - 1)
            up = bool(ctb_up or yb)
            left = bool(ctb_left or xb)
            ul = (left and up) if (xb or yb) else ctb_ul
            ur = (ctb_ur and not yb) if xb + w == ctb else up
            ur = ur and (x0 + w) < end_x
            bl = False if (y0 + h) >= end_y else left
            return int(bl) | int(left) << 1 | int(ul) << 2 | int(up) << 3 | int(ur) << 4

        def residual(log2, chroma):
            if rng.random() >= p_cbf:
                return None
            kind, f = hi.op_kind(rng, log2, chroma)
            c, lim = hi.decoder_block(rng, log2)
            if rng.random() < 0.5:                           # most blocks with small levels, as a parser leaves them
                c = (c.astype(np.int64) * int(rng.integers(1, 64)) // 32767).astype(np.int16)
            return kind, f, c, lim

        def add(x0, y0, log2c, c_idx, nab, r):
            mode = int(rng.integers(0, 35)) if rng.random() < 0.8 else int(rng.choice([0, 1, 10, 26, 2, 18, 34]))
            tus.append((x0, y0, log2c, c_idx, mode, nab))
            res.append(r)

        def chroma(pairs, log2c, w, h):                     # hevcdec.c:1395-1470 (with a residual) and 1485-1512 (without)
            nabs = [na(x, y, w, h) for x, y in pairs]
            rcb = [residual(log2c, True) for _ in pairs]
            rcr = [residual(log2c, True) for _ in pairs]
            return nabs, rcb, rcr

        def quad(x0, y0, log2, blk, xb, yb, intra):
            if x0 >= W or y0 >= H:
                return
            if intra is None and log2 <= 4:
                intra = rng.random() < p_intra
            must = log2 > 5 or x0 + (1 << log2) > W or y0 + (1 << log2) > H
            if log2 > 2 and (must or rng.random() < split * (1.2 if log2 > 3 else 0.8)):
                h = 1 << (log2 - 1)
                for k, (dx, dy) in enumerate(((0, 0), (h, 0), (0, h), (h, h))):
                    quad(x0 + dx, y0 + dy, log2 - 1, k, x0, y0, intra)
                return
            if intra is None:
                intra = rng.random() < p_intra
            if not intra:
                return
            rl = residual(log2, False)
            add(x0, y0, log2, 0, na(x0, y0, 1 << log2, 1 << log2), rl)
            if not cfmt:
                return
            if log2 > 2 or cfmt == 3:
                lc = log2 - (cfmt != 3)
                pairs = [(x0, y0 + (i << lc)) for i in range(2 if cfmt == 2 else 1)]
                nabs, rcb, rcr = chroma(pairs, lc, 1 << (lc + chs), 1 << (lc + cvs))
            elif blk == 3:
                lc = log2
                pairs = [(xb, yb + (i << log2)) for i in range(2 if cfmt == 2 else 1)]
                nabs, rcb, rcr = chroma(pairs, lc, 1 << (log2 + 1), 1 << (log2 + cvs))
            else:
                return
            if rl is not None or any(r is not None for r in rcb + rcr):
                for c_idx, rr in ((1, rcb), (2, rcr)):
                    for (x, y), nab, r in zip(pairs, nabs, rr):
                        add(x, y, lc, c_idx, nab, r)
            else:
                for (x, y), nab in zip(pairs, nabs):
                    add(x, y, lc, 1, nab, None)
                    add(x, y, lc, 2, nab, None)

        quad(xc, yc, log2_ctb, 0, xc, yc, None)

    ops = np.zeros(len(tus), RECON_DTYPE)
    chunks, off = [], 0
    for k, (x0, y0, log2, c_idx, mode, nab) in enumerate(tus):   # intra_pred's z-scan checks (pred_template.c:120-158)
        hs, vs = (chs, cvs) if c_idx else (0, 0)
        size = 1 << log2
        sth, stv = (size << hs) >> log2_min_tb, (size << vs) >> log2_min_tb
        x_tb, y_tb = (x0 >> log2_min_tb) & tb_mask, (y0 >> log2_min_tb) & tb_mask
        spin = int(c_idx != 0 and not stv and bool((2 * y0) & (1 << log2_min_tb)))
        cur = zs(x_tb, y_tb)
        bl = bool(nab & 1) and cur > zs(x_tb - 1, (y_tb + stv + spin) & tb_mask)
        ur = bool(nab & 16) and not spin and cur > zs((x_tb + sth) & tb_mask, y_tb - 1)
        f = (INTRA_CAND_BL if bl else 0) | (nab & (INTRA_CAND_L | INTRA_CAND_UL | INTRA_CAND_U)) | (INTRA_CAND_UR if ur else 0)
        f |= INTRA_LUMA if c_idx == 0 else 0
        f |= INTRA_SMOOTH if smoothing and (c_idx == 0 or cfmt == 3) else 0
        f |= INTRA_STRONG if strong else 0
        o = ops[k]
        o["x"], o["y"], o["plane"], o["log2_size"], o["mode"], o["flags"] = x0 >> hs, y0 >> vs, c_idx, log2, mode, f
        if res[k] is None:
            o["tu_kind"] = TU_NONE
        else:
            kind, tf, c, lim = res[k]
            o["tu_kind"], o["tu_flags"], o["col_limit"], o["coef_off"] = kind, tf, lim, off
            chunks.append(np.pad(c.ravel(), (0, (-c.size) % 8)))
            off += chunks[-1].size
    p.tus, p.ops = tus, ops
    p.coef = np.concatenate(chunks + [np.zeros(8, np.int16)])
    p.frames = [_frame(hp.content(rng, depth, p.dims(c)[1], p.dims(c)[0]), depth) for c in range(p.nplanes)]
    return p


# ---------------------------------------------------------------- runners
def _coef16(coef):
    """the coefficients in a 16-byte aligned buffer (the entry's requirement); returns (buffer, address)"""
    raw = coef.view(np.uint8)
    buf = np.zeros(raw.size + 32, np.uint8)
    start = -buf.ctypes.data % 16
    buf[start:start + raw.size] = raw
    return buf, buf.ctypes.data + start


def orc_picture(p, order=0, ops=None):
    """the checker's decode order (order 0) or its no-dependency order (1): the framed planes"""
    bufs = p.framed()
    ops = np.ascontiguousarray(p.ops if ops is None else ops)
    arr = (C.c_void_p * 3)(*p.ptrs(bufs))
    m = None if p.map is None else np.ascontiguousarray(p.map)
    ls_y, ls_uv = p.strides(bufs)
    assert orc().orc_hevc_intra_picture(p.depth, p.cfmt, p.W, p.H, arr, ls_y, ls_uv, len(ops), ops.ctypes.data, p.coef.ctypes.data,
                                        None if m is None else m.ctypes.data, 0 if m is None else m.strides[0], p.log2_min_pu, order) == 0
    return bufs


class RefReconTu(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("x0", "y0", "log2_size", "c_idx", "mode", "na")] + [("coef_off", C.c_int64)] + \
               [(n, C.c_int32) for n in ("kind", "flags", "col_limit", "pad")]


def ref_picture(p):
    """the reference's intra_pred and residual sequence TU by TU in decode order: the framed planes"""
    bufs = p.framed()
    tus = (RefReconTu * max(1, len(p.tus)))(*[RefReconTu(x0, y0, l2, c, m, nab, int(o["coef_off"]), int(o["tu_kind"]), int(o["tu_flags"]),
                                                         int(o["col_limit"]), 0)
                                               for (x0, y0, l2, c, m, nab), o in zip(p.tus, p.ops)])
    arr = (C.c_void_p * 3)(*p.ptrs(bufs))
    m = None if p.map is None else np.ascontiguousarray(p.map)
    ls_y, ls_uv = p.strides(bufs)
    assert ref().ffref_hevc_intra_picture(p.depth, p.cfmt, p.W, p.H, p.log2_ctb, p.log2_min_tb, p.log2_min_pu, arr, ls_y, ls_uv,
                                          len(p.tus), tus, C.c_void_p(p.coef.ctypes.data),
                                          None if m is None else C.c_void_p(m.ctypes.data), int(not p.smoothing), int(p.strong)) == 0
    return bufs


def level_batches(p):
    """the per-level path's calls: for each plane and each dependency level (hevcpredlib.schedule over the plane's ops in decode
    order), (plane, INTRA_DTYPE ops, the indices into p.ops)"""
    out = []
    for c in range(p.nplanes):
        sel = np.nonzero(p.ops["plane"] == c)[0]
        if not len(sel):
            continue
        io = np.zeros(len(sel), INTRA_DTYPE)
        for f in ("x", "y", "log2_size", "mode", "flags"):
            io[f] = p.ops[f][sel]
        pw, ph = p.dims(c)
        lv = hp.schedule(io, pw, ph)
        for level in range(int(lv.max()) + 1):
            k = np.nonzero(lv == level)[0]
            out.append((c, np.ascontiguousarray(io[k]), sel[k]))
    return out


def level_tu_ops(p, idx, stride):
    """B200HevcTuOp records of the ops idx that have a residual, for a plane of `stride` bytes"""
    idx = [k for k in idx if p.ops["tu_kind"][k] != TU_NONE]
    t = np.zeros(len(idx), TU_DTYPE)
    isz = 1 if p.depth == 8 else 2
    for i, k in enumerate(idx):
        o = p.ops[k]
        t[i]["dst_off"] = int(o["y"]) * stride + int(o["x"]) * isz
        t[i]["coef_off"], t[i]["log2_size"], t[i]["kind"], t[i]["flags"], t[i]["col_limit"] = o["coef_off"], o["log2_size"], o["tu_kind"], \
            o["tu_flags"], o["col_limit"]
    return t


# ---------------------------------------------------------------- fixture
FIXTURES = {   # name -> (depth, chroma_format_idc, W, H, log2_ctb, kwargs)
    "420-8": (8, 1, 200, 136, 5, dict(tiles=(2, 2), nslices=3)),
    "420-10-cip": (10, 1, 232, 120, 4, dict(cip=True, nslices=2)),
    "422-9": (9, 2, 200, 136, 6, dict(nslices=2, strong=False)),
    "422-12-cip": (12, 2, 136, 72, 5, dict(cip=True, tiles=(2, 1))),
    "444-8-cip": (8, 3, 136, 88, 4, dict(cip=True, smoothing=False)),
    "444-10": (10, 3, 200, 136, 5, dict(tiles=(2, 2), nslices=2)),
    "400-12": (12, 0, 200, 136, 6, dict(nslices=3)),
    "420-9-sparse": (9, 1, 264, 136, 5, dict(p_intra=0.3, cip=True)),
}
FIXTURE_NAMES = list(FIXTURES)


def fixture_case(name):
    depth, cfmt, W, H, l2, kw = FIXTURES[name]
    return picture(7000 + FIXTURE_NAMES.index(name), depth, cfmt, W, H, l2, **kw)


def fixture_hashes():
    out = {}
    for line in open(FIXTURE):
        name, h = line.split()
        out[name] = h
    return out
