"""Test infrastructure for the VP9 loop filter (the loop-filter members of VP9DSPContext and b200_vp9_loopfilter_frame_device): seeded
frames with decoder-shaped loop-filter records (mask_edges, vp9block.c:1142-1262, restated on random partitions, transform sizes, skip
flags and levels) or arbitrary masks, member calls, and runners of the checker (oracle/liboracle.so: orc_vp9_lf_member, orc_vp9_lf_frame)
and of the compiled reference (oracle/_ref/libffref_vp9lf.so, built by oracle/ref/Makefile).  The reference's results are kept as
digests in tests/golden/vp9lf_ref_digests.json (cpulibs.RefCheck) for machines without the reference."""
import ctypes as C
import hashlib
import os

import numpy as np

import cpulibs as cl
from ffmpeg_b200.vp9dsp import LF_DTYPE

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_LIB = "libffref_vp9lf"
REF_DIGESTS = os.path.join(ROOT, "tests", "golden", "vp9lf_ref_digests.json")
FIXTURE = os.path.join(ROOT, "tests", "golden", "vp9lf_hashes.txt")
DEPTHS = (8, 10, 12)
FORMATS = {"420": (1, 1), "422": (1, 0), "440": (0, 1), "444": (0, 0)}     # (ss_h, ss_v)
MARGIN = 8           # sentinel samples around every plane's area


def have_ref():
    return cl.have_ref(REF_LIB)


def ref():
    return cl.ref_lib(REF_LIB)


def RefCheck():
    return cl.RefCheck(REF_DIGESTS, REF_LIB)


def sdtype(depth):
    return np.uint8 if depth == 8 else np.uint16


def luts(sharp):
    """the decoder's filter_lut for a sharpness (vp9.c:684-697); entry 0 stays 0"""
    lim, mblim = np.zeros(64, np.uint8), np.zeros(64, np.uint8)
    for i in range(1, 64):
        limit = i
        if sharp > 0:
            limit = min(limit >> ((sharp + 3) >> 2), 9 - sharp)
        limit = max(limit, 1)
        lim[i], mblim[i] = limit, 2 * (i + 2) + limit
    return lim, mblim


# ---------------------------------------------------------------- records
def mask_edges(mask, ss_h, ss_v, row_and_7, col_and_7, w, h, col_end, row_end, tx, skip_inter):
    """vp9block.c:1142-1262 on mask = uint8 [2 (col / row)][8][4]"""
    wide_col, wide_row = (0x11, 0x01), (0x03, 0x07)
    if tx == 0 and (ss_v | ss_h):
        if h == ss_v:
            if row_and_7 & 1:
                return
            if not row_end:
                h += 1
        if w == ss_h:
            if col_and_7 & 1:
                return
            if not col_end:
                w += 1
    t = 1 << col_and_7
    m_col = ((t << w) - t) & 0xFF
    if tx == 0 and not skip_inter:
        m_row_8 = m_col & wide_col[ss_h]
        m_row_4 = m_col - m_row_8
        for y in range(row_and_7, h + row_and_7):
            col_mask_id = 2 - (0 if (y & wide_row[ss_v]) else 1)
            mask[0][y][1] |= m_row_8
            mask[0][y][2] |= m_row_4
            if (ss_h & ss_v) and (col_end & 1) and (y & 1):
                mask[1][y][col_mask_id] |= ((t << (w - 1)) - t) & 0xFF
            else:
                mask[1][y][col_mask_id] |= m_col
            if not ss_h:
                mask[0][y][3] |= m_col
            if not ss_v:
                if ss_h and (col_end & 1):
                    mask[1][y][3] |= ((t << (w - 1)) - t) & 0xFF
                else:
                    mask[1][y][3] |= m_col
    elif not skip_inter:
        mask_id = 1 if tx == 1 else 0
        masks = (0xFF, 0x55, 0x11, 0x01)
        l2 = tx + ss_h - 1
        m_row = m_col & masks[l2]
        if ss_h and tx > 1 and (w ^ (w - 1)) == 1:
            m_row_16 = ((t << (w - 1)) - t) & masks[l2]
            m_row_8 = m_row - m_row_16
            for y in range(row_and_7, h + row_and_7):
                mask[0][y][0] |= m_row_16
                mask[0][y][1] |= m_row_8
        else:
            for y in range(row_and_7, h + row_and_7):
                mask[0][y][mask_id] |= m_row
        l2 = tx + ss_v - 1
        step1d = 1 << l2
        if ss_v and tx > 1 and (h ^ (h - 1)) == 1:
            y = row_and_7
            while y < h + row_and_7 - 1:
                mask[1][y][0] |= m_col
                y += step1d
            if y - row_and_7 == h - 1:
                mask[1][y][1] |= m_col
        else:
            for y in range(row_and_7, h + row_and_7, step1d):
                mask[1][y][mask_id] |= m_col
    elif tx != 0:
        mask_id = 1 if (tx == 1 or h == ss_v) else 0
        mask[1][row_and_7][mask_id] |= m_col
        mask_id = 1 if (tx == 1 or w == ss_h) else 0
        for y in range(row_and_7, h + row_and_7):
            mask[0][y][mask_id] |= t
    else:
        t8 = t & wide_col[ss_h]
        t4 = t - t8
        for y in range(row_and_7, h + row_and_7):
            mask[0][y][2] |= t4
            mask[0][y][1] |= t8
        mask[1][row_and_7][2 - (0 if (row_and_7 & wide_row[ss_v]) else 1)] |= m_col


def decoder_records(rng, ss_h, ss_v, cols, rows, lstride):
    """LF_DTYPE [sb_rows, lstride]: every superblock split into blocks at random (64 .. 8 and the sub-8x8 partitions), each block with a
    random transform size its size allows, the chroma transform size the decoder derives (vp9block.c:1291-1292), a skip flag and a level
    (0 for about one block in ten: no edges), its edges marked as ff_vp9_decode_block does (vp9block.c:1425-1446)"""
    sbc, sbr = (cols + 7) >> 3, (rows + 7) >> 3
    rec = np.zeros((sbr, lstride), LF_DTYPE)
    rec["level"] = rng.integers(0, 64, rec["level"].shape)                    # stale levels where no block sets one
    for r in range(sbr):
        for c in range(sbc):
            lv = rec["level"][r, c].reshape(8, 8)
            mk = rec["mask"][r, c]
            blocks = []

            def split(x, y, s):                                                # x, y, s in 8x8 units
                if 8 * r + y >= rows or 8 * c + x >= cols:
                    return
                if s > 1 and rng.random() < 0.6:
                    h = s // 2
                    for dy in (0, h):
                        for dx in (0, h):
                            split(x + dx, y + dy, h)
                    return
                bp = int(rng.integers(0, 4))                                   # NONE, H, V, SPLIT (SPLIT only at 8x8)
                if s == 1:
                    blocks.append((x, y, 1, 1, bp != 0))
                elif bp == 1:
                    blocks.append((x, y, s, s // 2, False))
                    if 8 * r + y + s // 2 < rows:
                        blocks.append((x, y + s // 2, s, s // 2, False))
                elif bp == 2:
                    blocks.append((x, y, s // 2, s, False))
                    if 8 * c + x + s // 2 < cols:
                        blocks.append((x + s // 2, y, s // 2, s, False))
                else:
                    blocks.append((x, y, s, s, False))
            split(0, 0, 8)
            for x, y, w4, h4, sub8 in blocks:
                lvl = int(rng.integers(1, 64)) if rng.random() > 0.1 else 0
                if not lvl:
                    continue
                maxtx = 0 if sub8 else min(int(np.log2(8 * min(w4, h4))) - 2, 3)
                tx = int(rng.integers(0, maxtx + 1))
                uvtx = tx - int((ss_h and w4 * 2 == (1 << tx)) or (ss_v and h4 * 2 == (1 << tx)))
                skip = bool(rng.random() < 0.3)
                col, row = 8 * c + x, 8 * r + y
                x_end, y_end = min(cols - col, w4), min(rows - row, h4)
                lv[y:y + h4, x:x + w4] = lvl
                mask_edges(mk[0], 0, 0, y, x, x_end, y_end, 0, 0, tx, skip)
                if ss_h or ss_v:
                    mask_edges(mk[1], ss_h, ss_v, y, x, x_end, y_end, (cols & 7) if (cols & 1 and col + w4 >= cols) else 0,
                               (rows & 7) if (rows & 1 and row + h4 >= rows) else 0, max(uvtx, 0), skip)
    return rec


def area(ss, n8):
    """samples of a plane's area along one direction: n8 8x8 luma blocks, subsampled by ss, rounded up to 8"""
    return ((n8 * 8 >> ss) + 7) & ~7


def arbitrary_records(rng, ss_h, ss_v, cols, rows, lstride, density=0.35):
    """random mask bytes and levels, restricted to the picture (bits of 8x8 columns < cols and rows < rows) and, for the chroma masks of
    subsampled formats, to 16-wide edges whose 16 samples lie inside the chroma area (not 4 samples from its left or top edge, nor past
    its right or bottom edge) and inside the superblock (not at bit 7 / row 7 of a subsampled direction)"""
    sbc, sbr = (cols + 7) >> 3, (rows + 7) >> 3
    rec = np.zeros((sbr, lstride), LF_DTYPE)
    rec["level"] = rng.integers(0, 64, rec["level"].shape)
    bits = (rng.random((sbr, lstride, 2, 2, 8, 4, 8)) < density).astype(np.uint8)
    wc, hc = area(ss_h, cols), area(ss_v, rows)
    for r in range(sbr):
        for c in range(lstride):
            for k in range(8):
                for y in range(8):
                    if c >= sbc or 8 * c + k >= cols or 8 * r + y >= rows:
                        bits[r, c, :, :, y, :, k] = 0
                    if ss_h | ss_v:
                        x16, y16 = c * (64 >> ss_h) + k * (8 >> ss_h), r * (64 >> ss_v) + y * (8 >> ss_v)
                        if x16 + 8 > wc or x16 == 4 or (ss_h and k == 7):
                            bits[r, c, 1, 0, y, 0, k] = 0
                        if y16 + 8 > hc or y16 == 4 or (ss_v and y == 7):
                            bits[r, c, 1, 1, y, 0, k] = 0
    rec["mask"] = (bits << np.arange(8, dtype=np.uint8)).sum(-1).astype(np.uint8)
    return rec


# ---------------------------------------------------------------- frames
def content(rng, depth, h, w):
    """8x8 blocks of a smooth base with steps between them and per-block noise of several amplitudes, so that flat8out / flat8in / hev /
    the filter mask all go both ways"""
    sh = depth - 8
    by, bx = (h + 7) // 8, (w + 7) // 8
    yy, xx = np.mgrid[0:by, 0:bx]
    base = 128 + 60 * np.sin(xx / 5.0 + yy / 7.0) + rng.integers(-12, 13, (by, bx)) * (rng.random((by, bx)) < 0.6)
    amp = rng.choice([0, 0, 1, 2, 5, 60], (by, bx))
    img = np.kron(base, np.ones((8, 8)))[:h, :w] * (1 << sh)
    noise = rng.integers(-(1 << 20), 1 << 20, (h, w)) % (np.kron(amp, np.ones((8, 8), np.int64))[:h, :w] * (1 << sh) + 1)
    return np.clip(img + noise, 0, (1 << depth) - 1).astype(sdtype(depth))


class Frame:
    """one frame: planes (full arrays with MARGIN sentinel samples around the area), records, LUTs"""

    def __init__(self, seed, depth, fmt, width, height, kind="decoder", sharp=None, pad=0):
        rng = np.random.default_rng(seed)
        self.depth, self.fmt, self.width, self.height = depth, fmt, width, height
        self.ss_h, self.ss_v = FORMATS[fmt]
        self.cols, self.rows = (width + 7) >> 3, (height + 7) >> 3
        self.sbc, self.sbr = (self.cols + 7) >> 3, (self.rows + 7) >> 3
        self.lstride = self.sbc + int(rng.integers(0, 2))
        sent = 0x5A5 & ((1 << depth) - 1) if depth > 8 else 0x5A
        self.planes = []
        for p in range(3):
            sh, sv = (self.ss_h, self.ss_v) if p else (0, 0)
            W, H = area(sh, self.cols), area(sv, self.rows)
            a = np.full((H + 2 * MARGIN, W + 2 * MARGIN + pad), sent, sdtype(depth))
            a[MARGIN:MARGIN + H, MARGIN:MARGIN + W] = content(rng, depth, H, W)
            self.planes.append(a)
        rec = decoder_records if kind == "decoder" else arbitrary_records
        self.lflvl = rec(rng, self.ss_h, self.ss_v, self.cols, self.rows, self.lstride)
        self.lim, self.mblim = luts(int(rng.integers(0, 8)) if sharp is None else sharp)

    def ptrs(self, planes):
        return [p.ctypes.data + MARGIN * p.strides[0] + MARGIN * p.itemsize for p in planes]

    def strides(self):
        return self.planes[0].strides[0], self.planes[1].strides[0]


def _frame(L, name, f, order, planes=None):
    fn = getattr(L, name)
    fn.argtypes = [C.c_int] * 5 + [C.c_void_p, C.c_ssize_t, C.c_ssize_t, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int]
    out = [p.copy() for p in (planes or f.planes)]
    arr = (C.c_void_p * 3)(*f.ptrs(out))
    rec = np.ascontiguousarray(f.lflvl)
    ls_y, ls_uv = f.strides()
    assert fn(f.depth, f.ss_h, f.ss_v, f.width, f.height, arr, ls_y, ls_uv, rec.ctypes.data, f.lstride, f.lim.ctypes.data,
              f.mblim.ctypes.data, order) == 0
    return out


def orc_frame(f, order=0):
    """the checker: order 0 raster (the entry's result), k >= 1 wavefront c + k r, -1 frame-wide columns then rows"""
    return _frame(cl.oracle(), "orc_vp9_lf_frame", f, order)


def ref_frame(f, k=0):
    """the reference driver: k = 0 raster order, k >= 1 wavefront c + k r"""
    return _frame(ref(), "ffref_vp9_lf_frame", f, k)


def frame_case(name):
    """the frames behind tests/golden/vp9lf_hashes.txt: name = '<depth>-<fmt>-<kind>'"""
    d, fmt, kind = name.split("-")
    depth = int(d)
    seed = 700 + 10 * DEPTHS.index(depth) + list(FORMATS).index(fmt) + (0 if kind == "decoder" else 50)
    size = {"decoder": (328, 203), "arbitrary": (264, 136)}[kind]
    return Frame(seed, depth, fmt, *size, kind=kind)


FIXTURE_NAMES = [f"{d}-{fmt}-{kind}" for d in DEPTHS for fmt in FORMATS for kind in ("decoder", "arbitrary")]


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


# ---------------------------------------------------------------- members
MEMBERS = [("loop_filter_8", (wd, d)) for wd in range(3) for d in range(2)] + [("loop_filter_16", (d,)) for d in range(2)] + \
          [("loop_filter_mix2", (a, b, d)) for a in range(2) for b in range(2) for d in range(2)]    # index = orc / ffref member number


def member_calls(seed, depth, per=6):
    """(member index, E, I, H, block [32, 32] with the edge's q0 of line 0 at (16, 16)) for all 16 members; E / I / H over the byte range
    (mix2: two different bytes per half), the content a step between two noisy flat halves so every branch is taken"""
    rng = np.random.default_rng(seed)
    sh = depth - 8
    for m in range(16):
        dir = m & 1
        for it in range(per):
            if it % 3 == 2:
                E, I, H = (int(v) for v in rng.integers(0, 256, 3))
            else:
                E, I, H = int(rng.integers(0, 80)), int(rng.integers(0, 20)), int(rng.integers(0, 16))
            if m >= 8:
                E |= int(rng.integers(0, 256)) << 8
                I |= int(rng.integers(0, 64)) << 8
                H |= int(rng.integers(0, 64)) << 8
            amp = [0, 1, 3, 40][it % 4] << sh
            blk = int(rng.integers(40, 200)) << sh
            b = np.full((32, 32), blk, np.int64)
            step = int(rng.integers(-10, 11)) << sh
            if dir == 0:
                b[:, 16:] += step
            else:
                b[16:, :] += step
            b += rng.integers(0, amp + 1, b.shape)
            yield m, E, I, H, np.clip(b, 0, (1 << depth) - 1).astype(sdtype(depth))


def run_member(L, name, depth, call):
    m, E, I, H, blk = call
    f = getattr(L, name)
    f.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_ssize_t, C.c_int, C.c_int, C.c_int]
    d = blk.copy()
    assert f(depth, m, d.ctypes.data + 16 * d.strides[0] + 16 * d.itemsize, d.strides[0], E, I, H) == 0
    return d


def run_members(L, name, seed, depth):
    return [run_member(L, name, depth, c) for c in member_calls(seed, depth)]
