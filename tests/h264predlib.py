"""Test infrastructure for H.264 intra prediction (H264PredContext): the seeded case generator, runners of the checker
(oracle/liboracle.so, orc_h264_pred) and of the compiled reference (oracle/_ref/libffref_h264pred.so, built by oracle/ref/Makefile),
and RefCheck, which keeps the reference's results as digests in tests/golden/h264pred_ref_digests.json for machines without the
reference."""
import ctypes as C
import os

import numpy as np

import cpulibs as cl

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_LIB = "libffref_h264pred"
REF_DIGESTS = os.path.join(ROOT, "tests", "golden", "h264pred_ref_digests.json")


def have_ref():
    return cl.have_ref(REF_LIB)


def ref():
    return cl.ref_lib(REF_LIB)


def RefCheck():
    return cl.RefCheck(REF_DIGESTS, REF_LIB)


# ---------------------------------------------------------------- H.264 intra prediction (libavcodec/h264pred_template.c)
PRED_CELL = 32        # one op per 32 x 32 cell, block at (8, 8): the row above (to x + 15 with pred8x8l's top-right) and the column left stay inside
SCAN8_XY = [(0, 0), (1, 0), (0, 1), (1, 1), (2, 0), (3, 0), (2, 1), (3, 1), (0, 2), (1, 2), (0, 3), (1, 3), (2, 2), (3, 2), (2, 3), (3, 3)]
# batched table -> (orc_h264_pred / ffref_h264_pred table, chroma_format_idc to use; None = the case's)
PRED_TABLE_MAP = {0: (0, None), 1: (1, None), 2: (2, 1), 3: (2, 2), 4: (3, None)}
ADD_TABLE_MAP = {0: (4, None), 1: (5, None), 2: (6, None), 3: (7, 1), 4: (7, 2), 5: (8, None)}
PRED_CLASSES = ("noise", "flat", "zero", "max", "gradient", "split")


def h264pred_combos(idc, add):
    """every (batched table, mode, flags) the batch entry has for chroma_format_idc: the chroma table is 8x8 for idc <= 1, else 8x16"""
    if add:
        c = 4 if idc > 1 else 3
        return ([(0, m, 0) for m in (0, 1)] + [(1, m, 0) for m in (0, 1)] + [(2, m, f) for m in (0, 1) for f in range(4)] +
                [(c, m, 0) for m in (1, 2)] + [(5, m, 0) for m in (1, 2)])
    c = 3 if idc > 1 else 2
    return ([(0, m, f) for m in range(12) for f in (0, 2)] + [(1, m, f) for m in range(12) for f in range(4)] +
            [(c, m, 0) for m in range(11)] + [(4, m, 0) for m in range(7)])


def h264pred_case(seed, n, depth, idc=1, add=False, cols=16):
    """(pic uint8 / uint16 [rows*32, cols*32], kinds uint8 [n], flags uint8 [n], off int64 [n] (bytes), coef int16 / int32 [n, 256],
    coef_off int64 [n] (coefficients)): n independent ops cycling through every (table, mode, flags), each combination over the content
    classes in turn (uniform noise, flat, all 0, all max, gentle gradients, a maximal top row over a zero left column or the reverse,
    which drives the plane forms into both clips); coefficients over the whole int16 (8 bit) / int32 range, so the add forms wrap"""
    rng = np.random.default_rng(seed)
    combos = h264pred_combos(idc, add)
    maxv = (1 << depth) - 1
    rows = (n + cols - 1) // cols
    pic = np.zeros((rows * PRED_CELL, cols * PRED_CELL), np.uint8 if depth == 8 else np.uint16)
    bps = pic.itemsize
    for i in range(rows * cols):
        y, x = (i // cols) * PRED_CELL, (i % cols) * PRED_CELL
        cls = (i // len(combos)) % len(PRED_CLASSES)
        S = PRED_CELL
        if cls == 0:
            c = rng.integers(0, maxv + 1, (S, S))
        elif cls == 1:
            c = np.full((S, S), int(rng.integers(0, maxv + 1)))
        elif cls == 2:
            c = np.zeros((S, S), np.int64)
        elif cls == 3:
            c = np.full((S, S), maxv)
        elif cls == 4:
            step = 1 << (depth - 8)
            gy, gx = (int(v) * step for v in rng.integers(-4, 5, 2))
            c = int(rng.integers(0, maxv + 1)) + gy * np.arange(S)[:, None] + gx * np.arange(S)[None, :] + rng.integers(0, step + 1, (S, S))
        else:
            hi, lo = (maxv, 0) if rng.random() < 0.5 else (0, maxv)
            c = np.full((S, S), lo)
            c[:8, :] = hi
            c[:, :8] = lo
        pic[y:y + S, x:x + S] = np.clip(c, 0, maxv)
    i = np.arange(n)
    kinds = np.array([(combos[k % len(combos)][0] << 4) | combos[k % len(combos)][1] for k in range(n)], np.uint8)
    flags = np.array([combos[k % len(combos)][2] for k in range(n)], np.uint8)
    off = (((i // cols) * PRED_CELL + 8) * pic.strides[0] + ((i % cols) * PRED_CELL + 8) * bps).astype(np.int64)
    if depth == 8:
        coef = rng.integers(-32768, 32768, (n, 256)).astype(np.int16)
    else:
        coef = rng.integers(-(1 << 31), 1 << 31, (n, 256)).astype(np.int32)
    return pic, kinds, flags, off, coef, (i * 256).astype(np.int64)


def h264pred_fixture_case(depth, idc, add):
    """the seeded batch behind each line of tests/golden/h264pred_hashes.txt: every (table, mode, flags) over every content class, twice"""
    n = 2 * len(PRED_CLASSES) * len(h264pred_combos(idc, add))
    return h264pred_case(800 + 10 * depth + 2 * idc + add, n, depth, idc, add)


def pred_block_offsets(stride, bps, n=16):
    """the decoder's block_offset table (h264_slice.c:554-563) for the given line size: entry i = scan8 position i"""
    return np.array([4 * x * bps + 4 * y * stride for (x, y) in SCAN8_XY[:n]], np.int32)


def _h264pred_run(L, name, depth, idc, add, pic, kinds, flags, off, coef, coef_off):
    f = getattr(L, name)
    f.argtypes = [C.c_int] * 4 + [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_ssize_t]
    out, cf = pic.copy(), coef.copy()
    bps, stride = pic.itemsize, pic.strides[0]
    bo = pred_block_offsets(stride, bps)
    tr = np.zeros(4, pic.dtype)
    for i in range(len(kinds)):
        t, m = int(kinds[i]) >> 4, int(kinds[i]) & 15
        table, tidc = (ADD_TABLE_MAP if add else PRED_TABLE_MAP).get(t, (None, None))
        if table is None:
            continue
        src = out.ctypes.data + int(off[i])
        topright = None
        if not add and t == 0:
            if flags[i] & 2:
                topright = src + 4 * bps - stride
            else:
                tr[:] = np.frombuffer(C.string_at(src + 3 * bps - stride, bps), pic.dtype)[0]
                topright = tr.ctypes.data
        r = f(depth, tidc if tidc is not None else idc, table, m, src, topright, int(flags[i]),
              cf.ctypes.data + int(coef_off[i]) * cf.itemsize if add else None, bo.ctypes.data, stride)
        assert r in (0, -1)
    return out, cf


def orc_h264pred(depth, idc, add, *case):
    return _h264pred_run(cl.oracle(), "orc_h264_pred", depth, idc, add, *case)


def ref_h264pred(depth, idc, add, *case):
    return _h264pred_run(ref(), "ffref_h264_pred", depth, idc, add, *case)


