"""CPU replay of the tensor-core horizontal pass (csrc/sws_mma.cuh): the library's operand tables (b200_sws_mma_probe) are run through a
lane-by-lane model of mma.sync.m16n8k32 (PTX ISA fragment layouts: A row = lane/4 (+8), k = 4*(lane%4)+b (+16); B k likewise, n = lane/4;
D row = lane/4 (+8), columns 2*(lane%4), +1) with the kernel's addressing, and compared with hScale8To15_c (libswscale/swscale.c:128-142)
computed directly.  Filter banks: the library's own (every scaler / ratio of tests/cases.py) and random ones."""
import ctypes as C
import numpy as np
import pytest
import cpulibs as cl
from cases import SWS_PATH_CASES
from ffmpeg_b200._lib import lib


def mma_tables(coef, pos):
    n, size = coef.shape
    L = lib()
    ng = (n + 7) // 8
    ginfo = np.zeros((ng + 1, 2), np.int32)
    pitch = np.zeros(2, np.int32)
    words = L.b200_sws_mma_probe(cl.ptr(coef, cl.i16p), cl.ptr(pos, cl.i32p), n, size, cl.ptr(ginfo, cl.i32p), ginfo.size, None, 0, cl.ptr(pitch, cl.i32p))
    assert words > 0 and words % 128 == 0
    bfrag = np.zeros(words, np.uint32)
    assert L.b200_sws_mma_probe(cl.ptr(coef, cl.i16p), cl.ptr(pos, cl.i32p), n, size, None, 0,
                                bfrag.ctypes.data_as(C.POINTER(C.c_uint32)), words, None) == words
    return ginfo, bfrag.reshape(-1, 32, 4), pitch


def hscale_direct(src, coef, pos):
    n, size = coef.shape
    idx = pos[:, None] + np.arange(size)[None, :]
    acc = (src[:, idx].astype(np.int64) * coef[None].astype(np.int64)).sum(axis=2)
    return np.minimum(acc >> 7, 32767).astype(np.int16)


def replay_tiles(src, coef, pos, tile_groups):
    """The kernel's data flow: per tile the staged window [c0, c0 + 16 * nseg) (zeros beyond srcW), per group the chunked MMAs."""
    rows, srcW = src.shape
    n = coef.shape[0]
    ginfo, bfrag, pitch = mma_tables(coef, pos)
    ng = (n + 7) // 8
    SP = int(pitch[0] if tile_groups == 16 else pitch[1])
    assert SP % 32 == 16                                                      # 16 x odd: conflict-free fragment loads
    out = np.zeros((rows, ng * 8), np.int64)
    rpad = (rows + 15) & ~15
    for G0 in range(0, ng, tile_groups):
        gs = range(G0, min(G0 + tile_groups, ng))
        s = min(int(ginfo[G, 0]) for G in gs)
        e = max(int(ginfo[G, 0]) + 32 * int(ginfo[G + 1, 1] - ginfo[G, 1]) for G in gs)
        c0 = s & ~15
        nseg = (e - c0 + 15) >> 4
        assert nseg * 16 <= SP
        st = np.zeros((rpad, SP), np.uint8)
        w = max(0, min(srcW, c0 + 16 * nseg) - c0)
        st[:rows, :w] = src[:, c0:c0 + w]
        for G in gs:
            kstart, ch0 = int(ginfo[G, 0]), int(ginfo[G, 1])
            nch = int(ginfo[G + 1, 1]) - ch0
            assert kstart % 4 == 0
            krel = kstart - c0
            for rb in range(rpad // 16):
                hi = np.zeros((16, 8), np.int64); lo = np.zeros((16, 8), np.int64)
                for c in range(nch):
                    A = st[rb * 16:rb * 16 + 16, krel + 32 * c:krel + 32 * c + 32].astype(np.int64)      # 16 x 32 as the fragments address it
                    Bh = np.zeros((32, 8), np.int64); Bl = np.zeros((32, 8), np.int64)
                    for lane in range(32):
                        g, t = lane >> 2, lane & 3
                        wv = bfrag[ch0 + c, lane]
                        for half in range(2):
                            for b in range(4):
                                k = 16 * half + 4 * t + b
                                hb = (int(wv[half]) >> (8 * b)) & 0xff
                                Bh[k, g] = hb - 256 if hb >= 128 else hb                                  # .s8
                                Bl[k, g] = (int(wv[2 + half]) >> (8 * b)) & 0xff                          # .u8
                    hi += A @ Bh
                    lo += A @ Bl
                out[rb * 16:rb * 16 + 16, G * 8:G * 8 + 8][:max(0, min(16, rows - rb * 16))] = \
                    np.minimum((hi * 256 + lo) >> 7, 32767)[:max(0, min(16, rows - rb * 16))]
    return out[:, :n].astype(np.int16)


@pytest.mark.parametrize("srcW,dstW,flags", [(3840, 1920, 4 | 0x40000 | 0x80000), (1920, 1280, 4 | 0x40000 | 0x80000), (352, 200, 4 | 0x40000 | 0x80000),
                                             (640, 1280, 2), (1000, 96, 0x200 | 0x40000 | 0x80000), (720, 704, 0x20), (3840, 1280, 0x400 | 0x80000)])
def test_library_banks_replay(srcW, dstW, flags):
    rng = np.random.default_rng(srcW * 7 + dstW)
    L = lib()
    info = np.zeros(16, np.int32)
    assert L.b200_sws_plan_probe(srcW, 64, dstW, 64, flags, 0, None, None, 0, cl.ptr(info, cl.i32p)) >= 0
    for which, sw, n in ((0, srcW, dstW), (1, int(info[4]), int(info[6]))):
        size = int(info[which])
        f = np.zeros(n * size, np.int16); p = np.zeros(n, np.int32)
        assert L.b200_sws_plan_probe(srcW, 64, dstW, 64, flags, which, cl.ptr(f, cl.i16p), cl.ptr(p, cl.i32p), n, None) == n
        coef = f[:n * size].reshape(n, size).copy(); pos = p[:n].copy()
        assert int(pos.min()) >= 0 and int((pos + size).max()) <= sw
        src = rng.integers(0, 256, (37, sw), dtype=np.uint8)
        ref = hscale_direct(src, coef, pos)
        for tg in (16, 8):
            assert np.array_equal(replay_tiles(src, coef, pos, tg), ref), (which, tg)


MT_W, MT_TPB, MT_CPB, MT_HDR = 128, 128 * 4 + 32, 128 * 2 + 32, 16      # sws_mma.cuh


def case_banks(row, dest):
    """info (as b200_sws_info) and the four filter banks {0: hLum, 1: hChr, 2: vLum, 3: vChr} as (coef, pos) of a SWS_PATH_CASES row, from the
    oracle (whose tables test_host_filter_tables_match_oracle pins to the library's; this also covers `param` and `src_filter`)"""
    w, h, dw, dh = row["geom"]
    O = cl.oracle()
    fmt = 0 if dest == "yuv420p" else cl.PACKED_RGB_FORMATS[dest]
    ctx = cl._open_filters(O, "orc", row.get("src_fmt", 0), w, h, 0, fmt, dw, dh, 0, row["flags"], 1, (row.get("src_filter"), None), row.get("param"))
    assert ctx
    info = np.zeros(16, np.int32)
    O.orc_sws_info(ctx, cl.ptr(info, cl.i32p))
    banks = {}
    for which in range(4):
        size, n = int(info[which]), [dw, int(info[6]), dh, int(info[7])][which]
        f, p = np.zeros(n * size, np.int16), np.zeros(n, np.int32)
        O.orc_sws_get_filter(ctx, which, cl.ptr(f, cl.i16p), cl.ptr(p, cl.i32p), n)
        banks[which] = (f.reshape(n, size), p)
    O.orc_sws_close(ctx)
    return info, banks


def rows_needed(bank, srcH, dstH, TR):
    """fused_rows_needed (csrc/sws.cu): staged lines of the tallest tile of TR output lines, -1 when a tile's windows are not nested"""
    coef, pos = bank
    size, mx = coef.shape[1], 0
    win = [(min(max(max(1 - size, int(p)), 0), srcH - 1), min(max(max(1 - size, int(p)) + size - 1, 0), srcH - 1)) for p in pos]
    for dy0 in range(0, dstH, TR):
        ra, rb = win[dy0][0], win[min(dy0 + TR, dstH) - 1][1]
        if rb < ra or any(a < ra or b > rb for a, b in win[dy0:dy0 + TR]):
            return -1
        mx = max(mx, rb - ra + 1)
    return mx


def mma_tiles(row, dest):
    """The tile heights launch_batch / launch_planar3 pick for the tensor-core kernels at the row's geometry: [(TR, shared bytes)] for the
    packed-RGB kernel or for the luma and chroma plane kernels; (None, None) where no height fits (the other kernels take over)"""
    info, banks = case_banks(row, dest)
    w, h, dw, dh = row["geom"]
    csh = int(info[5])
    pitch = {k: mma_tables(*banks[k])[2] for k in (0, 1)}
    out = []
    if dest == "yuv420p":
        for k, sh, dhh in ((0, h, dh), (1, csh, int(info[7]))):
            SP = int(pitch[k][0])
            best, pick = 1e30, (None, None)
            for TR in range(32, 7, -1):
                r = rows_needed(banks[k + 2], sh, dhh, TR)
                sm = MT_HDR + ((r + 15) & ~15) * (SP + MT_TPB)
                if r <= 0 or sm > 112 * 1024:
                    continue
                cost = ((r + 15) >> 4) / TR * (1.0 + (0.15 if sm > 56 * 1024 else 0) + (0.15 if sm > 75 * 1024 else 0))
                if cost < best - 1e-9:
                    best, pick = cost, (TR, sm)
            out.append(pick)
        return out

    def need(TR):
        rl, rc = rows_needed(banks[2], h, dh, TR), rows_needed(banks[3], csh, dh, TR)
        return (rl, rc), MT_HDR + ((rl + 15) & ~15) * (int(pitch[0][0]) + MT_TPB) + 2 * ((rc + 15) & ~15) * (int(pitch[1][1]) + MT_CPB)
    (rl, rc), sm = need(16)
    if rl > 0 and rc > 0 and sm <= 80 * 1024:
        return [(16, sm)]
    best, pick = 1e30, (None, None)
    for TR in range(32, 7, -1):
        (rl, rc), sm = need(TR)
        if rl <= 0 or rc <= 0 or sm > 112 * 1024:
            continue
        cost = (((rl + 15) >> 4) + ((rc + 15) >> 4)) / TR * (1.0 + (0.15 if sm > 56 * 1024 else 0) + (0.15 if sm > 75 * 1024 else 0))
        if cost < best - 1e-9:
            best, pick = cost, (TR, sm)
    return [pick]


def _groups_nch(row):
    ginfo = mma_tables(*case_banks(row, "yuv420p")[1][0])[0]
    return np.diff(ginfo[:, 1])


def _clamps(row):
    """the luma horizontal pass over the `extremes` input, before hScale8To15_c's clamp, goes above 32767 and below 0"""
    coef, pos = case_banks(row, "yuv420p")[1][0]
    y = cl.yuv_frame(*row["geom"][:2], 0, "extremes")[0]
    acc = (y[:, pos[:, None] + np.arange(coef.shape[1])[None, :]].astype(np.int64) * coef[None].astype(np.int64)).sum(axis=2) >> 7
    return int(acc.max()) > 32767 and int(acc.min()) < 0


def _tile(row, dest, plane=0):
    return mma_tiles(row, dest)[plane][0] or 0


# What a SWS_PATH_CASES row says it reaches, checked on the host tables (chunks and tiles as csrc/sws.cu and sws_mma.cuh derive them)
REACHES = {
    "nch=1": lambda r: _groups_nch(r).max() == 1,                                           # every group one 32-column chunk
    "nch=2": lambda r: _groups_nch(r).max() == 2,                                           # the two-chunk instantiation
    "nch>=3": lambda r: _groups_nch(r).max() >= 3,                                          # the general chunk loop (NCH == 0)
    "up2x": lambda r: r["geom"][2] >= 2 * r["geom"][0],
    "dstH%TR": lambda r: all(_tile(r, d) and r["geom"][3] % _tile(r, d) for d in ("rgb24", "yuv420p")),
    "taps>16": lambda r: case_banks(r, "rgb24")[0][0] > 16,                                 # no CUDA-core fused kernel
    "smem>75K": lambda r: (mma_tiles(r, "rgb24")[0][1] or 0) > 75 * 1024,
    "no tile fits": lambda r: mma_tiles(r, "rgb24")[0][0] is None and mma_tiles(r, "yuv420p")[0][0] is None,
    "vfs=1": lambda r: case_banks(r, "yuv420p")[0][2] == 1,
    "hscaled": lambda r: case_banks(r, "yuv420p")[0][0] > 1,
    "2-tap": lambda r: 2 in [int(x) for x in case_banks(r, "yuv420p")[0][:4]],
    "srcW%16": lambda r: r["geom"][0] % 16 != 0,
    "odd chroma": lambda r: case_banks(r, "yuv420p")[0][4] % 2 == 1 and case_banks(r, "yuv420p")[0][5] % 2 == 1,
    "srcW<16": lambda r: r["geom"][0] < 16,
    "bicublin": lambda r: case_banks(r, "yuv420p")[0][1] < case_banks(r, "yuv420p")[0][0],
    "one tile of 2 groups": lambda r: (r["geom"][2] + 7) // 8 == 2,
    "second tile of 2 groups": lambda r: (r["geom"][2] + 7) // 8 % 16 == 2 and r["geom"][2] > 128,
    "partial column tile": lambda r: r["geom"][2] % 128 != 0,
    "ngc<8": lambda r: (case_banks(r, "rgb24")[0][6] + 7) // 8 - 8 * ((r["geom"][2] + 127) // 128 - 1) < 8,    # chroma groups of the last RGB tile
    "rgb row tile of 1": lambda r: _tile(r, "rgb24") and r["geom"][3] % _tile(r, "rgb24") == 1,
    "luma row tile of 1": lambda r: _tile(r, "yuv420p") and r["geom"][3] % _tile(r, "yuv420p") == 1,
    "chroma dstW%8": lambda r: r["geom"][2] % 8 == 0 and case_banks(r, "yuv420p")[0][6] % 8 != 0,                # plane kernels need dstW % 8
    "coef>16384": lambda r: int(case_banks(r, "yuv420p")[1][0][0].max()) > 16384,          # high byte of the split above 63
    "clamp": _clamps,
    "nv": lambda r: r.get("src_fmt", 0) in (23, 24),
}


@pytest.mark.parametrize("row", SWS_PATH_CASES, ids=lambda r: "x".join(map(str, r["geom"])) + f"-{r['flags']:x}-{r.get('src_fmt', 0)}")
def test_path_cases_reach_their_code(row):
    for what in row["reaches"]:
        assert REACHES[what](row), what


def test_path_cases_cover_chunks_and_kernels():
    """the rows between them take groups of one, two and three or more chunks, and expect each of the three kernels for every destination"""
    top = {int(_groups_nch(r).max()) for r in SWS_PATH_CASES}
    assert {1, 2} <= top and max(top) >= 3, top
    for dest in ("rgb24", "bgra", "yuv420p"):
        seen = {b for r in SWS_PATH_CASES for p in r["paths"].get(dest, ()) for b in (1, 2, 4) if p & b}
        assert seen == {1, 2, 4}, (dest, seen)


@pytest.mark.parametrize("row", SWS_PATH_CASES, ids=lambda r: "x".join(map(str, r["geom"])) + f"-{r['flags']:x}-{r.get('src_fmt', 0)}")
def test_path_case_banks_replay(row):
    """the library's operand tables of every SWS_PATH_CASES bank, through the lane-by-lane replay, against hScale8To15_c"""
    info, banks = case_banks(row, "yuv420p")
    rng = np.random.default_rng(sum(row["geom"]))
    for which, sw in ((0, row["geom"][0]), (1, int(info[4]))):
        coef, pos = banks[which]
        src = rng.integers(0, 256, (17, sw), dtype=np.uint8)
        ref = hscale_direct(src, coef, pos)
        for tg in (16, 8):
            assert np.array_equal(replay_tiles(src, coef, pos, tg), ref), (which, tg)


def test_random_banks_replay():
    rng = np.random.default_rng(5)
    for _ in range(12):
        n = int(rng.integers(9, 300)); size = int(rng.integers(1, 40))
        step = float(rng.uniform(0.3, 6.0))
        pos = np.floor(np.arange(n) * step + rng.integers(0, 3, n)).astype(np.int32)
        srcW = int(pos.max()) + size + int(rng.integers(0, 20))
        coef = rng.integers(-16384, 16384, (n, size)).astype(np.int16)
        src = rng.integers(0, 256, (21, srcW), dtype=np.uint8)
        ref = hscale_direct(src, coef, pos)
        for tg in (16, 8):
            assert np.array_equal(replay_tiles(src, coef, pos, tg), ref)
