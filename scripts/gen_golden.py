#!/usr/bin/env python
"""Generate tests/golden/*.npz from the UNMODIFIED reference (oracle/_ref/libffref.so, built by oracle/ref/Makefile
from /root/reference).  Run in the build container only; the fixtures travel to the GPU box.

    python scripts/gen_golden.py

Every fixture stores the inputs (or the seed + a sha256 of the inputs, for the larger cases) and the reference's
outputs, so the tests need neither /root/reference nor oracle/_ref at run time.
"""
import ctypes as C
import hashlib
import os
import sys
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import cpulibs as cl  # noqa: E402
import h264predlib as hp  # noqa: E402
import hevcmclib as hm  # noqa: E402
from cases import SWS_SMALL_CASES, SWS_HASH_CASES, idct_blocks  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def gen_sws():
    d = {}
    for i, (w, h, dw, dh, fl, kind) in enumerate(SWS_SMALL_CASES):
        y, u, v = cl.yuv_frame(w, h, 100 + i, kind)
        out = cl.ref_sws(w, h, dw, dh, fl, y, u, v)
        assert out is not None, (w, h, dw, dh, fl)
        d[f"c{i}_y"], d[f"c{i}_u"], d[f"c{i}_v"], d[f"c{i}_rgb"] = y, u, v, out
    np.savez_compressed(os.path.join(OUT, "sws_small.npz"), **d)
    lines = []
    for i, (w, h, dw, dh, fl, kind) in enumerate(SWS_HASH_CASES):
        y, u, v = cl.yuv_frame(w, h, 200 + i, kind)
        out = cl.ref_sws(w, h, dw, dh, fl, y, u, v)
        lines.append(f"{i} {w} {h} {dw} {dh} {fl} {kind} {sha(np.concatenate([y.ravel(), u.ravel(), v.ravel()]))} {sha(out)}")
    open(os.path.join(OUT, "sws_hashes.txt"), "w").write("\n".join(lines) + "\n")
    # colourspace variants on one small frame
    d = {}
    y, u, v = cl.yuv_frame(64, 48, 300, "random")
    d["y"], d["u"], d["v"] = y, u, v
    FATE = cl.SWS_BICUBIC | cl.SWS_ACCURATE_RND | cl.SWS_BITEXACT
    for j, cs in enumerate([(1, 0, 1, 0, 0, 1 << 16, 1 << 16), (5, 1, 5, 1, 0, 1 << 16, 1 << 16),
                            (9, 0, 9, 0, 3000, 70000, 80000), (7, 1, 7, 0, -2000, 60000, 50000)]):
        for k, fl in enumerate([FATE, cl.SWS_BICUBIC]):
            d[f"cs{j}_{k}"] = cl.ref_sws(64, 48, 64, 48, fl, y, u, v, colorspace=cs)
            d[f"cs{j}_{k}_s"] = cl.ref_sws(64, 48, 96, 80, fl, y, u, v, colorspace=cs)
    np.savez_compressed(os.path.join(OUT, "sws_colorspace.npz"), **d)


def gen_sws_formats():
    """bgr24 / rgba / bgra / argb / abgr outputs of the reference for SWS_FORMAT_CASES, as sha256 lines."""
    from cases import SWS_FORMAT_CASES
    lines = []
    for name, fmt in cl.PACKED_RGB_FORMATS.items():
        if name == "rgb24":
            continue
        for i, (w, h, dw, dh, fl, kind) in enumerate(SWS_FORMAT_CASES):
            y, u, v = cl.yuv_frame(w, h, 500 + i, kind)
            out = cl.ref_sws(w, h, dw, dh, fl, y, u, v, fmt=fmt)
            assert out is not None and out.shape == (dh, dw * cl.fmt_bpp(fmt))
            lines.append(f"{name} {i} {w} {h} {dw} {dh} {fl} {kind} {sha(out)}")
    open(os.path.join(OUT, "sws_format_hashes.txt"), "w").write("\n".join(lines) + "\n")


def gen_sws_planar():
    """yuv420p -> yuv420p outputs of the reference for SWS_PLANAR_CASES (sha256 of Y, U, V planes concatenated)."""
    from cases import SWS_PLANAR_CASES
    lines = []
    for i, (w, h, dw, dh, fl, kind) in enumerate(SWS_PLANAR_CASES):
        y, u, v = cl.yuv_frame(w, h, 600 + i, kind)
        out = cl.ref_sws_planar(w, h, dw, dh, fl, y, u, v)
        assert out is not None
        lines.append(f"{i} {w} {h} {dw} {dh} {fl} {kind} {sha(np.concatenate([p.ravel() for p in out]))}")
    open(os.path.join(OUT, "sws_planar_hashes.txt"), "w").write("\n".join(lines) + "\n")


def gen_sws_range():
    """yuv420p -> yuv420p with range conversion: the reference's outputs for SWS_RANGE_CASES."""
    from cases import SWS_RANGE_CASES
    lines = []
    for i, (w, h, dw, dh, fl, kind, ranges, details) in enumerate(SWS_RANGE_CASES):
        y, u, v = cl.yuv_frame(w, h, 1200 + i, kind)
        out = cl.ref_sws_planar(w, h, dw, dh, fl, y, u, v, ranges=ranges, details=details)
        lines.append(f"{i} {w} {h} {dw} {dh} {fl} {kind} {sha(np.concatenate([p.ravel() for p in out]))}")
    open(os.path.join(OUT, "sws_range_hashes.txt"), "w").write("\n".join(lines) + "\n")


def gen_unquant():
    """mpegvideo inverse quantisers: the reference's outputs for unquant_case(seed, variant)."""
    d = {}
    for variant in range(7):
        for seed in (11, 12):
            cfg, blocks, blk_n, q, last = cl.unquant_case(seed * 7 + variant, variant, nblocks=48)
            d[f"v{variant}_s{seed}"] = cl.ref_unquant(variant, cfg, blocks, blk_n, q, last)
    np.savez_compressed(os.path.join(OUT, "unquant.npz"), **d)


def gen_fdsp():
    """AVFloatDSPContext C functions: the reference's outputs for fdsp_case(seed, op, length)."""
    d = {}
    for op in range(12):
        for length in (16, 100, 1024):
            r, a = cl.ref_fdsp(op, *cl.fdsp_case(40 + op, op, length), length)
            d[f"op{op}_n{length}"] = r
            if op == 8:
                d[f"op{op}_n{length}_v2"] = a
    np.savez_compressed(os.path.join(OUT, "fdsp.npz"), **d)


def gen_idct_hbd():
    """10 / 12 bit simple IDCT: the reference's outputs (through ff_idctdsp_init) for idct_hbd_blocks(seed, depth, 60)."""
    d = {}
    for depth in (10, 12):
        blocks = cl.idct_hbd_blocks(70 + depth, depth, 60)
        dest = np.random.default_rng(depth).integers(0, 1 << depth, (8, 60 * 8), dtype=np.uint16)
        for kind in (0, 1, 2):
            b, o = cl.ref_idct_hbd(depth, kind, blocks, dest, dest.strides[0])
            d[f"d{depth}_k{kind}"] = b if kind == 0 else o
    np.savez_compressed(os.path.join(OUT, "idct_hbd.npz"), **d)


def gen_sws_rgbsrc():
    """packed RGB sources: the reference's outputs for SWS_RGBSRC_CASES (sha256; yuv420p planes concatenated / the rgb24 picture)."""
    from cases import SWS_RGBSRC_CASES
    lines = []
    for i, (w, h, dw, dh, fl, kind) in enumerate(SWS_RGBSRC_CASES):
        for name, sf in cl.PACKED_RGB_FORMATS.items():
            src = cl.rgb_frame(w, h, 2000 + i, cl.fmt_bpp(sf), kind)
            for ranges in ((0, 0), (0, 1)):
                pl = cl.ref_sws_planar(w, h, dw, dh, fl, src, src, src, src_fmt=sf, ranges=ranges)
                lines.append(f"{i} {name} yuv420p {ranges[1]} {sha(np.concatenate([p.ravel() for p in pl]))}")
            if (w, h) != (dw, dh) and cl.fmt_bpp(sf) == 3:
                lines.append(f"{i} {name} rgb24 0 {sha(cl.ref_sws(w, h, dw, dh, fl, src, src, src, fmt=cl.PIX_FMT_RGB24, src_fmt=sf))}")
    open(os.path.join(OUT, "sws_rgbsrc_hashes.txt"), "w").write("\n".join(lines) + "\n")


def gen_tx_pfa():
    """compound 15 x M float MDCT (Opus CELT sizes), then 7 x M and 9 x M: the reference's outputs, inverse and forward, two scales."""
    R = cl.ref()
    d = {}
    rng = np.random.default_rng(77)
    for n in (120, 240, 480, 960, 112, 448, 144, 576):
        for inv in (1, 0):
            x = (rng.random((2, n if inv else 2 * n), dtype=np.float32) * 2 - 1).astype(np.float32)
            d[f"in_{n}_{inv}"] = x
            for j, sc in enumerate((1.0 / n, -1.0)):
                h = R.ffref_tx_open(1, inv, n, sc, 0)
                out = np.zeros((2, n), np.float32)
                R.ffref_tx_run(h, out.ctypes.data, x.ctypes.data, 4, 2, out.strides[0], x.strides[0])
                R.ffref_tx_close(h)
                d[f"out_{n}_{inv}_{j}"] = out
    np.savez_compressed(os.path.join(OUT, "tx_pfa.npz"), **d)


PFA_FFT_SIZES = (6, 12, 96, 10, 160, 14, 224, 18, 288, 30, 120, 960, 1920)


def gen_tx_pfa_fft():
    """compound complex FFTs (fft_pfa over fft{3,5,7,9,15}_ns x 2^k; checkasm av_tx.c lengths 120 / 960 / 1920): the reference's
    outputs in both directions, plus the codelet tree it reports for each length (ffref_tx_describe)."""
    R = cl.ref()
    R.ffref_tx_describe.argtypes = [C.c_void_p, C.c_char_p, C.c_int]
    d = {}
    rng = np.random.default_rng(78)
    trees = []
    for n in PFA_FFT_SIZES:
        x = (rng.random((2, 2 * n), dtype=np.float32) * 2 - 1).astype(np.float32)
        d[f"in_{n}"] = x
        for inv in (0, 1):
            h = R.ffref_tx_open(0, inv, n, 1.0, 0)
            buf = C.create_string_buffer(2048)
            R.ffref_tx_describe(h, buf, 2048)
            trees.append(f"{n} {inv}: " + buf.value.decode().strip().replace("\n", " | "))
            out = np.zeros((2, 2 * n), np.float32)
            R.ffref_tx_run(h, out.ctypes.data, x.ctypes.data, 8, 2, out.strides[0], x.strides[0])
            R.ffref_tx_close(h)
            d[f"out_{n}_{inv}"] = out
    d["trees"] = np.array(trees)
    np.savez_compressed(os.path.join(OUT, "tx_pfa_fft.npz"), **d)


def hbd_chroma_cases():
    """(avg, idx, x, y, h) for the 16-bit chroma fixture; (bw, bh, sx, sy) for the 16-bit edge fixture"""
    rng = np.random.default_rng(31)
    ch = [(avg, idx, x, y, [4, 8, 16, 2][(x + y + idx) % 4]) for avg in (0, 1) for idx in range(3) for x in range(8) for y in range(8)]
    ed = [(int(rng.integers(1, 25)), int(rng.integers(1, 25)), int(rng.integers(-30, 60)), int(rng.integers(-30, 50))) for _ in range(80)]
    return ch, ed


def gen_pel_hbd_chroma():
    """h264chroma (ff_h264chroma_init(c, 10 / 16)) and emulated_edge_mc (ff_videodsp_init(ctx, 10)) for 16-bit samples: sha256 of the
    compiled reference's destination per case"""
    R = cl.ref()
    R.ffref_h264chroma_hbd.argtypes = [C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_ssize_t, C.c_int, C.c_int, C.c_int]
    R.ffref_emulated_edge_mc_hbd.argtypes = [C.c_void_p, C.c_void_p, C.c_ssize_t, C.c_ssize_t] + [C.c_int] * 6
    ch, ed = hbd_chroma_cases()
    lines = []
    for depth in (10, 16):
        img, d0 = cl.hbd_picture(depth, 0)
        for (avg, idx, x, y, h) in ch:
            d = d0.copy()
            off = (8 * 64 + 8) * 2
            R.ffref_h264chroma_hbd(depth, avg, idx, d.ctypes.data + off, img.ctypes.data + off, 128, h, x, y)
            lines.append(f"c {depth} {avg} {idx} {x} {y} {h} {sha(d)}")
    pic, _ = cl.hbd_picture(10, 0)
    for (bw, bh, sx, sy) in ed:
        out = np.zeros((bh, bw + 3), np.uint16)
        R.ffref_emulated_edge_mc_hbd(out.ctypes.data, pic.ctypes.data + sy * pic.strides[0] + sx * 2, out.strides[0], pic.strides[0], bw, bh, sx, sy, 64, 48)
        lines.append(f"e {bw} {bh} {sx} {sy} {sha(out)}")
    open(os.path.join(OUT, "pel_hbd_chroma_hashes.txt"), "w").write("\n".join(lines) + "\n")


def gen_h264_weight_hbd():
    """weight / biweight tables of ff_h264dsp_init(c, 9 / 10 / 12 / 14): sha256 of the compiled reference's block per case"""
    R = cl.ref()
    R.ffref_h264_weight_hbd.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_ssize_t] + [C.c_int] * 4
    R.ffref_h264_biweight_hbd.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_ssize_t] + [C.c_int] * 5
    lines = []
    for depth in (9, 10, 12, 14):
        img, d0 = cl.hbd_picture(depth, 0)
        for k, (bi, idx, h, d, wd, ws, off) in enumerate(cl.hbd_weight_cases(depth)):
            blk = d0.copy()
            o = (8 * 64 + 8) * 2
            if bi:
                R.ffref_h264_biweight_hbd(depth, idx, blk.ctypes.data + o, img.ctypes.data + o, 128, h, d, wd, ws, off)
            else:
                R.ffref_h264_weight_hbd(depth, idx, blk.ctypes.data + o, 128, h, d, wd, off)
            lines.append(f"{depth} {k} {sha(blk)}")
    open(os.path.join(OUT, "h264_weight_hbd_hashes.txt"), "w").write("\n".join(lines) + "\n")


def gen_h264_idct_hbd():
    """idct_add / idct8_add / idct_dc_add / idct8_dc_add of ff_h264dsp_init(c, 9 / 10 / 12 / 14): sha256 of the compiled reference's
    destination picture + the block it leaves behind, per case"""
    R = cl.ref()
    R.ffref_h264_idct_hbd.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_ssize_t]
    lines = []
    for depth in (9, 10, 12, 14):
        for kind in range(4):
            for k, (blk, dst) in enumerate(cl.h264_idct_hbd_cases(depth, kind)):
                b, d = blk.copy(), dst.copy()
                R.ffref_h264_idct_hbd(depth, kind, d.ctypes.data + (2 * 16 + 4) * 2, b.ctypes.data, 32)
                lines.append(f"{depth} {kind} {k} {sha(np.concatenate([d.view(np.uint8).ravel(), b.view(np.uint8).ravel()]))}")
    open(os.path.join(OUT, "h264_idct_hbd_hashes.txt"), "w").write("\n".join(lines) + "\n")


def gen_h264lf_hbd():
    """the loop-filter members of ff_h264dsp_init(c, 9 / 10 / 12 / 14, 1 / 2): sha256 of the picture after 1024 independent edges of all 16 kinds"""
    lines = []
    for depth in (9, 10, 12, 14):
        case = cl.h264lf_hbd_case(50 + depth, 1024, depth)
        lines.append(f"{depth} {sha(cl.ref_h264lf_hbd(depth, *case))}")
    open(os.path.join(OUT, "h264lf_hbd_hashes.txt"), "w").write("\n".join(lines) + "\n")


def gen_h264pred():
    """H264PredContext from ff_h264_pred_init(AV_CODEC_ID_H264, depth, 1 / 2): sha256 of the reference's picture followed by its
    coefficients after one seeded batch of predictions ("pred") and of lossless adds ("add"), per depth and 4:2:0 / 4:2:2"""
    lines = []
    for depth in (8, 9, 10, 12, 14):
        for idc in (1, 2):
            for add in (0, 1):
                pic, cf = hp.ref_h264pred(depth, idc, add, *hp.h264pred_fixture_case(depth, idc, add))
                h = hashlib.sha256(np.ascontiguousarray(pic).tobytes() + np.ascontiguousarray(cf).tobytes()).hexdigest()
                lines.append(f"{depth} {idc} {'add' if add else 'pred'} {h}")
    open(os.path.join(OUT, "h264pred_hashes.txt"), "w").write("\n".join(lines) + "\n")


def gen_hevcmc():
    """HEVC motion compensation: sha256 of the reference's destination picture after the seeded batch of hm.fixture_case (the decoder's
    emulated_edge_mc windows and put_hevc_* calls, oracle/ref/ref_hevcdsp.c) per depth x luma (qpel) / chroma (epel)"""
    lines = []
    for depth in hm.DEPTHS:
        for epel in (0, 1):
            lines.append(f"{depth} {'chroma' if epel else 'luma'} {hm.digest(hm.ref_batch(depth, epel, *hm.fixture_case(depth, epel)))}")
    open(os.path.join(OUT, "hevcmc_hashes.txt"), "w").write("\n".join(lines) + "\n")


def gen_tx_double():
    """AV_TX_DOUBLE_FFT / AV_TX_DOUBLE_MDCT, power-of-two lengths: the compiled reference's outputs (sha256 of the float64 bits)"""
    R = cl.ref()
    R.ffref_txd_open.restype, R.ffref_txd_open.argtypes = C.c_void_p, [C.c_int, C.c_int, C.c_int, C.c_double, C.c_uint]
    R.ffref_tx_run.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_ssize_t, C.c_int, C.c_ssize_t, C.c_ssize_t]
    lines = []
    for (typ, n, inv, sc) in cl.txd_cases():
        x = cl.txd_input(typ, n, inv)
        oute = 2 * n if typ == 2 else n
        out = np.zeros((x.shape[0], oute))
        h = R.ffref_txd_open(typ, inv, n, sc, 0)
        xin = x.copy()
        R.ffref_tx_run(h, out.ctypes.data, xin.ctypes.data, 16 if typ == 2 else 8, x.shape[0], out.strides[0], xin.strides[0])
        R.ffref_tx_close(h)
        lines.append(f"{typ} {n} {inv} {sc!r} {sha(out)}")
    open(os.path.join(OUT, "tx_double_hashes.txt"), "w").write("\n".join(lines) + "\n")


RGB2RGB_FLAGS = (4, 4 | 0x80000, 4 | 0x80000 | 0x40000, 16)


def gen_sws_rgb2rgb():
    """same-size packed RGB -> packed RGB (rgbToRgbWrapper / packedCopyWrapper, or the scaler where findRgbConvFn has nothing): sha256 of
    the reference's destination picture for every ordered pair of the six formats, two sizes, four flag sets."""
    lines = []
    for (w, h) in ((37, 10), (64, 8)):
        for sn, sf in cl.PACKED_RGB_FORMATS.items():
            src = cl.rgb_frame(w, h, 2600 + w, cl.fmt_bpp(sf), "random", pad=3)
            for dn, df in cl.PACKED_RGB_FORMATS.items():
                for fl in RGB2RGB_FLAGS:
                    out = cl.ref_sws(w, h, w, h, fl, src, src, src, fmt=df, src_fmt=sf)
                    lines.append(f"{w} {h} {sn} {dn} {fl} {sha(out)}")
    open(os.path.join(OUT, "sws_rgb2rgb_hashes.txt"), "w").write("\n".join(lines) + "\n")


def gen_pel_hbd():
    """h264qpel at 9 / 10 / 12 / 14 bit: the compiled reference's tables (ff_h264qpel_init(c, depth)) on one random and one two-level
    picture per depth, every position / size / put+avg; stored as sha256 of the destination picture per case."""
    R = cl.ref()
    R.ffref_h264qpel_hbd.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_ssize_t]
    lines = []
    for depth in (9, 10, 12, 14):
        for kind in range(2):
            img, d0 = cl.hbd_picture(depth, kind)
            for avg in (0, 1):
                for si in range(3):
                    for pos in range(16):
                        d = d0.copy()
                        off = (8 * 64 + 8) * 2
                        R.ffref_h264qpel_hbd(depth, avg, si, pos, d.ctypes.data + off, img.ctypes.data + off, 128)
                        lines.append(f"{depth} {kind} {avg} {si} {pos} {sha(d)}")
    open(os.path.join(OUT, "pel_hbd_hashes.txt"), "w").write("\n".join(lines) + "\n")


def gen_tx_full_imdct():
    """AV_TX_FULL_IMDCT: the reference's 2 * len outputs of the inverse float MDCT, power-of-two and compound lengths, two scales."""
    R = cl.ref()
    d = {}
    rng = np.random.default_rng(79)
    for n in (4, 64, 256, 1024, 120, 144):
        x = (rng.random((2, n), dtype=np.float32) * 2 - 1).astype(np.float32)
        d[f"in_{n}"] = x
        for j, sc in enumerate((1.0 / n, -1.0)):
            h = R.ffref_tx_open(1, 1, n, sc, 4)
            assert h
            out = np.zeros((2, 2 * n), np.float32)
            R.ffref_tx_run(h, out.ctypes.data, x.ctypes.data, 4, 2, out.strides[0], x.strides[0])
            R.ffref_tx_close(h)
            d[f"out_{n}_{j}"] = out
    np.savez_compressed(os.path.join(OUT, "tx_full_imdct.npz"), **d)


def gen_tx_dct():
    """AV_TX_FLOAT_DCT: the reference's DCT-II (len points) and DCT-III (asked for len / 2) outputs, two scales."""
    R = cl.ref()
    d = {}
    rng = np.random.default_rng(78)
    for n in (8, 64, 512):
        x = (rng.random((2, n + 2), dtype=np.float32) * 2 - 1).astype(np.float32)
        x[:, n:] = 0
        d[f"in_{n}"] = x
        for inv, asked in ((0, n), (1, n // 2)):
            for j, sc in enumerate((1.0, 0.5 / n)):
                h = R.ffref_tx_open(9, inv, asked, sc, 0)
                out, xin = np.zeros((2, n + 2), np.float32), x.copy()
                R.ffref_tx_run(h, out.ctypes.data, xin.ctypes.data, 4, 2, out.strides[0], xin.strides[0])
                R.ffref_tx_close(h)
                d[f"out_{n}_{inv}_{j}"] = out[:, :n].copy()
    np.savez_compressed(os.path.join(OUT, "tx_dct.npz"), **d)


def gen_tx_int32():
    """AV_TX_INT32_FFT / AV_TX_INT32_MDCT: the reference's outputs (full-range FFT inputs, so the wrapping sums are exercised)."""
    R = cl.ref()
    d = {}
    rng = np.random.default_rng(79)
    for n in (8, 64, 1024):
        x = rng.integers(-(1 << 31), 1 << 31, (2, 2 * n)).astype(np.int32)
        d[f"in_{n}"] = x
        for inv in (0, 1):
            h = R.ffref_tx_open(4, inv, n, 1.0, 0)
            out, xin = np.zeros((2, 2 * n), np.int32), x.copy()
            R.ffref_tx_run(h, out.ctypes.data, xin.ctypes.data, 8, 2, out.strides[0], xin.strides[0])
            R.ffref_tx_close(h)
            d[f"fft_{n}_{inv}"] = out
        xs = (x >> 6).astype(np.int32)
        for j, sc in enumerate((1.0 / n, -1.0 / 32768)):
            for inv in (1, 0):
                xi = np.ascontiguousarray(xs[:, :n]) if inv else xs
                h = R.ffref_tx_open(5, inv, n, sc, 0)
                out, xin = np.zeros((2, n), np.int32), xi.copy()
                R.ffref_tx_run(h, out.ctypes.data, xin.ctypes.data, 4, 2, out.strides[0], xin.strides[0])
                R.ffref_tx_close(h)
                d[f"mdct_{n}_{inv}_{j}"] = out
    np.savez_compressed(os.path.join(OUT, "tx_int32.npz"), **d)


def gen_pixelutils():
    """av_pixelutils_get_sad_fn: the reference's sums for pixelutils_case(50 + bits, bits, 200), sizes 2 ... 32."""
    d = {}
    for bits in range(1, 6):
        d[f"sad_{bits}"] = cl.ref_pixelutils(bits, *cl.pixelutils_case(50 + bits, bits, 200))
    np.savez_compressed(os.path.join(OUT, "pixelutils.npz"), **d)


def gen_sws_float_kernels():
    """gauss / sinc / lanczos / spline / experimental scalers: sha256 of the reference's rgb24 and yuv420p outputs per case."""
    import hashlib
    from cases import SWS_FLOAT_KERNEL_CASES
    with open(os.path.join(OUT, "sws_float_kernel_hashes.txt"), "w") as f:
        for i, (w, h, dw, dh, fl, kind) in enumerate(SWS_FLOAT_KERNEL_CASES):
            y, u, v = cl.yuv_frame(w, h, 4100 + i, kind)
            rgb = cl.ref_sws(w, h, dw, dh, fl, y, u, v)
            yuv = np.concatenate([p.ravel() for p in cl.ref_sws_planar(w, h, dw, dh, fl, y, u, v)])
            f.write(f"{i} {hashlib.sha256(rgb.tobytes()).hexdigest()} {hashlib.sha256(yuv.tobytes()).hexdigest()}\n")


def gen_h264lf():
    """H264DSPContext loop filters, 8 bit: the reference's picture after the 512 edges of h264lf_case(seed, 512) (sha256, plus the first
    64 x 512 pixels of seed 0 for a readable diff)."""
    import hashlib
    d = {}
    for seed in (0, 1, 2):
        pic, kinds, off, alpha, beta, tc0 = cl.h264lf_case(40 + seed, 512)
        out = cl.ref_h264lf(pic, kinds, off, alpha, beta, tc0)
        assert not np.array_equal(out, pic)
        d[f"sha_{seed}"] = np.frombuffer(hashlib.sha256(out.tobytes()).digest(), np.uint8)
        if seed == 0:
            d["head_0"] = out[:64].copy()
    np.savez_compressed(os.path.join(OUT, "h264lf.npz"), **d)


def gen_prores():
    """ProresDSPContext.idct_put at 10 and 12 bit: the reference's pixels for prores_case(seed, bits, 60)."""
    d = {}
    for bits in (10, 12):
        for seed in (0, 1, 2):
            blocks, qmat = cl.prores_case(90 + seed, bits, 60)
            _, px = cl.ref_prores(bits, blocks, qmat, np.zeros((8, 60 * 8), np.uint16), 60 * 16)
            d[f"b{bits}_s{seed}"] = px
    np.savez_compressed(os.path.join(OUT, "prores.npz"), **d)


def gen_sws_fastbil():
    from cases import SWS_FASTBIL_CASES
    lines = []
    for i, (w, h, dw, dh, fl, kind) in enumerate(SWS_FASTBIL_CASES):
        y, u, v = cl.yuv_frame(w, h, 800 + i, kind)
        rgb = cl.ref_sws(w, h, dw, dh, fl, y, u, v)
        pl = cl.ref_sws_planar(w, h, dw, dh, fl, y, u, v)
        lines.append(f"{i} {w} {h} {dw} {dh} {fl} {kind} {sha(rgb)} {sha(np.concatenate([p.ravel() for p in pl]))}")
    open(os.path.join(OUT, "sws_fastbil_hashes.txt"), "w").write("\n".join(lines) + "\n")


def gen_sws_nv():
    from cases import SWS_NV_CASES
    lines = []
    for i, (w, h, dw, dh, fl, kind) in enumerate(SWS_NV_CASES):
        y, u, v = cl.yuv_frame(w, h, 1000 + i, kind)
        for sf, name in ((cl.PIX_FMT_NV12, "nv12"), (cl.PIX_FMT_NV21, "nv21")):
            uv = cl.nv_interleave(u, v, sf)
            rgb = cl.ref_sws(w, h, dw, dh, fl, y, uv, uv, src_fmt=sf)
            bgra = cl.ref_sws(w, h, dw, dh, fl, y, uv, uv, src_fmt=sf, fmt=cl.PIX_FMT_BGRA)
            pl = cl.ref_sws_planar(w, h, dw, dh, fl, y, uv, uv, src_fmt=sf)
            lines.append(f"{name} {i} {w} {h} {dw} {dh} {fl} {kind} {sha(rgb)} {sha(bgra)} {sha(np.concatenate([p.ravel() for p in pl]))}")
    open(os.path.join(OUT, "sws_nv_hashes.txt"), "w").write("\n".join(lines) + "\n")


def gen_idct():
    R = cl.ref()
    d = {}
    for kind in ("dense", "wide", "extreme", "sparse", "dc63", "dconly"):
        blk = idct_blocks(kind, 256, seed=7)
        rng = np.random.default_rng(11)
        dest0 = rng.integers(0, 256, (8, 256 * 8), dtype=np.uint8)
        off = (np.arange(256) * 8).astype(np.int64)
        d[f"{kind}_in"] = blk
        d[f"{kind}_dest"] = dest0
        for op in (0, 1, 2):
            b, de = blk.copy(), dest0.copy()
            R.ffref_idct_batch(op, cl.ptr(b, cl.i16p), 256, cl.ptr(de), 256 * 8, cl.ptr(off, cl.i64p))
            d[f"{kind}_op{op}"] = b if op == 0 else de
    np.savez_compressed(os.path.join(OUT, "idct.npz"), **d)


def h264_blocks(kind, n, seed):
    """coefficient blocks for the H.264 transforms: dequantised-residual-like, full-range, sparse and saturating ones"""
    rng = np.random.default_rng(seed)
    nc = 16 if kind in (0, 2) else 64
    b = np.zeros((n, nc), np.int16)
    for i in range(n):
        m = i % 4
        if m == 0:
            b[i] = rng.integers(-512, 513, nc)
        elif m == 1:
            b[i] = rng.integers(-32768, 32768, nc)
        elif m == 2:
            k = rng.integers(0, nc, 3)
            b[i, k] = rng.integers(-2000, 2001, 3)
        else:
            b[i] = rng.integers(0, 2, nc) * rng.choice([-32768, 32767], nc)
    if kind >= 2:
        b[:, 1:] = 0
    return b


def gen_h264idct():
    R = cl.ref()
    d = {}
    for kind in range(4):
        n, N = 64, 4 if kind in (0, 2) else 8
        blk = h264_blocks(kind, n, 30 + kind)
        dst0 = np.random.default_rng(40 + kind).integers(0, 256, (N, n * 8), dtype=np.uint8)
        out, b2 = dst0.copy(), blk.copy()
        for i in range(n):
            R.ffref_h264_idct(kind, C.cast(out.ctypes.data + 8 * i, cl.u8p), C.cast(b2.ctypes.data + i * b2.strides[0], cl.i16p), n * 8)
        d[f"k{kind}_in"], d[f"k{kind}_dst"], d[f"k{kind}_out"], d[f"k{kind}_blk_after"] = blk, dst0, out, b2
    np.savez_compressed(os.path.join(OUT, "h264idct.npz"), **d)


def gen_h264weight():
    """weight / biweight for every width, a grid of (log2_denom, weights, offset) incl. the extremes the bitstream allows"""
    R = cl.ref()
    rng = np.random.default_rng(25)
    src = rng.integers(0, 256, (20, 32), dtype=np.uint8)
    dst0 = rng.integers(0, 256, (20, 32), dtype=np.uint8)
    cases = []
    for idx in range(4):
        for (d, w1, w2, off) in ((0, 1, 1, 0), (5, 32, 32, 0), (7, -128, 127, -128), (6, 127, -128, 127), (3, 10, -3, 5), (1, -1, 3, -7), (7, 64, 64, 1), (2, 0, 0, 9)):
            cases.append((idx, (2, 4, 8, 16)[(idx + d) % 4], d, w1, w2, off))
    d = {"src": src, "dst0": dst0, "cases": np.array(cases, np.int32)}
    ps = C.cast(src.ctypes.data + 2 * 32 + 8, cl.u8p)
    for k, (idx, h, ld, w1, w2, off) in enumerate(cases):
        a, b = dst0.copy(), dst0.copy()
        R.ffref_h264_weight(idx, C.cast(a.ctypes.data + 2 * 32 + 8, cl.u8p), 32, h, ld, w1, off)
        R.ffref_h264_biweight(idx, C.cast(b.ctypes.data + 2 * 32 + 8, cl.u8p), ps, 32, h, ld, w1, w2, off)
        d[f"w{k}"], d[f"b{k}"] = a, b
    np.savez_compressed(os.path.join(OUT, "h264weight.npz"), **d)


def gen_mecmp():
    R = cl.ref()
    rng = np.random.default_rng(21)
    img1 = rng.integers(0, 256, (64, 64), dtype=np.uint8)          # tests/checkasm/motion.c:38-88: 64x64 random images
    img2 = rng.integers(0, 256, (64, 64), dtype=np.uint8)
    rows = []
    for fn, idxs in ((0, (0, 1)), (1, (0, 1, 2)), (2, range(8))):
        for idx in idxs:
            for _ in range(12):
                x1, y1, x2, y2 = (int(v) for v in rng.integers(0, 40, 4))
                h = int(rng.choice([4, 8, 16]))
                v = R.ffref_me_cmp(fn, idx, C.cast(img1.ctypes.data + y1 * 64 + x1, cl.u8p), C.cast(img2.ctypes.data + y2 * 64 + x2, cl.u8p), 64, h)
                rows.append((fn, idx, x1, y1, x2, y2, h, v))
    d = {"img1": img1, "img2": img2, "cases": np.array(rows, np.int32)}
    # exhaustive search: shifted + noisy reference, a flat pair (all ties) and an identical pair (early exit)
    W, H = 96, 64
    cur = rng.integers(0, 256, (H, W), dtype=np.uint8)
    ref_ = np.roll(cur, (2, -3), (0, 1)).copy()
    ref_[::5, ::3] ^= 5
    flat = np.full((H, W), 99, np.uint8)
    d["esa_cur"], d["esa_ref"] = cur, ref_
    for name, (a, b) in {"shift": (cur, ref_), "flat": (flat, flat), "same": (cur, cur)}.items():
        for mb, sp in ((16, 7), (8, 4), (16, 32), (4, 3)):
            bw, bh = W // mb, H // mb
            mv = np.zeros((bh * bw, 2), np.int32)
            cost = np.zeros(bh * bw, np.uint64)
            R.ffref_esa_frame(cl.ptr(a), cl.ptr(b), W, W, H, mb, sp, 0, bh, cl.ptr(mv, cl.i32p), cl.ptr(cost, cl.u64p))
            d[f"esa_{name}_{mb}_{sp}_mv"], d[f"esa_{name}_{mb}_{sp}_cost"] = mv, cost
    np.savez_compressed(os.path.join(OUT, "mecmp.npz"), **d)


def gen_chroma():
    """h264chroma put/avg, all three widths, every (x, y) eighth-pel phase, h in {2,4,8,16} per width."""
    R = cl.ref()
    rng = np.random.default_rng(23)
    src = rng.integers(0, 256, (40, 48), dtype=np.uint8)
    dst0 = rng.integers(0, 256, (40, 48), dtype=np.uint8)
    d = {"src": src, "dst0": dst0}
    ps = C.cast(src.ctypes.data + 8 * 48 + 8, cl.u8p)
    for avg in (0, 1):
        for idx in (0, 1, 2):
            for h in ((4, 8, 16), (2, 4, 8), (2, 4))[idx]:
                outs = []
                for xy in range(64):
                    o = dst0.copy()
                    assert R.ffref_h264chroma(avg, idx, C.cast(o.ctypes.data + 8 * 48 + 8, cl.u8p), ps, 48, h, xy & 7, xy >> 3) == 0
                    assert np.array_equal(o[:8], dst0[:8]) and np.array_equal(o[8 + h:], dst0[8 + h:])
                    outs.append(o[8:24, 8:16].copy())
                d[f"c_{avg}_{idx}_{h}"] = np.stack(outs)
    np.savez_compressed(os.path.join(OUT, "chroma.npz"), **d)


def gen_edge():
    from cases import EDGE_PIC, EDGE_CASES
    R = cl.ref()
    W, H, LS = EDGE_PIC
    pic = np.random.default_rng(24).integers(0, 256, (H, LS), dtype=np.uint8)
    d = {"pic": pic}
    for i, (bw, bh, sx, sy) in enumerate(EDGE_CASES):
        b = np.full((24, 32), 0x5A, np.uint8)
        R.ffref_emulated_edge_mc(cl.ptr(b), pic.ctypes.data + sy * LS + sx, 32, LS, bw, bh, sx, sy, W, H)
        d[f"e{i}"] = b
    np.savez_compressed(os.path.join(OUT, "edge.npz"), **d)


def gen_satd():
    """hadamard8_diff[0] (16 wide, h 8 / 16) and [1] (8x8) on the checkasm-style 64x64 random images of mecmp.npz"""
    R = cl.ref()
    g = np.load(os.path.join(OUT, "mecmp.npz"))
    img1, img2 = g["img1"], g["img2"]
    rng = np.random.default_rng(26)
    rows = []
    for idx in (0, 1):
        for _ in range(40):
            x1, y1, x2, y2 = (int(v) for v in rng.integers(0, 40, 4))
            h = int(rng.choice([8, 16]))
            v = R.ffref_me_cmp(3, idx, C.cast(img1.ctypes.data + y1 * 64 + x1, cl.u8p), C.cast(img2.ctypes.data + y2 * 64 + x2, cl.u8p), 64, h)
            rows.append((3, idx, x1, y1, x2, y2, h, v))
    np.savez_compressed(os.path.join(OUT, "satd.npz"), cases=np.array(rows, np.int32))


def gen_mecmp_dct():
    """dct_sad / dct_max (ff_jpeg_fdct_islow_8 and ff_fdct_ifast) and dct264_sad, [0] 16 wide (h 8 / 16) and [1] 8x8, from the compiled reference
    (encoder context with fdsp / pdsp / sum_abs_dctelem set up by ffref_me_cmp_set_dct_algo) on the 64x64 images of mecmp.npz and on a
    saturated pair (255 against 0 in a checkerboard: the largest coefficients the transforms see)"""
    R = cl.ref()
    g = np.load(os.path.join(OUT, "mecmp.npz"))
    chk = ((np.add.outer(np.arange(64), np.arange(64)) & 1) * 255).astype(np.uint8)
    pairs = [(g["img1"], g["img2"]), (chk, np.ascontiguousarray(255 - chk)), (np.full((64, 64), 255, np.uint8), np.zeros((64, 64), np.uint8))]
    rng = np.random.default_rng(2310)
    rows = []
    for algo in (0, 1):
        R.ffref_me_cmp_set_dct_algo(algo)
        for pi, (img1, img2) in enumerate(pairs):
            for fn in (8, 9, 10):
                if fn == 10 and algo == 1:
                    continue
                for idx in (0, 1):
                    for _ in range(12 if pi == 0 else 3):
                        x1, y1, x2, y2 = (int(v) for v in rng.integers(0, 40, 4))
                        h = int(rng.choice([8, 16]))
                        v = R.ffref_me_cmp(fn, idx, C.cast(img1.ctypes.data + y1 * 64 + x1, cl.u8p), C.cast(img2.ctypes.data + y2 * 64 + x2, cl.u8p), 64, h)
                        rows.append((fn, idx, algo, pi, x1, y1, x2, y2, h, v))
    R.ffref_me_cmp_set_dct_algo(0)
    np.savez_compressed(os.path.join(OUT, "mecmp_dct.npz"), cases=np.array(rows, np.int32))


def gen_fdct():
    """FDCTDSPContext.fdct / fdct248 of the compiled reference (islow 8 / 10 bit, ifast) on the blocks of test_cuda_emu.fdct_blocks: sha256 per set"""
    from test_cuda_emu import fdct_blocks
    R = cl.ref()
    lines = []
    for algo, bits in ((0, 8), (1, 8), (0, 10), (1, 9)):
        for is248 in (0, 1):
            x = fdct_blocks(bits, 200, 7000 + 10 * algo + bits + is248)
            for i in range(x.shape[0]):
                R.ffref_fdct(algo, bits, is248, cl.ptr(x[i], cl.i16p))
            lines.append(f"{algo} {bits} {is248} {sha(x)}")
    open(os.path.join(OUT, "fdct_hashes.txt"), "w").write("\n".join(lines) + "\n")


def gen_pel():
    R = cl.ref()
    rng = np.random.default_rng(22)
    src = rng.integers(0, 256, (40, 48), dtype=np.uint8)
    dst0 = rng.integers(0, 256, (40, 48), dtype=np.uint8)
    d = {"src": src, "dst0": dst0}
    ps = C.cast(src.ctypes.data + 8 * 48 + 8, cl.u8p)
    for avg in (0, 1):
        for sz in (0, 1, 2):
            for pos in range(16):
                o = dst0.copy()
                R.ffref_h264qpel(avg, sz, pos, C.cast(o.ctypes.data + 8 * 48 + 8, cl.u8p), ps, 48)
                d[f"q_{avg}_{sz}_{pos}"] = o[8:24, 8:24].copy()
    for tab in range(4):
        for sz in range(4):
            for xy in range(4):
                for h in ((8, 16) if sz < 2 else (2, 8)):
                    o = dst0.copy()
                    if R.ffref_hpel(tab, sz, xy, C.cast(o.ctypes.data + 8 * 48 + 8, cl.u8p), ps, 48, h) == 0:
                        d[f"h_{tab}_{sz}_{xy}_{h}"] = o[8:24, 8:24].copy()
    np.savez_compressed(os.path.join(OUT, "pel.npz"), **d)


def gen_tx():
    R = cl.ref()
    rng = np.random.default_rng(23)
    d = {}

    def run(typ, inv, n, scale, x, out_floats):
        h = R.ffref_tx_open(typ, inv, n, scale, 0)
        assert h
        out = np.zeros((x.shape[0], out_floats), np.float32)
        R.ffref_tx_run(h, out.ctypes.data, x.ctypes.data, 8 if typ == 0 else 4, x.shape[0], out.strides[0], x.strides[0])
        R.ffref_tx_close(h)
        return out
    for n in (2, 4, 8, 16, 32, 64, 256, 1024, 2048):            # tests/checkasm/av_tx.c:38-40 power-of-two lengths + BASELINE sizes
        x = rng.random((2, 2 * n), dtype=np.float32)            # in[i] = rnd()/UINT_MAX like checkasm (av_tx.c:33-41)
        d[f"fft_in_{n}"] = x
        for inv in (0, 1):
            d[f"fft_{n}_{inv}"] = run(0, inv, n, 1.0, x, 2 * n)
    for n in (8, 16, 64, 256, 1024, 2048):
        x = rng.random((2, n), dtype=np.float32)
        x2 = rng.random((2, 2 * n), dtype=np.float32)
        d[f"imdct_in_{n}"], d[f"mdct_in_{n}"] = x, x2
        for j, sc in enumerate((1.0 / n, -1.0, 1.0)):
            d[f"imdct_{n}_{j}"] = run(1, 1, n, sc, x, n)
            d[f"mdct_{n}_{j}"] = run(1, 0, n, sc, x2, n)
    np.savez_compressed(os.path.join(OUT, "tx.npz"), **d)
    # AV_TX_FLOAT_RDFT: forward r2c (len floats -> len/2+1 complex) and inverse c2r; the inverse rewrites its input
    d = {}
    for n in (4, 8, 16, 64, 256, 1024, 2048, 4096):
        for j, sc in enumerate((1.0, 1.0 / n)):
            x = (rng.random((2, n), dtype=np.float32) * 2 - 1).astype(np.float32)
            xc = (rng.random((2, n + 2), dtype=np.float32) * 2 - 1).astype(np.float32)
            d[f"r2c_in_{n}_{j}"], d[f"c2r_in_{n}_{j}"] = x.copy(), xc.copy()
            d[f"r2c_{n}_{j}"] = run(6, 0, n, sc, x, n + 2)
            d[f"c2r_{n}_{j}"] = run(6, 1, n, sc, xc, n)
            d[f"c2r_in_after_{n}_{j}"] = xc
    np.savez_compressed(os.path.join(OUT, "tx_rdft.npz"), **d)


def gen_vsynth1():
    """Frame 0 of FATE's vsynth1 (tests/videogen.c -> tests/vsynth1/00.pgm, a pgmyuv file: Y plane, then rows of U|V),
    converted by the reference with the FATE flags: the exact picture filter-pixfmts-{null,copy,...} hash for rgb24
    (tests/ref/fate/filter-pixfmts-null:93) before it is wrapped in NUT."""
    import subprocess, tempfile
    vg = os.path.join(ROOT, "oracle", "_ref", "videogen")
    with tempfile.TemporaryDirectory() as td:
        subprocess.run([vg, td + "/"], check=True)
        raw = open(os.path.join(td, "00.pgm"), "rb").read()
    hdr, rest = raw.split(b"\n255\n", 1)
    assert hdr.split()[0] == b"P5" and hdr.split()[1:] == [b"352", b"432"], hdr
    a = np.frombuffer(rest, np.uint8).reshape(432, 352)
    y = np.ascontiguousarray(a[:288])
    u = np.ascontiguousarray(a[288:, :176])
    v = np.ascontiguousarray(a[288:, 176:])
    FATE = cl.SWS_BICUBIC | cl.SWS_ACCURATE_RND | cl.SWS_BITEXACT
    d = {"y": y, "u": u, "v": v}
    d["rgb_same"] = cl.ref_sws(352, 288, 352, 288, FATE, y, u, v)
    d["rgb_200x100"] = cl.ref_sws(352, 288, 200, 100, FATE, y, u, v)          # filter-pixfmts-scale geometry
    d["rgb_lut"] = cl.ref_sws(352, 288, 352, 288, cl.SWS_BICUBIC, y, u, v)
    np.savez_compressed(os.path.join(OUT, "vsynth1_f0.npz"), **d)


def gen_sws_slices():
    """sws_scale() fed with top-down bands: the reference's per-call return values (lines written) and final picture."""
    R = cl.ref()
    FATE = cl.SWS_BICUBIC | cl.SWS_ACCURATE_RND | cl.SWS_BITEXACT
    d = {}
    y, u, v = cl.yuv_frame(64, 48, 400, "random")
    d["y"], d["u"], d["v"] = y, u, v
    from cases import SWS_SLICE_CASES
    for ci, (dw, dh, fl, bands) in enumerate(SWS_SLICE_CASES):
        ctx = R.ffref_sws_open(64, 48, dw, dh, fl, 1)
        out = np.full((dh, dw * 3), 0xA5, np.uint8)
        rets = []
        for (sy, sh) in bands:
            rets.append(R.ffref_sws_scale(ctx, C.cast(y.ctypes.data + sy * 64, cl.u8p), 64, C.cast(u.ctypes.data + (sy // 2) * 32, cl.u8p), 32,
                                          C.cast(v.ctypes.data + (sy // 2) * 32, cl.u8p), 32, sy, sh, cl.ptr(out), dw * 3))
        R.ffref_sws_close(ctx)
        d[f"s{ci}_rets"] = np.array(rets, np.int32)
        d[f"s{ci}_rgb"] = out
    np.savez_compressed(os.path.join(OUT, "sws_slices.npz"), **d)


if __name__ == "__main__":
    assert cl.have_ref(), "build oracle/_ref first: make -C oracle/ref"
    os.makedirs(OUT, exist_ok=True)
    if len(sys.argv) > 1:                                           # python scripts/gen_golden.py tx_pfa_fft ...: only those fixtures
        for name in sys.argv[1:]:
            globals()["gen_" + name]()
        sys.exit(0)
    gen_sws()
    gen_sws_formats()
    gen_sws_planar()
    gen_sws_fastbil()
    gen_sws_nv()
    gen_idct()
    gen_h264idct()
    gen_h264weight()
    gen_mecmp()
    gen_satd()
    gen_mecmp_dct()
    gen_fdct()
    gen_pel()
    gen_chroma()
    gen_edge()
    gen_tx()
    gen_h264lf()
    gen_sws_float_kernels()
    gen_pixelutils()
    gen_vsynth1()
    gen_sws_slices()
    gen_sws_range()
    gen_unquant()
    gen_fdsp()
    gen_idct_hbd()
    gen_sws_rgbsrc()
    gen_tx_pfa()
    gen_tx_pfa_fft()
    gen_pel_hbd()
    gen_pel_hbd_chroma()
    gen_h264_weight_hbd()
    gen_h264_idct_hbd()
    gen_h264lf_hbd()
    gen_h264pred()
    gen_hevcmc()
    gen_tx_double()
    gen_sws_rgb2rgb()
    gen_tx_full_imdct()
    gen_tx_dct()
    gen_tx_int32()
    gen_prores()
    for f in sorted(os.listdir(OUT)):
        print(f, os.path.getsize(os.path.join(OUT, f)))
