"""Side-by-side timing of two builds of libb200dsp.so on the IDCT and inverse-quantiser kernels whose machine code a change to the
shared arithmetic (csrc/simple_idct.cuh, csrc/mpv_unquant.cuh) can move.  Both libraries run on one stream, alternately, 12 runs
each; every run restores its inputs first (outside the timed window, which is CUDA events around the one call), and the outputs of
the two builds' last runs are compared bit for bit.  Prints card name, power limit and max SM clock, then one line per case:
median [min - max] in microseconds for each build.

Cases: b200_idct_mb420_device put / add at 1920x1088, 64 frames, luma plane 8 bytes off 16-byte alignment (the warp kernel);
b200_idct_hbd_batch_device at 10 and 12 bit, kinds 0 / 1 / 2, 2^20 blocks; b200_prores_idct_put_batch_device at 10 and 12 bit,
2^20 blocks; b200_mpv_unquant_idct_mb420_device put, every variant, 1920x1088, 16 frames; b200_mpv_unquantize_batch_device, every
variant, 2^20 blocks.

usage: python scripts/bench_idct_arith.py --base <other libb200dsp.so> [--lib <libb200dsp.so>]"""
import argparse
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from ffmpeg_b200._lib import PROTOTYPES, MpvUnquant  # noqa: E402

RUNS = 12


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip()


def load(path, stream):
    L = C.CDLL(path)
    for name in ("b200_device_open", "b200_last_error", "b200_idct_mb420_device", "b200_idct_hbd_batch_device",
                 "b200_prores_idct_put_batch_device", "b200_mpv_unquant_idct_mb420_device", "b200_mpv_unquantize_batch_device"):
        f = getattr(L, name)
        f.restype, f.argtypes = PROTOTYPES[name]
    dev = C.c_void_p()
    assert L.b200_device_open(C.byref(dev), 0, C.c_void_p(stream)) == 0, L.b200_last_error()
    return L, dev


def ptr(t, off=0):
    return C.c_void_p(t.data_ptr() + off)


def planes420(mb_w, mb_h, nf, luma_off):
    """three uint8 planes for nf frames of mb_w x mb_h macroblocks: (buffers, pointer offsets, line sizes, frame strides)"""
    ls = [mb_w * 16 + 64, mb_w * 8 + 64, mb_w * 8 + 64]
    hs = [mb_h * 16, mb_h * 8, mb_h * 8]
    fs = [ls[i] * hs[i] for i in range(3)]
    bufs = [torch.randint(0, 256, (nf * fs[i] + 64,), dtype=torch.uint8, device="cuda") for i in range(3)]
    return bufs, [luma_off, 0, 0], ls, fs


def coefficients(rng, nblocks, lo=-300, hi=300):
    """int16 blocks: sparse AC, every fourth block DC-only"""
    b = rng.integers(lo, hi, (nblocks, 64)).astype(np.int16)
    b[rng.random((nblocks, 64)) < 0.6] = 0
    b[::4, 1:] = 0
    return torch.from_numpy(b).cuda()


def time_pair(libs, inputs, outputs, call):
    """inputs: (work tensor, master copy) pairs restored before every run; returns per-build times (us) and last outputs"""
    times = [[] for _ in libs]
    last = [None] * len(libs)
    for _ in range(RUNS):
        for k, (L, dev) in enumerate(libs):
            for w, m in inputs:
                w.copy_(m)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            rc = call(L, dev)
            e1.record()
            assert rc == 0, (rc, L.b200_last_error())
            torch.cuda.synchronize()
            times[k].append(e0.elapsed_time(e1) * 1e3)
            last[k] = [o.clone() for o in outputs]
    same = all(torch.equal(a, b) for a, b in zip(last[0], last[1]))
    return times, same


def report(name, times, same):
    cols = []
    for t in times:
        t = np.array(t)
        cols.append(f"{np.median(t):9.1f} [{t.min():.1f} - {t.max():.1f}]")
    print(f"{name:34s} base {cols[0]:>30s}   this {cols[1]:>30s}   outputs {'identical' if same else 'DIFFER'}", flush=True)
    return same


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--base", required=True)
    ap.add_argument("--lib", default=os.path.join(ROOT, "ffmpeg_b200", "libb200dsp.so"))
    a = ap.parse_args()
    print(card(), flush=True)
    stream = torch.cuda.Stream()              # not the legacy default stream: a null handle makes each library open a stream of its own
    torch.cuda.set_stream(stream)
    libs = [load(a.base, stream.cuda_stream), load(a.lib, stream.cuda_stream)]
    rng = np.random.default_rng(1)
    ok = True

    # warp route: luma plane 8 bytes off, so the tiled kernel refuses the frames
    mb_w, mb_h, nf = 120, 68, 64
    blocks = coefficients(rng, mb_w * mb_h * 6 * nf)
    bufs, offs, ls, fs = planes420(mb_w, mb_h, nf, 8)
    masters = [b.clone() for b in bufs]
    PL = C.c_void_p * 3
    for kind, kname in ((1, "put"), (2, "add")):
        call = lambda L, dev: L.b200_idct_mb420_device(dev, kind, ptr(blocks), mb_w, mb_h, nf,  # noqa: E731
                                                       PL(*[b.data_ptr() + o for b, o in zip(bufs, offs)]), (C.c_int * 3)(*ls), (C.c_int64 * 3)(*fs))
        ok &= report(f"warp mb420 {kname} 1920x1088x64", *time_pair(libs, list(zip(bufs, masters)), bufs, call))
    del blocks, bufs, masters

    # 10 / 12 bit and ProRes, one 8 x 8 block of 16-bit samples per destination tile, 1024 x 1024 tiles
    n = 1 << 20
    row_bytes = 1024 * 16
    i = torch.arange(n, dtype=torch.int64, device="cuda")
    off = (i // 1024) * 8 * row_bytes + (i % 1024) * 16
    dest = torch.zeros(n * 128, dtype=torch.uint8, device="cuda")
    for depth in (10, 12):
        coef = coefficients(rng, n, -2000, 2000)
        cwork = coef.clone()
        dmaster = torch.randint(0, 1 << depth, (n * 64,), dtype=torch.int16, device="cuda").view(torch.uint8)
        for kind in (0, 1, 2):
            call = lambda L, dev: L.b200_idct_hbd_batch_device(dev, depth, kind, ptr(cwork), n, ptr(dest), ptr(off), None, row_bytes)  # noqa: E731
            ok &= report(f"hbd {depth} bit kind {kind}", *time_pair(libs, [(cwork, coef), (dest, dmaster)], [cwork, dest], call))
        qmat = torch.from_numpy(rng.integers(1, 9, 64).astype(np.int16)).cuda()
        coef_p = coefficients(rng, n, -512, 512)
        call = lambda L, dev: L.b200_prores_idct_put_batch_device(dev, depth, ptr(coef_p), n, ptr(qmat), ptr(dest), ptr(off), None, row_bytes)  # noqa: E731
        ok &= report(f"prores {depth} bit put", *time_pair(libs, [(dest, dmaster)], [dest], call))
    del dest, off

    # quantiser, alone and fused in front of the tiled IDCT
    p = MpvUnquant()
    for i in range(64):
        p.intra_matrix[i] = int(rng.integers(8, 64))
        p.inter_matrix[i] = int(rng.integers(8, 64))
        p.permutated[i] = i
        p.raster_end[i] = i
    p.y_dc_scale, p.c_dc_scale, p.q_scale_type, p.h263_aic, p.ac_pred = 8, 8, 1, 0, 0
    lv = coefficients(rng, n, -40, 40)
    lwork = lv.clone()
    qs = torch.from_numpy(rng.integers(1, 32, n).astype(np.uint8)).cuda()
    last = torch.from_numpy(rng.integers(-1, 64, n).astype(np.int8)).cuda()
    for v in range(7):
        call = lambda L, dev: L.b200_mpv_unquantize_batch_device(dev, v, C.byref(p), ptr(lwork), n, None, ptr(qs), ptr(last))  # noqa: E731
        ok &= report(f"unquant variant {v}", *time_pair(libs, [(lwork, lv)], [lwork], call))
    del lwork
    mb_w, mb_h, nf = 120, 68, 16
    nb = mb_w * mb_h * 6 * nf
    fl = coefficients(rng, nb, -40, 40)
    fq = torch.from_numpy(rng.integers(1, 32, nb).astype(np.uint8)).cuda()
    fla = torch.from_numpy(rng.integers(-1, 64, nb).astype(np.int8)).cuda()
    bufs, offs, ls, fs = planes420(mb_w, mb_h, nf, 0)
    masters = [b.clone() for b in bufs]
    for v in range(7):
        call = lambda L, dev: L.b200_mpv_unquant_idct_mb420_device(dev, v, C.byref(p), 1, ptr(fl), ptr(fq), ptr(fla), mb_w, mb_h, nf,  # noqa: E731
                                                                    PL(*[b.data_ptr() + o for b, o in zip(bufs, offs)]), (C.c_int * 3)(*ls),
                                                                    (C.c_int64 * 3)(*fs))
        ok &= report(f"fused put variant {v} 1920x1088x16", *time_pair(libs, list(zip(bufs, masters)), bufs, call))
    print("all outputs identical" if ok else "OUTPUTS DIFFER", flush=True)
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
