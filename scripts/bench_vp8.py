"""Benchmark of b200_vp8_mc_frame_device and b200_vp8_residual_frame_device (ffmpeg_b200/csrc/vp8mc.cu, vp8idct.cu) on cuda:0: CUDA
events around each call after warm-up, the inputs evicted from L2 (a 256 MB buffer rewritten) before every timed call, the median and
p10 / p90 over the calls reported.

Cases: decoder-shaped inter frames of 3840x2160 (240 x 135 MBs) and 1920x1088 (120 x 68) built by tests/vp8dsplib.py (mostly 16x16,
some 16x8 / 8x16 / 8x8 and 4x4 splits, motion within +-16 samples), with the epel and the bilinear table; the residual entry on the same
frames (decoder-shaped nnz caches: Y2 on most MBs, a mix of DC-only and full blocks); and one macroblock-row call of each entry (the
240 MBs of a 3840-wide row), which is launch-bound.  Bytes are counted from shapes: MC reads the (w + 5) x (h + 5) window of each op and
plane (w x h for full-pel), writes w x h and reads the 24-byte op; the residual reads 800 coefficient bytes and the 48-byte op per MB and
reads and writes the 4x4 blocks it adds to.  The fraction is of the H100 SXM data sheet's 3.35 TB/s.  Prints card name, power limit and
max SM clock first."""
import argparse
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
PEAK = 3.35e12


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip()


def mc_bytes(ops):
    w, h = ops["w"].astype(np.int64), ops["h"].astype(np.int64)
    full = (ops["mx"] == 0) & (ops["my"] == 0)
    win = np.where(full, w * h, (w + 5) * (h + 5))
    planes = np.where(ops["plane"] == 1, 2, 1)
    return int((planes * (win + w * h)).sum()) + 24 * len(ops)


def res_bytes(ops):
    nz = ops["nnz"].reshape(len(ops), 24) > 0
    luma = (ops["flags"] & 1).astype(bool)
    blocks = int(nz[:, 16:].sum() + (nz[:, :16] & luma[:, None]).sum())
    return len(ops) * (800 + 48) + blocks * 32


def timed(dev, st, flush, fn, warmup, iters):
    import torch
    times = []
    for it in range(warmup + iters):
        flush.fill_(it & 0xFF)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(st)
        fn()
        e1.record(st)
        dev.sync()
        if it >= warmup:
            times.append(e0.elapsed_time(e1) / 1e3)
    return np.median(times), np.percentile(times, 10), np.percentile(times, 90)


def report(name, n, nbytes, t):
    t, lo, hi = t
    print(f"{name:44s} ops {n:7d}  median {t * 1e6:8.1f} us  (p10 {lo * 1e6:.1f}, p90 {hi * 1e6:.1f})  {nbytes / t / 1e9:7.1f} GB/s  "
          f"{nbytes / t / PEAK:.3f} of 3.35 TB/s", flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    args = ap.parse_args()
    import torch
    import ffmpeg_b200 as fb
    from ffmpeg_b200 import vp8dsp
    import vp8dsplib as v8
    print("card:", card(), flush=True)
    dev = fb.Device(0)
    dev.set_default()
    st = torch.cuda.ExternalStream(dev.stream)
    with torch.cuda.stream(st):
        flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
        for label, mbw, mbh in (("3840x2160", 240, 135), ("1920x1088", 120, 68)):
            rng = np.random.default_rng(mbw)
            refs = v8.ref_frames(rng, mbw, mbh, 3, pad=0)
            ops = v8.mc_ops(v8.mb_partitions(rng, mbw, mbh, 3, far=0, intra=0.0))
            drefs = [tuple(torch.from_numpy(p).cuda() for p in r) for r in refs]
            rl = [(y, u, v, 16 * mbw, 8 * mbw) for (y, u, v) in drefs]
            dst = [torch.zeros(16 * mbh * 16 * mbw, dtype=torch.uint8, device="cuda")] + \
                  [torch.zeros(8 * mbh * 8 * mbw, dtype=torch.uint8, device="cuda") for _ in range(2)]
            row = ops[ops["dst_y"] < np.where(ops["plane"] == 0, 16, 8)]
            for bil in (0, 1):
                for nm, o in ((f"mc {label} {'bilinear' if bil else 'epel'}", ops), (f"mc one MB row {label[:4]}w {'bilinear' if bil else 'epel'}", row)):
                    do = torch.from_numpy(np.ascontiguousarray(o).view(np.uint8)).cuda()
                    t = timed(dev, st, flush, lambda: vp8dsp.vp8_mc_frame_device(dev, bil, mbw, mbh, rl, len(o), do, dst, 16 * mbw, 8 * mbw),
                              args.warmup, args.iters)
                    report(nm, len(o), mc_bytes(o), t)
            rops, coef = v8.residual_case(mbw + 1, mbw, mbh, 0, skip=0.0)
            dc = torch.from_numpy(coef).cuda()
            rrow = rops[rops["mb_y"] == 0]
            for nm, o in ((f"residual {label} vp8", rops), (f"residual one MB row {label[:4]}w vp8", rrow)):
                do = torch.from_numpy(np.ascontiguousarray(o).view(np.uint8)).cuda()
                t = timed(dev, st, flush, lambda: vp8dsp.vp8_residual_frame_device(dev, 0, len(o), do, dc, dst, 16 * mbw, 8 * mbw),
                          args.warmup, args.iters)
                report(nm, len(o), res_bytes(o), t)
    dev.close()


if __name__ == "__main__":
    main()
