"""Benchmark of b200_vc1_mc_frame_device and b200_vc1_residual_frame_device (ffmpeg_b200/csrc/vc1mc.cu, vc1idct.cu) on cuda:0: CUDA
events around each call after warm-up, the inputs evicted from L2 (a 256 MB buffer rewritten) before every timed call, the median and
p10 / p90 over the calls reported.

Cases: decoder-shaped progressive pictures of 3840x2160 (240 x 135 MBs) and 1920x1088 (120 x 68) built by tests/vc1dsplib.py: a P picture
(1MV and 4MV macroblocks, mspel, rnd 1) and a B picture (forward, backward and interpolated 1MV macroblocks, mspel, rnd 0), motion
mostly within +-24 samples; the residual entry on the six blocks of every macroblock with decoder-shaped coefficients and a mix of the
four transform types.  Bytes are counted from the op list: MC reads the footprint of each source (n + 3 samples in a direction mspel
filters, n + 1 for hpel, n otherwise; chroma 9 or 8) and the 40-byte op, and writes the block (for an interpolated op: reads and
writes it once more); the residual reads the 128 coefficient bytes and the 16-byte op and reads and writes the 64 samples.  The
fraction is of the H100 SXM data sheet's 3.35 TB/s.  Prints card name, power limit and max SM clock first, read in the same run."""
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
    from ffmpeg_b200.vc1dsp import MC_1MV, MC_CHROMA8, MSPEL, AVG
    total = 40 * len(ops)
    for o in ops:
        ms = bool(o["flags"] & MSPEL)
        for s in range(2 if o["flags"] & AVG else 1):
            S = o["src"][s]
            if o["kind"] != MC_CHROMA8:
                n = 16 if o["kind"] == MC_1MV else 8
                ext = lambda f: n + (3 if ms else 1) if (f if ms else f & 2) else n  # noqa: E731
                total += ext(int(S["mx"])) * ext(int(S["my"])) + n * n * (1 + s)
            if o["kind"] != 1:
                total += 2 * ((8 + (S["uvmx"] > 0)) * (8 + (S["uvmy"] > 0)) + 64 * (1 + s))
    return int(total)


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
    print(f"{name:36s} ops {n:7d}  median {t * 1e6:8.1f} us  (p10 {lo * 1e6:.1f}, p90 {hi * 1e6:.1f})  {nbytes / t / 1e9:7.1f} GB/s  "
          f"{nbytes / t / PEAK:.3f} of 3.35 TB/s", flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    args = ap.parse_args()
    import torch
    import ffmpeg_b200 as fb
    from ffmpeg_b200 import vc1dsp
    import vc1dsplib as v1
    print("card:", card(), flush=True)
    dev = fb.Device(0)
    dev.set_default()
    st = torch.cuda.ExternalStream(dev.stream)
    with torch.cuda.stream(st):
        flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
        for label, w, h in (("3840x2160", 3840, 2160), ("1920x1088", 1920, 1088)):
            mbw, mbh = w // 16, h // 16
            for pic, b, rnd in (("P", False, 1), ("B", True, 0)):
                refs, ops, dst, H, V = v1.mc_case(w + b, mbw, mbh, w, h, b, 1, rnd)
                bufs = [[torch.from_numpy(p).cuda() for p in r.planes] for r in refs]
                descs = [r.desc([int(x.data_ptr()) for x in bb]) for r, bb in zip(refs, bufs)]
                dd = [torch.from_numpy(p).cuda() for p in dst]
                do = torch.from_numpy(np.ascontiguousarray(ops).view(np.uint8)).cuda()
                t = timed(dev, st, flush, lambda: vc1dsp.vc1_mc_frame_device(dev, descs, dd, dst[0].strides[0], dst[1].strides[0], mbw, mbh, H, V,
                                                                             len(ops), do), args.warmup, args.iters)
                report(f"mc {label} {pic} mspel", len(ops), mc_bytes(ops), t)
            rops, coef = v1.residual_case(w + 7, mbw, mbh, "decoder", skip=0.0)
            dc = torch.from_numpy(coef).cuda()
            do = torch.from_numpy(np.ascontiguousarray(rops).view(np.uint8)).cuda()
            t = timed(dev, st, flush, lambda: vc1dsp.vc1_residual_frame_device(dev, dd, dst[0].strides[0], dst[1].strides[0], mbw, mbh, dc,
                                                                               len(rops), do), args.warmup, args.iters)
            report(f"residual {label}", len(rops), len(rops) * (128 + 16 + 128), t)
    dev.close()


if __name__ == "__main__":
    main()
