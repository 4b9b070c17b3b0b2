"""Benchmark of b200_vp9_mc_batch_device (ffmpeg_b200/csrc/vp9mc.cu) on cuda:0: CUDA events around each call after warm-up, the
inputs evicted from L2 (a 256 MB buffer rewritten) before every timed call, the median and the spread over the calls reported.

Cases: a 3840x2160 8-bit luma plane tiled with 16x16 single, 16x16 compound, 64x64 single and 8x8 single blocks; 16x16 single and
compound at 10 bit; the 1920x1080 4:2:0 chroma plane as 8x8 single; one scaled case (a reference of twice the size, step 32 in both
directions, 16x16 single); and one superblock-row call (the 60 64x64 superblocks of a 3840-wide row as 960 16x16 compound ops), which is
launch-bound.  Regular 8-tap bank, motion vectors seeded within +-32 samples, phases uniform in 0..15.  Bytes are counted from shapes:
the reference window each slot reads (8-tap span only in directions it filters), the block written and the 40-byte descriptor; the
fraction is of the H100 SXM data sheet's 3.35 TB/s of HBM3 bandwidth.  Prints card name, power limit and max SM clock first."""
import argparse
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
PEAK = 3.35e12

from ffmpeg_b200.vp9dsp import OP_DTYPE  # noqa: E402


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip()


def make_case(rng, W, H, unit, compound, depth, step, rows=None):
    """ops tiling a W x H plane with unit x unit blocks (the first `rows` lines only, if given) and the bytes the call has to move"""
    xy = np.array([(x, y) for y in range(0, H if rows is None else rows, unit) for x in range(0, W, unit)])
    n = len(xy)
    ops = np.zeros(n, OP_DTYPE)
    bps = 1 if depth == 8 else 2
    ops["dst_off"] = (xy[:, 1] * W + xy[:, 0]) * bps
    ops["w"] = ops["h"] = unit
    ops["kind"] = 1 if compound else 0
    ops["filter"] = 1
    rd = 0
    for r in range(2 if compound else 1):
        ops["ref"][:, r] = r
        ops["x"][:, r] = (xy[:, 0] + rng.integers(-32, 33, n)) * step // 16
        ops["y"][:, r] = (xy[:, 1] + rng.integers(-32, 33, n)) * step // 16
        ops["mx"][:, r] = rng.integers(0, 16, n)
        ops["my"][:, r] = rng.integers(0, 16, n)
        mx, my = ops["mx"][:, r].astype(np.int64), ops["my"][:, r].astype(np.int64)
        wc = np.where((mx > 0) | (step != 16), (((unit - 1) * step + mx) >> 4) + 8, unit)
        wr = np.where((my > 0) | (step != 16), (((unit - 1) * step + my) >> 4) + 8, unit)
        rd += int((wc * wr).sum())
    return ops, rd * bps + n * unit * unit * bps + n * OP_DTYPE.itemsize


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    args = ap.parse_args()
    import torch
    import ffmpeg_b200 as fb
    from ffmpeg_b200 import vp9dsp
    print("card:", card(), flush=True)
    dev = fb.Device(0)
    dev.set_default()
    st = torch.cuda.ExternalStream(dev.stream)
    rng = np.random.default_rng(1)
    cases = [("luma 8bit 16x16 single", 8, 3840, 2160, 16, False, 16, None), ("luma 8bit 16x16 compound", 8, 3840, 2160, 16, True, 16, None),
             ("luma 8bit 64x64 single", 8, 3840, 2160, 64, False, 16, None), ("luma 8bit 8x8 single", 8, 3840, 2160, 8, False, 16, None),
             ("luma 10bit 16x16 single", 10, 3840, 2160, 16, False, 16, None), ("luma 10bit 16x16 compound", 10, 3840, 2160, 16, True, 16, None),
             ("chroma 8bit 8x8 single", 8, 1920, 1080, 8, False, 16, None), ("luma 8bit 16x16 single, step 32", 8, 3840, 2160, 16, False, 32, None),
             ("superblock row luma 8bit 16x16 compound", 8, 3840, 2160, 16, True, 16, 64)]
    with torch.cuda.stream(st):
        flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
        for name, depth, W, H, unit, compound, step, rows in cases:
            ops, nbytes = make_case(rng, W, H, unit, compound, depth, step, rows)
            dt = torch.uint8 if depth == 8 else torch.int16
            bps = 1 if depth == 8 else 2
            RW, RH = W * step // 16, H * step // 16
            planes = [torch.randint(0, 1 << depth, (RH * RW,), dtype=torch.int32, device="cuda").to(dt) for _ in range(2)]
            refs = [(p, RW * bps, RW, RH, step, step) for p in planes]
            dst = torch.zeros(H * W, dtype=dt, device="cuda")
            dops = torch.from_numpy(ops.view(np.uint8)).cuda()
            times = []
            for it in range(args.warmup + args.iters):
                flush.fill_(it & 0xFF)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(st)
                vp9dsp.vp9_mc_batch_device(dev, depth, refs, len(ops), dops, dst, W * bps)
                e1.record(st)
                dev.sync()
                if it >= args.warmup:
                    times.append(e0.elapsed_time(e1) / 1e3)
            t, lo, hi = np.median(times), np.percentile(times, 10), np.percentile(times, 90)
            print(f"{name:42s} ops {len(ops):7d}  median {t * 1e6:8.1f} us  (p10 {lo * 1e6:.1f}, p90 {hi * 1e6:.1f})  {len(ops) / t / 1e9:6.3f} G ops/s  "
                  f"{nbytes / t / 1e9:7.1f} GB/s  {nbytes / t / PEAK:.3f} of 3.35 TB/s", flush=True)
    dev.close()


if __name__ == "__main__":
    main()
