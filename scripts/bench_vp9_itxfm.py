"""Benchmark of b200_vp9_itxfm_add_batch_device (ffmpeg_b200/csrc/vp9itxfm.cu) on cuda:0: CUDA events around each call after warm-up,
the inputs evicted from L2 (a 256 MB buffer rewritten) before every timed call, the median and the spread over the calls reported.

Cases: a 3840x2160 8-bit plane tiled with one transform size (4x4, 8x8, 16x16, 32x32), DCT_DCT, then the 4x4..16x16 planes with the
four types mixed; a 3840x2160 plane of mixed sizes (64x64 superblocks split at random down to 4x4) and types at 8, 10 and 12 bit; the
1920x1080 4:2:0 chroma plane of mixed sizes at 8 bit.  Dense coefficients, eob = sz * sz, so every block runs both passes.  Bytes are
counted from shapes: the coefficients read (2 bytes each at 8 bit, 4 above), the block of dst read and written, the 24-byte descriptor;
the fraction is of the H100 SXM data sheet's 3.35 TB/s of HBM3 bandwidth.  Prints card name, power limit and max SM clock first."""
import argparse
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
PEAK = 3.35e12

from ffmpeg_b200.vp9dsp import TX_DTYPE  # noqa: E402


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip()


def make_case(rng, W, H, depth, unit=None, mixed_types=False):
    """ops tiling a W x H plane with unit x unit blocks (unit None: 64x64 superblocks split at random down to 4x4), the coefficient
    count and the bytes the call has to move"""
    units = []
    if unit:
        units = [(x, y, unit) for y in range(0, H - unit + 1, unit) for x in range(0, W - unit + 1, unit)]
    else:
        def split(x, y, s):
            if s > 32 or (s > 4 and rng.random() < 0.5):
                for dy in (0, s // 2):
                    for dx in (0, s // 2):
                        split(x + dx, y + dy, s // 2)
            elif x + s <= W and y + s <= H:
                units.append((x, y, s))
        for y in range(0, H, 64):
            for x in range(0, W, 64):
                split(x, y, 64)
    u = np.array(units)
    n = len(u)
    bps, cs = (1, 2) if depth == 8 else (2, 4)
    ops = np.zeros(n, TX_DTYPE)
    ops["dst_off"] = (u[:, 1] * W + u[:, 0]) * bps
    ops["tx"] = np.log2(u[:, 2]).astype(int) - 2
    ops["type"] = rng.integers(0, 4, n) if (mixed_types or not unit) else 0
    sizes = u[:, 2].astype(np.int64) ** 2
    ops["eob"] = sizes
    ops["coef_off"] = np.concatenate([[0], np.cumsum(sizes)[:-1]])
    ncoef = int(sizes.sum())
    return ops, ncoef, ncoef * cs + 2 * ncoef * bps + n * TX_DTYPE.itemsize


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
    cases = [(f"luma 8bit {s}x{s} DCT_DCT", 8, 3840, 2160, s, False) for s in (4, 8, 16, 32)]
    cases += [(f"luma 8bit {s}x{s} mixed types", 8, 3840, 2160, s, True) for s in (4, 8, 16)]
    cases += [(f"luma {d}bit mixed sizes and types", d, 3840, 2160, None, True) for d in (8, 10, 12)]
    cases += [("chroma 8bit 1920x1080 mixed sizes and types", 8, 1920, 1080, None, True)]
    with torch.cuda.stream(st):
        flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
        for name, depth, W, H, unit, mixed in cases:
            ops, ncoef, nbytes = make_case(rng, W, H, depth, unit, mixed)
            dt, ct = (torch.uint8, torch.int16) if depth == 8 else (torch.int16, torch.int32)
            bps = 1 if depth == 8 else 2
            coef = torch.randint(-(1 << (depth + 2)), 1 << (depth + 2), (ncoef + 16,), dtype=torch.int32, device="cuda").to(ct)
            dst = torch.randint(0, 1 << depth, (H * W,), dtype=torch.int32, device="cuda").to(dt)
            dops = torch.from_numpy(ops.view(np.uint8)).cuda()
            times = []
            for it in range(args.warmup + args.iters):
                flush.fill_(it & 0xFF)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(st)
                vp9dsp.vp9_itxfm_add_batch_device(dev, depth, len(ops), dops, coef, dst, W * bps)
                e1.record(st)
                dev.sync()
                if it >= args.warmup:
                    times.append(e0.elapsed_time(e1) / 1e3)
            t, lo, hi = np.median(times), np.percentile(times, 10), np.percentile(times, 90)
            print(f"{name:44s} ops {len(ops):7d}  median {t * 1e6:8.1f} us  (p10 {lo * 1e6:.1f}, p90 {hi * 1e6:.1f})  "
                  f"{ncoef / t / 1e9:6.1f} G samples/s  {nbytes / t / 1e9:7.1f} GB/s  {nbytes / t / PEAK:.3f} of 3.35 TB/s", flush=True)
    dev.close()


if __name__ == "__main__":
    main()
