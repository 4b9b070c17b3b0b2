"""Benchmark of b200_hevc_mc_batch_device (ffmpeg_b200/csrc/hevcmc.cu) on cuda:0: CUDA events around back-to-back calls after warm-up.

Cases: a 3840x2160 luma plane (qpel) at 8 and 10 bit tiled with 8x8, 16x16 and 64x64 units, all uni or all bi; the matching 4:2:0
chroma plane (1920x1080, epel) with 4x4, 8x8 and 32x32 units; and one CTU-row call (the 60 64x64 CTUs of a 3840-wide row as 16x16 bi units),
which is launch-bound.  Motion vectors are seeded within +-32 samples.  Bytes are counted from shapes: the reference windows each op
reads ((w + taps - 1) x (h + taps - 1) samples per reference, only in filtered directions), the block written, and the 64-byte
descriptor; the fraction is of the H100 SXM's 3.35 TB/s.  Prints card name, power limit and max SM clock first."""
import argparse
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
PEAK = 3.35e12

from ffmpeg_b200.hevcdsp import OP_DTYPE  # noqa: E402


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip()


def make_case(rng, W, H, unit, bi, depth, epel, rows=None):
    P, T = (8, 4) if epel else (4, 8)
    ys = range(0, H if rows is None else rows, unit)
    xy = np.array([(x, y) for y in ys for x in range(0, W, unit)])
    n = len(xy)
    ops = np.zeros(n, OP_DTYPE)
    bps = 1 if depth == 8 else 2
    ops["dst_off"] = (xy[:, 1] * W + xy[:, 0]) * bps
    ops["w"] = ops["h"] = unit
    ops["kind"] = 2 if bi else 0
    ops["ref_off"][:, 0] = -W * H * bps
    for r in (0, 1):
        ops["x"][:, r] = xy[:, 0] + rng.integers(-32, 33, n)
        ops["y"][:, r] = xy[:, 1] + rng.integers(-32, 33, n)
        ops["mx"][:, r] = rng.integers(0, P, n)
        ops["my"][:, r] = rng.integers(0, P, n)
    nref = 2 if bi else 1
    rd = 0
    for r in range(nref):
        rd += int((((unit + np.where(ops["mx"][:, r] > 0, T - 1, 0)) * (unit + np.where(ops["my"][:, r] > 0, T - 1, 0)))).sum())
    nbytes = rd * bps + n * unit * unit * bps + n * 64
    return ops, nbytes


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()
    import torch
    import ffmpeg_b200 as fb
    from ffmpeg_b200 import hevcdsp
    print("card:", card(), flush=True)
    dev = fb.Device(0)
    dev.set_default()
    st = torch.cuda.ExternalStream(dev.stream)
    rng = np.random.default_rng(1)
    cases = []
    for depth in (8, 10):
        for unit in (8, 16, 64):
            for bi in (False, True):
                cases.append((f"luma {depth}bit {unit}x{unit} {'bi' if bi else 'uni'}", depth, 0, 3840, 2160, unit, bi, None))
        for unit in (4, 8, 32):
            for bi in (False, True):
                cases.append((f"chroma {depth}bit {unit}x{unit} {'bi' if bi else 'uni'}", depth, 1, 1920, 1080, unit, bi, None))
    cases.append(("CTU row luma 8bit 16x16 bi", 8, 0, 3840, 2160, 16, True, 64))
    with torch.cuda.stream(st):
        for name, depth, epel, W, H, unit, bi, rows in cases:
            ops, nbytes = make_case(rng, W, H, unit, bi, depth, epel, rows)
            dt = torch.uint8 if depth == 8 else torch.int16
            ref = torch.randint(0, 1 << depth, (2 * H * W,), dtype=torch.int32, device="cuda").to(dt)
            dst = torch.zeros(H * W, dtype=dt, device="cuda")
            dops = torch.from_numpy(ops.view(np.uint8)).cuda()
            bps = 1 if depth == 8 else 2
            refp = ref.data_ptr() + H * W * bps

            def call():
                hevcdsp.hevc_mc_batch_device(dev, depth, epel, len(ops), dops, dst, W * bps, refp, W * bps, W, H)
            for _ in range(args.warmup):
                call()
            dev.sync()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(st)
            for _ in range(args.iters):
                call()
            e1.record(st)
            dev.sync()
            t = e0.elapsed_time(e1) / 1e3 / args.iters
            print(f"{name:44s} ops {len(ops):7d}  {t * 1e6:9.1f} us  {len(ops) / t / 1e9:6.3f} G ops/s  {nbytes / t / 1e9:7.1f} GB/s  "
                  f"{nbytes / t / PEAK:.3f} of 3.35 TB/s", flush=True)
    dev.close()


if __name__ == "__main__":
    main()
