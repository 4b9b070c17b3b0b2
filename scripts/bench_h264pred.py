#!/usr/bin/env python
"""Throughput and per-call latency of the batched H.264 intra prediction entries (b200_h264_pred_batch_device,
b200_h264_pred_add_batch_device) on cuda:0.

    python scripts/bench_h264pred.py [--iters 200] [--warmup 20]

Cases:
  - a whole 3840x2160 luma frame (240 x 135 macroblocks) of independent ops: 32 400 pred16x16 ops (modes 0-6 in turn), 518 400 pred4x4
    ops (modes 0-11, top-right available on every other op), and 32 400 pred16x16_add ops (lossless), at 8 and 10 bit;
  - one wavefront step of 120 pred16x16 ops, and of 120 pred4x4 ops: what a decoder issues per call.  These are launch-bound.
The blocks sit on a grid with a gutter of one row and four columns between them, so every op reads neighbours no op writes (one
call = one independent set, as the entries require) and every block row starts on a 4-sample boundary, as in a decoder's picture.
Bytes are counted from shapes: neighbour samples read + block written (+ coefficients read and cleared for the add forms) + the
per-op kind, flags and offsets; the fraction is of 3.35 TB/s (H100 SXM data sheet).
Times are CUDA events around `iters` back-to-back calls after `warmup` calls.  The card's name, power limit and maximum SM clock are
read in the same run and printed first.  Prints one JSON line per case."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PEAK_BYTES = 3.35e12


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown (nvidia-smi failed)"


def neighbours(table, mode, flags, W, H):
    """samples the reference function of (table, mode) reads (pred_needs in h264pred.cu)"""
    if table in (0, 1):
        need = {0: "T", 10: "T", 1: "L", 8: "L", 9: "L", 2: "TL", 3: "TR", 7: "TR", 4: "TLC", 5: "TLC", 6: "TLC"}.get(mode, "")
    else:
        need = {0: "TL", 7: "TL", 8: "TL", 1: "L", 4: "L", 9: "L", 10: "L", 2: "T", 5: "T", 3: "TLC"}.get(mode, "")
    n = ("T" in need) * W + ("L" in need) * H + ("C" in need)
    if "R" in need:
        n += 4 if table == 0 else (8 if flags & 2 else 0)
    return n


def grid_ops(depth, nx, ny, W, H, table, modes, flags_of):
    """ops on an nx x ny grid of W x H blocks (gutter: one row, four columns): picture, kinds, flags, byte offsets, bytes moved per call"""
    bps = 1 if depth == 8 else 2
    pw, ph = nx * (W + 4) + 4 + 16, ny * (H + 1) + 1
    rng = np.random.default_rng(1)
    pic = rng.integers(0, 1 << depth, (ph, pw)).astype(np.uint8 if depth == 8 else np.uint16)
    n = nx * ny
    i = np.arange(n)
    kinds = np.array([(table << 4) | modes[k % len(modes)] for k in range(n)], np.uint8)
    flags = np.array([flags_of(k) for k in range(n)], np.uint8)
    off = (((i // nx) * (H + 1) + 1) * pic.strides[0] + ((i % nx) * (W + 4) + 4) * bps).astype(np.int64)
    moved = 0
    for k in range(n):
        moved += (neighbours(table, int(kinds[k]) & 15, int(flags[k]), W, H) + W * H) * bps
    moved += n * (1 + 1 + 8)
    return pic, kinds, flags, off, moved


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    a = ap.parse_args()
    import torch
    import ffmpeg_b200 as fb
    from ffmpeg_b200 import pel
    print(json.dumps({"card": card()}), flush=True)
    dev = fb.Device(0)
    dev.set_default()
    st = torch.cuda.ExternalStream(dev.stream)
    cases = []
    for depth in (8, 10):
        cases.append(("pred16x16 3840x2160", depth, False, 240, 135, 16, 16, 4, list(range(7)), lambda k: 0))
        cases.append(("pred4x4 3840x2160", depth, False, 960, 540, 4, 4, 0, list(range(12)), lambda k: 2 * (k & 1)))
        cases.append(("pred16x16_add 3840x2160", depth, True, 240, 135, 16, 16, 5, [1, 2], lambda k: 0))
    cases.append(("pred16x16 wavefront", 8, False, 120, 1, 16, 16, 4, list(range(7)), lambda k: 0))
    cases.append(("pred4x4 wavefront", 8, False, 120, 1, 4, 4, 0, list(range(12)), lambda k: 2 * (k & 1)))
    with torch.cuda.stream(st):
        for (name, depth, add, nx, ny, W, H, table, modes, flags_of) in cases:
            pic, kinds, flags, off, moved = grid_ops(depth, nx, ny, W, H, table, modes, flags_of)
            n = len(kinds)
            dp = torch.from_numpy(pic.view(np.int16) if depth > 8 else pic).cuda()
            dk, df, do = torch.from_numpy(kinds).cuda(), torch.from_numpy(flags).cuda(), torch.from_numpy(off).cuda()
            if add:
                ctype = np.int16 if depth == 8 else np.int32
                coef = torch.zeros((n, 256), dtype=torch.int16 if depth == 8 else torch.int32, device="cuda")
                dco = torch.arange(n, dtype=torch.int64, device="cuda") * 256
                moved += n * (2 * W * H * np.dtype(ctype).itemsize + 8)
                call = lambda: pel.h264_pred_add_batch_device(dev, depth, n, dk, df, dp, do, pic.strides[0], coef, dco)
            else:
                call = lambda: pel.h264_pred_batch_device(dev, depth, n, dk, df, dp, do, pic.strides[0])
            for _ in range(a.warmup):
                call()
            dev.sync()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(st)
            for _ in range(a.iters):
                call()
            e1.record(st)
            e1.synchronize()
            sec = e0.elapsed_time(e1) / 1e3 / a.iters
            print(json.dumps({"case": name, "bit_depth": depth, "ops": n, "us_per_call": round(sec * 1e6, 2), "ops_per_s": round(n / sec),
                              "bytes_per_call": int(moved), "GB_per_s": round(moved / sec / 1e9, 1),
                              "fraction_of_3.35TB_s": round(moved / sec / PEAK_BYTES, 4)}), flush=True)
    dev.close()


if __name__ == "__main__":
    main()
