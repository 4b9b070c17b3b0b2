"""Benchmark of b200_hevc_transform_add_batch_device (ffmpeg_b200/csrc/hevcidct.cu) on cuda:0: CUDA events around calls after warm-up.

Cases: a 3840x2160 plane at 8 and 10 bit tiled with TUs of one size (4x4 .. 32x32), all IDCT (dense coefficients, full col_limit) or all
IDCT_DC; a mixed plane (sizes and kinds in a decoder-like proportion); a 1920x1080 chroma plane of 8x8 IDCT.  An 8-bit 4K plane's
coefficients and samples (about 33 MB) fit in the 50 MB L2, so each timed call works on the next of FRAMES independent frames (more
than 3x the L2 in total) and reads what the previous calls evicted.  Bytes are the algorithm's: 2 B of coefficient read per sample,
the sample read and written, and the 32-byte descriptor per op.  The integer-ALU bound counts the partial butterfly's multiply-adds and
add / subtracts per sample (both passes, with the rounding, shift and clip) at 64 INT32 lanes per SM and the card's maximum SM clock.
Prints card name, power limit and max SM clock first."""
import argparse
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
PEAK = 3.35e12
FRAMES = 6

from ffmpeg_b200.hevcdsp import TU_DTYPE, IDCT, IDCT_DC, SKIP  # noqa: E402


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip()


def int_ops_per_sample(n, kind):
    """integer operations per output sample of one TU of size n: the two butterfly passes of IDCT, or the add alone"""
    if kind != IDCT:
        return 3
    line = 8 + sum((m // 2) ** 2 + m for m in (8, 16, 32) if m <= n)    # 4-point core, then each level's odd products and butterflies
    return 2 * (line / n + 3) + 3


def tiling(W, H, sizes, rng):
    """(x, y, log2) of TUs covering the plane: 32x32 blocks split down to the sizes drawn from `sizes` (a {log2: weight} dict)"""
    tus = []
    logs, w = np.array(list(sizes)), np.array(list(sizes.values()), float)

    def fill(x, y, l):
        if x >= W or y >= H:
            return
        pick = int(rng.choice(logs, p=w / w.sum()))
        if (pick >= l and x + (1 << l) <= W and y + (1 << l) <= H) or l == 2:
            tus.append((x, y, l))
            return
        s = 1 << (l - 1)
        for dy in (0, s):
            for dx in (0, s):
                fill(x + dx, y + dy, l - 1)
    for y in range(0, H, 32):
        for x in range(0, W, 32):
            fill(x, y, 5)
    return np.array(tus)


def make_case(rng, W, H, depth, sizes, kinds):
    """ops (frame-local offsets), nbytes, int ops, samples"""
    t = tiling(W, H, sizes, rng)
    n, bps = len(t), 1 if depth == 8 else 2
    ops = np.zeros(n, TU_DTYPE)
    ops["dst_off"] = (t[:, 1] * W + t[:, 0]) * bps
    ops["log2_size"] = t[:, 2]
    sz = (1 << t[:, 2].astype(np.int64)) ** 2
    ops["coef_off"] = np.concatenate([[0], np.cumsum(sz)[:-1]])
    ops["kind"] = rng.choice(kinds, n)
    ops["col_limit"] = 1 << t[:, 2]
    samples = int(sz.sum())
    iops = sum(int_ops_per_sample(1 << int(l), int(k)) * (1 << (2 * int(l))) for l, k in zip(ops["log2_size"], ops["kind"]))
    return ops, samples * (2 + 2 * bps) + 32 * n, iops, samples


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=60)
    ap.add_argument("--warmup", type=int, default=12)
    args = ap.parse_args()
    import torch
    import ffmpeg_b200 as fb
    from ffmpeg_b200 import hevcdsp
    c = card()
    print("card:", c, flush=True)
    clock = float(c.split(",")[-1].strip().split()[0]) * 1e6 if c else 1.98e9
    alu = 132 * 64 * clock
    dev = fb.Device(0)
    dev.set_default()
    st = torch.cuda.ExternalStream(dev.stream)
    rng = np.random.default_rng(1)
    cases = []
    for depth in (8, 10):
        for l in (2, 3, 4, 5):
            for kind, kn in ((IDCT, "idct"), (IDCT_DC, "dc")):
                cases.append((f"3840x2160 {depth}bit {1 << l}x{1 << l} {kn}", depth, 3840, 2160, {l: 1}, [kind]))
        cases.append((f"3840x2160 {depth}bit mixed", depth, 3840, 2160, {2: 3, 3: 3, 4: 2, 5: 1}, [IDCT] * 6 + [IDCT_DC] * 3 + [SKIP]))
    cases.append(("1920x1080 chroma 8bit 8x8 idct", 8, 1920, 1080, {3: 1}, [IDCT]))
    with torch.cuda.stream(st):
        for name, depth, W, H, sizes, kinds in cases:
            ops, nbytes, iops, samples = make_case(rng, W, H, depth, sizes, kinds)
            dt = torch.uint8 if depth == 8 else torch.int16
            frames = []
            for _ in range(FRAMES):
                coef = torch.randint(-2048, 2048, (samples + 8,), dtype=torch.int16, device="cuda")
                dst = torch.randint(0, 1 << depth, (H * W,), dtype=torch.int32, device="cuda").to(dt)
                frames.append((torch.from_numpy(ops.view(np.uint8)).cuda(), coef, dst))
            bps = 1 if depth == 8 else 2
            k = [0]

            def call():
                do, dc, dd = frames[k[0] % FRAMES]
                k[0] += 1
                hevcdsp.hevc_transform_add_batch_device(dev, depth, len(ops), do, dc, dd, W * bps)
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
            tb, ta = nbytes / PEAK, iops / alu
            print(f"{name:36s} ops {len(ops):7d}  {t * 1e6:8.1f} us  {samples / t / 1e9:6.1f} G samples/s  {nbytes / t / 1e9:7.1f} GB/s  "
                  f"{tb / t:.3f} of 3.35 TB/s  int-ALU bound {ta * 1e6:6.1f} us ({ta / t:.3f})  bound by {'ALU' if ta > tb else 'HBM'}",
                  flush=True)
            del frames
            torch.cuda.empty_cache()
    dev.close()


if __name__ == "__main__":
    main()
