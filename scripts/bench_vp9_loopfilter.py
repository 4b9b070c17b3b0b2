"""Benchmark of b200_vp9_loopfilter_frame_device (ffmpeg_b200/csrc/vp9lf.cu) on cuda:0: CUDA events around each call after warm-up, the
inputs evicted from L2 (a 256 MB buffer rewritten) before every timed call, the median and the spread over the calls reported.

Cases: 1920x1080 and 3840x2160 4:2:0 frames at 8 and 10 bit with decoder-shaped loop-filter records (tests/vp9lflib.py).  The work is a
wavefront of superblocks: its critical path is sb_cols + 2 (sb_rows - 1) superblock steps (62 for 1080p, 126 for 2160p), each a column
pass and a row pass of one 64 x 64 luma superblock by one CTA.  The time per step is printed beside the total; the bytes moved (each
plane read and written once) are printed as a fraction of the H100 SXM data sheet's 3.35 TB/s to show that HBM bandwidth is not what
binds.  Prints card name, power limit and max SM clock first."""
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    args = ap.parse_args()
    import torch
    import ffmpeg_b200 as fb
    from ffmpeg_b200 import vp9dsp
    import vp9lflib as vl
    print("card:", card(), flush=True)
    dev = fb.Device(0)
    dev.set_default()
    st = torch.cuda.ExternalStream(dev.stream)
    with torch.cuda.stream(st):
        flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
        for depth in (8, 10):
            for W, H in ((1920, 1080), (3840, 2160)):
                f = vl.Frame(1000 + depth + H, depth, "420", W, H)
                planes = [torch.from_numpy(np.ascontiguousarray(p).view(np.int16 if depth > 8 else np.uint8)).cuda() for p in f.planes]
                ptrs = [t.data_ptr() + vl.MARGIN * p.strides[0] + vl.MARGIN * p.itemsize for t, p in zip(planes, f.planes)]
                rec = torch.from_numpy(np.ascontiguousarray(f.lflvl).view(np.uint8)).cuda()
                ls_y, ls_uv = f.strides()
                nbytes = 2 * sum(p.nbytes for p in f.planes) + f.lflvl.nbytes
                steps = f.sbc + 2 * (f.sbr - 1)
                times = []
                for it in range(args.warmup + args.iters):
                    flush.fill_(it & 0xFF)
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record(st)
                    vp9dsp.vp9_loopfilter_frame_device(dev, depth, 1, 1, W, H, ptrs, ls_y, ls_uv, rec, f.lstride, f.lim, f.mblim)
                    e1.record(st)
                    dev.sync()
                    if it >= args.warmup:
                        times.append(e0.elapsed_time(e1) / 1e3)
                t, lo, hi = np.median(times), np.percentile(times, 10), np.percentile(times, 90)
                print(f"{W}x{H} 4:2:0 {depth:2d} bit  median {t * 1e6:8.1f} us  (p10 {lo * 1e6:.1f}, p90 {hi * 1e6:.1f})  "
                      f"{steps} steps: {t * 1e6 / steps:6.2f} us / step  {nbytes / t / 1e9:6.1f} GB/s = {nbytes / t / PEAK:.3f} of 3.35 TB/s",
                      flush=True)
    dev.close()


if __name__ == "__main__":
    main()
