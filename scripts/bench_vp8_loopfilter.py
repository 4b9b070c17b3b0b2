"""Benchmark of b200_vp8_loopfilter_frame_device (ffmpeg_b200/csrc/vp8lf.cu) on cuda:0: CUDA events around each call after warm-up, the
unfiltered planes copied back and the inputs evicted from L2 (a 256 MB buffer rewritten) before every timed call, the median and p10 /
p90 over the calls reported.

Cases: 3840x2160 (240 x 135 MBs) and 1920x1088 (120 x 68) frames built by tests/vp8lflib.py with decoder-shaped records
(filter_level_for_mb on random segmentation, deltas, sharpness, modes and skip flags), VP8 normal, VP8 simple and VP7 normal, inter
frames.  Bytes are counted from shapes: each plane read and written once (luma only for the simple filter), plus 3 bytes per MB.  The
critical path of the slope-2 wavefront is mb_width + 2 (mb_height - 1) MB steps; the time per step is the median over that count.  The
fraction is of the H100 SXM data sheet's 3.35 TB/s.  Prints card name, power limit and max SM clock first."""
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
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()
    import torch
    import ffmpeg_b200 as fb
    from ffmpeg_b200 import vp8dsp
    import vp8lflib as vl
    print("card:", card(), flush=True)
    dev = fb.Device(0)
    dev.set_default()
    st = torch.cuda.ExternalStream(dev.stream)
    with torch.cuda.stream(st):
        flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
        for label, mbw, mbh in (("3840x2160", 240, 135), ("1920x1088", 120, 68)):
            for codec, is_vp7, simple in (("vp8 normal", 0, 0), ("vp8 simple", 0, 1), ("vp7 normal", 1, 0)):
                f = vl.Frame(mbw + 3 * is_vp7 + simple, mbw, mbh, is_vp7, simple, 0, "decoder")
                areas = [np.ascontiguousarray(a) for a in f.area(f.planes)]
                src = [torch.from_numpy(a).cuda() for a in areas]
                planes = [s.clone() for s in src]
                rec = torch.from_numpy(np.ascontiguousarray(f.f).view(np.uint8).ravel()).cuda()
                times = []
                for it in range(args.warmup + args.iters):
                    for p, s in zip(planes, src):
                        p.copy_(s)
                    flush.fill_(it & 0xFF)
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record(st)
                    vp8dsp.vp8_loopfilter_frame_device(dev, is_vp7, simple, 0, mbw, mbh, planes, 16 * mbw, 8 * mbw, rec, f.fstride)
                    e1.record(st)
                    dev.sync()
                    if it >= args.warmup:
                        times.append(e0.elapsed_time(e1) / 1e3)
                t, lo, hi = np.median(times), np.percentile(times, 10), np.percentile(times, 90)
                nbytes = 2 * (256 if simple else 384) * mbw * mbh + 3 * mbw * mbh
                steps = mbw + 2 * (mbh - 1)
                print(f"loop filter {label} {codec:10s} MBs {mbw * mbh:6d}  median {t * 1e6:8.1f} us  (p10 {lo * 1e6:.1f}, p90 {hi * 1e6:.1f})  "
                      f"{nbytes / t / 1e9:6.1f} GB/s  {nbytes / t / PEAK:.4f} of 3.35 TB/s  {steps} steps, {t / steps * 1e9:.0f} ns per step",
                      flush=True)
        assert vp8dsp.vp8_loopfilter_timeouts(dev) == 0
    dev.close()


if __name__ == "__main__":
    main()
