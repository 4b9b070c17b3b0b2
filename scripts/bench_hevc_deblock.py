"""Benchmark of b200_hevc_deblock_plane_device (ffmpeg_b200/csrc/hevcdbk.cu) on cuda:0: CUDA events around calls after warm-up.

Cases: a 3840x2160 luma plane at 8 and 10 bit and a 1920x1080 (4:2:0) chroma plane at 8 bit, with decoder-shaped grids and content
(tests/hevcdbklib.py: CU quadtree, boundary strengths, table beta / tc).  A plane and its grids (about 10 MB at 8 bit) fit in the 50 MB
L2, so each timed call works on the next of FRAMES independent copies (more than the L2 in total) and reads what the previous calls
evicted.  Calls filter their copy in place again and again, as a timing loop must; the decisions then see already filtered edges.
Bytes are the algorithm's least: the plane read and written once plus both grids read once.  Prints card name, power limit and max SM
clock first."""
import argparse
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
PEAK = 3.35e12
L2 = 50 << 20


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
    from ffmpeg_b200 import hevcdsp
    import hevcdbklib as hd
    print("card:", card(), flush=True)
    dev = fb.Device(0)
    dev.set_default()
    st = torch.cuda.ExternalStream(dev.stream)
    cases = (("3840x2160 luma 8bit", 8, 0, 3840, 2160), ("3840x2160 luma 10bit", 10, 0, 3840, 2160),
             ("1920x1080 chroma 420 8bit", 8, 1, 1920, 1080))
    with torch.cuda.stream(st):
        for name, depth, chroma, W, H in cases:
            buf, vg, hg = hd.plane_case(3 + depth + chroma, depth, W, H, bool(chroma), ctb=64)
            plane = np.ascontiguousarray(buf[hd.MARGIN:hd.MARGIN + H, hd.MARGIN:hd.MARGIN + W])
            bps = plane.itemsize
            nbytes = 2 * plane.nbytes + vg.nbytes + hg.nbytes
            frames_n = max(4, -(-3 * L2 // nbytes) // 2 * 2)
            p0 = torch.from_numpy(plane.view(np.int16) if bps == 2 else plane).cuda()
            frames = [(p0.clone(), torch.from_numpy(vg.view(np.uint8)).cuda(), torch.from_numpy(hg.view(np.uint8)).cuda())
                      for _ in range(frames_n)]
            k = [0]

            def call():
                dp, dv, dh = frames[k[0] % frames_n]
                k[0] += 1
                hevcdsp.hevc_deblock_plane_device(dev, depth, chroma, dp, W * bps, W, H, dv, vg.shape[1], dh, hg.shape[1])
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
            tb = nbytes / PEAK
            print(f"{name:28s} {t * 1e6:8.1f} us  {nbytes / 1e6:6.1f} MB  {nbytes / t / 1e9:7.1f} GB/s  HBM bound {tb * 1e6:5.1f} us "
                  f"({tb / t:.3f} of 3.35 TB/s)  frames {frames_n}", flush=True)
            del frames, p0
            torch.cuda.empty_cache()
    dev.close()


if __name__ == "__main__":
    main()
