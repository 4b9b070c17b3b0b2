"""Benchmark of b200_hevc_sao_plane_device (ffmpeg_b200/csrc/hevcsao.cu) on cuda:0: CUDA events around calls after warm-up.

Cases: a 3840x2160 luma plane at 8 and 10 bit and a 1920x1080 (4:2:0) chroma plane at 8 bit, with decoder-shaped records
(tests/hevcsaolib.py: CTB 64, a mix of NONE, BAND and EDGE CTBs, slices, a PCM map).  A source and destination plane (about 17 MB at
8 bit) fit in the 50 MB L2, so each timed call works on the next of FRAMES independent (src, dst) pairs (more than the L2 in total)
and reads what the previous calls evicted.  Bytes are the algorithm's least: the plane read once and written once plus the records.
Prints card name, power limit and max SM clock first.  The 8-bit luma plane is then timed again with every CTB NONE, BAND or EDGE
(no keep map), which shows what each path costs."""
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
    import hevcsaolib as hl
    print("card:", card(), flush=True)
    dev = fb.Device(0)
    dev.set_default()
    st = torch.cuda.ExternalStream(dev.stream)
    cases = (("3840x2160 luma 8bit", 8, 0, None), ("3840x2160 luma 10bit", 10, 0, None), ("1920x1080 chroma 420 8bit", 8, 1, None),
             ("  every CTB NONE", 8, 0, hl.SAO_NONE), ("  every CTB BAND", 8, 0, hl.SAO_BAND), ("  every CTB EDGE", 8, 0, hl.SAO_EDGE))
    with torch.cuda.stream(st):
        for name, depth, c, only in cases:
            p = hl.picture_case(3 + depth, depth, 3840, 2160, 6, 1, nslices=8, lf_slices=(1, 0), pcm=True)
            W, H, hs, vs = hl.comp_geometry(p, c)
            plane, g, k = p.planes[c], hl.records(p, c), hl.keep_map(p)
            if only is not None:
                g["type"] = only
                g["cls"] = g["cls"] & 3 if only == hl.SAO_EDGE else g["cls"]
            bps = plane.itemsize
            nbytes = 2 * plane.nbytes + p.cw * p.ch * 16
            frames_n = max(4, -(-3 * L2 // nbytes))
            s0 = torch.from_numpy(plane.view(np.int16) if bps == 2 else plane).cuda()
            frames = [(s0.clone(), torch.empty_like(s0)) for _ in range(frames_n)]
            dg, dk = torch.from_numpy(g.view(np.uint8)).cuda(), torch.from_numpy(k).cuda()
            n = [0]

            def call():
                s, d = frames[n[0] % frames_n]
                n[0] += 1
                hevcdsp.hevc_sao_plane_device(dev, depth, d, W * bps, s, W * bps, W, H, 6, hs, vs, dg, g.shape[1],
                                              dk if only is None else None, k.shape[1], 2)
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
            del frames, s0
            torch.cuda.empty_cache()
    dev.close()


if __name__ == "__main__":
    main()
