"""HEVC intra prediction on the GPU (b200_hevc_intra_pred_batch_device), timed with CUDA events; prints one JSON line.
(a) independent-op throughput: ops on a 2x2-spaced TU grid (every other TU position in both directions, so that no op reads what
    another writes) over a 3840x2160 luma plane at 8 and 10 bit and a 1920x1080 4:2:0 chroma plane, per size and mixed; bytes from the
    op footprints (the 4 * size + 1 neighbours read, the size^2 samples written, the 16-byte record).  Each call works on the next of
    enough plane copies (with their own op records) that together exceed twice the 50 MB L2, so L2 holds none of a call's inputs.
(b) decoder-shaped intra pictures (1920x1080 and 3840x2160 luma, CTB 32, tests/hevcpredlib.py's quadtrees): one prediction call
    and one BYPASS residual-add call per dependency level; levels, launches and the total time.
The card's name and power limit are read in the same run.  usage: python scripts/bench_hevc_pred.py [--reps N] [--out FILE]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

HBM = 3.35e12


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                              text=True).stdout.strip()
    except OSError:
        return "unknown"


def grid_ops(rng, pw, ph, log2s, luma):
    import hevcpredlib as hl
    out = []
    flags = 0x1F | (hl.INTRA_LUMA | hl.INTRA_SMOOTH | hl.INTRA_STRONG if luma else 0)
    for log2 in log2s:
        s = 1 << log2
        ys, xs = np.mgrid[s:ph - 2 * s + 1:2 * s, s:pw - 2 * s + 1:2 * s]
        o = np.zeros(xs.size, hl.INTRA_DTYPE)
        o["x"], o["y"], o["log2_size"], o["flags"] = xs.ravel(), ys.ravel(), log2, flags
        o["mode"] = rng.integers(0, 35, xs.size)
        out.append(o)
    o = np.concatenate(out)
    if len(log2s) > 1:                                     # mixed: keep only ops whose blocks and footprints do not meet
        taken = np.zeros((ph, pw), bool)
        keep = []
        for k in range(len(o)):
            x, y, s = int(o[k]["x"]), int(o[k]["y"]), 1 << int(o[k]["log2_size"])
            if not taken[y - 1:y + 2 * s, x - 1:x + 2 * s].any():
                taken[y - 1:y + 2 * s, x - 1:x + 2 * s] = True
                keep.append(k)
        o = o[keep]
    return o


def timed(fn, reps):
    import torch
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e3 / reps                   # µs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    import ffmpeg_b200 as fb
    from ffmpeg_b200 import hevcdsp
    import hevcpredlib as hl
    dev = fb.Device(0)
    dev.set_default()
    st = torch.cuda.ExternalStream(dev.stream)
    rng = np.random.default_rng(1)
    res = {"card": card(), "a": {}, "b": {}}
    with torch.cuda.stream(st):
        for name, depth, W, H, hs, vs in (("luma8_3840x2160", 8, 3840, 2160, 0, 0), ("luma10_3840x2160", 10, 3840, 2160, 0, 0),
                                          ("chroma8_1920x1080", 8, 3840, 2160, 1, 1)):
            pw, ph = W >> hs, H >> vs
            bps = 1 if depth == 8 else 2
            plane = torch.randint(0, 1 << depth, (ph, pw), dtype=torch.int32, device="cuda").to(torch.uint8 if depth == 8 else torch.int16)
            for label, log2s in (("4x4", (2,)), ("8x8", (3,)), ("16x16", (4,)), ("32x32", (5,)), ("mixed", (2, 3, 4, 5))):
                o = grid_ops(rng, pw, ph, log2s, hs == 0)
                ncopy = max(2, -(-100_000_000 // (pw * ph * bps + o.nbytes)))
                copies = [(plane.clone(), torch.from_numpy(o.view(np.uint8)).cuda()) for _ in range(ncopy)]
                size = 1 << o["log2_size"].astype(np.int64)
                nbytes = int(((4 * size + 1 + size * size) * bps + 16).sum())
                it = [0]

                def call():
                    pl, do = copies[it[0] % ncopy]
                    it[0] += 1
                    hevcdsp.hevc_intra_pred_batch_device(dev, depth, pl, pw * bps, W, H, hs, vs, len(o), do)
                us = timed(call, max(args.reps, 2 * ncopy))
                del copies
                res["a"][f"{name}_{label}"] = {"ops": len(o), "us": round(us, 2), "bytes": nbytes, "GBps": round(nbytes / us / 1e3, 1),
                                               "hbm_frac": round(nbytes / (us * 1e-6) / HBM, 3)}
        for W, H in ((1920, 1080), (3840, 2160)):
            p = hl.picture_case(7, 8, W, H - H % 8, 5, 0, 0, split=0.5)
            buf = torch.from_numpy(hl.framed(p.plane, 8)).cuda()
            stride = buf.shape[1]
            pix = buf.data_ptr() + hl.MARGIN * stride + hl.MARGIN
            coef, base = hl.packed_residuals(p)
            coef = torch.from_numpy(coef).cuda()
            nl = int(p.levels.max()) + 1
            lv = []
            for k in range(nl):
                sel = np.nonzero(p.levels == k)[0]
                lv.append((len(sel), torch.from_numpy(np.ascontiguousarray(p.ops[sel]).view(np.uint8)).cuda(),
                           torch.from_numpy(hl.tu_ops(p, sel, stride, base).view(np.uint8)).cuda()))

            def picture():
                for n, dops, dtu in lv:
                    hevcdsp.hevc_intra_pred_batch_device(dev, 8, pix, stride, p.W, p.H, 0, 0, n, dops)
                    hevcdsp.hevc_transform_add_batch_device(dev, 8, n, dtu, coef, pix, stride)
            us = timed(picture, max(3, args.reps // 10))
            res["b"][f"luma8_{W}x{H}"] = {"tus": len(p.ops), "levels": nl, "launches": 2 * nl, "us": round(us, 1),
                                          "us_per_launch": round(us / (2 * nl), 2)}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
