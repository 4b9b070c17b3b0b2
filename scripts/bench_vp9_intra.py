"""VP9 intra reconstruction on the device: b200_vp9_intra_recon_frame_device on decoder-shaped frames (tests/vp9intralib.py), one call per
frame against the same ops issued as one call per dependency level (the scheme of the HEVC intra entry: every level's ops depend only on
earlier levels), the two forms alternated in one run.  Per frame it prints the op count, the longest dependency chain computed from the
ops, the median frame time of both forms (CUDA events, inputs evicted from L2 before every call) and the time per chain step.  The GPU's
name and power limit are read in the same run.

    python scripts/bench_vp9_intra.py [--reps 15] [--out file.json]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)

import vp9intralib as vi  # noqa: E402

# IntraPredMode after mode_conv: what the mode reads (check_intra_mode's edges[]): left, top, top-left, top-right
NEEDS = {0: "t", 1: "l", 2: "lt", 3: "tr", 4: "ltx", 5: "ltx", 6: "ltx", 7: "tr", 8: "l", 9: "ltx", 10: "l", 11: "t", 12: "", 13: "", 14: ""}


def conv(m, hl, ht):
    if m in (0, 3, 7):
        return m if ht else 13
    if m in (1, 8):
        return m if hl else 14
    if m == 2:
        return (2 if ht else 10) if hl else (11 if ht else 12)
    if m == 9:
        return (9 if ht else 1) if hl else (0 if ht else 14)
    return m


def levels(f):
    """each op's dependency level (1 + the largest level of the earlier ops that write a 4x4 cell its mode reads)"""
    owner = [np.full((f.H[p] // 4, f.W[p] // 4), -1, np.int64) for p in range(3)]
    lev = np.zeros(len(f.ops), np.int64)
    o = f.ops
    for k in range(len(o)):
        p, x, y, t, fl = int(o["plane"][k]), int(o["x"][k]), int(o["y"][k]), int(o["tx"][k]), int(o["flags"][k])
        n, ht, hl, hr = 4 << t, y > 0, bool(fl & 1), bool(fl & 2)
        need = NEEDS[conv(int(o["mode"][k]), hl, ht)]
        nh, nv = f.W[p] - x, f.H[p] - y
        cells = []
        if "t" in need and ht:
            x1 = x + min(n, nh) - 1
            if n == 4 and "r" in need and hr and nh >= 8:
                x1 = x + 7
            cells += [((y - 1) >> 2, c) for c in range(x >> 2, (x1 >> 2) + 1)]
        if "x" in need and ht and hl:
            cells.append(((y - 1) >> 2, (x - 1) >> 2))
        if "l" in need and hl:
            cells += [(r, (x - 1) >> 2) for r in range(y >> 2, ((y + min(n, nv) - 1) >> 2) + 1)]
        w = owner[p]
        lv = 0
        for cy, cx in cells:
            j = w[cy, cx]
            if j >= 0:
                lv = max(lv, lev[j] + 1)
        lev[k] = lv
        w[y >> 2:min(y + n, f.H[p]) >> 2, x >> 2:min(x + n, f.W[p]) >> 2] = k
    return lev


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    import ffmpeg_b200 as fb
    from ffmpeg_b200 import vp9dsp
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    print("gpu:", gpu)
    dev = fb.Device(0)
    dev.set_default()
    st = torch.cuda.ExternalStream(dev.stream)
    scrub = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")     # 256 MB: more than the 50 MB L2
    cases = [(f"{w}x{h} {d}-bit 4:2:0 {sz}", dict(seed=s, depth=d, fmt="420", width=w, height=h, sizes=sz))
             for s, (w, h) in enumerate(((1920, 1080), (3840, 2160))) for d in (8, 10) for sz in ("4x4", "mixed")]
    cases.append(("1920x1080 8-bit 4:2:0 inter, ~10% intra", dict(seed=9, depth=8, fmt="420", width=1920, height=1080, kind="inter",
                                                                  p_intra=0.1)))
    results = []
    with torch.cuda.stream(st):
        for name, kw in cases:
            f = vi.Frame(kw.pop("seed") + 50, kw.pop("depth"), kw.pop("fmt"), kw.pop("width"), kw.pop("height"), **kw)
            lev = levels(f)
            order = np.argsort(lev, kind="stable")
            bounds = np.searchsorted(lev[order], np.arange(lev.max() + 2))
            ts = [torch.from_numpy(p.view(np.int16) if p.dtype == np.uint16 else p).cuda() for p in f.planes]
            ptrs = [t.data_ptr() + vi.MARGIN * p.strides[0] + vi.MARGIN * p.itemsize for t, p in zip(ts, f.planes)]
            one = torch.from_numpy(np.ascontiguousarray(f.ops).view(np.uint8)).cuda()
            byl = torch.from_numpy(np.ascontiguousarray(f.ops[order]).view(np.uint8)).cuda()
            coef = torch.from_numpy(f.coef).cuda()
            ls_y, ls_uv = f.strides()

            def call_one():
                vp9dsp.vp9_intra_recon_frame_device(dev, f.depth, f.ss_h, f.ss_v, f.width, f.height, ptrs, ls_y, ls_uv, len(f.ops), one, coef)

            def call_levels():
                for a, b in zip(bounds[:-1], bounds[1:]):
                    if b > a:
                        vp9dsp.vp9_intra_recon_frame_device(dev, f.depth, f.ss_h, f.ss_v, f.width, f.height, ptrs, ls_y, ls_uv, int(b - a),
                                                            byl.data_ptr() + 32 * int(a), coef)
            # both forms give the checker's frame
            want = vi.orc_frame(f)
            for fn in (call_one, call_levels):
                for t, p in zip(ts, f.planes):
                    t.copy_(torch.from_numpy(p.view(np.int16) if p.dtype == np.uint16 else p))
                fn()
                dev.sync()
                got = [t.cpu().numpy().view(p.dtype) for t, p in zip(ts, f.planes)]
                assert all(np.array_equal(a, b) for a, b in zip(got, want)), (name, fn.__name__)
            times = {"one": [], "levels": []}
            for r in range(args.reps + 2):
                for key, fn in (("one", call_one), ("levels", call_levels)) if r % 2 == 0 else (("levels", call_levels), ("one", call_one)):
                    scrub.zero_()
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record(st)
                    fn()
                    e1.record(st)
                    e1.synchronize()
                    if r >= 2:
                        times[key].append(e0.elapsed_time(e1) * 1000.0)
            chain = int(lev.max()) + 1
            one_us, lev_us = float(np.median(times["one"])), float(np.median(times["levels"]))
            row = {"frame": name, "ops": int(len(f.ops)), "chain": chain, "one_call_us": round(one_us, 1),
                   "one_call_spread_us": [round(min(times["one"]), 1), round(max(times["one"]), 1)], "per_level_us": round(lev_us, 1),
                   "per_level_calls": int((np.diff(bounds) > 0).sum()), "us_per_chain_step": round(one_us / chain, 3),
                   "speedup": round(lev_us / one_us, 2)}
            print(json.dumps(row))
            results.append(row)
    from ffmpeg_b200 import vp9dsp as v
    out = {"gpu": gpu, "reps": args.reps, "timeouts": v.vp9_intra_timeouts(dev), "results": results}
    print(json.dumps({"gpu": gpu, "timeouts": out["timeouts"]}))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        json.dump(out, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()
