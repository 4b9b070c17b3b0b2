"""Times b200_hevc_intra_recon_picture_device (one call per picture) against the per-level path of the batch entries (per plane and
dependency level, b200_hevc_intra_pred_batch_device then b200_hevc_transform_add_batch_device) on the same decoder-shaped 4:2:0 pictures:
1080p and 4K intra pictures at 8 and 10 bit with every TU kind, and a 1080p inter picture with a fifth of its CUs intra.  Both forms are
checked against the checker first, then timed alternately (CUDA events, L2 scrubbed before every call).  Per picture: ops, the longest
dependency chain over the planes, the per-level path's levels and launches, the median time of both forms and the one-call time per
dependency step.  The GPU's name and power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)

import hevcintralib as hl  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=9)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    import ffmpeg_b200 as fb
    from ffmpeg_b200 import hevcdsp
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    print("gpu:", gpu)
    dev = fb.Device(0)
    dev.set_default()
    st = torch.cuda.ExternalStream(dev.stream)
    scrub = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")     # 256 MB: more than the 50 MB L2
    cases = [(f"{w}x{h} {d}-bit 4:2:0 intra", dict(seed=s, depth=d, W=w, H=h)) for s, (w, h) in enumerate(((1920, 1080), (3840, 2160)))
             for d in (8, 10)]
    cases.append(("1920x1080 8-bit 4:2:0 inter, 20% intra CUs", dict(seed=9, depth=8, W=1920, H=1080, p_intra=0.2)))
    results = []

    def dev_t(a):
        return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8)).cuda()

    with torch.cuda.stream(st):
        for name, kw in cases:
            p = hl.picture(kw.pop("seed") + 40, kw.pop("depth"), 1, kw.pop("W"), kw.pop("H"), 6, nslices=4, split=0.6, **kw)
            bufs = p.framed()
            ts = [torch.from_numpy(b.view(np.int16) if b.dtype == np.uint16 else b).cuda() for b in bufs]
            ptrs = [t.data_ptr() + hl.MARGIN * b.strides[0] + hl.MARGIN * b.itemsize for t, b in zip(ts, bufs)]
            ls_y, ls_uv = p.strides(bufs)
            ops, coef = dev_t(p.ops), torch.from_numpy(p.coef).cuda()
            calls = []
            for c, io, idx in hl.level_batches(p):
                hs, vs = p.shifts(c)
                tu = hl.level_tu_ops(p, idx, bufs[c].strides[0])
                calls.append((c, hs, vs, len(io), dev_t(io), len(tu), dev_t(tu) if len(tu) else None))
            levels = [sum(1 for c in calls if c[0] == k) for k in range(3)]
            launches = sum(1 + (c[5] > 0) for c in calls)

            def call_one():
                hevcdsp.hevc_intra_recon_picture_device(dev, p.depth, 1, p.W, p.H, ptrs, ls_y, ls_uv, len(p.ops), ops, coef)

            def call_levels():
                for c, hs, vs, n, io, ntu, tu in calls:
                    s = bufs[c].strides[0]
                    hevcdsp.hevc_intra_pred_batch_device(dev, p.depth, ptrs[c], s, p.W, p.H, hs, vs, n, io)
                    if ntu:
                        hevcdsp.hevc_transform_add_batch_device(dev, p.depth, ntu, tu, coef, ptrs[c], s)
            want = hl.orc_picture(p)
            for fn in (call_one, call_levels):
                for t, b in zip(ts, bufs):
                    t.copy_(torch.from_numpy(b.view(np.int16) if b.dtype == np.uint16 else b))
                fn()
                dev.sync()
                got = [t.cpu().numpy().view(b.dtype) for t, b in zip(ts, bufs)]
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
            chain = max(levels)
            one_us, lev_us = float(np.median(times["one"])), float(np.median(times["levels"]))
            row = {"picture": name, "ops": int(len(p.ops)), "levels_y_cb_cr": levels, "per_level_launches": launches,
                   "one_call_us": round(one_us, 1), "one_call_spread_us": [round(min(times["one"]), 1), round(max(times["one"]), 1)],
                   "per_level_us": round(lev_us, 1), "us_per_dependency_step": round(one_us / chain, 3), "speedup": round(lev_us / one_us, 2)}
            print(json.dumps(row))
            results.append(row)
    out = {"gpu": gpu, "reps": args.reps, "timeouts": hevcdsp.hevc_intra_timeouts(dev), "results": results}
    print(json.dumps({"gpu": gpu, "timeouts": out["timeouts"]}))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        json.dump(out, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()
