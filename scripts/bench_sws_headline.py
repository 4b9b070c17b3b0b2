#!/usr/bin/env python
"""The headline swscale workload of bench.py (256 x 4K yuv420p -> rgb24, FATE flags) timed on its own, beside the nv12-source
and rgba-output variants and plain streaming moves of the same byte volumes (the bandwidth the card reaches at all).

    python scripts/bench_sws_headline.py [--root DIR ...] [--rounds 3] [--seconds 2]

Every --root names a tree whose ffmpeg_b200 is imported (default: this one); with several, the trees are timed one after the
other, round after round, so that a difference between two builds is measured on the same card under the same conditions.
Each measurement runs in a process of its own.  Printed: the card, its power limit and maximum SM clock (read only), then
median / min / max over the rounds of frames/s, GB/s over the algorithmic bytes and the fraction of the 3.35 TB/s data sheet
and of the best streaming move."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
W4K, H4K, BATCH = 3840, 2160, 256
FRAME_IN, FRAME_OUT = W4K * H4K * 3 // 2, W4K * H4K * 3
FRAME_BYTES = FRAME_IN + FRAME_OUT               # 37 324 800 B / frame
FRAME_BYTES_RGBA = FRAME_IN + W4K * H4K * 4
FATE = 4 | 0x40000 | 0x80000                     # SWS_BICUBIC | SWS_ACCURATE_RND | SWS_BITEXACT
DATASHEET_GBS = 3350.0                           # H100 SXM, HBM3


def timed(call, seconds, warmup=3):
    """CUDA-event time of back-to-back calls over a window of at least `seconds`; returns (calls, ms)"""
    import torch
    for _ in range(warmup):
        call()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    call()
    e1.record()
    e1.synchronize()
    n = max(3, int(seconds * 1e3 / max(e0.elapsed_time(e1), 1e-3)) + 1)
    e0.record()
    for _ in range(n):
        call()
    e1.record()
    e1.synchronize()
    return n, e0.elapsed_time(e1)


def child_sws(root, seconds):
    sys.path.insert(0, root)
    import torch
    import ffmpeg_b200 as fb
    from ffmpeg_b200 import swscale as sw
    assert os.path.dirname(os.path.abspath(fb.__file__)) == os.path.join(os.path.abspath(root), "ffmpeg_b200"), fb.__file__
    stream = torch.cuda.Stream()
    dev = fb.Device(0, stream=stream.cuda_stream)
    out = {}
    with torch.cuda.stream(stream):
        g = torch.Generator(device="cuda")
        g.manual_seed(1)                                     # the inputs of bench.py
        Y = torch.randint(0, 256, (BATCH, H4K, W4K), dtype=torch.uint8, device="cuda", generator=g)
        U = torch.randint(0, 256, (BATCH, H4K // 2, W4K // 2), dtype=torch.uint8, device="cuda", generator=g)
        V = torch.randint(0, 256, (BATCH, H4K // 2, W4K // 2), dtype=torch.uint8, device="cuda", generator=g)
        UV = torch.stack((U, V), dim=3).reshape(BATCH, H4K // 2, W4K).contiguous()
        OUT = torch.empty((BATCH, H4K, W4K * 3), dtype=torch.uint8, device="cuda")
        OUT4 = torch.empty((BATCH, H4K, W4K * 4), dtype=torch.uint8, device="cuda")
        for name, src_fmt, fmt, planes, strides, fstrides, o, bpf in (
                ("yuv420p->rgb24", sw.AV_PIX_FMT_YUV420P, sw.AV_PIX_FMT_RGB24, [Y, U, V], [W4K, W4K // 2, W4K // 2],
                 [W4K * H4K, W4K * H4K // 4, W4K * H4K // 4], OUT, FRAME_BYTES),
                ("nv12->rgb24", sw.AV_PIX_FMT_NV12, sw.AV_PIX_FMT_RGB24, [Y, UV], [W4K, W4K], [W4K * H4K, W4K * H4K // 2], OUT, FRAME_BYTES),
                ("yuv420p->rgba", sw.AV_PIX_FMT_YUV420P, sw.AV_PIX_FMT_RGBA, [Y, U, V], [W4K, W4K // 2, W4K // 2],
                 [W4K * H4K, W4K * H4K // 4, W4K * H4K // 4], OUT4, FRAME_BYTES_RGBA)):
            ctx = sw.sws_getContext(dev, W4K, H4K, src_fmt, W4K, H4K, fmt, FATE)
            bpp = ctx.bpp
            n, ms = timed(lambda: ctx.scale_batch_device(planes, strides, fstrides, o, W4K * bpp, W4K * H4K * bpp, BATCH), seconds)
            ctx.free()
            out[name] = {"fps": n * BATCH / (ms / 1e3), "gbs": n * BATCH * bpf / (ms / 1e3) / 1e9, "calls": n, "ms": ms}
    dev.close()
    return out


def child_probes(seconds):
    """copy_ of the input volume (12.4 MB read + 12.4 MB written per frame), fill_ of the output volume (24.9 MB written),
    and a 1:2 move (12.4 MB read, each 4-byte word written twice: 24.9 MB) over the same 256-frame buffers"""
    import torch
    src = torch.randint(0, 256, (BATCH * FRAME_IN,), dtype=torch.uint8, device="cuda")
    dst_in = torch.empty_like(src)
    dst_out = torch.empty((BATCH * FRAME_OUT,), dtype=torch.uint8, device="cuda")
    s32, d32 = src.view(torch.int32).view(-1, 1), dst_out.view(torch.int32).view(-1, 2)
    res = {}
    for name, call, nbytes in (("copy_ 12.4 MB/frame", lambda: dst_in.copy_(src), 2 * BATCH * FRAME_IN),
                               ("fill_ 24.9 MB/frame", lambda: dst_out.fill_(7), BATCH * FRAME_OUT),
                               ("read:write 1:2", lambda: d32.copy_(s32.expand(-1, 2)), BATCH * (FRAME_IN + FRAME_OUT))):
        n, ms = timed(call, seconds)
        res[name] = {"gbs": n * nbytes / (ms / 1e3) / 1e9, "calls": n, "ms": ms}
    return res


def card():
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip()
    except Exception as ex:
        return f"nvidia-smi unavailable ({ex})"


def stats(v):
    return statistics.median(v), min(v), max(v)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--root", action="append", help="tree to import ffmpeg_b200 from (repeatable; default: this tree)")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--seconds", type=float, default=2.0, help="least length of each timed window")
    ap.add_argument("--child", choices=["sws", "probes"], help=argparse.SUPPRESS)
    ap.add_argument("--json", help="also write every sample to this file")
    args = ap.parse_args()
    if args.child == "sws":
        print(json.dumps(child_sws(args.root[0], args.seconds)))
        return
    if args.child == "probes":
        print(json.dumps(child_probes(args.seconds)))
        return

    roots = [os.path.abspath(r) for r in (args.root or [ROOT])]
    print("card (name, power.limit, clocks.max.sm):", card(), flush=True)
    samples = {r: {} for r in roots}
    probes = {}

    def run(extra):
        r = subprocess.run([sys.executable, os.path.abspath(__file__), "--seconds", str(args.seconds)] + extra, capture_output=True, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout[-2000:] + r.stderr[-4000:])
            raise SystemExit(f"child {extra} failed")
        return json.loads(r.stdout.strip().splitlines()[-1])

    for rnd in range(args.rounds):
        for name, v in run(["--child", "probes"]).items():
            probes.setdefault(name, []).append(v["gbs"])
        for root in roots:
            for name, v in run(["--child", "sws", "--root", root]).items():
                samples[root].setdefault(name, []).append(v)
            print(f"round {rnd}: {root}: " + ", ".join(f"{k} {v[-1]['fps']:.0f} fps" for k, v in samples[root].items()), flush=True)

    print("\nstreaming moves on the same buffers (GB/s, median / min / max):")
    for name, v in probes.items():
        print(f"  {name:22s} {stats(v)[0]:7.0f} / {stats(v)[1]:7.0f} / {stats(v)[2]:7.0f}   {stats(v)[0] / DATASHEET_GBS:.3f} of the data sheet")
    ceiling = max(stats(v)[0] for v in probes.values())
    print(f"  reachable bound: {ceiling:.0f} GB/s = {ceiling / DATASHEET_GBS:.3f} of {DATASHEET_GBS:.0f} GB/s")
    for root in roots:
        print(f"\n{root}:")
        for name, v in samples[root].items():
            f, gb = [s["fps"] for s in v], [s["gbs"] for s in v]
            print(f"  {name:15s} frames/s {stats(f)[0]:8.0f} (min {stats(f)[1]:.0f}, max {stats(f)[2]:.0f})   {stats(gb)[0]:6.0f} GB/s = "
                  f"{stats(gb)[0] / DATASHEET_GBS:.3f} of the data sheet, {stats(gb)[0] / ceiling:.3f} of the streaming bound")
    if len(roots) == 2:
        a, b = roots
        for name in samples[a]:
            fa, fb_ = [s["fps"] for s in samples[a][name]], [s["fps"] for s in samples[b][name]]
            print(f"  {name}: {os.path.basename(b)} / {os.path.basename(a)} median {stats(fb_)[0] / stats(fa)[0]:.3f}, "
                  f"every {os.path.basename(b)} run faster: {min(fb_) > max(fa)}")
    if args.json:
        with open(args.json, "w") as fh:
            json.dump({"card": card(), "probes": probes, "samples": samples}, fh, indent=1)


if __name__ == "__main__":
    main()
