"""Timing of two builds of libb200dsp.so side by side: the H.264 residual adds (b200_h264_idct_batch_device, b200_h264_idct_hbd_batch_device)
and emulated_edge_mc (b200_emulated_edge_mc_batch_device, b200_emulated_edge_mc_hbd_batch_device) on cuda:0.

    python scripts/bench_h264_residual_edge.py --lib before=PATH --lib after=PATH [--runs 12] [--steps 10]

Residual adds: bench.py's h264_idct set-up, a block on every 4x4 or 8x8 cell of 32 1920x1088 luma planes, coefficients refilled and
evicted from L2 before every timed call and CUDA events around the call alone; all four kinds at 8 bit and at 10 bit (int32
coefficients, uint16 samples).  emulated_edge_mc: 98304 windows of 21x21 samples on a 1920x1088 picture, half of them crossing a border,
at 8 and 16 bit; events around `steps` back-to-back calls.  The libraries take turns within each run (the order swaps every run); a run
gives the mean time per call, and the figures are the median and [min-max] over the runs.  Each case is first run once from the same
inputs by every library and the outputs compared bit for bit.  Prints the card name, power limit and max SM clock first."""
import argparse
import ctypes as C
import statistics
import subprocess

import numpy as np

W, H, PLANES = 1920, 1088, 32
NWIN, WIN = 98304, 21


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip()


def open_lib(path, stream):
    L = C.CDLL(path)
    vp = C.c_void_p
    L.b200_device_open.argtypes = [C.POINTER(vp), C.c_int, vp]
    L.b200_h264_idct_batch_device.argtypes = [vp, C.c_int, C.c_int64, vp, vp, vp, vp, C.c_ssize_t]
    L.b200_h264_idct_hbd_batch_device.argtypes = [vp, C.c_int, C.c_int, C.c_int64, vp, vp, vp, vp, C.c_ssize_t]
    edge = [vp, C.c_int64, vp, vp, C.c_ssize_t, vp, vp, C.c_ssize_t, vp, C.c_int, C.c_int]
    L.b200_emulated_edge_mc_batch_device.argtypes = edge
    L.b200_emulated_edge_mc_hbd_batch_device.argtypes = edge
    dev = vp()
    assert L.b200_device_open(C.byref(dev), 0, vp(stream)) == 0, path
    return L, dev


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", required=True, metavar="NAME=PATH")
    ap.add_argument("--runs", type=int, default=12)
    ap.add_argument("--steps", type=int, default=10)
    args = ap.parse_args()
    import torch
    print("card:", card(), flush=True)
    st = torch.cuda.Stream()
    libs = [(s.split("=", 1)[0],) + open_lib(s.split("=", 1)[1], st.cuda_stream) for s in args.lib]
    g = torch.Generator(device="cuda").manual_seed(5)
    p = lambda t: C.c_void_p(t.data_ptr())
    cases = []                                             # (name, reset(), call(L, dev), outputs(), timed with an L2 flush)
    with torch.cuda.stream(st):
        flush = torch.empty(192 << 20, dtype=torch.uint8, device="cuda")
        for depth in (8, 10):
            sdt = torch.uint8 if depth == 8 else torch.int16
            planes0 = torch.randint(0, 1 << depth, (PLANES, H, W), dtype=torch.int32, device="cuda", generator=g).to(sdt)
            planes = planes0.clone()
            for kind, N in ((0, 4), (1, 8), (2, 4), (3, 8)):
                nb = PLANES * (H // N) * (W // N)
                keep = torch.randint(-600, 601, (nb, N * N), dtype=torch.int16 if depth == 8 else torch.int32, device="cuda", generator=g)
                coef = keep.clone()
                bi = torch.arange(nb, device="cuda", dtype=torch.int64)
                per = (H // N) * (W // N)
                fr, r = bi // per, bi % per
                bps = planes.element_size()
                doff = ((fr * (H * W) + (r // (W // N)) * (N * W) + (r % (W // N)) * N) * bps).contiguous()
                boff = (bi * (N * N)).contiguous()

                def call(L, dev, kind=kind, nb=nb, coef=coef, boff=boff, doff=doff, planes=planes, depth=depth, bps=bps):
                    if depth == 8:
                        rc = L.b200_h264_idct_batch_device(dev, kind, nb, p(coef), p(boff), p(planes), p(doff), W)
                    else:
                        rc = L.b200_h264_idct_hbd_batch_device(dev, depth, kind, nb, p(coef), p(boff), p(planes), p(doff), W * bps)
                    assert rc == 0

                def reset(coef=coef, keep=keep, planes=planes, planes0=planes0):
                    coef.copy_(keep)
                    planes.copy_(planes0)
                name = f"{['idct4 add', 'idct8 add', 'idct4 dc add', 'idct8 dc add'][kind]}, {depth} bit, {nb} blocks"
                cases.append((name, reset, call, lambda coef=coef, planes=planes: (coef.clone(), planes.clone()),
                              lambda coef=coef, keep=keep: coef.copy_(keep)))
        rng = np.random.default_rng(7)
        inside = np.stack([rng.integers(0, W - WIN + 1, NWIN // 2), rng.integers(0, H - WIN + 1, NWIN // 2)], 1)
        side = rng.integers(0, 4, NWIN // 2)                 # left, top, right, bottom
        cross = np.stack([rng.integers(-WIN + 1, W, NWIN // 2), rng.integers(-WIN + 1, H, NWIN // 2)], 1)
        cross[side == 0, 0] = rng.integers(-WIN + 1, 0, (side == 0).sum())
        cross[side == 1, 1] = rng.integers(-WIN + 1, 0, (side == 1).sum())
        cross[side == 2, 0] = rng.integers(W - WIN + 1, W, (side == 2).sum())
        cross[side == 3, 1] = rng.integers(H - WIN + 1, H, (side == 3).sum())
        xy = np.concatenate([inside, cross])[rng.permutation(NWIN)]
        geom = torch.from_numpy(np.concatenate([np.full((NWIN, 2), WIN), xy], 1).astype(np.int32)).cuda()
        origin = torch.zeros(NWIN, dtype=torch.int64, device="cuda")
        for bits in (8, 16):
            sdt, bps = (torch.uint8, 1) if bits == 8 else (torch.int16, 2)
            pic = torch.randint(0, 256, (H, W), dtype=torch.int32, device="cuda", generator=g).to(sdt)
            buf = torch.zeros((NWIN * WIN, 32), dtype=sdt, device="cuda")
            boff = torch.arange(NWIN, dtype=torch.int64, device="cuda") * (WIN * 32 * bps)

            def call(L, dev, bits=bits, pic=pic, buf=buf, boff=boff, bps=bps):
                fn = L.b200_emulated_edge_mc_batch_device if bits == 8 else L.b200_emulated_edge_mc_hbd_batch_device
                assert fn(dev, NWIN, p(buf), p(boff), 32 * bps, p(pic), p(origin), W * bps, p(geom), W, H) == 0
            cases.append((f"emulated_edge_mc, {bits} bit, {NWIN} windows of {WIN}x{WIN}", buf.zero_, call,
                          lambda buf=buf: (buf.clone(),), None))
    st.synchronize()

    for name, reset, call, outputs, prep in cases:
        got = []
        for lname, L, dev in libs:
            with torch.cuda.stream(st):
                reset()
                call(L, dev)
                got.append(outputs())
            st.synchronize()
        same = all(torch.equal(a, b) for o in got[1:] for a, b in zip(got[0], o))
        times = {lname: [] for lname, _, _ in libs}
        for run in range(args.runs + 1):                   # run 0 is the warm-up
            order = libs if run % 2 == 0 else libs[::-1]
            for lname, L, dev in order:
                with torch.cuda.stream(st):
                    if prep is None:
                        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        e0.record(st)
                        for _ in range(args.steps):
                            call(L, dev)
                        e1.record(st)
                        evs = [(e0, e1)]
                    else:
                        evs = []
                        for _ in range(args.steps):
                            prep()
                            flush.fill_(1)
                            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                            e0.record(st)
                            call(L, dev)
                            e1.record(st)
                            evs.append((e0, e1))
                st.synchronize()
                if run:
                    times[lname].append(1e3 * sum(a.elapsed_time(b) for a, b in evs) / args.steps)
        cols = "  ".join(f"{lname} {statistics.median(t):9.2f} [{min(t):.2f}-{max(t):.2f}] us" for lname, t in times.items())
        print(f"{name:52s} {cols}  outputs {'identical' if same else 'DIFFER'}", flush=True)


if __name__ == "__main__":
    main()
