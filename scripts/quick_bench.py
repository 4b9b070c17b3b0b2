#!/usr/bin/env python
"""Time one path quickly on the GPU box: python scripts/quick_bench.py qpel|idct|sws|lut|tx|esa [reps]"""
import json, os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
import ffmpeg_b200 as fb
from ffmpeg_b200 import swscale as sw, idctdsp, pel, tx, me_cmp

what = sys.argv[1]
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 10
stream = torch.cuda.Stream()
dev = fb.Device(0, stream=stream.cuda_stream)
g = torch.Generator(device="cuda"); g.manual_seed(1)


def hbm_peak():
    """the peak bench.py divides by: MEASURED_PEAKS.json hbm_gbs, else the H100 SXM data sheet (3.35 TB/s)"""
    try:
        return float(json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"])
    except Exception:
        return 3350.0


PEAK_GBS = hbm_peak()


def timed(call, n_units, unit, bytes_per_unit=None):
    with torch.cuda.stream(stream):
        for _ in range(3):
            call()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(reps):
            call()
        e1.record(stream)
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    line = f"{what}: {n_units / ms / 1e6:.3f} G{unit}/s  ({ms:.3f} ms)"
    if bytes_per_unit:
        line += f"  {n_units * bytes_per_unit / ms / 1e6:.0f} GB/s = {n_units * bytes_per_unit / ms / 1e6 / PEAK_GBS:.3f} of peak"
    print(line)


with torch.cuda.stream(stream):
    if what == "qpel":
        nfr, W, H, ap = 64, 1920, 1088, 32
        PW, PH = W + 2 * ap, H + 2 * ap
        refp = torch.randint(0, 256, (nfr, PH, PW), dtype=torch.uint8, device="cuda", generator=g)
        dstp = torch.randint(0, 256, (nfr, PH, PW), dtype=torch.uint8, device="cuda", generator=g)
        fi = torch.arange(nfr, device="cuda").view(-1, 1, 1)
        by = torch.arange(H // 16, device="cuda").view(1, -1, 1); bx = torch.arange(W // 16, device="cuda").view(1, 1, -1)
        base = fi * (PH * PW) + (by * 16 + ap) * PW + bx * 16 + ap
        dx = torch.randint(-16, 17, base.shape, device="cuda", generator=g); dy = torch.randint(-16, 17, base.shape, device="cuda", generator=g)
        doff = base.reshape(-1).to(torch.int64).contiguous(); soff = (base + dy * PW + dx).reshape(-1).to(torch.int64).contiguous()
        ops = (torch.randint(0, 2, (doff.numel(),), device="cuda", generator=g) | (torch.randint(0, 16, (doff.numel(),), device="cuda", generator=g) << 3)).to(torch.uint8)
        n = doff.numel()
        timed(lambda: pel.h264qpel_batch_device(dev, n, ops, dstp, doff, refp, soff, PW), n, "blocks", 825)
    elif what == "chroma":
        nfr, W, H, ap = 128, 960, 544, 16
        PW, PH = W + 2 * ap, H + 2 * ap
        refp = torch.randint(0, 256, (nfr, PH, PW), dtype=torch.uint8, device="cuda", generator=g)
        dstp = torch.randint(0, 256, (nfr, PH, PW), dtype=torch.uint8, device="cuda", generator=g)
        fi = torch.arange(nfr, device="cuda").view(-1, 1, 1)
        by = torch.arange(H // 8, device="cuda").view(1, -1, 1); bx = torch.arange(W // 8, device="cuda").view(1, 1, -1)
        base = fi * (PH * PW) + (by * 8 + ap) * PW + bx * 8 + ap
        dx = torch.randint(-8, 9, base.shape, device="cuda", generator=g); dy = torch.randint(-8, 9, base.shape, device="cuda", generator=g)
        doff = base.reshape(-1).to(torch.int64).contiguous(); soff = (base + dy * PW + dx).reshape(-1).to(torch.int64).contiguous()
        n = doff.numel()
        ops = torch.randint(0, 2, (n,), device="cuda", generator=g).to(torch.uint8)
        hs = torch.full((n,), 8, dtype=torch.uint8, device="cuda")
        xys = torch.randint(0, 64, (n,), device="cuda", generator=g).to(torch.uint8)
        timed(lambda: pel.h264chroma_batch_device(dev, n, ops, hs, xys, dstp, doff, refp, soff, PW), n, "blocks", 177)
    elif what == "scale":
        W, H, B = 3840, 2160, 32
        Y = torch.randint(0, 256, (B, H, W), dtype=torch.uint8, device="cuda", generator=g)
        U = torch.randint(0, 256, (B, H // 2, W // 2), dtype=torch.uint8, device="cuda", generator=g)
        V = torch.randint(0, 256, (B, H // 2, W // 2), dtype=torch.uint8, device="cuda", generator=g)
        FATE = 4 | 0x40000 | 0x80000
        for (dw, dh, fmt, name) in ((1920, 1080, 0, "4k->1080p yuv420p"), (1920, 1080, 2, "4k->1080p rgb24"), (1280, 720, 0, "4k->720p yuv420p")):
            what = "scale " + name
            ctx = sw.sws_getContext(dev, W, H, 0, dw, dh, fmt, FATE)
            if fmt == 0:
                oY = torch.empty((B, dh, dw), dtype=torch.uint8, device="cuda")
                oU = torch.empty((B, dh // 2, dw // 2), dtype=torch.uint8, device="cuda"); oV = torch.empty_like(oU)
                call = lambda: ctx.scale_batch_device_planar([Y, U, V], [W, W // 2, W // 2], [W * H, W * H // 4, W * H // 4], [oY, oU, oV],
                                                             [dw, dw // 2, dw // 2], [dw * dh, dw * dh // 4, dw * dh // 4], B)
                ob = dw * dh * 3 // 2
            else:
                o = torch.empty((B, dh, dw * 3), dtype=torch.uint8, device="cuda")
                call = lambda: ctx.scale_batch_device([Y, U, V], [W, W // 2, W // 2], [W * H, W * H // 4, W * H // 4], o, dw * 3, dw * dh * 3, B)
                ob = dw * dh * 3
            timed(call, B, "frames", W * H * 3 // 2 + ob)
            ctx.free()
    elif what == "e2e":
        import time
        W, H, B = 3840, 2160, 256
        sys.path.insert(0, ROOT)
        import bench
        bind = os.environ.get("E2E_BIND", "1") == "1"
        ctxm = bench.near_gpu(0) if bind else bench.near_gpu.__new__(bench.near_gpu)
        if not bind:
            ctxm.cpus = None
        print("bind:", bind, "cpus:", len(ctxm.cpus) if ctxm.cpus else None)
        ctxm.__enter__()
        hY = torch.randint(0, 256, (B, H, W), dtype=torch.uint8).pin_memory()
        hU = torch.randint(0, 256, (B, H // 2, W // 2), dtype=torch.uint8).pin_memory()
        hV = torch.randint(0, 256, (B, H // 2, W // 2), dtype=torch.uint8).pin_memory()
        hO = torch.empty((B, H, W * 3), dtype=torch.uint8).pin_memory()
        hO.zero_()
        ctxm.__exit__()
        ctx = sw.sws_getContext(dev, W, H, 0, W, H, 2, 4 | 0x40000 | 0x80000)
        call = lambda: ctx.scale_batch_host([hY.data_ptr(), hU.data_ptr(), hV.data_ptr()], [W, W // 2, W // 2],
                                            [W * H, W * H // 4, W * H // 4], hO.data_ptr(), W * 3, W * H * 3, B)
        call()
        t0 = time.perf_counter()
        for _ in range(reps):
            call()
        torch.cuda.synchronize()
        dt = (time.perf_counter() - t0) / reps
        print(f"e2e: {B / dt:.1f} frames/s  ({dt * 1e3:.1f} ms per 256-frame step, D2H {B * W * H * 3 / dt / 1e9:.1f} GB/s, H2D {B * W * H * 1.5 / dt / 1e9:.1f} GB/s)")
        dY, dU, dV = hY[:2].cuda(), hU[:2].cuda(), hV[:2].cuda()
        o = torch.empty((2, H, W * 3), dtype=torch.uint8, device="cuda")
        ctx.scale_batch_device([dY, dU, dV], [W, W // 2, W // 2], [W * H, W * H // 4, W * H // 4], o, W * 3, W * H * 3, 2)
        dev.sync()
        print("matches device path:", bool(torch.equal(o.cpu(), hO[:2])))
    elif what == "idct":
        mbw, mbh, fr = 120, 68, 256
        n = mbw * mbh * 6 * fr
        blk = torch.randint(-256, 257, (n, 64), dtype=torch.int16, device="cuda", generator=g)
        pl = [torch.zeros((fr, mbh * 16, mbw * 16), dtype=torch.uint8, device="cuda"), torch.zeros((fr, mbh * 8, mbw * 8), dtype=torch.uint8, device="cuda"),
              torch.zeros((fr, mbh * 8, mbw * 8), dtype=torch.uint8, device="cuda")]
        for kind, name, b in ((1, "put", 192), (2, "add", 256)):
            what = "idct_" + name
            timed(lambda: idctdsp.idct_mb420_device(dev, kind, blk, mbw, mbh, fr, pl, [mbw * 16, mbw * 8, mbw * 8],
                                                    [mbw * 16 * mbh * 16, mbw * 8 * mbh * 8, mbw * 8 * mbh * 8]), n, "blocks", b)
    elif what in ("sws", "lut"):
        W, H, nf = 3840, 2160, 128
        Y = torch.randint(0, 256, (nf, H, W), dtype=torch.uint8, device="cuda", generator=g)
        U = torch.randint(0, 256, (nf, H // 2, W // 2), dtype=torch.uint8, device="cuda", generator=g)
        V = torch.randint(0, 256, (nf, H // 2, W // 2), dtype=torch.uint8, device="cuda", generator=g)
        O = torch.empty((nf, H, W * 3), dtype=torch.uint8, device="cuda")
        c = sw.sws_getContext(dev, W, H, 0, W, H, 2, (4 | 0x40000 | 0x80000) if what == "sws" else 4)
        timed(lambda: c.scale_batch_device([Y, U, V], [W, W // 2, W // 2], [W * H, W * H // 4, W * H // 4], O, W * 3, W * H * 3, nf), nf, "frames", 37324800)
    elif what == "tx":
        for n in [int(v) for v in os.environ.get("QB_TX_SIZES", "1024,2048").split(",")]:
            cnt = (1 << 28) // (2 * n)
            x = torch.rand((cnt, 2 * n), device="cuda", generator=g); y = torch.empty_like(x)
            c = tx.av_tx_init(0, 0, n, device=dev); what = f"fft{n}"
            timed(lambda: c.batch_device(y, x, 8, cnt, 8 * n, 8 * n), cnt, "tx", 16 * n); c.uninit()
            c = tx.av_tx_init(1, 1, n, scale=1.0 / n, device=dev); what = f"imdct{n}"
            timed(lambda: c.batch_device(y, x, 4, cnt, 4 * n, 4 * n), cnt, "tx", 8 * n); c.uninit()
    elif what == "h264":
        Hh, Wh, hn = 1088, 1920, 32
        planes_h = torch.randint(0, 256, (hn, Hh, Wh), dtype=torch.uint8, device="cuda", generator=g)
        for kind, N in ((0, 4), (1, 8)):
            nb = hn * (Hh // N) * (Wh // N)
            coef = torch.randint(-600, 601, (nb, N * N), dtype=torch.int16, device="cuda", generator=g)
            bi = torch.arange(nb, device="cuda", dtype=torch.int64)
            per = (Hh // N) * (Wh // N)
            fr, r = bi // per, bi % per
            hdoff = (fr * (Hh * Wh) + (r // (Wh // N)) * (N * Wh) + (r % (Wh // N)) * N).contiguous()
            hboff = (bi * (N * N)).contiguous()
            what = f"h264 idct{N} add (coefficients left cleared: dc-free blocks after the first pass)"
            timed(lambda: idctdsp.h264_idct_batch_device(dev, kind, nb, coef, hboff, planes_h, hdoff, Wh), nb, "blocks", 2 * N * N * 2 + 2 * N * N)
    elif what == "esa":
        W, H, npairs = 3840, 2160, 4
        cur = torch.randint(0, 256, (npairs, H, W), dtype=torch.uint8, device="cuda", generator=g)
        ref = torch.roll(cur, shifts=(7, -13), dims=(1, 2)).contiguous()
        nmb = (W // 16) * (H // 16)
        mv = torch.zeros((npairs, nmb, 2), dtype=torch.int32, device="cuda"); cost = torch.zeros((npairs, nmb), dtype=torch.int64, device="cuda")
        timed(lambda: me_cmp.me_esa_device(dev, cur, ref, W, W, H, W * H, npairs, 16, 32, mv, cost), npairs, "pairs")
    elif what == "fdct":
        from ffmpeg_b200 import fdctdsp
        nb = 4 * 1024 * 1024                                    # 512 MB of coefficients: larger than L2
        blocks = torch.randint(-255, 256, (nb, 64), dtype=torch.int16, device="cuda", generator=g)
        for algo, bits, is248, name in ((0, 8, 0, "islow_8"), (1, 8, 0, "ifast"), (0, 10, 0, "islow_10"), (0, 8, 1, "islow_8 2-4-8")):
            what = f"fdct {name} (in place: 128 B read + 128 B written per block)"
            timed(lambda: fdctdsp.fdct_batch_device(dev, blocks, nb, algo, bits, is248), nb, "blocks", 256)
    elif what == "dctcmp":
        W, H = 3840, 2160
        f1 = torch.randint(0, 256, (H, W), dtype=torch.uint8, device="cuda", generator=g)
        f2 = torch.randint(0, 256, (H, W), dtype=torch.uint8, device="cuda", generator=g)
        n = 2 * 1024 * 1024
        o1 = (torch.randint(0, H - 16, (n,), device="cuda", generator=g) * W + torch.randint(0, W - 16, (n,), device="cuda", generator=g)).to(torch.int64)
        o2 = (torch.randint(0, H - 16, (n,), device="cuda", generator=g) * W + torch.randint(0, W - 16, (n,), device="cuda", generator=g)).to(torch.int64)
        out = torch.zeros(n, dtype=torch.int32, device="cuda")
        for fn, name in ((8, "dct_sad"), (9, "dct_max"), (10, "dct264_sad"), (3, "hadamard8_diff")):
            what = f"me_cmp {name}16 (h = 16, random offsets in a 4K frame pair)"
            timed(lambda: me_cmp.me_cmp_batch_device(dev, fn, 0, f1, f2, W, 16, o1, o2, n, out), n, "cmp")
dev.close()
