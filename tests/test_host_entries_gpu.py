"""GPU tier: the pipelined HOST-buffer entry points (what bench.py's e2e legs time) against the oracle: b200_tx_batch_host,
b200_h264qpel_frames_host, b200_me_esa_host.  The tx and qpel batches span several chunks and every pipeline slot; the 5 frames of
the search fit in one chunk (several chunks and a reused slot: tests/test_me_search_gpu.py)."""
import ctypes as C

import numpy as np
import pytest

import cpulibs as cl

pytestmark = pytest.mark.gpu


def test_tx_batch_host_vs_oracle(device):
    from ffmpeg_b200 import tx
    O = cl.oracle()
    rng = np.random.default_rng(77)

    def orc(typ, inv, n, scale, x, of):
        h = O.orc_tx_open(typ, inv, n, scale, 0)
        out = np.zeros((x.shape[0], of), np.float32)
        O.orc_tx_run(h, out.ctypes.data, x.ctypes.data, 8 if typ == 0 else 4, x.shape[0], out.strides[0], x.strides[0])
        O.orc_tx_close(h)
        return out
    for n, cnt in ((1024, 7000), (2048, 2500), (64, 11)):          # 7000 x 16 KB = 4 chunks of 48 MB staging
        x = rng.random((cnt, 2 * n), dtype=np.float32)
        c = tx.av_tx_init(tx.AV_TX_FLOAT_FFT, 0, n, device=device)
        out = np.zeros_like(x)
        c.batch_host(out, x, 8, cnt, 8 * n, 8 * n)
        assert np.array_equal(out, orc(0, 0, n, 1.0, x, 2 * n)), ("fft", n)
        c.uninit()
        xi = np.ascontiguousarray(x[:, :n])
        c = tx.av_tx_init(tx.AV_TX_FLOAT_MDCT, 1, n, scale=1.0 / n, device=device)
        out = np.zeros((cnt, n), np.float32)
        c.batch_host(out, xi, 4, cnt, 4 * n, 4 * n)
        assert np.array_equal(out, orc(1, 1, n, 1.0 / n, xi, n)), ("imdct", n)
        assert c.batch_host(out, xi, 4, 0, 4 * n, 4 * n) == 0       # empty batch
        c.uninit()


def test_h264qpel_frames_host_vs_oracle(device):
    from ffmpeg_b200 import pel
    O = cl.oracle()
    rng = np.random.default_rng(78)
    W, H, nfr = 352, 288, 700                                       # 700 frames x 2 x 101 KB: several chunks
    fb = W * H
    src = rng.integers(0, 256, (nfr, H, W), dtype=np.uint8)
    dst = rng.integers(0, 256, (nfr, H, W), dtype=np.uint8)
    exp = dst.copy()
    ops, doffs, soffs, begin = [], [], [], [0]
    for f in range(nfr):
        k = int(rng.integers(0, 40)) if f % 50 else 0               # some frames have no operation at all
        used = set()
        for _ in range(k):
            by, bx = int(rng.integers(1, H // 16 - 1)), int(rng.integers(1, W // 16 - 1))
            if (by, bx) in used:
                continue
            used.add((by, bx))
            op = pel.qpel_op(int(rng.integers(0, 2)), int(rng.integers(0, 3)), int(rng.integers(0, 16)))
            dx, dy = (int(v) for v in rng.integers(-10, 11, 2))
            ops.append(op); doffs.append(f * fb + by * 16 * W + bx * 16); soffs.append(f * fb + (by * 16 + dy) * W + bx * 16 + dx)
        begin.append(len(ops))
    ops_a, do_a, so_a, bg = np.array(ops, np.uint8), np.array(doffs, np.int64), np.array(soffs, np.int64), np.array(begin, np.int64)
    e8, s8 = exp.reshape(-1), src.reshape(-1)
    for op, do, so in zip(ops, doffs, soffs):
        O.orc_h264qpel(op & 1, (op >> 1) & 3, (op >> 3) & 15, C.cast(e8.ctypes.data + do, cl.u8p), C.cast(s8.ctypes.data + so, cl.u8p), W)
    pel.h264qpel_frames_host(device, nfr, fb, bg, ops_a, dst, do_a, src, so_a, W)
    assert np.array_equal(dst, exp), int((dst != exp).sum())


def test_me_esa_host_vs_oracle_and_device(device):
    from ffmpeg_b200 import me_cmp
    O = cl.oracle()
    rng = np.random.default_rng(79)
    nf, W, H, mb, sp = 5, 320, 192, 16, 16
    cur = rng.integers(0, 256, (nf, H, W), dtype=np.uint8)
    ref_ = np.stack([np.roll(cur[i], (3 - 2 * i, -4 + 3 * i), (0, 1)) for i in range(nf)])
    ref_ = (ref_.astype(np.int16) + rng.integers(-2, 3, ref_.shape)).clip(0, 255).astype(np.uint8)
    bw, bh = W // mb, H // mb
    mv = np.zeros((nf, bw * bh, 2), np.int32)
    cost = np.zeros((nf, bw * bh), np.uint64)
    me_cmp.me_esa_host(device, cur, ref_, W, W, H, W * H, nf, mb, sp, mv, cost)
    for i in range(nf):
        emv, ec = np.zeros((bh * bw, 2), np.int32), np.zeros(bh * bw, np.uint64)
        O.orc_esa_frame(cl.ptr(cur[i]), cl.ptr(ref_[i]), W, W, H, mb, sp, 0, bh, cl.ptr(emv, cl.i32p), cl.ptr(ec, cl.u64p))
        assert np.array_equal(mv[i], emv) and np.array_equal(cost[i], ec), i
