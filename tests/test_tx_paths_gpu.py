"""GPU tier: every route b200_tx_batch_device takes for the power-of-two float FFT / MDCT / RDFT, bit for bit against the checker.

Each case is built so that the dispatcher in csrc/tx.cu picks a known kernel, named first in the case id:
  r16    tx_r16_kernel (512 ... 4096-point FFT and inverse MDCT): in and in_step 16-byte aligned, out 8-byte aligned, MDCT stride 4
  level  the level-by-level kernels (tx_fft_kernel, tx_mdct_inv/fwd_kernel, tx_rdft_r2c/c2r_kernel): every other size, or a
         512 ... 4096-point call that r16 refuses (input 8 but not 16-byte aligned, in_step padded by 8 bytes, MDCT stride 8 / 12)
Inputs mix seven classes row by row (uniform, 2^U(-60, 60), subnormal, signed zeros, impulse, constant, near 2^100), all finite.
The gaps out_step leaves between outputs, the rows past `count` and 256 bytes past the batch hold a sentinel that must survive,
and the input must come back unchanged.  Every non-subnormal row is also held to the float64 definition (tests/txref.py)."""
import numpy as np
import pytest

import txref as T

pytestmark = pytest.mark.gpu

SENT = T.SENT
H100_SMS, R16_CTAS_PER_SM = 132, 3         # shared memory holds at most 3 CTAs of tx_r16_kernel per SM
MDCT_SCALES = ("1/len", 1.0, -1.0, -1.0 / 32768, 0.5)


def r16_count(n):
    """transforms enough for four rounds of every thread group of a full r16 grid (n / 16 threads per group), plus an odd tail"""
    return 4 * H100_SMS * R16_CTAS_PER_SM * (256 // (n // 16)) + 7


def level_counts(points):
    """1 transform, partial last CTAs of the 4- and 2-transform CTAs, and a batch with an odd tail"""
    return (1, 2, 3, 5, 301 if points <= 4096 else 37)


def _cases():
    cs = []

    def add(route, kind, inv, ln, counts, stride=4, in_off=0, in_pad=0, out_pad=0, tag=""):
        cid = f"{route}-{kind}-{ln}" + (f"-{tag}" if tag else "")
        cs.append(pytest.param(kind, inv, ln, counts, stride, in_off, in_pad, out_pad, id=cid))
    for n in (512, 1024, 2048, 4096):
        for inv in (0, 1):
            add("r16", "ifft" if inv else "fft", inv, n, (1, r16_count(n)), out_pad=8 * inv)
        add("r16", "imdct", 1, 2 * n, (1, r16_count(n)))
    for lg in range(1, 15):
        n = 1 << lg
        for inv in (0, 1):
            k = "ifft" if inv else "fft"
            if 512 <= n <= 4096:
                add("level", k, inv, n, level_counts(n), in_off=8, tag="in8")
                add("level", k, inv, n, level_counts(n), in_pad=8, out_pad=8, tag="step+8")
            else:
                add("level", k, inv, n, level_counts(n))
    for lg in range(2, 16):
        ln = 1 << lg
        if 1024 <= ln <= 8192:
            add("level", "imdct", 1, ln, level_counts(ln // 2), stride=8, tag="stride8")
            add("level", "imdct", 1, ln, level_counts(ln // 2), stride=12, tag="stride12")
            add("level", "imdct", 1, ln, level_counts(ln // 2), in_pad=4, out_pad=8, tag="step+4")
        else:
            add("level", "imdct", 1, ln, level_counts(ln // 2))
        for st in (4, 8, 12):
            add("level", "mdct", 0, ln, level_counts(ln // 2), stride=st, out_pad=4 * (st == 4), tag=f"stride{st}")
        for inv in (0, 1):
            k = "c2r" if inv else "r2c"
            add("level", k, inv, ln, level_counts(ln // 2))
            add("level", k, inv, ln, level_counts(ln // 2), in_pad=8, out_pad=8, tag="step+8")
    return cs


# logical floats per transform in / out, the av_tx type, and which side is strided (MDCT)
def _shape(kind, ln):
    return {"fft": (2 * ln, 2 * ln, 0), "ifft": (2 * ln, 2 * ln, 0), "imdct": (ln, ln, 1), "mdct": (2 * ln, ln, 1),
            "r2c": (ln, ln + 2, 6), "c2r": (ln + 2, ln, 6)}[kind]


def _float64(kind, x, scale):
    if kind in ("fft", "ifft"):
        return T.fft(x, kind == "ifft")
    if kind == "imdct":
        return T.imdct(x, scale)
    if kind == "mdct":
        return T.mdct(x, scale)
    return T.rdft(x, kind == "c2r", scale)


@pytest.mark.parametrize("kind, inv, ln, counts, stride, in_off, in_pad, out_pad", _cases())
def test_tx_path_vs_checker(device, kind, inv, ln, counts, stride, in_off, in_pad, out_pad):
    import torch
    from ffmpeg_b200 import tx
    in_w, out_w, typ = _shape(kind, ln)
    in_elem = stride if kind == "imdct" else 4
    out_elem = stride if kind == "mdct" else 4
    in_step, out_step = in_w * in_elem + in_pad, out_w * out_elem + out_pad
    rows = max(counts)
    rng = np.random.default_rng([typ, inv, ln, stride, in_off, in_pad, out_pad])
    x, cls = T.rows(rng, rows, in_w)
    pin = T.positions(rows, in_w, in_step, in_off, in_elem)
    pout = T.positions(rows, out_w, out_step, 0, out_elem)
    host_in = np.full(pin.max() + 1 + 64, SENT, np.uint32)
    host_in[pin] = x.view(np.uint32)
    out_len = pout.max() + 1 + 64
    check = [r for r in range(rows) if cls[r] != "subnormal"]
    scales = MDCT_SCALES if typ == 1 else (1.0, 1.0 / ln) if typ == 6 else (1.0,)
    with torch.cuda.stream(torch.cuda.ExternalStream(device.stream)):
        din = torch.from_numpy(host_in.view(np.int32)).cuda()
        dout = torch.empty(out_len, dtype=torch.int32, device="cuda")
        for sc in scales:
            sc = 1.0 / ln if sc == "1/len" else sc
            exp = T.checker(typ, inv, ln, sc, x, out_w)
            c = tx.av_tx_init(typ, inv, ln, scale=None if typ == 0 else sc, device=device)
            try:                                                 # a failing check must not leave the context to outlive the device
                for cnt in counts:
                    dout.fill_(SENT)
                    c.batch_device(dout.data_ptr(), din.data_ptr() + in_off, stride if typ == 1 else 8 if typ == 0 else 4,
                                   cnt, out_step, in_step)
                    device.sync()
                    got = dout.cpu().numpy().view(np.uint32)
                    o = got[pout[:cnt]]
                    bad = np.nonzero((o != exp[:cnt].view(np.uint32)).any(axis=1))[0]
                    assert not len(bad), f"scale {sc} count {cnt}: {len(bad)} transforms differ from the checker, first {bad[:8].tolist()} ({[cls[r] for r in bad[:8]]})"
                    rest = got.copy()
                    rest[pout[:cnt]] = SENT
                    assert (rest == SENT).all(), f"scale {sc} count {cnt}: writes outside the outputs at float {np.nonzero(rest != SENT)[0][:8].tolist()}"
            finally:
                c.uninit()
            if check:
                err = T.rel_l2(o[check].view(np.float32), _float64(kind, x[check], sc))
                assert err.max() <= T.bound(ln), f"scale {sc}: relative L2 error {err.max():.3g} > {T.bound(ln):.3g} ({cls[check[int(err.argmax())]]})"
        assert np.array_equal(din.cpu().numpy().view(np.uint32), host_in), "the input buffer changed"


def test_tx_fft1024_batch_over_2g(device):
    """one launch of about 300 k 1024-point FFTs: input and output each larger than 2^31 bytes.  Sampled transforms (the first, the
    last, those around the 2^31-byte offset and a random sample) equal the checker bit for bit."""
    import torch
    from ffmpeg_b200 import tx
    n, cnt = 1024, 300_001
    step = 8 * n
    assert cnt * step > 2 ** 31
    edge = 2 ** 31 // step
    rng = np.random.default_rng(31)
    pick = np.unique(np.concatenate([[0, 1, cnt - 2, cnt - 1], np.arange(edge - 3, edge + 4), rng.integers(0, cnt, 200)]))
    with torch.cuda.stream(torch.cuda.ExternalStream(device.stream)):
        g = torch.Generator(device="cuda").manual_seed(7)
        din = torch.rand((cnt, 2 * n), device="cuda", generator=g) * 2 - 1
        dout = torch.full((cnt + 1, 2 * n), float("nan"), device="cuda")
        c = tx.av_tx_init(tx.AV_TX_FLOAT_FFT, 0, n, device=device)
        try:
            c.batch_device(dout, din, 8, cnt, step, step)
            device.sync()
        finally:
            c.uninit()
        sel = torch.from_numpy(pick).cuda()
        x, got = din[sel].cpu().numpy(), dout[sel].cpu().numpy()
        assert bool(torch.isnan(dout[cnt]).all()), "the row after the batch was written"
        del din, dout
        torch.cuda.empty_cache()
    exp = T.checker(0, 0, n, 1.0, x, 2 * n)
    bad = np.nonzero((got.view(np.uint32) != exp.view(np.uint32)).any(axis=1))[0]
    assert not len(bad), f"transforms {pick[bad][:8].tolist()} differ from the checker"
