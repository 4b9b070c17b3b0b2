"""GPU tier: the compound, DCT, int32 and double routes of b200_tx_batch_device, bit for bit against the checker at every length the
library builds.  The case id names the route first:
  pfa-fft   tx_fft_pfa_kernel: all 45 lengths N x m (N = 3, 5, 7, 9, 15; m = 2 ... 512) both ways; at m = 64 also output strides of 16
            and 24 bytes, steps padded by 8 bytes, and AV_TX_INPLACE
  pfa-mdct  tx_mdct_pfa_inv / fwd_kernel: all 45 lengths 2 N m both ways, five scales (negative ones shift the twiddle phase); at m = 64
            also inverse input / forward output strides of 8 and 12 bytes, and AV_TX_FULL_IMDCT
  dct2/3    the DCT stages around the nested RDFT: 4 ... 32768 points, scales 1, 0.5 / n, -1, padded steps at some sizes; one call of
            65537 transforms crosses the 65535-transform chunk of tx_dct_launch
  i32-*     tx_i32_kernel<0, 1, 2>: FFT 2 ... 4096, MDCT len 4 ... 8192 both ways (scales 1 / len, 1, -1 / 32768), strides 8 / 12 bytes
  dbl-*     tx_dbl_*_kernel: FFT 2 ... 8192, MDCT len 4 ... 16384 both ways (scales 1 / len, 1, -1, 0.5), strides 16 / 24 bytes
The compound, int32 and double kernels cap their grid at 8 CTAs per SM and loop over the batch, so the largest count,
2 * 8 * 132 + 7, makes every CTA of an H100 run at least two transforms; it runs at the first scale, the other scales at 3 and
301 transforms.  The DCT has no grid cap (it runs 1, 3 and 301).  One context runs the counts in increasing order, so the DCT's
scratch area grows between calls.

Each call checks: every transform equal to the checker (contiguous: a forward MDCT with an output stride writes the values of the
contiguous transform at that stride, see DESIGN.md), a sentinel intact in every gap, in the rows past `count` and 256 bytes past the
batch, and the input unchanged.  The rows of an eligible class among the first and last 128 of the largest count are also held to
the high-precision definition of tests/txref.py (float64; long double for the double types)."""
import numpy as np
import pytest

import txref as T

pytestmark = pytest.mark.gpu

H100_SMS, CTAS_PER_SM = 132, 8
CAP_COUNT = 2 * CTAS_PER_SM * H100_SMS + 7                  # every CTA of the capped grid runs two transforms or more
COUNTS, DCT_COUNTS = (1, 3, CAP_COUNT), (1, 3, 301)
PFA_MDCT_SCALES = ("1/len", 1.0, -1.0, -1.0 / 32768, 0.5)
DCT_SCALES = (1.0, "0.5/n", -1.0)
I32_SCALES = ("1/len", 1.0, -1.0 / 32768)
DBL_SCALES = ("1/len", 1.0, -1.0, 0.5)
LATER_COUNTS = (3, 301)                                     # the scales after the first: the grid loop does not depend on them
DEF_ROWS = 128                                              # rows of each end of the batch the high-precision definition checks


class Case:
    """one transform setup: av_tx type / direction / length, element layout of input and output, the counts and scales to run"""

    def __init__(self, typ, inv, ln, counts, scales=(1.0,), stride=None, flags=0, in_pad=0, out_pad=0, out_stride=None, inplace=False):
        self.typ, self.inv, self.ln, self.counts, self.scales, self.flags = typ, inv, ln, counts, scales, flags
        self.in_pad, self.out_pad, self.inplace = in_pad, out_pad, inplace
        dbl = typ in (2, 3)
        self.word = 8 if dbl else 4
        self.dtype = np.float64 if dbl else np.int32 if typ in (4, 5) else np.float32
        full = flags & 4
        if typ in (0, 2, 4):                                 # complex FFT: 2 ln words, in contiguous, out with a stride (bytes per complex)
            self.in_w = self.out_w = 2 * ln
            self.in_elem, self.in_group = 2 * self.word, 2
            self.stride = out_stride or 2 * self.word
            self.out_elem, self.out_group = self.stride, 2
        elif typ == 9:                                       # DCT: n floats both ways
            self.in_w = self.out_w = ln
            self.in_elem = self.out_elem = 4
            self.in_group = self.out_group = 1
            self.stride = 4
        else:                                                # MDCT: the inverse's input and the forward's output carry the stride
            self.stride = stride or self.word
            self.in_w, self.out_w = (ln, 2 * ln if full else ln) if inv else (2 * ln, ln)
            self.in_elem, self.out_elem = (self.stride, self.word) if inv else (self.word, self.stride)
            self.in_group = self.out_group = 1
        self.in_step = self.in_w // self.in_group * self.in_elem + in_pad
        self.out_step = self.out_w // self.out_group * self.out_elem + out_pad


def _cases():
    cs = []

    def add(route, c, tag=""):
        d = "inv" if c.inv else "fwd"
        cs.append(pytest.param(c, id=f"{route}-{c.ln}-{d}" + (f"-{tag}" if tag else "")))
    for nf in (3, 5, 7, 9, 15):
        for m in (1 << k for k in range(1, 10)):
            n = nf * m
            for inv in (0, 1):
                add("pfa-fft", Case(0, inv, n, COUNTS))
                add("pfa-mdct", Case(1, inv, 2 * n, COUNTS, PFA_MDCT_SCALES))
                if m != 64:
                    continue
                add("pfa-fft", Case(0, inv, n, COUNTS, out_stride=16), "ostride16")
                add("pfa-fft", Case(0, inv, n, COUNTS, out_stride=24), "ostride24")
                add("pfa-fft", Case(0, inv, n, COUNTS, in_pad=8, out_pad=8), "step+8")
                add("pfa-fft", Case(0, inv, n, COUNTS, flags=1, inplace=True), "inplace")
                for st in (8, 12):
                    add("pfa-mdct", Case(1, inv, 2 * n, COUNTS, PFA_MDCT_SCALES, stride=st, in_pad=4 * inv, out_pad=8), f"stride{st}")
                if inv:
                    add("pfa-mdct", Case(1, 1, 2 * n, COUNTS, ("1/len", -1.0), flags=4), "full")
    for lg in range(2, 16):
        n = 1 << lg
        for inv in (0, 1):
            add("dct3" if inv else "dct2", Case(9, inv, n, DCT_COUNTS, DCT_SCALES))
            if n in (16, 1024, 32768):
                add("dct3" if inv else "dct2", Case(9, inv, n, DCT_COUNTS, DCT_SCALES, in_pad=4, out_pad=8), "step+pad")
    for inv in (0, 1):
        add("dct3" if inv else "dct2", Case(9, inv, 16, (65537,), (1.0,)), "count65537")
    for lg in range(1, 14):
        n = 1 << lg
        for inv in (0, 1):
            if n <= 4096:
                add("i32-fft", Case(4, inv, n, COUNTS))
            if n >= 4:
                add("i32-mdct", Case(5, inv, n, COUNTS, I32_SCALES))
                if n in (16, 1024, 8192):
                    for st in (8, 12):
                        add("i32-mdct", Case(5, inv, n, COUNTS, I32_SCALES, stride=st), f"stride{st}")
    for lg in range(1, 15):
        n = 1 << lg
        for inv in (0, 1):
            if n <= 8192:
                add("dbl-fft", Case(2, inv, n, COUNTS))
            if n >= 4:
                add("dbl-mdct", Case(3, inv, n, COUNTS, DBL_SCALES))
                if n in (16, 1024, 16384):
                    for st in (16, 24):
                        add("dbl-mdct", Case(3, inv, n, COUNTS, DBL_SCALES, stride=st), f"stride{st}")
    return cs


def _inputs(c, rows, rng):
    """(rows x in_w input, class per row, rows the definition check takes)"""
    if c.typ in (4, 5):
        x, cls = T.rows_i32(rng, rows, c.in_w, T.i32_headroom(c.typ, c.inv, c.ln))
        return x, cls, [r for r in range(rows) if cls[r] == "headroom"]
    if c.typ in (2, 3):
        x, cls = T.rows_dbl(rng, rows, c.in_w)
        return x, cls, [r for r in range(rows) if cls[r] != "subnormal"]
    x, cls = T.rows(rng, rows, c.in_w)
    skip = ("subnormal", "constant") if c.typ == 9 else ("subnormal",)
    return x, cls, [r for r in range(rows) if cls[r] not in skip]


def _expected(c, x, sc):
    if c.typ == 9:                                             # the checker's DCT reads and writes n + 2 floats per transform
        xp = np.zeros((x.shape[0], c.ln + 2), np.float32)
        xp[:, :c.ln] = x
        return T.checker(9, c.inv, c.ln // 2 if c.inv else c.ln, sc, xp, c.ln + 2)[:, :c.ln]
    return T.checker(c.typ, c.inv, c.ln, sc, x, c.out_w, c.flags & 4)         # in place or not, the same values


def _definition(c, x, sc):
    """(high-precision result, relative error function, bound)"""
    if c.typ == 9:
        return T.dct(x, c.inv, sc), T.rel_l2, T.dct_bound(c.ln)
    if c.typ in (4, 5):
        return T.i32_transform(c.typ, c.inv, x, sc), T.rel_l2_i32, T.bound(c.ln, T.I32_TOL_C)
    ld = c.typ in (2, 3)
    eps, tol = (2.0 ** -53, T.DBL_TOL_C) if ld else (2.0 ** -24, T.TOL_C)
    if c.typ in (0, 2):
        ref = T.fft(x, c.inv, ld)
    elif c.inv:
        ref = (T.imdct_full if c.flags & 4 else T.imdct)(x, sc, ld)
    else:
        ref = T.mdct(x, sc, ld)
    return ref, T.rel_l2, T.bound(c.ln, tol, eps)


@pytest.mark.parametrize("c", _cases())
def test_tx_route_vs_checker(device, c):
    import torch
    from ffmpeg_b200 import tx
    rows = max(c.counts)
    rng = np.random.default_rng([c.typ, c.inv, c.ln, c.stride, c.flags, c.in_pad, c.out_pad, int(c.inplace)])
    x, cls, check = _inputs(c, rows, rng)
    wt, st, tt = (np.uint64, np.int64, torch.int64) if c.word == 8 else (np.uint32, np.int32, torch.int32)
    sent = np.array(SENT_WORD[c.word], wt)
    pin = T.positions(rows, c.in_w, c.in_step, 0, c.in_elem, c.word, c.in_group)
    pout = T.positions(rows, c.out_w, c.out_step, 0, c.out_elem, c.word, c.out_group)
    host_in = np.full(pin.max() + 1 + 256 // c.word, sent, wt)
    host_in[pin] = x.view(wt)
    out_len = pout.max() + 1 + 256 // c.word
    with torch.cuda.stream(torch.cuda.ExternalStream(device.stream)):
        din = torch.from_numpy(host_in.view(st)).cuda()
        dout = din if c.inplace else torch.empty(out_len, dtype=tt, device="cuda")
        pout_d = torch.from_numpy(pout).cuda()
        sent_d = torch.tensor(int(sent.view(st)), dtype=tt, device="cuda")
        for k, sc in enumerate(c.scales):
            sc = 1.0 / c.ln if sc == "1/len" else 0.5 / c.ln if sc == "0.5/n" else sc
            counts = c.counts if k == 0 else LATER_COUNTS
            exp = _expected(c, x[:max(counts)], sc)
            kw = {} if c.typ == 0 else {"scale": sc}
            ctx = tx.av_tx_init(c.typ, c.inv, c.ln // 2 if c.typ == 9 and c.inv else c.ln, flags=c.flags, device=device, **kw)
            try:                                                 # a failing check must not leave the context to outlive the device
                for cnt in counts:
                    if c.inplace:
                        din.copy_(torch.from_numpy(host_in.view(st)))
                    else:
                        dout.fill_(sent_d.item())
                    ctx.batch_device(dout.data_ptr(), din.data_ptr(), c.stride, cnt, c.out_step, c.in_step)
                    device.sync()
                    o = dout[pout_d[:cnt]].cpu().numpy().view(wt)
                    bad = np.nonzero((o != exp[:cnt].view(wt)).any(axis=1))[0]
                    assert not len(bad), f"scale {sc} count {cnt}: {len(bad)} transforms differ from the checker, first {bad[:8].tolist()} ({[cls[r] for r in bad[:8]]})"
                    keep = torch.ones(out_len if not c.inplace else din.numel(), dtype=torch.bool, device="cuda")
                    keep[pout_d[:cnt].reshape(-1)] = False
                    if c.inplace:                                # rows past `count` keep their input
                        keep[torch.from_numpy(pin[cnt:].reshape(-1)).cuda()] = False
                    stray = torch.nonzero(keep & (dout != sent_d)).reshape(-1)
                    assert not stray.numel(), f"scale {sc} count {cnt}: writes outside the outputs at word {stray[:8].tolist()}"
            finally:
                ctx.uninit()
            rs = [r for r in check if r < cnt]
            rs = rs[:DEF_ROWS] + rs[DEF_ROWS:][-DEF_ROWS:]
            if rs:
                ref, err_fn, bnd = _definition(c, x[rs], sc)
                err = err_fn(o[rs].view(c.dtype), ref)
                assert err.max() <= bnd, f"scale {sc}: relative L2 error {float(err.max()):.3g} > {bnd:.3g} ({cls[rs[int(err.argmax())]]})"
        if not c.inplace:
            assert np.array_equal(din.cpu().numpy().view(wt), host_in), "the input buffer changed"


SENT_WORD = {4: T.SENT, 8: (T.SENT << 32) | T.SENT}
