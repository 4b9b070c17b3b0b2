"""High-precision definitions of the tx transforms, the input classes their tests feed them, and the error bounds the kernels are
held to (test infrastructure only).

The relative L2 error of a float32 transform of n points against its float64 value grows like log2(n) * 2^-24; TOL_C is the
constant c of the bound c * log2(n) * 2^-24, calibrated on the checker (tests/test_oracle_more.py records the worst c it sees
and keeps 4x margin under TOL_C).  The CUDA kernels equal the checker bit for bit, so the same bound holds for them.
The other routes have their own constants, calibrated the same way (worst value measured in the comment beside each):
  DCT_TOL_C  float32 DCT-II / DCT-III, c * sqrt(n) * 2^-24: the DCT-II's odd outputs are a running sum over n / 2 terms and the
             DCT-III multiplies by 1 / (2 sin((2i + 1) pi / 2n)), up to n / pi, so the error grows faster than log2(n).  Constant rows
             are left out: their DCT-III cancels to a few large outputs, and its relative error grows like n
  I32_TOL_C  int32 FFT / MDCT, c * log2(n) * 2^-24 relative to max(||ref||, 2^24 sqrt(width)): the Q31 tables are rounded through
             float (2^-24 relative), and every product rounds to an integer (a floor of about one unit per output and level)
  DBL_TOL_C  double FFT / MDCT, c * log2(n) * 2^-53 against a long double definition"""
import numpy as np

TOL_C = 6.0              # worst measured 1.25 (power-of-two routes), 0.79 (compound routes)
DCT_TOL_C = 12.0         # worst measured 2.70 (DCT-II)
I32_TOL_C = 10.0         # worst measured 2.13 (forward MDCT: the >> 6 fold rounds before the transform)
DBL_TOL_C = 8.0          # worst measured 1.88 (forward MDCT)
CLASSES = ("uniform", "wide", "subnormal", "zeros", "impulse", "constant", "huge")
DCT_CLASSES = ("uniform", "wide", "zeros", "impulse", "huge")
I32_CLASSES = ("headroom", "full", "extremes", "impulse", "constant", "zeros")
DBL_CLASSES = ("uniform", "wide", "subnormal", "zeros", "impulse", "huge")
PI_L = np.longdouble("3.14159265358979323846264338327950288")


def rows(rng, count, width, classes=CLASSES):
    """count x width float32 rows; row r is of class classes[r % len(classes)].  Returns (x, class index per row)."""
    x = np.empty((count, width), np.float32)
    kind = np.arange(count) % len(classes)
    for k, name in enumerate(classes):
        sel = np.nonzero(kind == k)[0]
        m = len(sel)
        if not m:
            continue
        sign = rng.choice(np.array([-1.0, 1.0]), (m, width))
        if name == "uniform":
            v = rng.uniform(-1, 1, (m, width))
        elif name == "wide":                                     # sign x 2^U(-60, 60)
            v = sign * np.exp2(rng.uniform(-60, 60, (m, width)))
        elif name == "subnormal":                                # almost every value below 2^-126
            v = rng.uniform(-1, 1, (m, width)) * 2.0 ** -130
        elif name == "zeros":                                    # +0.0 and -0.0
            v = sign * 0.0
        elif name == "impulse":
            v = np.zeros((m, width))
            v[np.arange(m), rng.integers(0, width, m)] = rng.uniform(0.5, 1, m) * rng.choice([-1.0, 1.0], m)
        elif name == "constant":
            v = np.repeat(rng.uniform(-1, 1, (m, 1)), width, axis=1)
        elif name == "huge":                                     # magnitudes near 2^100
            v = sign * rng.uniform(0.5, 1, (m, width)) * 2.0 ** 100
        else:
            raise ValueError(name)
        x[sel] = v.astype(np.float32)
    return x, [classes[k] for k in kind]


def rows_i32(rng, count, width, headroom, classes=I32_CLASSES):
    """count x width int32 rows, row r of class classes[r % len(classes)]: `headroom` uniform in +-2^headroom (no sum of the transform
    wraps), `full` uniform over the whole int32 range (sums wrap modulo 2^32), `extremes` runs of INT32_MIN / INT32_MAX / -1 / 0,
    impulses, constants and zeros.  Returns (x, class name per row)."""
    x = np.zeros((count, width), np.int64)
    kind = np.arange(count) % len(classes)
    lo, hi = -(1 << 31), (1 << 31) - 1
    for k, name in enumerate(classes):
        sel = np.nonzero(kind == k)[0]
        m = len(sel)
        if not m:
            continue
        if name == "headroom":
            v = rng.integers(-(1 << headroom), 1 << headroom, (m, width))
        elif name == "full":
            v = rng.integers(lo, hi, (m, width), endpoint=True)
        elif name == "extremes":
            v = np.repeat(rng.choice(np.array([lo, hi, -1, 0]), (m, (width + 7) // 8)), 8, axis=1)[:, :width]
        elif name == "impulse":
            v = np.zeros((m, width), np.int64)
            v[np.arange(m), rng.integers(0, width, m)] = rng.integers(lo, hi, m)
        elif name == "constant":
            v = np.repeat(rng.integers(-(1 << headroom), 1 << headroom, (m, 1)), width, axis=1)
        elif name == "zeros":
            v = np.zeros((m, width), np.int64)
        else:
            raise ValueError(name)
        x[sel] = v
    return x.astype(np.int32), [classes[k] for k in kind]


def rows_dbl(rng, count, width, classes=DBL_CLASSES):
    """count x width float64 rows: uniform, sign x 2^U(-500, 500), subnormal (below 2^-1022), +0.0 / -0.0, impulses, near 2^1000"""
    x = np.empty((count, width))
    kind = np.arange(count) % len(classes)
    for k, name in enumerate(classes):
        sel = np.nonzero(kind == k)[0]
        m = len(sel)
        if not m:
            continue
        sign = rng.choice(np.array([-1.0, 1.0]), (m, width))
        if name == "uniform":
            v = rng.uniform(-1, 1, (m, width))
        elif name == "wide":
            v = sign * np.exp2(rng.uniform(-500, 500, (m, width)))
        elif name == "subnormal":
            v = rng.uniform(-1, 1, (m, width)) * 2.0 ** -1030
        elif name == "zeros":
            v = sign * 0.0
        elif name == "impulse":
            v = np.zeros((m, width))
            v[np.arange(m), rng.integers(0, width, m)] = rng.uniform(0.5, 1, m) * rng.choice([-1.0, 1.0], m)
        elif name == "huge":
            v = sign * rng.uniform(0.5, 1, (m, width)) * 2.0 ** 1000
        else:
            raise ValueError(name)
        x[sel] = v
    return x, [classes[k] for k in kind]


def _wide(x, ld):
    return np.asarray(x, np.longdouble if ld else np.float64)


def cpx(x, ld=False):
    x = _wide(x, ld)
    return x[..., 0::2] + 1j * x[..., 1::2]


def interleave(z):
    out = np.empty(z.shape[:-1] + (2 * z.shape[-1],), z.real.dtype)
    out[..., 0::2], out[..., 1::2] = z.real, z.imag
    return out


def _dft(z, inv):
    """unnormalised DFT along the last axis, in the precision of z (scipy keeps long double)"""
    import scipy.fft as sf
    return sf.ifft(z, axis=-1, norm="forward") if inv else sf.fft(z, axis=-1)


def _pi(ld):
    return PI_L if ld else np.pi


def fft(x, inv, ld=False):
    """complex FFT of n points (2n interleaved floats); the inverse is unnormalised, like av_tx.  ld: in long double"""
    z = cpx(x, ld)
    if ld:
        return interleave(_dft(z, inv))
    return interleave(np.fft.ifft(z, axis=-1) * z.shape[-1] if inv else np.fft.fft(z, axis=-1))


def rdft(x, inv, scale):
    """r2c: len real -> len/2 + 1 complex (len + 2 floats); c2r: len/2 + 1 complex -> len real, times len (unnormalised) and scale"""
    if not inv:
        return interleave(np.fft.rfft(np.asarray(x, np.float64), axis=-1)) * scale
    z = cpx(x)
    n = 2 * (z.shape[-1] - 1)
    return np.fft.irfft(z, n, axis=-1) * n * scale


def mdct(x, scale, ld=False):
    """forward MDCT, 2 len inputs -> len outputs: y[k] = scale * sum_i x[i] cos(pi / len (i + 1/2 + len/2)(k + 1/2))"""
    x, pi = _wide(x, ld), _pi(ld)
    n = x.shape[-1] // 2
    i = np.arange(2 * n)
    u = _dft(x * np.exp(-1j * pi * i / (2 * n)), 0)[..., :n]
    k = np.arange(n)
    return _wide(scale, ld) * (np.exp(-1j * pi * (0.5 + n / 2) * (k + 0.5) / n) * u).real


def imdct_full(x, scale, ld=False):
    """inverse MDCT as AV_TX_FULL_IMDCT computes it, len inputs -> 2 len outputs:
    y[i] = -scale * sum_k x[k] cos(pi / len (i + 1/2 + len/2)(k + 1/2))  (av_tx's inverse has the opposite sign of the forward one)"""
    x, pi = _wide(x, ld), _pi(ld)
    n = x.shape[-1]
    k = np.arange(n)
    v = np.zeros(x.shape[:-1] + (2 * n,), np.clongdouble if ld else complex)
    v[..., :n] = x * np.exp(1j * pi * (0.5 + n / 2) * k / n)
    w = _dft(v, 1)
    i = np.arange(2 * n)
    return -_wide(scale, ld) * (np.exp(1j * pi * (i + 0.5 + n / 2) / (2 * n)) * w).real


def imdct(x, scale, ld=False):
    """the non-full inverse MDCT: the middle half of imdct_full (ff_tx_mdct_inv_full puts it at out[len/2 .. 3 len/2))"""
    n = np.asarray(x).shape[-1]
    return imdct_full(x, scale, ld)[..., n // 2: n // 2 + n]


def dct(x, inv, scale):
    """AV_TX_FLOAT_DCT on n points: DCT-II y[k] = scale * 2 sum_i x[i] cos(pi k (2i + 1) / 2n); the inverse (asked for n / 2) is the
    DCT-III y[k] = scale * (x[0] + 2 sum_{i>0} x[i] cos(pi i (2k + 1) / 2n)) -- scipy's unnormalised types 2 and 3"""
    import scipy.fft as sf
    return scale * sf.dct(np.asarray(x, np.float64), 3 if inv else 2, axis=-1)


def i32_transform(typ, inv, x, scale):
    """AV_TX_INT32_FFT (typ 4) / AV_TX_INT32_MDCT (typ 5) without rounding or wrapping: the FFT is the plain DFT (the Q31 twiddles
    carry no gain), the MDCT is scaled by `scale`, and the forward MDCT folds its input with (a + b + 32) >> 6, i.e. divides by 64"""
    if typ == 4:
        return fft(x, inv)
    return imdct(x, scale) if inv else mdct(x, scale) / 64


def rel_l2_i32(got, ref):
    """per row ||got - ref|| / max(||ref||, 2^24 sqrt(width)): relative where the output is large, one unit per sample where it is not"""
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    floor = 2.0 ** 24 * np.sqrt(ref.shape[-1])
    return np.linalg.norm(got - ref, axis=-1) / np.maximum(np.linalg.norm(ref, axis=-1), floor)


def rel_l2(got, ref):
    """per-row ||got - ref|| / ||ref||; rows whose reference is exactly zero give 0 when got is zero too, inf otherwise"""
    dt = np.result_type(np.asarray(got).dtype, np.asarray(ref).dtype, np.float64)      # a long double reference keeps its precision
    got, ref = np.asarray(got, dt), np.asarray(ref, dt)
    num, den = np.linalg.norm(got - ref, axis=-1), np.linalg.norm(ref, axis=-1)
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(den > 0, num / np.where(den > 0, den, 1), np.where(num > 0, np.inf, 0.0))


def bound(n, c=TOL_C, eps=2.0 ** -24):
    """c * log2(n) * eps for an n-point transform (TOL_C and float32 unless told otherwise)"""
    return c * max(1, int(np.log2(n))) * eps


def dct_bound(n):
    """DCT_TOL_C * sqrt(n) * 2^-24 for an n-point DCT-II / DCT-III"""
    return DCT_TOL_C * np.sqrt(n) * 2.0 ** -24


# ---------------------------------------------------------------------------------------------- harness of the batched GPU route tests
SENT = 0x7FC0DEAD                          # a NaN payload (the double tests fill 64-bit words with two of it): no finite input makes a kernel write it


def positions(count, width, step, off, elem, word=4, group=1):
    """word index of logical element j of transform r in a buffer of `word`-byte words: element j is word j % group of sample j // group,
    and sample s of transform r starts at byte off + r * step + s * elem"""
    j = np.arange(width, dtype=np.int64)
    return (off + np.arange(count, dtype=np.int64)[:, None] * step + (j // group * elem + j % group * word)[None, :]) // word


def checker(typ, inv, ln, scale, x, out_w, flags=0):
    """the CPU checker's result of av_tx type `typ` on the rows of x, contiguous (stride one sample, complex for the FFTs): float and
    int32 types through orc_tx / orc_txi, double through orc_txd.  The input array is left alone (c2r and the DCT rewrite theirs)."""
    import ctypes as C
    import cpulibs as cl
    O = cl.oracle()
    pre = {2: "orc_txd", 3: "orc_txd", 4: "orc_txi", 5: "orc_txi"}.get(typ, "orc_tx")
    op, run, close = (getattr(O, pre + s) for s in ("_open", "_run", "_close"))
    op.restype = C.c_void_p
    op.argtypes = [C.c_int, C.c_int, C.c_int, C.c_double if pre == "orc_txd" else C.c_float, C.c_uint]
    run.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_ssize_t, C.c_int, C.c_ssize_t, C.c_ssize_t]
    close.argtypes = [C.c_void_p]
    h = op(typ, inv, ln, scale, flags)
    assert h, (typ, inv, ln, scale, flags)
    out, xin = np.zeros((x.shape[0], out_w), x.dtype), x.copy()
    stride = {0: 8, 2: 16, 4: 8}.get(typ, x.dtype.itemsize)
    run(h, out.ctypes.data, xin.ctypes.data, stride, x.shape[0], out.strides[0], xin.strides[0])
    close(h)
    return out


def i32_headroom(typ, inv, n):
    """log2 of the largest input magnitude at which no sum of an int32 transform of n points (len n for the MDCT) can wrap"""
    lg = int(np.log2(n))
    return 29 - lg if typ == 4 else 30 - lg if inv else min(30, 34 - lg)
