"""Float64 definitions of the power-of-two float transforms and the input classes their tests feed them (test infrastructure only).

The relative L2 error of a float32 transform of n points against its float64 value grows like log2(n) * 2^-24; TOL_C is the
constant c of the bound c * log2(n) * 2^-24, calibrated on the checker (tests/test_oracle_more.py records the worst c it sees
and keeps 4x margin under TOL_C).  The CUDA kernels equal the checker bit for bit, so the same bound holds for them."""
import numpy as np

TOL_C = 6.0
CLASSES = ("uniform", "wide", "subnormal", "zeros", "impulse", "constant", "huge")


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


def cpx(x):
    x = np.asarray(x, np.float64)
    return x[..., 0::2] + 1j * x[..., 1::2]


def interleave(z):
    out = np.empty(z.shape[:-1] + (2 * z.shape[-1],))
    out[..., 0::2], out[..., 1::2] = z.real, z.imag
    return out


def fft(x, inv):
    """complex FFT of n points (2n interleaved floats); the inverse is unnormalised, like av_tx"""
    z = cpx(x)
    return interleave(np.fft.ifft(z, axis=-1) * z.shape[-1] if inv else np.fft.fft(z, axis=-1))


def rdft(x, inv, scale):
    """r2c: len real -> len/2 + 1 complex (len + 2 floats); c2r: len/2 + 1 complex -> len real, times len (unnormalised) and scale"""
    if not inv:
        return interleave(np.fft.rfft(np.asarray(x, np.float64), axis=-1)) * scale
    z = cpx(x)
    n = 2 * (z.shape[-1] - 1)
    return np.fft.irfft(z, n, axis=-1) * n * scale


def mdct(x, scale):
    """forward MDCT, 2 len inputs -> len outputs: y[k] = scale * sum_i x[i] cos(pi / len (i + 1/2 + len/2)(k + 1/2))"""
    x = np.asarray(x, np.float64)
    n = x.shape[-1] // 2
    i = np.arange(2 * n)
    u = np.fft.fft(x * np.exp(-1j * np.pi * i / (2 * n)), axis=-1)[..., :n]
    k = np.arange(n)
    return scale * (np.exp(-1j * np.pi * (0.5 + n / 2) * (k + 0.5) / n) * u).real


def imdct_full(x, scale):
    """inverse MDCT as AV_TX_FULL_IMDCT computes it, len inputs -> 2 len outputs:
    y[i] = -scale * sum_k x[k] cos(pi / len (i + 1/2 + len/2)(k + 1/2))  (av_tx's inverse has the opposite sign of the forward one)"""
    x = np.asarray(x, np.float64)
    n = x.shape[-1]
    k = np.arange(n)
    v = np.zeros(x.shape[:-1] + (2 * n,), complex)
    v[..., :n] = x * np.exp(1j * np.pi * (0.5 + n / 2) * k / n)
    w = np.fft.ifft(v, axis=-1) * (2 * n)
    i = np.arange(2 * n)
    return -scale * (np.exp(1j * np.pi * (i + 0.5 + n / 2) / (2 * n)) * w).real


def imdct(x, scale):
    """the non-full inverse MDCT: the middle half of imdct_full (ff_tx_mdct_inv_full puts it at out[len/2 .. 3 len/2))"""
    n = np.asarray(x).shape[-1]
    return imdct_full(x, scale)[..., n // 2: n // 2 + n]


def rel_l2(got, ref):
    """per-row ||got - ref|| / ||ref||; rows whose reference is exactly zero give 0 when got is zero too, inf otherwise"""
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    num, den = np.linalg.norm(got - ref, axis=-1), np.linalg.norm(ref, axis=-1)
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(den > 0, num / np.where(den > 0, den, 1), np.where(num > 0, np.inf, 0.0))


def bound(n):
    """TOL_C * log2(n) * 2^-24 for an n-point transform"""
    return TOL_C * max(1, int(np.log2(n))) * 2.0 ** -24
