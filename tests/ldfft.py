"""Mixed-radix FFT in extended precision (np.clongdouble): the reference the TMA kernel tests measure against.

Decimation in time, radix = smallest prime factor (4 where it divides), any 2..13-smooth length, along any axis, either sign,
unnormalised.  Twiddles are exp(sign*2*pi*i*(r*k mod N)/N) with the index reduced exactly in integers and the angle formed
from a long-double pi literal (np.pi is only a double), so each twiddle is correct to the long-double epsilon (~1.1e-19 on
x86-64, 64-bit mantissa).  `dtype` and `round_bits` exist for the self-test only: they run the same algorithm in another
precision, optionally with the twiddles of one recursion level rounded to fewer mantissa bits."""
import numpy as np

PI_L = np.longdouble("3.14159265358979323846264338327950288419716939937510")
LD_EPS_MAX = 1e-18   # the references are meaningless for the fp64 bounds unless long double is wider than double

_tw_cache = {}


def _radix(n):
    if n % 4 == 0 and n > 4:
        return 4
    for p in (2, 3, 5, 7, 11, 13):
        if n % p == 0:
            return p
    raise ValueError(f"length {n} is not 2..13-smooth")


def _expi(num, den, sign):
    """exp(sign * 2 pi i * num / den) in long double, num an integer array"""
    num = np.asarray(num, dtype=np.int64) % den
    ang = (2 * PI_L) * num.astype(np.longdouble) / np.longdouble(den)
    return np.cos(ang) + (1j * sign) * np.sin(ang)


def _round_mantissa(z, bits):
    def r(v):
        m, e = np.frexp(v)
        return np.ldexp(np.round(np.ldexp(m, bits)), e - bits)
    return (r(z.real) + 1j * r(z.imag)).astype(z.dtype)


def _twiddles(n, p, sign, dtype, round_bits):
    key = (n, p, sign, np.dtype(dtype).str, round_bits)
    if key not in _tw_cache:
        m = n // p
        r = np.arange(p)
        tw = _expi(np.outer(r, np.arange(m)), n, sign).astype(dtype)   # (p, m): W_N^{r k}
        dft = _expi(np.outer(r, r), p, sign).astype(dtype)             # (p, p): W_p^{q r}
        if round_bits is not None:
            tw = _round_mantissa(tw, round_bits)
        _tw_cache[key] = (tw, dft)
    return _tw_cache[key]


def _fft_last(x, sign, dtype, perturb, level=0):
    n = x.shape[-1]
    if n == 1:
        return x
    p = _radix(n)
    m = n // p
    # x[j*p + r] -> sub-sequence r; transform each (length m), then combine: X[q*m + k] = sum_r W_p^{qr} W_N^{rk} Y_r[k]
    y = _fft_last(np.ascontiguousarray(np.swapaxes(x.reshape(x.shape[:-1] + (m, p)), -1, -2)), sign, dtype, perturb, level + 1)
    tw, dft = _twiddles(n, p, sign, dtype, perturb[1] if perturb and perturb[0] == level else None)
    z = y * tw
    out = np.empty_like(z)
    for q in range(p):
        acc = z[..., 0, :].copy()
        for r in range(1, p):
            acc += dft[q, r] * z[..., r, :]
        out[..., q, :] = acc
    return out.reshape(x.shape)


def fft(x, axis=-1, sign=-1, dtype=np.clongdouble, perturb=None):
    """1-D transform of `x` along `axis`: sum_j x[j] exp(sign 2 pi i j k / N).  perturb = (level, bits): round the twiddles
    of that recursion level to `bits` mantissa bits (self-test)."""
    x = np.moveaxis(np.asarray(x).astype(dtype), axis, -1)
    return np.moveaxis(_fft_last(np.ascontiguousarray(x), sign, dtype, perturb), -1, axis)


def fftn(x, sign=-1, dtype=np.clongdouble, perturb=None):
    """transform over every axis (the perturbation, if any, on the longest axis only)"""
    y = np.asarray(x).astype(dtype)
    longest = int(np.argmax(y.shape))
    for ax in range(y.ndim):
        y = fft(y, ax, sign, dtype, perturb if ax == longest else None)
    return y


def errors(got, ref, linf_scale="rms"):
    """(rel_l2, linf): ||got - ref||_2 / ||ref||_2 and max|got - ref| / rms(ref), evaluated in long double.  For a spectrum
    that is one spike, rms(ref) is sqrt(Ntot) times below the spike and says little: linf_scale="max" divides by max|ref|"""
    ref = np.asarray(ref, dtype=np.clongdouble).ravel()
    d = np.asarray(got).astype(np.clongdouble).ravel() - ref
    ad2 = d.real ** 2 + d.imag ** 2
    ar2 = ref.real ** 2 + ref.imag ** 2
    n2 = np.sum(ar2)
    scale2 = np.max(ar2) if linf_scale == "max" else n2 / ref.size
    return float(np.sqrt(np.sum(ad2) / n2)), float(np.sqrt(np.max(ad2) / scale2))


EPS = {"double": 2.0 ** -53, "float": 2.0 ** -24}
REL_L2_K, LINF_K = 1.0, 4.0   # bounds, in units of eps * log2(Ntot): numpy's own fp64 FFT sits near 0.14 and 0.6


def ratios(got, ref, eps, ntot, linf_scale="rms"):
    """the two errors as multiples of eps * log2(ntot)"""
    rl2, linf = errors(got, ref, linf_scale)
    u = eps * np.log2(ntot)
    return rl2 / u, linf / u
