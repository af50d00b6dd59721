"""numpy restatement of the signal conditioner (b200_iq_set_conditioner): gr::filter::freq_xlating_fir_filter_ccf(D, h, IF, fs)
written in absolute stream indices,

    y[j] = r(j) sum_{k<T} c[k] x[j D - k],  c[k] = h[k] e^{+i k w},  r(j) = e^{-i w D j},  w = 2 pi IF / fs,  x[m < 0] = 0.

condition_f32 is the float32 loop in the device kernel's order (k ascending from zero, every product and sum rounded on its
own; real taps at IF = 0, complex taps otherwise, then the rotator in double, rounded once), so the destination band can be
checked bit for bit at IF = 0 and to a few float ulps elsewhere.  condition_f64 is the formula in float64 with the rotator's
phase reduced exactly (rational arithmetic on the two doubles IF and fs), the truth both are held to."""
from fractions import Fraction

import numpy as np


def composite_taps(h, if_hz: float, fs: float) -> np.ndarray:
    """c[k] = h[k] e^{+i k w} in double, each component rounded once to float32 (complex64)"""
    h64 = np.asarray(h, np.float32).astype(np.float64)
    kw = np.arange(h64.size, dtype=np.float64) * (2.0 * np.pi * if_hz / fs)
    return (h64 * np.cos(kw)).astype(np.float32) + 1j * (h64 * np.sin(kw)).astype(np.float32)


def rotator_step(if_hz: float, fs: float, d: int) -> int:
    """D |IF| / fs mod 1 as a 128-bit binary fraction, truncated, and negated mod 2^128 for a negative IF"""
    q = Fraction(abs(if_hz)) * d / Fraction(fs)
    f = ((q.numerator % q.denominator) << 128) // q.denominator
    return (-f) % (1 << 128) if if_hz < 0 else f


def rotator_phase(step: int, j: np.ndarray) -> np.ndarray:
    """phi(j) in cycles, float64 in [-1/2, 1/2): the top 64 bits of j * step mod 2^128 as a signed fraction"""
    top = [((int(jj) * step) >> 64) & ((1 << 64) - 1) for jj in j]
    return np.array([float(t - (1 << 64) if t >= 1 << 63 else t) for t in top]) * 2.0 ** -64


def _gather(x, x0: int, m: np.ndarray):
    """x[m] for absolute indices m; zeros below 0; samples of [0, x0) are not held and must not be needed"""
    assert np.all((m < 0) | (m >= x0)), "the span reaches samples the host does not hold"
    i = m - x0
    ok = m >= 0
    return np.where(ok, x[np.clip(i, 0, x.size - 1)], 0)


def condition_f32(x, x0: int, h, d: int, if_hz: float, fs: float, j0: int, n_out: int) -> np.ndarray:
    """outputs j0 .. j0 + n_out - 1 as the device computes them; x[i] is absolute sample x0 + i (complex64)"""
    x = np.asarray(x, np.complex64)
    xr, xi = np.ascontiguousarray(x.real), np.ascontiguousarray(x.imag)
    c = composite_taps(h, if_hz, fs)
    cr, ci = c.real.astype(np.float32), c.imag.astype(np.float32)
    j = j0 + np.arange(n_out, dtype=np.int64)
    re, im = np.zeros(n_out, np.float32), np.zeros(n_out, np.float32)
    for k in range(c.size):
        m = j * d - k
        vr, vi = _gather(xr, x0, m).astype(np.float32), _gather(xi, x0, m).astype(np.float32)
        if if_hz == 0:
            re = re + cr[k] * vr
            im = im + cr[k] * vi
        else:
            re = re + (cr[k] * vr - ci[k] * vi)
            im = im + (cr[k] * vi + ci[k] * vr)
    if if_hz == 0:
        return (re + 1j * im).astype(np.complex64)
    phi = rotator_phase(rotator_step(if_hz, fs, d), j)
    cs, sn = np.cos(np.pi * (2.0 * phi)), np.sin(np.pi * (2.0 * phi))
    re64, im64 = re.astype(np.float64), im.astype(np.float64)
    yr = re64 * cs + im64 * sn
    yi = im64 * cs - re64 * sn
    return yr.astype(np.float32) + 1j * yi.astype(np.float32)


def exact_phase(if_hz: float, fs: float, d: int, j: np.ndarray) -> np.ndarray:
    """frac(j D IF / fs) in cycles, from the exact rational value of the two doubles"""
    q = Fraction(if_hz) * d / Fraction(fs)
    p, r = q.numerator % q.denominator, q.denominator
    return np.array([((int(jj) * p) % r) / r for jj in j])


def condition_f64(x, x0: int, h, d: int, if_hz: float, fs: float, j0: int, n_out: int):
    """-> (y, scale): the formula in float64 for the float32 taps h, and sum_k |c[k]| |x[j D - k]|, the size the float32
    loop's rounding is measured against"""
    x = np.asarray(x).astype(np.complex128)
    h64 = np.asarray(h, np.float32).astype(np.float64)
    c = h64 * np.exp(1j * np.arange(h64.size) * (2.0 * np.pi * if_hz / fs))
    j = j0 + np.arange(n_out, dtype=np.int64)
    acc = np.zeros(n_out, np.complex128)
    scale = np.zeros(n_out)
    for k in range(c.size):
        v = _gather(x, x0, j * d - k)
        acc += c[k] * v
        scale += abs(c[k]) * np.abs(v)
    return acc * np.exp(-2j * np.pi * exact_phase(if_hz, fs, d, j)), scale


def ceil_div(a: int, b: int) -> int:
    return -(-a // b)
