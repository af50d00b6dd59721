"""numpy restatement of the acquisition resampler (GNSS-SDR.use_acquisition_resampler, gnss_flowgraph.cc:1117-1212): the
decimation rule and gr::filter::firdes::low_pass with its default Hamming window in float64, and the float32 decimating
FIR in the order b200_acq_set_band_resampler's kernel computes it, so the GPU's decimated vector can be checked bit for
bit.  GNU Radio is not part of the reference tree: the filter design is restated from its formula, not from its bits."""
import math

import numpy as np


def decimation(fs_in: int, opt_acq_fs: int) -> int:
    """floor(fs_in / opt_acq_fs), lowered until it divides fs_in; 1 (no resampler) when opt_acq_fs >= fs_in"""
    if opt_acq_fs >= fs_in:
        return 1
    d = int(math.floor(float(fs_in) / float(opt_acq_fs)))
    while fs_in % d:
        d -= 1
    return d


def low_pass(gain: float, fs: float, cutoff: float, transition: float) -> np.ndarray:
    """firdes::low_pass with the Hamming window, in float64: ntaps = int(53 fs / (22 transition)) made odd, windowed
    sinc around M = (ntaps - 1) / 2, scaled to a DC gain of `gain`"""
    ntaps = int(53.0 * fs / (22.0 * transition))
    ntaps += 1 - ntaps % 2
    m = (ntaps - 1) // 2
    n = np.arange(-m, m + 1, dtype=np.float64)
    w = 0.54 - 0.46 * np.cos(2.0 * np.pi * np.arange(ntaps) / (ntaps - 1))
    fw = 2.0 * np.pi * cutoff / fs
    nz = np.where(n == 0, 1.0, n)
    h = np.where(n == 0, fw / np.pi, np.sin(n * fw) / (nz * np.pi)) * w
    return h * (gain / h.sum())


def design(fs_in: int, opt_acq_fs: int):
    """-> (decimation, float64 taps) of the resampler the reference inserts; (1, empty) where it inserts none"""
    d = decimation(fs_in, opt_acq_fs)
    if d <= 1:
        return 1, np.zeros(0)
    fs_dec = fs_in / d
    return d, low_pass(1.0, float(fs_in), fs_dec / 2.1, fs_dec / 2.0)


def decimate_f32(x: np.ndarray, taps: np.ndarray, d: int, start: int, n_out: int) -> np.ndarray:
    """y[j] = sum_k taps[k] x[start + j d - k], j < n_out, in float32: k ascending from a zero accumulator, every product and
    sum rounded on its own (what the device kernel computes).  x: complex samples indexed from 0."""
    h = np.asarray(taps, np.float32)
    xr, xi = np.ascontiguousarray(x.real, np.float32), np.ascontiguousarray(x.imag, np.float32)
    idx = start + d * np.arange(n_out)
    assert idx[0] - (h.size - 1) >= 0 and idx[-1] < x.size
    re, im = np.zeros(n_out, np.float32), np.zeros(n_out, np.float32)
    for k in range(h.size):
        re = re + h[k] * xr[idx - k]
        im = im + h[k] * xi[idx - k]
    return (re + 1j * im).astype(np.complex64)
