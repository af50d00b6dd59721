"""numpy restatement of the pulse blanker (b200_iq_set_pulse_blanking): pulse_blanking_cc(pfa, L, E, R) in float32, segment
by segment from the blanker's origin.

    e = sum_{i<L} (re_i re_i + im_i im_i)                       (each square and sum rounded, i ascending from 0.0)
    n < E and not last_filtered:  est = (float(n) est + e / float(2L)) / float(n + 1), copied
    else if e / est > thres:      zeroed, last_filtered = True
    else:                         copied, last_filtered = False, n = 0 if n > R
    n += 1

Energies are accumulated column by column in float32 (np.sum would sum pairwise), and the state machine steps through the
segments with np.float32 scalars, so every operation rounds on its own as in the block and in the device kernels."""
import ctypes as C
import os

import numpy as np

FILTER_SO = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "liboracle_ref_filter.so")


def threshold(pfa: float, length: int) -> np.float32:
    """the block's thres_: the chi-squared upper quantile with 2L degrees of freedom at the float pfa, rounded to float"""
    from scipy.stats import chi2
    return np.float32(chi2.isf(float(np.float32(pfa)), 2 * length))


def segment_energies(x: np.ndarray, length: int) -> np.ndarray:
    """float32 energies of the len(x) // length whole segments of x"""
    k = x.size // length
    seg = np.ascontiguousarray(x[:k * length], np.complex64).reshape(k, length)
    re, im = seg.real.astype(np.float32), seg.imag.astype(np.float32)
    mag = re * re + im * im
    e = np.zeros(k, np.float32)
    for i in range(length):
        e = e + mag[:, i]
    return e


class Blanker:
    """The block from its initial state.  push(x) takes the next samples of the stream and returns the output of the whole
    segments they complete (samples of an incomplete segment wait for the next push)."""

    def __init__(self, pfa: float, length: int, segments_est: int, segments_reset: int, thres=None):
        self.length = int(length)
        self.n_est, self.n_reset = int(segments_est), int(segments_reset)
        self.thres = threshold(pfa, length) if thres is None else np.float32(thres)
        self.n = 0
        self.est = np.float32(0.0)
        self.last_filtered = False
        self.segments = 0
        self.blanked = 0
        self._pending = np.zeros(0, np.complex64)

    def push(self, x) -> np.ndarray:
        x = np.concatenate([self._pending, np.asarray(x, np.complex64)])
        L = self.length
        k = x.size // L
        self._pending = x[k * L:].copy()
        out = x[:k * L].copy()
        e = segment_energies(out, L)
        two_l = np.float32(2 * L)
        with np.errstate(divide="ignore", invalid="ignore"):
            for s in range(k):
                if self.n < self.n_est and not self.last_filtered:
                    self.est = np.float32((np.float32(self.n) * self.est + e[s] / two_l) / np.float32(self.n + 1))
                elif np.float32(e[s] / self.est) > self.thres:
                    out[s * L:(s + 1) * L] = 0
                    self.last_filtered = True
                    self.blanked += 1
                else:
                    self.last_filtered = False
                    if self.n > self.n_reset:
                        self.n = 0
                self.n += 1
        self.segments += k
        return out

    def state(self) -> dict:
        """the fields of b200_iq_pulse_blanking_status that the state machine determines"""
        return {"segments": self.segments, "blanked": self.blanked, "n": self.n, "noise_power": self.est,
                "last_filtered": int(self.last_filtered)}


def blank(x, pfa: float, length: int, segments_est: int, segments_reset: int, thres=None) -> np.ndarray:
    """the output of the whole segments of x, for a block started at x[0]"""
    return Blanker(pfa, length, segments_est, segments_reset, thres).push(x)


def reference_filter():
    """the reference's pulse_blanking_cc compiled in place (oracle/_ref/liboracle_ref_filter.so), or None where it is not built"""
    if not os.path.exists(FILTER_SO):
        return None
    lib = C.CDLL(FILTER_SO)
    lib.ref_pulse_blanking.argtypes = [C.c_float, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_uint64, C.c_void_p, C.c_int,
                                       C.c_void_p, C.POINTER(C.c_uint64), C.POINTER(C.c_float), C.c_void_p, C.POINTER(C.c_float)]
    lib.ref_pulse_blanking.restype = C.c_int
    lib.ref_pulse_blanking_threshold.argtypes = [C.c_float, C.c_int32]
    lib.ref_pulse_blanking_threshold.restype = C.c_float
    return lib


def reference_block(lib, x, pfa, length, est, reset, chunk_ends):
    """the reference block over x fed in chunks ending at chunk_ends: (its published output, thres, (n, last_filtered, est))"""
    x = np.ascontiguousarray(x, np.complex64)
    ends = np.ascontiguousarray(chunk_ends, np.uint64)
    out = np.zeros(x.size, np.complex64)
    n_out, thres, e = C.c_uint64(0), C.c_float(0), C.c_float(0)
    state = np.zeros(2, np.int64)
    assert lib.ref_pulse_blanking(pfa, length, est, reset, x.ctypes.data, x.size, ends.ctypes.data, ends.size, out.ctypes.data,
                                  C.byref(n_out), C.byref(thres), state.ctypes.data, C.byref(e)) == 0
    return out[:n_out.value], np.float32(thres.value), (int(state[0]), int(state[1]), np.float32(e.value))
