"""Shared helpers of the DLL/PLL loop tests: synthetic correlator outputs, CPU correlators behind one call shape,
and the closed loop `prepare -> correlate -> update` over a host sample buffer."""
import numpy as np

from gnss_sdr_b200.abi import TRK_DUMP_RECORD_DTYPE


def synthetic_taps(n_epochs, n_taps, seed, amp=4000.0, weak_from=None):
    """E,P,L (or VE,E,P,L,VL) of a tracked signal with data bit flips, phase jitter and noise; from epoch
    weak_from on only noise (drives the lock detectors to a loss of lock)."""
    rng = np.random.default_rng(seed)
    shape = {3: [0.5, 1.0, 0.5], 5: [0.25, 0.6, 1.0, 0.6, 0.25]}[n_taps]
    out = np.zeros((n_epochs, n_taps), np.complex64)
    bit = 1.0
    for k in range(n_epochs):
        if k % 20 == 0 and rng.random() < 0.5:
            bit = -bit
        a = amp if (weak_from is None or k < weak_from) else 0.0
        ph = rng.normal(0, 0.15)
        skew = rng.normal(0, 0.02)
        t = np.array([s * (1 + (skew if i > n_taps // 2 else -skew if i < n_taps // 2 else 0)) for i, s in enumerate(shape)])
        out[k] = (a * bit * t * np.exp(1j * ph) + rng.normal(0, 150, n_taps) + 1j * rng.normal(0, 150, n_taps)).astype(np.complex64)
    return out


class RefCorrelator:
    """The reference's Cpu_Multicorrelator_Real_Codes (oracle.ref)."""

    def __init__(self, ref, code, shifts, max_len):
        self.ref, self.taps = ref, len(shifts)
        self.h = ref.mc_create(max_len, self.taps)
        self.code = np.ascontiguousarray(code, np.float32)
        self.shifts = np.ascontiguousarray(shifts, np.float32)
        ref.mc_set_code(self.h, self.code, self.shifts)

    def __call__(self, block, p6, n):
        return self.ref.mc_correlate(self.h, block, self.taps, float(p6[0]), float(p6[1]), float(p6[2]), float(p6[3]),
                                     float(p6[4]), float(p6[5]), n)


class PortCorrelator:
    """oracle.port restatement of the same correlator (a_avx/u_avx association), for boxes without oracle/_ref."""

    def __init__(self, port, code, shifts):
        self.port, self.code, self.shifts = port, np.ascontiguousarray(code, np.float32), np.ascontiguousarray(shifts, np.float32)

    def __call__(self, block, p6, n):
        return self.port.multicorrelator(1, block, self.code, self.shifts, float(p6[0]), float(p6[1]), float(p6[3]), float(p6[4]), n)


def run_closed_loop(loop, correlate, iq, n_epochs):
    """-> structured array of the dump records of the logged cycles"""
    recs = []
    for _ in range(n_epochs):
        item = loop.prepare()
        if item is None:
            break
        s, n, p6 = item
        if s + n > len(iq):
            break
        taps = correlate(iq[s:s + n], p6, n)
        logged, r = loop.update(taps)
        if logged:
            recs.append(r)
    return np.array(recs, TRK_DUMP_RECORD_DTYPE)
