"""Exact references of the tracking correlator tests: the integer correlation over the reference's chip indices, the
small-integer code tables the integer-exact tests correlate, and the reference's own AVX correlator (the C port where
oracle/_ref is not built)."""
import numpy as np


def int_oracle(x_int, code_int, idx):
    """exact integer correlation given chip indices (taps x n)."""
    return np.array([np.sum(x_int * code_int[idx[t]]) for t in range(idx.shape[0])], dtype=np.int64)


def chip_indices(oracle, code, rem, step, shifts, n):
    """the reference's chip index of every tap and sample (taps x n): its resampler with the a_avx association"""
    return oracle.port.resampler(1, np.asarray(code, np.float32), rem, step, shifts, n, return_idx=True)[1]


def exact_taps(oracle, x_int, code_int, rem, step, shifts, n):
    """exact integer taps of the n samples x_int against the small-integer table code_int, at the reference's indices"""
    return int_oracle(x_int, code_int, chip_indices(oracle, code_int, rem, step, shifts, n))


def int_code(L, salt=0, nonzero=False):
    """((k * (7919 + 2 salt)) mod 31) - 15 for k < L, values in [-15, 15]; nonzero: its zeros replaced by 16"""
    c = ((np.arange(L) * (7919 + 2 * salt)) % 31) - 15
    if nonzero:
        c[c == 0] = 16
    return c


def ref_or_port_avx(oracle, iq, code, shifts, rem_carr, dphi, rem_code, step):
    if oracle.ref is not None:
        oracle.ref.select_arch("a_avx")
        h = oracle.ref.mc_create(len(iq), len(shifts), high_dyn=False)
        oracle.ref.mc_set_code(h, code, shifts)
        out = oracle.ref.mc_correlate(h, iq, len(shifts), rem_carr, dphi, 0.0, rem_code, step, 0.0)
        oracle.ref.mc_destroy(h)
        return out
    return oracle.port.multicorrelator(1, iq, code, shifts, rem_carr, dphi, rem_code, step)
