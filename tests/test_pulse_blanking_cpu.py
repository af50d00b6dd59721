"""The pulse blanker's host side, without a GPU: b200_iq_pulse_blanking_threshold against scipy and against the reference
block's own threshold, and the numpy restatement the GPU tests hold the device to, byte for byte against the reference's
pulse_blanking_cc compiled in place (oracle/_ref/liboracle_ref_filter.so): pulsed and pulse-free noise, resets forced by
small segments_est / segments_reset, segments_est = 0, all-zero input and chunkings that do not align with the segments."""
import ctypes as C

import numpy as np
import pytest

import pulse_blanking_np as pnp

ERR_ARG = -1

PFAS = [1e-6, 1e-4, 1e-3, 0.01, 0.04, 0.1, 0.5]
LENGTHS = [1, 8, 32, 100, 1024]


@pytest.fixture(scope="module")
def reflib():
    lib = pnp.reference_filter()
    if lib is None:
        pytest.skip("oracle/_ref/liboracle_ref_filter.so not built (make -C oracle filter; needs the reference tree)")
    return lib


def noise_with_pulses(n, seed, pulses=True, scale=1.0):
    """complex64 unit noise, with strong DME-like pulse pairs (12 us apart at 4 Msps, each a few segments long) when pulses"""
    rng = np.random.default_rng(seed)
    x = ((rng.standard_normal(n) + 1j * rng.standard_normal(n)) * (scale / np.sqrt(2))).astype(np.complex64)
    if pulses:
        for start in rng.integers(0, n - 200, n // 2000):
            for off in (0, 48):
                w = np.exp(-0.5 * ((np.arange(40) - 20) / 6.0) ** 2) * 30.0 * scale
                x[start + off:start + off + 40] += (w * np.exp(1j * rng.uniform(0, 2 * np.pi))).astype(np.complex64)
    return x


def test_threshold_matches_scipy_and_the_reference_block(reflib):
    from gnss_sdr_b200 import capi
    for pfa in PFAS:
        for L in LENGTHS:
            got = np.float32(capi.pulse_blanking_threshold(pfa, L))
            assert got == pnp.threshold(pfa, L), (pfa, L)
            assert got == np.float32(reflib.ref_pulse_blanking_threshold(pfa, L)), (pfa, L)


def test_status_layout_matches_header():
    from gnss_sdr_b200 import capi
    assert C.sizeof(capi.PulseBlankingStatus) == 48


def test_threshold_refusals():
    from gnss_sdr_b200 import capi
    t = C.c_float(0)
    for pfa, L in [(0.0, 32), (1.0, 32), (-0.1, 32), (float("nan"), 32), (0.04, 0), (0.04, -1),
                   (0.04, capi.B200_IQ_MAX_BLANKING_LENGTH + 1)]:
        assert capi.lib.b200_iq_pulse_blanking_threshold(pfa, L, C.byref(t)) == ERR_ARG, (pfa, L)
    assert capi.lib.b200_iq_pulse_blanking_threshold(0.04, 32, None) == ERR_ARG
    assert capi.lib.b200_iq_pulse_blanking_threshold(0.04, capi.B200_IQ_MAX_BLANKING_LENGTH, C.byref(t)) == 0


def check_against_block(lib, x, pfa, length, est, reset, chunk_ends):
    got, thres, (n, lf, e) = pnp.reference_block(lib, x, pfa, length, est, reset, chunk_ends)
    assert got.size % length == 0 and got.size < x.size
    b = pnp.Blanker(pfa, length, est, reset)
    assert b.thres == thres
    mine = b.push(x[:got.size])
    assert mine.tobytes() == got.tobytes()
    assert (b.n, int(b.last_filtered)) == (n, lf)
    assert b.est.tobytes() == e.tobytes()
    return b


CASES = [
    # pfa, L, E, R, pulses
    (0.04, 32, 12500, 5000000, True),  # the adapter's defaults: all estimation at this length
    (0.04, 32, 1000, 5000000, True),
    (0.04, 32, 200, 5000000, False),
    (0.01, 7, 50, 120, True),         # dozens of resets: the n = 1 blend after each
    (0.04, 32, 3, 9, True),
    (0.1, 1, 40, 300, True),
    (0.04, 301, 4, 11, True),
    (0.04, 32, 0, 5000000, True),     # E = 0: est stays 0, e / 0 = inf blanks
    (0.04, 16, 1, 0, True),
]


@pytest.mark.parametrize("pfa,length,est,reset,pulses", CASES, ids=[f"L{c[1]}_E{c[2]}_R{c[3]}_{'p' if c[4] else 'n'}" for c in CASES])
def test_restatement_matches_the_reference_block(reflib, pfa, length, est, reset, pulses):
    n = 120_000
    x = noise_with_pulses(n, seed=length * 7 + est, pulses=pulses)
    b = check_against_block(reflib, x, pfa, length, est, reset, [n])
    if pulses and 0 < est < b.segments // 2:
        assert b.blanked > 0
    if reset < 1000:
        assert (b.segments - est) // (reset + 1) >= 2  # several reset cycles


@pytest.mark.parametrize("length", [1, 7, 32])
def test_restatement_matches_the_block_over_unaligned_chunks(reflib, length):
    n = 60_000
    x = noise_with_pulses(n, seed=11 + length)
    rng = np.random.default_rng(length)
    ends = np.cumsum(rng.integers(1, 3 * length + 500, 4000))
    ends = np.append(ends[ends < n], n)
    check_against_block(reflib, x, 0.02, length, 30, 200, ends)
    # the restatement's own pushes, at another chunking, give the same bytes
    b1, b2 = pnp.Blanker(0.02, length, 30, 200), pnp.Blanker(0.02, length, 30, 200)
    whole = b1.push(x)
    parts = np.concatenate([b2.push(x[a:c]) for a, c in zip(np.append(0, ends[:-1]), ends)])
    assert whole.tobytes() == parts.tobytes()


def test_all_zero_input(reflib):
    x = np.zeros(20_000, np.complex64)
    for est in (0, 5):  # 0 / 0 = NaN is not above the threshold: copied
        b = check_against_block(reflib, x, 0.04, 32, est, 40, [x.size])
        assert b.blanked == 0


def test_e0_with_zero_segments_mixed(reflib):
    """E = 0 and segments of zeros among noise: e / 0 is +inf (blanked) for noise and NaN (copied) for zeros"""
    x = noise_with_pulses(16_000, seed=5, pulses=False)
    x[3200:6400] = 0
    b = check_against_block(reflib, x, 0.04, 32, 0, 10, [x.size])
    assert 0 < b.blanked < b.segments
