"""The signal conditioner's host side, without a GPU: b200_iq_conditioner_lowpass (the input filter's filter_type = lowpass
branch) against the float64 firdes::low_pass restatement, its defaults and refusals, and its identity with the acquisition
resampler's design, which shares the one restatement in the library; and the numpy restatements the GPU tests hold the
device to: at IF = 0 the float32 loop is the acquisition resampler's, the rotator's phase step is exact, and the float32
loop stays within the stated bound of the float64 truth at output indices past 2^40."""
import ctypes as C

import numpy as np
import pytest

import acq_resampler_np as rnp
import iq_conditioner_np as cnp

ERR_ARG, ERR_RANGE = -1, -5

# (fs, decimation, bw, tw, taps): bw / tw 0 take the adapter's defaults bw = fs / D / 2, tw = bw / 10
ROWS = [
    (25e6, 5, 0.0, 0.0, 241),
    (25e6, 10, 0.0, 0.0, 481),
    (50e6, 25, 1.0e6, 1.0e6, 121),
    (4e6, 2, 0.0, 2e5, 49),
    (16.368e6, 8, 0.9e6, 0.0, 439),
]


@pytest.mark.parametrize("fs,d,bw,tw,t", ROWS, ids=[f"{int(r[0])}_d{r[1]}_{r[4]}" for r in ROWS])
def test_lowpass_matches_the_float64_restatement(fs, d, bw, tw, t):
    from gnss_sdr_b200 import capi
    taps = capi.iq_conditioner_lowpass(fs, d, bw, tw)
    bw_ = bw if bw > 0 else (fs / d) / 2
    tw_ = tw if tw > 0 else bw_ / 10.0
    want = rnp.low_pass(1.0, fs, bw_, tw_)
    assert taps.dtype == np.float32 and taps.size == want.size == t
    assert np.max(np.abs(taps.astype(np.float64) - want)) < 1e-6
    assert np.array_equal(taps, taps[::-1])
    assert abs(float(np.sum(taps.astype(np.float64))) - 1.0) < 1e-5


@pytest.mark.parametrize("fs,opt", [(25_000_000, 2_000_000), (50_000_000, 10_000_000), (16_368_000, 2_000_000)])
def test_lowpass_is_the_acquisition_resamplers_design(fs, opt):
    """both entry points run the same firdes::low_pass: the same cutoff and transition give the same float32 taps"""
    from gnss_sdr_b200 import capi
    d, taps = capi.acq_resampler_design(fs, opt)
    fs_d = fs / d
    got = capi.iq_conditioner_lowpass(float(fs), d, fs_d / 2.1, fs_d / 2.0)
    assert got.tobytes() == taps.tobytes()


def test_lowpass_refusals():
    from gnss_sdr_b200 import capi
    fn = capi.lib.b200_iq_conditioner_lowpass
    n = C.c_uint32(0)
    buf = np.zeros(240, np.float32)
    assert fn(25e6, 5, 0.0, 0.0, buf.size, buf.ctypes.data, C.byref(n)) == ERR_RANGE
    assert n.value == 241 and "241 taps needed" in capi.lib.b200_last_error().decode()
    assert not buf.any()
    for args in ((0.0, 5, 0.0, 0.0, 0, None), (-1.0, 5, 0.0, 0.0, 0, None), (25e6, 0, 0.0, 0.0, 0, None),
                 (float("nan"), 5, 0.0, 0.0, 0, None), (25e6, 5, float("inf"), 0.0, 0, None), (25e6, 5, 0.0, 0.0, 8, None)):
        assert fn(*args, C.byref(n)) == ERR_ARG, args
    assert fn(25e6, 5, 0.0, 0.0, 0, None, None) == ERR_ARG
    assert fn(25e6, 5, 0.0, 1e-300, 0, None, C.byref(n)) == ERR_RANGE      # no buffer holds that many taps


def test_f32_restatement_at_if_zero_is_the_resamplers_loop():
    rng = np.random.default_rng(1)
    x = (rng.normal(0, 100, 5000) + 1j * rng.normal(0, 100, 5000)).astype(np.complex64)
    h = rng.normal(0, 1, 37).astype(np.float32)
    d, j0, n = 5, 40, 900
    got = cnp.condition_f32(x, 0, h, d, 0.0, 25e6, j0, n)
    assert got.tobytes() == rnp.decimate_f32(x, h, d, j0 * d, n).tobytes()
    # zero history below index 0
    y = cnp.condition_f32(x, 0, h, d, 0.0, 25e6, 0, 3)
    assert y[0] == np.complex64(h[0] * x[0])


@pytest.mark.parametrize("if_hz,fs,d,want", [(1.25e6, 25e6, 5, 1 << 126), (-1.25e6, 25e6, 5, 3 << 126), (0.0, 25e6, 5, 0),
                                             (3e6, 8e6, 3, 1 << 125)])
def test_rotator_step_is_exact(if_hz, fs, d, want):
    assert cnp.rotator_step(if_hz, fs, d) == want


@pytest.mark.parametrize("if_hz", [2.1e6, -3.3e6, 4_092_000.0])
def test_f32_restatement_follows_the_f64_truth_past_2_40(if_hz):
    rng = np.random.default_rng(2)
    fs, d = 25e6, 5
    h = cnp.composite_taps(np.hanning(31) / 16, 0.0, fs).real
    j0 = (1 << 40) + 12_345
    x0 = j0 * d - (h.size - 1)
    x = (rng.normal(0, 30, 4000) + 1j * rng.normal(0, 30, 4000)).astype(np.complex64)
    n = (x.size - h.size) // d
    got = cnp.condition_f32(x, x0, h, d, if_hz, fs, j0, n)
    want, scale = cnp.condition_f64(x, x0, h, d, if_hz, fs, j0, n)
    bound = (h.size + 4) * 2.0 ** -23 * scale
    assert np.all(np.abs(got - want) <= bound)
    # the rotator is what it claims to be: its phase step per output reproduces the exact phase to 2^-60 cycles
    j = j0 + np.arange(n)
    err = (cnp.rotator_phase(cnp.rotator_step(if_hz, fs, d), j) - cnp.exact_phase(if_hz, fs, d, j) + 0.5) % 1.0 - 0.5
    assert np.max(np.abs(err)) < 2.0 ** -50
