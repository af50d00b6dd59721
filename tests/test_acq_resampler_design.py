"""b200_acq_resampler_design (host only) against the float64 restatement of the reference's acquisition resampler:
decimation and tap count exact, the cases where the reference inserts no filter, every tap within 1e-6, symmetric taps of
unit DC gain, and a too-small tap buffer refused with the count it needs.  GNU Radio's own float32 tap bits are not
available offline, so nothing here claims them."""
import ctypes as C

import numpy as np
import pytest

import acq_resampler_np as rnp

ERR_ARG, ERR_RANGE = -1, -5

# (fs_in, optimal acquisition rate, decimation, taps): the rows worked out by hand from the reference's rule
ROWS = [
    (4_000_000, 2_000_000, 2, 9),
    (16_368_000, 2_000_000, 8, 39),
    (25_000_000, 2_000_000, 10, 49),
    (50_000_000, 2_000_000, 25, 121),
    (50_000_000, 10_000_000, 5, 25),
    (100_000_000, 2_000_000, 50, 241),
    (20_000_000, 2_000_000, 10, 49),
    (25_000_000, 10_000_000, 2, 9),
]


@pytest.mark.parametrize("fs,opt,d,t", ROWS, ids=[f"{r[0]}_to_{r[1]}" for r in ROWS])
def test_design_matches_the_float64_restatement(fs, opt, d, t):
    from gnss_sdr_b200 import capi
    got_d, taps = capi.acq_resampler_design(fs, opt)
    want_d, want = rnp.design(fs, opt)
    assert (got_d, taps.size) == (want_d, want.size) == (d, t)
    assert taps.dtype == np.float32
    assert np.max(np.abs(taps.astype(np.float64) - want)) < 1e-6
    assert np.array_equal(taps, taps[::-1])
    assert abs(float(np.sum(taps.astype(np.float64))) - 1.0) < 1e-6


@pytest.mark.parametrize("fs,opt", [(3_000_000, 2_000_000), (2_000_000, 2_000_000), (2_000_000, 10_000_000)],
                         ids=["decimation_1", "equal_rates", "optimal_above_input"])
def test_no_filter_where_the_reference_inserts_none(fs, opt):
    from gnss_sdr_b200 import capi
    d, taps = capi.acq_resampler_design(fs, opt)
    assert (d, taps.size) == (1, 0) == (rnp.design(fs, opt)[0], rnp.design(fs, opt)[1].size)


def test_too_small_tap_buffer_is_refused_with_the_count_needed():
    from gnss_sdr_b200 import capi
    d, n = C.c_uint32(0), C.c_uint32(0)
    buf = np.zeros(48, np.float32)
    rc = capi.lib.b200_acq_resampler_design(25_000_000, 2_000_000, buf.size, C.byref(d), buf.ctypes.data, C.byref(n))
    assert rc == ERR_RANGE
    assert (d.value, n.value) == (10, 49)
    assert "49 taps needed" in capi.lib.b200_last_error().decode()
    assert not buf.any()
    buf = np.zeros(49, np.float32)
    assert capi.lib.b200_acq_resampler_design(25_000_000, 2_000_000, buf.size, C.byref(d), buf.ctypes.data, C.byref(n)) == 0
    assert buf.any()


def test_bad_arguments():
    from gnss_sdr_b200 import capi
    d, n = C.c_uint32(0), C.c_uint32(0)
    for fs, opt in ((0, 2_000_000), (25_000_000, 0), (-1, 2_000_000)):
        assert capi.lib.b200_acq_resampler_design(fs, opt, 0, C.byref(d), None, C.byref(n)) == ERR_ARG
    assert capi.lib.b200_acq_resampler_design(25_000_000, 2_000_000, 64, C.byref(d), None, C.byref(n)) == ERR_ARG
    assert capi.lib.b200_acq_resampler_design(25_000_000, 2_000_000, 0, None, None, C.byref(n)) == ERR_ARG
