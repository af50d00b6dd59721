"""GPU parity tests for the acquisition options at chirp-z transform sizes (fft_size with a prime factor above 7, e.g.
16 368 = 2^4 * 3 * 11 * 31 at 16.368 Msps): bit transition, the zero-padded code layout, two-step acquisition and the
cshort entry points, all through the C ABI.

Oracle and contract as in test_acq_gpu.py: oracle/acq_np.py (pcps_acquisition.cc restated in numpy); exact index_time,
index_doppler and doppler; statistics within 1e-4 relative; magnitude grid within 2e-5 of its peak, element-wise.
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from gnss_synth import make_iq  # noqa: E402
from gpu_fixtures import capi, engine  # noqa: E402,F401
import acq_rig as ar  # noqa: E402


def _sampled(table, fs, n, chip_rate=1.023e6):
    """`table` (one value per chip) sampled at fs for n samples, as a complex64 local code"""
    idx = np.floor(np.arange(n, dtype=np.float64) * chip_rate / fs).astype(np.int64) % len(table)
    return table[idx].astype(np.complex64)


def test_bit_transition_gps_l1_16368(capi, engine, oracle):
    """bit_transition_flag at 16.368 Msps: 2 ms of samples, code in the second half of N = 32 736, magnitudes from
    [16 368, 32 736) of the correlation (pcps_acquisition.cc:107-112, :230-235, :544)."""
    fs, dmax, dstep, prn = 16.368e6, 5000, 250, 7
    codes = {p: oracle.port.gps_ca_code(p) for p in (7, 21)}
    svs = [dict(prn=7, doppler=1760.0, code_phase_chips=321.4, cn0=45.0, phase0=1.0, symbols=[1.0, -1.0], periods_per_symbol=1),
           dict(prn=21, doppler=-1230.0, code_phase_chips=77.7, cn0=45.0, phase0=2.0)]
    iq = make_iq(codes, fs, 2 * 16368, svs, seed=71)
    code2 = ar.ca_code(oracle.port, prn, fs, 2)
    p = ar.params(fs, doppler_max=dmax, doppler_step=dstep, bit_transition_flag=True, keep_grid=True)
    o = ar.oracle(p, code2, pfa=0.001)
    want = o.acquisition_core(iq)
    acq = capi.PcpsAcquisition(engine, **p)
    assert (acq.conf.fft_size, acq.conf.effective_fft_size, acq.conf.consumed_samples, acq.conf.code_layout) == (32736, 16368, 32736, 1)
    acq.set_local_code(0, code2)
    ar.check(acq.search(iq, [0])[0], want)
    ar.check_grid(acq.read_grid(0), o.magnitude_grid, cols=16368)
    assert abs(want["doppler"] - 1760.0) <= dstep
    acq.close()


def test_bit_transition_galileo_e1_shaped_5456(capi, engine, oracle):
    """A Galileo-E1-shaped search at 5.456 Msps: 4 ms code (4092 chips), 4 ms coherent integration, bit_transition_flag:
    N = 43 648 = 2^7 * 11 * 31, effective size 21 824."""
    fs, dmax, dstep = 5.456e6, 5000, 125
    rng = np.random.default_rng(43)
    table = rng.choice([-1.0, 1.0], 4092).astype(np.float32)
    sv = dict(prn="e", doppler=-2140.0, code_phase_chips=1234.5, cn0=42.0, phase0=0.4, symbols=[1.0, -1.0, -1.0], periods_per_symbol=1)
    iq = make_iq({"e": table}, fs, 2 * 21824, [sv], seed=44)
    local = _sampled(table, fs, 21824)
    p = ar.params(fs, doppler_max=dmax, doppler_step=dstep, sampled_ms=4, ms_per_code=4, bit_transition_flag=True, keep_grid=True)
    o = ar.oracle(p, np.tile(local, 2), samples_per_code=4 * p["samples_per_ms"], pfa=0.001)
    want = o.acquisition_core(iq)
    acq = capi.PcpsAcquisition(engine, **p)
    assert (acq.conf.fft_size, acq.conf.effective_fft_size, acq.conf.consumed_samples) == (43648, 21824, 43648)
    acq.set_local_code(0, local)
    ar.check(acq.search(iq, [0])[0], want)
    ar.check_grid(acq.read_grid(0), o.magnitude_grid, cols=21824)
    assert abs(want["doppler"] + 2140.0) <= dstep
    acq.close()


@pytest.mark.parametrize("fs,dmax,dstep", [(16.368e6, 5000, 250), (5.456e6, 5000, 500)])
def test_zero_padded_layout_dwells_and_doppler_center(capi, engine, oracle, fs, dmax, dstep):
    """sampled_ms = 2 with ms_per_code = 1: 2 ms of samples zero-padded to N = 4 code periods, code at [N - consumed, N)
    (:243-246).  Two dwells accumulate on the grid, then a Doppler-centre change rebuilds the chirped wipe-off rows.  The
    searched code sits in slot 1, so the grid rows of slot 1 must land where read_grid looks for them."""
    p = ar.params(fs, doppler_max=dmax, doppler_step=dstep, max_dwells=2, keep_grid=True, n_code_slots=2, sampled_ms=2,
                  ms_per_code=1)
    n1 = int(p["samples_per_ms"])
    prn = 7
    codes = {p: oracle.port.gps_ca_code(p) for p in (7, 21)}
    svs = [dict(prn=7, doppler=dstep * round(0.6 * dmax / dstep) + 10.0, code_phase_chips=321.4, cn0=44.0, phase0=1.0),
           dict(prn=21, doppler=-dstep * round(0.3 * dmax / dstep) + 20.0, code_phase_chips=77.7, cn0=44.0, phase0=2.0)]
    iq = make_iq(codes, fs, 4 * n1, svs, seed=int(fs / 1e3) + 2)
    code2 = ar.ca_code(oracle.port, prn, fs, 2)
    o = ar.oracle(p, code2, pfa=0.001)
    acq = capi.PcpsAcquisition(engine, **p)
    assert (acq.conf.fft_size, acq.conf.effective_fft_size, acq.conf.consumed_samples, acq.conf.code_layout) == (4 * n1, 4 * n1, 2 * n1, 2)
    acq.set_local_code(1, code2)
    acq.set_local_code(0, ar.ca_code(oracle.port, 21, fs, 2))
    want = o.acquisition_core(iq[:2 * n1])
    both = acq.search(iq[:2 * n1], [0, 1])
    ar.check(both[1], want)
    ar.check_grid(acq.read_grid(1), o.magnitude_grid, cols=4 * n1)
    assert abs(want["doppler"] - svs[0]["doppler"]) <= dstep
    assert abs(int(both[0]["doppler"]) - svs[1]["doppler"]) <= dstep
    # second dwell accumulates on the grid
    o.num_noncoherent_integrations_counter = 1   # keep accumulating whatever the threshold decided
    want2 = o.acquisition_core(iq[2 * n1:])
    ar.check(acq.search(iq[2 * n1:], [1], dwell_counter=2)[0], want2)
    ar.check_grid(acq.read_grid(1), o.magnitude_grid, cols=4 * n1)
    # assisted acquisition
    center = 2 * dstep
    want3 = ar.oracle(p, code2, pfa=0.001, max_dwells=1, center=center).acquisition_core(iq[:2 * n1])
    acq.set_doppler_center(center)
    ar.check(acq.search(iq[:2 * n1], [1])[0], want3)
    acq.close()


def test_two_step_acquisition_16368(capi, engine, oracle):
    """make_2_steps at 16.368 Msps (pcps_acquisition.cc:294-301, :605-626): step two searches 4 bins of 125 Hz around the
    step-one Doppler on the next buffer, keeps the step-one input power and uses the float Doppler formula.  The narrow
    grid comes back through read_grid as for a mixed-radix object (the first num_doppler_bins_step2 rows)."""
    fs, prn = 16.368e6, 8
    sv = dict(prn=prn, doppler=2310.0, code_phase_chips=512.3, cn0=46.0, phase0=0.7)
    iq = make_iq({prn: oracle.port.gps_ca_code(prn)}, fs, 2 * 16368, [sv], seed=88)
    code = ar.ca_code(oracle.port, prn, fs)
    p = ar.params(fs, doppler_max=5000, doppler_step=500, keep_grid=True)
    o = ar.oracle(p, code, pfa=0.001, pfa2=0.001, make_2_steps=True, doppler_step2=125.0, num_doppler_bins_step2=4)
    w1 = o.acquisition_core(iq[:16368])
    assert not w1["positive"] and o.step_two          # first step passed the threshold, second pending
    w2 = o.acquisition_core(iq[16368:])
    assert w2["positive"] and w2["step_two"]
    acq = capi.PcpsAcquisition(engine, **p)
    acq.set_local_code(0, code)
    with pytest.raises(capi.B200Error):               # step two before set_step_two
        acq.search_step_two(iq[16368:], 0, 1.0)
    g1 = acq.search(iq[:16368], [0])[0]
    ar.check(g1, w1)
    acq.set_step_two(float(g1["doppler"]), 125.0, 4)
    g2 = acq.search_step_two(iq[16368:], 0, float(g1["input_power"]))
    ar.check(g2, w2)
    assert g2["input_power"] == g1["input_power"]
    ar.check_grid(acq.read_grid(0), o.magnitude_grid, rows=4, cols=16368)
    assert abs(w2["doppler"] - sv["doppler"]) < abs(w1["doppler"] - sv["doppler"]) + 63   # refined (within half a fine bin)
    # a first-step search after the second one is back on the wide grid
    g3 = acq.search(iq[:16368], [0])[0]
    assert g3.tobytes() == g1.tobytes()
    acq.close()


def test_cshort_entry_points_match_float_path(capi, engine, oracle):
    """b200_acq_search_i16 / _step_two_i16 at chirp-z sizes: the int16 pairs are converted on the device, so the result
    records equal those of the float entry points on the converted samples, byte for byte.  The engine's launch counter
    grows by exactly the launches issued: 5 + 5 per slot for a chirp-z search, plus the conversion."""
    fs, prn = 16.368e6, 3
    sv = dict(prn=prn, doppler=-1480.0, code_phase_chips=700.2, cn0=47.0, phase0=0.2)
    iq = make_iq({prn: oracle.port.gps_ca_code(prn)}, fs, 4 * 16368, [sv], seed=33)
    sc = ar.to_int(iq, np.int16, 64.0)
    conv = ar.from_int(sc)

    # bit transition through b200_acq_search_i16
    acq = ar.make(capi, engine, fs, doppler_max=5000, doppler_step=250, bit_transition_flag=True)
    acq.set_local_code(0, ar.ca_code(oracle.port, prn, fs, 2))
    n = acq.conf.consumed_samples
    k0 = engine.launch_count()
    want = acq.search(conv[:n], [0])
    k1 = engine.launch_count()
    got = ar.search_i16(acq, sc[:2 * n], [0])
    k2 = engine.launch_count()
    assert got.tobytes() == want.tobytes()
    assert abs(int(got[0]["doppler"]) - sv["doppler"]) <= 250
    assert k1 - k0 == 5 + 5 * 1 and k2 - k1 == k1 - k0 + 1
    acq.close()

    # step two through b200_acq_search_step_two_i16
    acq = ar.make(capi, engine, fs, doppler_max=5000, doppler_step=500)
    acq.set_local_code(0, ar.ca_code(oracle.port, prn, fs))
    g1 = acq.search(conv[:16368], [0])[0]
    acq.set_step_two(float(g1["doppler"]), 125.0, 4)
    k0 = engine.launch_count()
    want2 = acq.search_step_two(conv[16368:2 * 16368], 0, float(g1["input_power"]))
    k1 = engine.launch_count()
    got2 = ar.search_step_two_i16(acq, sc[2 * 16368:4 * 16368], 0, float(g1["input_power"]))
    k2 = engine.launch_count()
    assert got2.tobytes() == want2.tobytes()
    assert abs(int(want2["doppler"]) - sv["doppler"]) <= 125
    assert k1 - k0 == 5 + 5 * 1 and k2 - k1 == k1 - k0 + 1
    acq.close()


@pytest.mark.parametrize("n", [5456, 16368])
def test_round_trip_every_layout(capi, engine, n):
    """A random +-1 code searched against itself delayed by k samples peaks at the delay with zero Doppler, for each code
    layout (plain, bit transition, zero-padded) at two chirp-z sizes.  The correlation index of the delay is k shifted by
    where the layout places the code (N - consumed for the zero-padded layout) and by the bit-transition window offset."""
    for layout in (0, 1, 2):
        rng = np.random.default_rng(n + layout)
        kw = {0: {}, 1: dict(bit_transition_flag=True), 2: dict(sampled_ms=2, ms_per_code=1)}[layout]
        acq = ar.make(capi, engine, n * 1000, doppler_max=1000, doppler_step=500, **kw)
        c = acq.conf
        assert c.code_layout == layout
        need = ar.code_len(c)
        code = (rng.choice([-1.0, 1.0], need).astype(np.float32) * 1j).astype(np.complex64)
        acq.set_local_code(0, code)
        k = int(rng.integers(0, need // 2))
        iq = np.roll(np.tile(code, c.consumed_samples // need), k)
        r = acq.search(iq, [0])[0]
        place = {0: 0, 1: c.fft_size // 2, 2: c.fft_size - c.consumed_samples}[layout]
        off = c.effective_fft_size if layout == 1 else 0
        assert int(r["index_time"]) == (k + place - off) % c.fft_size, (n, layout, k)
        assert int(r["doppler"]) == 0
        acq.close()


def test_chirp_z_limits_stay(capi, engine):
    """What chirp-z sizes still refuse: the first/second-peak statistic, and fft_size above 5 x 27 648 = 138 240 points.
    Both are named in the error text."""
    # 16.368 Msps, 5 ms, bit transition: N = 163 680
    with pytest.raises(capi.B200Error) as ei:
        ar.make(capi, engine, 16368000, doppler_max=1000, doppler_step=500, sampled_ms=5, ms_per_code=5, bit_transition_flag=True)
    assert "use_cfar = 1" in str(ei.value) and "138240" in str(ei.value)
    with pytest.raises(capi.B200Error) as ei:
        ar.make(capi, engine, 16368000, doppler_max=1000, doppler_step=500, bit_transition_flag=True, use_CFAR_algorithm_flag=False)
    assert "use_cfar = 1" in str(ei.value)
