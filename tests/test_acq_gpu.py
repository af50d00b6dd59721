"""GPU parity tests for the PCPS acquisition grid search, through the C ABI.

Oracle: oracle/acq_np.py (numpy restatement of pcps_acquisition.cc with pocketfft float32 FFTs) plus
the reference's own sincos kernel for the wipe-off carriers.  Contract (SURVEY 8c):
  * wipe-off carriers BIT-EXACT with volk_gnsssdr_s32f_sincos_32fc a_avx2 (for the n - n%8 samples
    the AVX2 loop produces; the <8-sample libm tail is within 1 ulp);
  * (index_time, index_doppler, doppler) EXACT;
  * test_statistics / grid_maximum / input_power / second_peak within 1e-4 relative
    (different FFT summation order; the reference pins nothing at the FFT boundary);
  * full magnitude grid within 2e-5 of the grid peak, element-wise.
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from gnss_synth import make_iq  # noqa: E402
from gpu_fixtures import capi, engine  # noqa: E402,F401
import acq_rig as ar  # noqa: E402


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def _signal(oracle, prns_present, fs, n, seed, cn0=45.0):
    rng = np.random.default_rng(seed)
    codes = {p: oracle.port.gps_ca_code(p) for p in prns_present}
    svs = [dict(prn=p, doppler=float(rng.uniform(-4500, 4500)), code_phase_chips=float(rng.uniform(0, 1023)), cn0=cn0,
                phase0=float(rng.uniform(0, 6.28))) for p in prns_present]
    return make_iq(codes, fs, n, svs, seed=seed), svs


@pytest.mark.parametrize("fs,dmax,dstep,center", [(4e6, 5000, 250, 0), (4e6, 5000, 100, 0), (25e6, 10125, 250, 0),
                                                   (4e6, 5000, 250, 1375), (2.048e6, 5000, 500, 0)])
def test_wipeoff_grid_bitexact(capi, engine, oracle, fs, dmax, dstep, center):
    import ctypes as C
    acq = ar.make(capi, engine, fs, doppler_max=dmax, doppler_step=dstep)
    if center:
        acq.set_doppler_center(center, 0)
    got = acq.read_wipeoffs()
    n, bins = acq.conf.fft_size, acq.conf.num_doppler_bins
    want = np.empty((bins, n), np.complex64)
    oracle.port.lib.port_acq_wipeoff_grid(C.c_int(1), C.c_void_p(want.ctypes.data), C.c_uint(n), C.c_uint(bins),
                                          C.c_int32(dmax), C.c_int32(center), C.c_int32(dstep), C.c_int32(0),
                                          C.c_int64(int(fs)))
    body = (n // 8) * 8
    assert np.array_equal(_bits(got[:, :body]), _bits(want[:, :body]))
    if body < n:
        assert np.max(np.abs(got[:, body:] - want[:, body:])) < 3e-7
    if oracle.ref is not None:   # and the port is the reference's kernel, bit for bit
        d = bins // 3
        doppler = -dmax + center + dstep * d
        inc = -np.float32(np.float32(2 * np.pi) * np.float32(doppler) / np.float32(fs))
        r, _ = oracle.ref.sincos("a_avx2", float(inc), 0.0, n)
        assert np.array_equal(_bits(r[:body]), _bits(got[d, :body]))
    acq.close()


@pytest.mark.parametrize("fs,dmax,dstep,cfar", [(4e6, 10000, 250, True), (4e6, 5000, 100, False), (25e6, 10125, 250, True),
                                                 (25e6, 5000, 250, False), (8e6, 5000, 500, True), (2.048e6, 5000, 250, True),
                                                 (12.5e6, 5000, 250, True), (5e6, 5000, 250, False)])
def test_single_prn_acquisition_parity(capi, engine, oracle, fs, dmax, dstep, cfar):
    p = ar.params(fs, doppler_max=dmax, doppler_step=dstep, use_CFAR_algorithm_flag=cfar, keep_grid=True)
    prn = 7
    iq, svs = _signal(oracle, [7, 12, 20], fs, int(p["samples_per_ms"]), seed=int(fs / 1e3) + dstep)
    code = ar.ca_code(oracle.port, prn, fs)
    o = ar.oracle(p, code, pfa=0.001 if cfar else 0.0)
    want = o.acquisition_core(iq)
    acq = capi.PcpsAcquisition(engine, **p)
    acq.set_local_code(0, code)
    got = acq.search(iq, [0])[0]
    ar.check(got, want, ar.CFAR_STATS if cfar else ar.PEAK_STATS)
    # the satellite is really there: Doppler within a bin, code phase within half a chip
    sv = svs[0]
    assert abs(want["doppler"] - sv["doppler"]) <= 666   # the reference test's own Doppler tolerance (1 ms main lobe)
    # whole magnitude grid
    ar.check_grid(acq.read_grid(0), o.magnitude_grid, cols=acq.conf.effective_fft_size)
    acq.close()


def test_multi_prn_sweep_shares_forward_ffts(capi, engine, oracle):
    """32 PRNs on the same samples in one call == 32 independent single-PRN searches."""
    fs, dmax, dstep = 4e6, 5000, 250
    present = [3, 9, 17, 22, 31]
    iq, _ = _signal(oracle, present, fs, 4000, seed=44, cn0=46.0)
    p = ar.params(fs, doppler_max=dmax, doppler_step=dstep, n_code_slots=32)
    acq = capi.PcpsAcquisition(engine, **p)
    ar.load_codes(acq, [ar.ca_code(oracle.port, prn, fs) for prn in range(1, 33)])
    res = acq.search(iq, np.arange(32))
    # arbitrary slot subsets / orders give the same per-PRN answers
    sub = [30, 2, 16, 8]
    res2 = acq.search(iq, sub)
    for k, s in enumerate(sub):
        assert res2[k] == res[s]
    from oracle.acq_np import compute_threshold
    th = compute_threshold(0.001, 4000, acq.conf.num_doppler_bins, 1)
    detected = {prn for prn in range(1, 33) if res[prn - 1]["test_statistics"] > th}
    assert detected == set(present)
    for prn in (3, 17, 5, 28):
        want = ar.oracle(p, ar.ca_code(oracle.port, prn, fs), pfa=0.001).acquisition_core(iq)
        ar.check(res[prn - 1], want, ("test_statistics",))
    acq.close()


def test_noncoherent_dwells_accumulate(capi, engine, oracle):
    """max_dwells = 3: magnitudes accumulate across dwells (pcps_acquisition.cc:545-553) and the
    CFAR input power is divided by the dwell counter (:431)."""
    fs, dmax, dstep, prn = 4e6, 5000, 250, 11
    iq, _ = _signal(oracle, [prn], fs, 12000, seed=77, cn0=38.0)
    p = ar.params(fs, doppler_max=dmax, doppler_step=dstep, max_dwells=3)
    code = ar.ca_code(oracle.port, prn, fs)
    o = ar.oracle(p, code, pfa=0.001)
    acq = capi.PcpsAcquisition(engine, **p)
    acq.set_local_code(0, code)
    for k in range(3):
        seg = iq[4000 * k: 4000 * (k + 1)]
        if k > 0:
            # keep accumulating regardless of the threshold decision, like a block below threshold would
            o.num_noncoherent_integrations_counter = k
        want = o.acquisition_core(seg)
        got = acq.search(seg, [0], dwell_counter=k + 1)[0]
        ar.check(got, want, ("test_statistics",))
        o.num_noncoherent_integrations_counter = k + 1
    ar.check_grid(acq.read_grid(0), o.magnitude_grid, cols=4000)
    acq.close()


def test_bit_transition_and_padded_layouts(capi, engine, oracle):
    """bit_transition_flag (2x input, code in the second half, magnitudes from the second half,
    :107-112,:230-235,:544) and sampled_ms != ms_per_code (zero-padded FFT, :243-246)."""
    fs, dmax, dstep, prn = 4e6, 5000, 250, 5
    # (a) bit transition
    iq, _ = _signal(oracle, [prn], fs, 8000, seed=5, cn0=47.0)
    code2 = ar.ca_code(oracle.port, prn, fs, 2)
    p = ar.params(fs, doppler_max=dmax, doppler_step=dstep, bit_transition_flag=True)
    want = ar.oracle(p, code2, pfa=0.001).acquisition_core(iq)
    acq = capi.PcpsAcquisition(engine, **p)
    assert (acq.conf.fft_size, acq.conf.effective_fft_size, acq.conf.consumed_samples) == (8000, 4000, 8000)
    acq.set_local_code(0, code2)
    ar.check(acq.search(iq, [0])[0], want, ("test_statistics",))
    acq.close()
    # (b) sampled_ms = 2 with ms_per_code = 1 ... equal -> plain; use ms_per_code=4 analogue: sampled 1, code 4
    p = ar.params(fs, doppler_max=dmax, doppler_step=dstep, sampled_ms=2, ms_per_code=4)
    want = ar.oracle(p, code2, pfa=0.001).acquisition_core(iq)
    acq = capi.PcpsAcquisition(engine, **p)
    assert (acq.conf.fft_size, acq.conf.consumed_samples, acq.conf.code_layout) == (16000, 8000, 2)
    acq.set_local_code(0, code2)
    ar.check(acq.search(iq, [0])[0], want, ("test_statistics",))
    acq.close()


def test_doppler_center_assisted(capi, engine, oracle):
    fs, prn = 4e6, 14
    iq, svs = _signal(oracle, [prn], fs, 4000, seed=14)
    center = int(round(svs[0]["doppler"] / 250.0)) * 250
    p = ar.params(fs, doppler_max=1000, doppler_step=125)
    code = ar.ca_code(oracle.port, prn, fs)
    want = ar.oracle(p, code, pfa=0.001, center=center).acquisition_core(iq)
    acq = capi.PcpsAcquisition(engine, **p)
    acq.set_doppler_center(center, 0)
    acq.set_local_code(0, code)
    ar.check(acq.search(iq, [0])[0], want, stats=())
    assert abs(want["doppler"] - svs[0]["doppler"]) <= 666
    acq.close()


def test_fft_round_trip_property_all_supported_radices(capi, engine, oracle):
    """Size-independent property at sizes up to the single-CTA maximum: searching the local code
    against ITSELF delayed by k samples must peak exactly at index k with zero Doppler,
    for sizes exercising radices 2,3,4,5,7,8."""
    rng = np.random.default_rng(9)
    for n in (4096, 6000, 8400, 16000, 25000, 27000, 27648, 2 * 3 * 5 * 7, 4802):
        acq = ar.make(capi, engine, n * 1000, doppler_max=1000, doppler_step=500)
        code = rng.choice([-1.0, 1.0], n).astype(np.float32).astype(np.complex64) * 1j
        acq.set_local_code(0, code)
        k = int(rng.integers(0, n))
        iq = np.roll(code, k)
        r = acq.search(iq, [0])[0]
        assert int(r["index_time"]) == k, (n, k)
        assert int(r["doppler"]) == 0
        assert abs(r["grid_maximum"] - float(n) ** 4) / float(n) ** 4 < 1e-4   # |sum of n unit products|^2 * n^2 (unnormalised IFFT)
        acq.close()


def test_acq_error_paths(capi, engine):
    with pytest.raises(capi.B200Error):   # 16368 = 2^4*3*11*31 goes through chirp-z, which has the CFAR statistic only
        ar.make(capi, engine, 16368000, doppler_max=5000, doppler_step=250, use_CFAR_algorithm_flag=False)
    with pytest.raises(capi.B200Error):   # beyond 8 x 27648 points
        ar.make(capi, engine, 300000000, samples_per_chip=290, doppler_max=1000, doppler_step=500)
    acq = ar.make(capi, engine, 4000000, doppler_max=5000, doppler_step=250)
    with pytest.raises(capi.B200Error):   # search before set_local_code
        acq.search(np.zeros(4000, np.complex64), [0])
    acq.set_local_code(0, np.ones(4000, np.complex64))
    with pytest.raises(capi.B200Error):   # dwell accumulation without a grid
        acq.search(np.zeros(4000, np.complex64), [0], dwell_counter=2)
    acq.close()


def test_two_step_acquisition(capi, engine, oracle):
    """make_2_steps (pcps_acquisition.cc:294-301,:605-626): the second step searches 4 bins of 125 Hz
    around the first step's Doppler on the next buffer, keeps the first step's input power, and uses the
    float Doppler formula."""
    fs, prn = 4e6, 8
    iq, svs = _signal(oracle, [prn], fs, 8000, seed=88, cn0=47.0)
    p = ar.params(fs, doppler_max=5000, doppler_step=500)
    code = ar.ca_code(oracle.port, prn, fs)
    o = ar.oracle(p, code, pfa=0.001, pfa2=0.001, make_2_steps=True, doppler_step2=125.0, num_doppler_bins_step2=4)
    w1 = o.acquisition_core(iq[:4000])
    assert not w1["positive"] and o.step_two          # first step passed the threshold, second pending
    w2 = o.acquisition_core(iq[4000:8000])
    assert w2["positive"] and w2["step_two"]
    acq = capi.PcpsAcquisition(engine, **p)
    acq.set_local_code(0, code)
    g1 = acq.search(iq[:4000], [0])[0]
    ar.check(g1, w1, stats=())
    acq.set_step_two(float(g1["doppler"]), 125.0, 4)
    g2 = acq.search_step_two(iq[4000:8000], 0, float(g1["input_power"]))
    ar.check(g2, w2, ("test_statistics",))
    assert abs(w2["doppler"] - svs[0]["doppler"]) < abs(w1["doppler"] - svs[0]["doppler"]) + 63   # refined (within half a fine bin)
    acq.close()


@pytest.mark.parametrize("fs,sampled_ms,dmax,dstep,cfar", [
    (50e6, 1, 5000, 500, True),       # N = 50000  = 2 x 25000
    (25e6, 4, 2000, 250, True),       # N = 100000 = 4 x 25000   (4 ms coherent)
    (50e6, 4, 1000, 250, False),      # N = 200000 = 8 x 25000   (Galileo E1 size at 50 Msps), first/second peak
    (8e6, 4, 2000, 500, True),        # N = 32000  = 2 x 16000
    (8e6, 7, 1000, 500, True),        # N = 56000  = 7 x 8000 -> radix-7 global stage
])
def test_two_level_fft_sizes(capi, engine, oracle, fs, sampled_ms, dmax, dstep, cfar):
    """fft_size above the single-CTA limit: one radix-n1 stage through global memory + in-shared-memory
    blocks.  Same contract as the small sizes: exact indices, statistics within 1e-4, grid within 2e-5."""
    p = ar.params(fs, doppler_max=dmax, doppler_step=dstep, use_CFAR_algorithm_flag=cfar, sampled_ms=sampled_ms,
                  ms_per_code=sampled_ms, keep_grid=True)
    spms = int(p["samples_per_ms"])
    n = spms * sampled_ms
    prn = 7
    codes = {q: oracle.port.gps_ca_code(q) for q in (7, 21)}
    svs = [dict(prn=7, doppler=dstep * round(0.6 * dmax / dstep) + 10.0, code_phase_chips=321.4, cn0=42.0, phase0=1.0),
           dict(prn=21, doppler=-0.3 * dmax, code_phase_chips=77.7, cn0=42.0, phase0=2.0)]
    iq = make_iq(codes, fs, n, svs, seed=int(fs / 1e3) + sampled_ms)
    local = ar.ca_code(oracle.port, prn, fs, sampled_ms)
    o = ar.oracle(p, local, pfa=0.001 if cfar else 0.0)
    want = o.acquisition_core(iq)
    acq = capi.PcpsAcquisition(engine, **p)
    assert acq.conf.fft_size == n
    acq.set_local_code(0, local)
    got = acq.search(iq, [0])[0]
    # with sampled_ms code periods in the buffer the correlation has sampled_ms mathematically equal peaks one
    # code period apart; which one wins is rounding noise, and update_synchro folds it away
    # (Acq_delay_samples = fmod(index_time, samples_per_code), pcps_acquisition.cc:582)
    ar.check(got, want, ("grid_maximum", "test_statistics"), period=spms)
    ar.check_grid(acq.read_grid(0), o.magnitude_grid, cols=acq.conf.effective_fft_size)
    assert abs(want["doppler"] - svs[0]["doppler"]) <= max(dstep, 666 / sampled_ms)
    acq.close()


@pytest.mark.parametrize("fs,sampled_ms,dmax,dstep", [
    (16.368e6, 1, 5000, 250),     # N = 16368 = 2^4 * 3 * 11 * 31   (the classic 16.368 Msps front end)  -> M = 32768
    (5.456e6, 1, 5000, 500),      # N = 5456  = 2^4 * 11 * 31
    (16.368e6, 2, 2000, 250),     # N = 32736 -> M = 65536: two-level M
    (13e6, 1, 4000, 500),         # N = 13000 = 2^3 * 5^3 * 13
])
def test_chirp_z_sizes_with_large_prime_factors(capi, engine, oracle, fs, sampled_ms, dmax, dstep):
    """fft_size with prime factors above 7: every N-point transform becomes a circular convolution with a chirp, done with
    M-point transforms (M >= 2N - 1).  Same contract as the other sizes (exact indices, statistics 1e-4, grid 2e-5 of the
    peak), plus two dwells and a Doppler-centre change through the same path."""
    kw = dict(sampled_ms=sampled_ms, ms_per_code=sampled_ms) if sampled_ms > 1 else {}
    p = ar.params(fs, doppler_max=dmax, doppler_step=dstep, use_CFAR_algorithm_flag=True, keep_grid=True, max_dwells=2,
                  n_code_slots=2, **kw)
    spms = int(p["samples_per_ms"])
    n = spms * sampled_ms
    prn = 7
    codes = {q: oracle.port.gps_ca_code(q) for q in (7, 21)}
    svs = [dict(prn=7, doppler=dstep * round(0.6 * dmax / dstep) + 10.0, code_phase_chips=321.4, cn0=47.0, phase0=1.0),
           dict(prn=21, doppler=-dstep * round(0.3 * dmax / dstep) + 20.0, code_phase_chips=77.7, cn0=47.0, phase0=2.0)]
    iq = make_iq(codes, fs, 2 * n, svs, seed=int(fs / 1e3) + sampled_ms)
    local = ar.ca_code(oracle.port, prn, fs, sampled_ms)
    o = ar.oracle(p, local, pfa=0.001)
    want = o.acquisition_core(iq[:n])
    acq = capi.PcpsAcquisition(engine, **p)
    assert acq.conf.fft_size == n
    acq.set_local_code(1, local)
    acq.set_local_code(0, ar.ca_code(oracle.port, 21, fs, sampled_ms))
    both = acq.search(iq[:n], [0, 1])
    ar.check(both[1], want, period=spms)
    ar.check_grid(acq.read_grid(1), o.magnitude_grid, cols=acq.conf.effective_fft_size)
    assert abs(want["doppler"] - svs[0]["doppler"]) <= max(dstep, 666 / sampled_ms)
    assert abs(int(both[0]["doppler"]) - svs[1]["doppler"]) <= max(dstep, 666 / sampled_ms)
    # second dwell accumulates on the grid
    o.num_noncoherent_integrations_counter = 1   # keep accumulating whatever the threshold decided
    want2 = o.acquisition_core(iq[n:])
    got2 = acq.search(iq[n:], [1], dwell_counter=2)[0]
    ar.check(got2, want2, ("test_statistics",), period=spms)
    # assisted acquisition: moving the Doppler centre rebuilds the chirped wipe-off rows
    want3 = ar.oracle(p, local, pfa=0.001, max_dwells=1, center=875).acquisition_core(iq[:n])
    acq.set_doppler_center(875)
    got3 = acq.search(iq[:n], [1])[0]
    ar.check(got3, want3, ("test_statistics",), period=spms)
    acq.close()


@pytest.mark.gpu
def test_async_search_matches_synchronous_and_guards_misuse(oracle):
    """b200_acq_search_submit / _wait: same results as b200_acq_search, one sweep in flight per object."""
    from gnss_sdr_b200 import capi
    import gnss_synth as gs
    fs, n = 4e6, 4000
    code = gs.gps_ca_code(3)
    iq = gs.make_iq({3: code}, fs, n, [dict(prn=3, doppler=2100.0, code_phase_chips=400.0, cn0=48.0)], seed=8)
    e = capi.Engine()
    a, b = (ar.make(capi, e, fs, samples_per_chip=4, doppler_max=5000, doppler_step=250, n_code_slots=2) for _ in range(2))
    for o in (a, b):
        ar.load_codes(o, [ar.ca_code(gs, prn, fs) for prn in (3, 4)])
    want = a.search(iq, [0, 1])
    a.search_submit(iq, [0, 1])
    b.search_submit(iq, [1, 0])
    with pytest.raises(capi.B200Error) as ei:
        a.search_submit(iq, [0])
    assert ei.value.code == ar.ERR_STATE
    ra, rb = a.search_wait(), b.search_wait()
    assert ra.tobytes() == want.tobytes()
    assert rb[::-1].tobytes() == want.tobytes()
    with pytest.raises(capi.B200Error):
        a.search_wait()
    a.close()
    b.close()
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("entry", ["search", "search_i16", "search_step_two", "search_step_two_i16",
                                   "search_submit", "search_band", "search_band_submit", "search_step_two_band"])
def test_host_searches_refused_while_a_sweep_is_in_flight(entry):
    """Every search that returns results to the host is B200_ERR_STATE while a submitted sweep is in flight, and the
    sweep's results are still the synchronous search's."""
    from gnss_sdr_b200 import capi
    import gnss_synth as gs
    fs, n, band = 4e6, 4000, 0
    iq = gs.make_iq({3: gs.gps_ca_code(3)}, fs, n, [dict(prn=3, doppler=2100.0, code_phase_chips=400.0, cn0=48.0)], seed=8)
    raw = ar.to_int(iq, np.int16, 100)
    e = capi.Engine()
    e.iq_create(band, 8192)
    e.iq_push(band, iq)
    a = ar.make(capi, e, fs, samples_per_chip=4, doppler_max=5000, doppler_step=250, n_code_slots=2)
    ar.load_codes(a, [ar.ca_code(gs, prn, fs) for prn in (3, 4)])
    a.set_step_two(2100.0, 125.0, 4)   # so that a step-two call is otherwise legal
    want = a.search(iq, [0, 1])
    calls = {
        "search": lambda: a.search(iq, [0]),
        "search_i16": lambda: ar.search_i16(a, raw, [0]),
        "search_step_two": lambda: a.search_step_two(iq, 0, 1.0),
        "search_step_two_i16": lambda: ar.search_step_two_i16(a, raw, 0, 1.0),
        "search_submit": lambda: a.search_submit(iq, [0]),
        "search_band": lambda: a.search_band(band, 0, [0]),
        "search_band_submit": lambda: a.search_band_submit(band, 0, [0]),
        "search_step_two_band": lambda: a.search_step_two_band(band, 0, 0, 1.0),
    }
    a.search_submit(iq, [0, 1])
    with pytest.raises(capi.B200Error) as ei:
        calls[entry]()
    assert ei.value.code == ar.ERR_STATE
    assert a.search_wait().tobytes() == want.tobytes()
    a.close()
    e.close()
