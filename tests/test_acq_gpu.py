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


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def _signal(oracle, prns_present, fs, n, seed, cn0=45.0):
    rng = np.random.default_rng(seed)
    codes = {p: oracle.port.gps_ca_code(p) for p in prns_present}
    svs = [dict(prn=p, doppler=float(rng.uniform(-4500, 4500)), code_phase_chips=float(rng.uniform(0, 1023)), cn0=cn0,
                phase0=float(rng.uniform(0, 6.28))) for p in prns_present]
    return make_iq(codes, fs, n, svs, seed=seed), svs


def _oracle_acq(oracle, fs, spms, spchip, dmax, dstep, prn, iq, cfar=True, dwells=1, center=0, **kw):
    from oracle.acq_np import AcqConf, PcpsAcquisitionOracle
    conf = AcqConf(fs_in=int(fs), samples_per_ms=spms, samples_per_code=spms, samples_per_chip=spchip, doppler_max=dmax,
                   doppler_step=dstep, pfa=0.001 if cfar else 0.0, threshold=0.0, use_CFAR_algorithm_flag=cfar,
                   max_dwells=dwells, **kw)
    o = PcpsAcquisitionOracle(conf)
    if center:
        o.set_doppler_center(center)
    o.set_local_code(oracle.port.gps_ca_code_complex_sampled(prn, int(fs)) if kw.get("sampled_ms", 1) == 1 else
                     np.tile(oracle.port.gps_ca_code_complex_sampled(prn, int(fs)), kw["sampled_ms"]))
    return o


@pytest.mark.parametrize("fs,dmax,dstep,center", [(4e6, 5000, 250, 0), (4e6, 5000, 100, 0), (25e6, 10125, 250, 0),
                                                   (4e6, 5000, 250, 1375), (2.048e6, 5000, 500, 0)])
def test_wipeoff_grid_bitexact(capi, engine, oracle, fs, dmax, dstep, center):
    import ctypes as C
    spms = fs / 1000.0
    acq = capi.PcpsAcquisition(engine, fs_in=int(fs), samples_per_ms=spms, samples_per_chip=int(fs / 1.023e6),
                               doppler_max=dmax, doppler_step=dstep)
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
    spms = fs / 1000.0
    n = int(spms)
    spchip = int(fs / 1.023e6)
    prn = 7
    iq, svs = _signal(oracle, [7, 12, 20], fs, n, seed=int(fs / 1e3) + dstep)
    o = _oracle_acq(oracle, fs, spms, spchip, dmax, dstep, prn, iq, cfar=cfar)
    want = o.acquisition_core(iq)
    acq = capi.PcpsAcquisition(engine, fs_in=int(fs), samples_per_ms=spms, samples_per_chip=spchip, doppler_max=dmax,
                               doppler_step=dstep, use_CFAR_algorithm_flag=cfar, keep_grid=True)
    acq.set_local_code(0, oracle.port.gps_ca_code_complex_sampled(prn, int(fs)))
    got = acq.search(iq, [0])[0]
    assert int(got["index_time"]) == want["index_time"]
    assert int(got["index_doppler"]) == want["index_doppler"]
    assert int(got["doppler"]) == want["doppler"]
    assert abs(got["grid_maximum"] - want["grid_maximum"]) / want["grid_maximum"] < 1e-4
    assert abs(got["test_statistics"] - want["test_statistics"]) / want["test_statistics"] < 1e-4
    if cfar:
        assert abs(got["input_power"] - want["input_power"]) / want["input_power"] < 1e-4
    else:
        assert abs(got["second_peak"] - want["second_peak"]) / want["second_peak"] < 1e-4
    # the satellite is really there: Doppler within a bin, code phase within half a chip
    sv = svs[0]
    assert abs(want["doppler"] - sv["doppler"]) <= 666   # the reference test's own Doppler tolerance (1 ms main lobe)
    # whole magnitude grid
    g = acq.read_grid(0)
    ref_g = o.magnitude_grid[:, :acq.conf.effective_fft_size]
    assert np.max(np.abs(g - ref_g)) / ref_g.max() < 2e-5
    acq.close()


def test_multi_prn_sweep_shares_forward_ffts(capi, engine, oracle):
    """32 PRNs on the same samples in one call == 32 independent single-PRN searches."""
    fs, dmax, dstep = 4e6, 5000, 250
    present = [3, 9, 17, 22, 31]
    iq, _ = _signal(oracle, present, fs, 4000, seed=44, cn0=46.0)
    acq = capi.PcpsAcquisition(engine, fs_in=int(fs), samples_per_ms=4000.0, samples_per_chip=3, doppler_max=dmax,
                               doppler_step=dstep, n_code_slots=32)
    for p in range(1, 33):
        acq.set_local_code(p - 1, oracle.port.gps_ca_code_complex_sampled(p, int(fs)))
    res = acq.search(iq, np.arange(32))
    # arbitrary slot subsets / orders give the same per-PRN answers
    sub = [30, 2, 16, 8]
    res2 = acq.search(iq, sub)
    for k, s in enumerate(sub):
        assert res2[k] == res[s]
    from oracle.acq_np import compute_threshold
    th = compute_threshold(0.001, 4000, acq.conf.num_doppler_bins, 1)
    detected = {p for p in range(1, 33) if res[p - 1]["test_statistics"] > th}
    assert detected == set(present)
    for p in (3, 17, 5, 28):
        o = _oracle_acq(oracle, fs, 4000.0, 3, dmax, dstep, p, iq)
        want = o.acquisition_core(iq)
        got = res[p - 1]
        assert (int(got["index_time"]), int(got["index_doppler"])) == (want["index_time"], want["index_doppler"])
        assert abs(got["test_statistics"] - want["test_statistics"]) / want["test_statistics"] < 1e-4
    acq.close()


def test_noncoherent_dwells_accumulate(capi, engine, oracle):
    """max_dwells = 3: magnitudes accumulate across dwells (pcps_acquisition.cc:545-553) and the
    CFAR input power is divided by the dwell counter (:431)."""
    fs, dmax, dstep, prn = 4e6, 5000, 250, 11
    iq, _ = _signal(oracle, [prn], fs, 12000, seed=77, cn0=38.0)
    o = _oracle_acq(oracle, fs, 4000.0, 3, dmax, dstep, prn, iq, dwells=3)
    acq = capi.PcpsAcquisition(engine, fs_in=int(fs), samples_per_ms=4000.0, samples_per_chip=3, doppler_max=dmax,
                               doppler_step=dstep, max_dwells=3)
    acq.set_local_code(0, oracle.port.gps_ca_code_complex_sampled(prn, int(fs)))
    for k in range(3):
        seg = iq[4000 * k: 4000 * (k + 1)]
        want = o.acquisition_core(seg) if k == 0 else None
        if k > 0:
            # keep accumulating regardless of the threshold decision, like a block below threshold would
            o.num_noncoherent_integrations_counter = k
            want = o.acquisition_core(seg)
        got = acq.search(seg, [0], dwell_counter=k + 1)[0]
        assert (int(got["index_time"]), int(got["index_doppler"])) == (want["index_time"], want["index_doppler"])
        assert abs(got["test_statistics"] - want["test_statistics"]) / want["test_statistics"] < 1e-4
        o.num_noncoherent_integrations_counter = k + 1
    g = acq.read_grid(0)
    assert np.max(np.abs(g - o.magnitude_grid[:, :4000])) / o.magnitude_grid.max() < 2e-5
    acq.close()


def test_bit_transition_and_padded_layouts(capi, engine, oracle):
    """bit_transition_flag (2x input, code in the second half, magnitudes from the second half,
    :107-112,:230-235,:544) and sampled_ms != ms_per_code (zero-padded FFT, :243-246)."""
    fs, dmax, dstep, prn = 4e6, 5000, 250, 5
    # (a) bit transition
    iq, _ = _signal(oracle, [prn], fs, 8000, seed=5, cn0=47.0)
    from oracle.acq_np import AcqConf, PcpsAcquisitionOracle
    conf = AcqConf(fs_in=int(fs), samples_per_ms=4000.0, samples_per_code=4000.0, samples_per_chip=3, doppler_max=dmax,
                   doppler_step=dstep, pfa=0.001, bit_transition_flag=True)
    o = PcpsAcquisitionOracle(conf)
    code = oracle.port.gps_ca_code_complex_sampled(prn, int(fs))
    code2 = np.tile(code, 2)
    o.set_local_code(code2)
    want = o.acquisition_core(iq)
    acq = capi.PcpsAcquisition(engine, fs_in=int(fs), samples_per_ms=4000.0, samples_per_chip=3, doppler_max=dmax,
                               doppler_step=dstep, bit_transition_flag=True)
    assert (acq.conf.fft_size, acq.conf.effective_fft_size, acq.conf.consumed_samples) == (8000, 4000, 8000)
    acq.set_local_code(0, code2)
    got = acq.search(iq, [0])[0]
    assert (int(got["index_time"]), int(got["index_doppler"])) == (want["index_time"], want["index_doppler"])
    assert abs(got["test_statistics"] - want["test_statistics"]) / want["test_statistics"] < 1e-4
    acq.close()
    # (b) sampled_ms = 2 with ms_per_code = 1 ... equal -> plain; use ms_per_code=4 analogue: sampled 1, code 4
    conf = AcqConf(fs_in=int(fs), samples_per_ms=4000.0, samples_per_code=4000.0, samples_per_chip=3, doppler_max=dmax,
                   doppler_step=dstep, pfa=0.001, sampled_ms=2, ms_per_code=4)
    o = PcpsAcquisitionOracle(conf)
    o.set_local_code(code2)
    want = o.acquisition_core(iq)
    acq = capi.PcpsAcquisition(engine, fs_in=int(fs), samples_per_ms=4000.0, samples_per_chip=3, doppler_max=dmax,
                               doppler_step=dstep, sampled_ms=2, ms_per_code=4)
    assert (acq.conf.fft_size, acq.conf.consumed_samples, acq.conf.code_layout) == (16000, 8000, 2)
    acq.set_local_code(0, code2)
    got = acq.search(iq, [0])[0]
    assert (int(got["index_time"]), int(got["index_doppler"])) == (want["index_time"], want["index_doppler"])
    assert abs(got["test_statistics"] - want["test_statistics"]) / want["test_statistics"] < 1e-4
    acq.close()


def test_doppler_center_assisted(capi, engine, oracle):
    fs, prn = 4e6, 14
    iq, svs = _signal(oracle, [prn], fs, 4000, seed=14)
    center = int(round(svs[0]["doppler"] / 250.0)) * 250
    o = _oracle_acq(oracle, fs, 4000.0, 3, 1000, 125, prn, iq, center=center)
    want = o.acquisition_core(iq)
    acq = capi.PcpsAcquisition(engine, fs_in=int(fs), samples_per_ms=4000.0, samples_per_chip=3, doppler_max=1000,
                               doppler_step=125)
    acq.set_doppler_center(center, 0)
    acq.set_local_code(0, oracle.port.gps_ca_code_complex_sampled(prn, int(fs)))
    got = acq.search(iq, [0])[0]
    assert int(got["doppler"]) == want["doppler"]
    assert int(got["index_time"]) == want["index_time"]
    assert abs(want["doppler"] - svs[0]["doppler"]) <= 666
    acq.close()


def test_fft_round_trip_property_all_supported_radices(capi, engine, oracle):
    """Size-independent property at sizes up to the single-CTA maximum: searching the local code
    against ITSELF delayed by k samples must peak exactly at index k with zero Doppler,
    for sizes exercising radices 2,3,4,5,7,8."""
    rng = np.random.default_rng(9)
    for n in (4096, 6000, 8400, 16000, 25000, 27000, 27648, 2 * 3 * 5 * 7, 4802):
        fs = n * 1000
        acq = capi.PcpsAcquisition(engine, fs_in=fs, samples_per_ms=float(n), samples_per_chip=max(1, n // 1023),
                                   doppler_max=1000, doppler_step=500)
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
        capi.PcpsAcquisition(engine, fs_in=16368000, samples_per_ms=16368.0, samples_per_chip=16, doppler_max=5000, doppler_step=250,
                             use_CFAR_algorithm_flag=False)
    with pytest.raises(capi.B200Error):   # beyond 8 x 27648 points
        capi.PcpsAcquisition(engine, fs_in=300000000, samples_per_ms=300000.0, samples_per_chip=290, doppler_max=1000, doppler_step=500)
    acq = capi.PcpsAcquisition(engine, fs_in=4000000, samples_per_ms=4000.0, samples_per_chip=3, doppler_max=5000, doppler_step=250)
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
    from oracle.acq_np import AcqConf, PcpsAcquisitionOracle
    fs, prn = 4e6, 8
    iq, svs = _signal(oracle, [prn], fs, 8000, seed=88, cn0=47.0)
    conf = AcqConf(fs_in=int(fs), samples_per_ms=4000.0, samples_per_code=4000.0, samples_per_chip=3, doppler_max=5000,
                   doppler_step=500, pfa=0.001, pfa2=0.001, make_2_steps=True, doppler_step2=125.0, num_doppler_bins_step2=4)
    o = PcpsAcquisitionOracle(conf)
    code = oracle.port.gps_ca_code_complex_sampled(prn, int(fs))
    o.set_local_code(code)
    w1 = o.acquisition_core(iq[:4000])
    assert not w1["positive"] and o.step_two          # first step passed the threshold, second pending
    w2 = o.acquisition_core(iq[4000:8000])
    assert w2["positive"] and w2["step_two"]
    acq = capi.PcpsAcquisition(engine, fs_in=int(fs), samples_per_ms=4000.0, samples_per_chip=3, doppler_max=5000, doppler_step=500)
    acq.set_local_code(0, code)
    g1 = acq.search(iq[:4000], [0])[0]
    assert (int(g1["index_time"]), int(g1["doppler"])) == (w1["index_time"], w1["doppler"])
    acq.set_step_two(float(g1["doppler"]), 125.0, 4)
    g2 = acq.search_step_two(iq[4000:8000], 0, float(g1["input_power"]))
    assert (int(g2["index_time"]), int(g2["index_doppler"]), int(g2["doppler"])) == (w2["index_time"], w2["index_doppler"], w2["doppler"])
    assert abs(g2["test_statistics"] - w2["test_statistics"]) / w2["test_statistics"] < 1e-4
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
    spms = fs / 1000.0
    n = int(spms) * sampled_ms
    spchip = int(fs / 1.023e6)
    prn = 7
    codes = {p: oracle.port.gps_ca_code(p) for p in (7, 21)}
    svs = [dict(prn=7, doppler=dstep * round(0.6 * dmax / dstep) + 10.0, code_phase_chips=321.4, cn0=42.0, phase0=1.0),
           dict(prn=21, doppler=-0.3 * dmax, code_phase_chips=77.7, cn0=42.0, phase0=2.0)]
    iq = make_iq(codes, fs, n, svs, seed=int(fs / 1e3) + sampled_ms)
    o = _oracle_acq(oracle, fs, spms, spchip, dmax, dstep, prn, iq, cfar=cfar, sampled_ms=sampled_ms, ms_per_code=sampled_ms)
    want = o.acquisition_core(iq)
    acq = capi.PcpsAcquisition(engine, fs_in=int(fs), samples_per_ms=spms, samples_per_chip=spchip, doppler_max=dmax,
                               doppler_step=dstep, use_CFAR_algorithm_flag=cfar, sampled_ms=sampled_ms, ms_per_code=sampled_ms,
                               keep_grid=True)
    assert acq.conf.fft_size == n
    acq.set_local_code(0, np.tile(oracle.port.gps_ca_code_complex_sampled(prn, int(fs)), sampled_ms))
    got = acq.search(iq, [0])[0]
    # with sampled_ms code periods in the buffer the correlation has sampled_ms mathematically equal peaks one
    # code period apart; which one wins is rounding noise, and update_synchro folds it away
    # (Acq_delay_samples = fmod(index_time, samples_per_code), pcps_acquisition.cc:582)
    assert int(got["index_time"]) % int(spms) == want["index_time"] % int(spms)
    assert int(got["index_doppler"]) == want["index_doppler"]
    assert abs(got["grid_maximum"] - want["grid_maximum"]) / want["grid_maximum"] < 1e-4
    assert abs(got["test_statistics"] - want["test_statistics"]) / want["test_statistics"] < 1e-4
    g = acq.read_grid(0)
    ref_g = o.magnitude_grid[:, :acq.conf.effective_fft_size]
    assert np.max(np.abs(g - ref_g)) / ref_g.max() < 2e-5
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
    spms = fs / 1000.0
    n = int(spms) * sampled_ms
    spchip = int(fs / 1.023e6)
    prn = 7
    codes = {p: oracle.port.gps_ca_code(p) for p in (7, 21)}
    svs = [dict(prn=7, doppler=dstep * round(0.6 * dmax / dstep) + 10.0, code_phase_chips=321.4, cn0=47.0, phase0=1.0),
           dict(prn=21, doppler=-dstep * round(0.3 * dmax / dstep) + 20.0, code_phase_chips=77.7, cn0=47.0, phase0=2.0)]
    iq = make_iq(codes, fs, 2 * n, svs, seed=int(fs / 1e3) + sampled_ms)
    kw = dict(sampled_ms=sampled_ms, ms_per_code=sampled_ms) if sampled_ms > 1 else {}
    o = _oracle_acq(oracle, fs, spms, spchip, dmax, dstep, prn, iq, cfar=True, dwells=2, **kw)
    want = o.acquisition_core(iq[:n])
    acq = capi.PcpsAcquisition(engine, fs_in=int(fs), samples_per_ms=spms, samples_per_chip=spchip, doppler_max=dmax,
                               doppler_step=dstep, use_CFAR_algorithm_flag=True, keep_grid=True, max_dwells=2, n_code_slots=2, **kw)
    assert acq.conf.fft_size == n
    local = oracle.port.gps_ca_code_complex_sampled(prn, int(fs))
    acq.set_local_code(1, np.tile(local, sampled_ms))
    acq.set_local_code(0, np.tile(oracle.port.gps_ca_code_complex_sampled(21, int(fs)), sampled_ms))
    both = acq.search(iq[:n], [0, 1])
    got = both[1]
    assert int(got["index_time"]) % int(spms) == want["index_time"] % int(spms)
    assert int(got["index_doppler"]) == want["index_doppler"]
    assert int(got["doppler"]) == want["doppler"]
    assert abs(got["grid_maximum"] - want["grid_maximum"]) / want["grid_maximum"] < 1e-4
    assert abs(got["test_statistics"] - want["test_statistics"]) / want["test_statistics"] < 1e-4
    assert abs(got["input_power"] - want["input_power"]) / want["input_power"] < 1e-4
    g = acq.read_grid(1)
    ref_g = o.magnitude_grid[:, :acq.conf.effective_fft_size]
    assert np.max(np.abs(g - ref_g)) / ref_g.max() < 2e-5
    assert abs(want["doppler"] - svs[0]["doppler"]) <= max(dstep, 666 / sampled_ms)
    assert abs(int(both[0]["doppler"]) - svs[1]["doppler"]) <= max(dstep, 666 / sampled_ms)
    # second dwell accumulates on the grid
    o.num_noncoherent_integrations_counter = 1   # keep accumulating whatever the threshold decided
    want2 = o.acquisition_core(iq[n:])
    got2 = acq.search(iq[n:], [1], dwell_counter=2)[0]
    assert int(got2["index_doppler"]) == want2["index_doppler"]
    assert abs(got2["test_statistics"] - want2["test_statistics"]) / want2["test_statistics"] < 1e-4
    # assisted acquisition: moving the Doppler centre rebuilds the chirped wipe-off rows
    o3 = _oracle_acq(oracle, fs, spms, spchip, dmax, dstep, prn, iq, cfar=True, center=875, **kw)
    want3 = o3.acquisition_core(iq[:n])
    acq.set_doppler_center(875)
    got3 = acq.search(iq[:n], [1])[0]
    assert int(got3["doppler"]) == want3["doppler"]
    assert abs(got3["test_statistics"] - want3["test_statistics"]) / want3["test_statistics"] < 1e-4
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
    a = capi.PcpsAcquisition(e, fs_in=int(fs), samples_per_ms=float(n), samples_per_chip=4, doppler_max=5000, doppler_step=250, n_code_slots=2)
    b = capi.PcpsAcquisition(e, fs_in=int(fs), samples_per_ms=float(n), samples_per_chip=4, doppler_max=5000, doppler_step=250, n_code_slots=2)
    for o in (a, b):
        o.set_local_code(0, gs.gps_ca_code_complex_sampled(3, int(fs)))
        o.set_local_code(1, gs.gps_ca_code_complex_sampled(4, int(fs)))
    want = a.search(iq, [0, 1])
    a.search_submit(iq, [0, 1])
    b.search_submit(iq, [1, 0])
    with pytest.raises(capi.B200Error) as ei:
        a.search_submit(iq, [0])
    assert ei.value.code == -4
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
    import ctypes as C
    from gnss_sdr_b200 import capi
    import gnss_synth as gs
    fs, n, band = 4e6, 4000, 0
    iq = gs.make_iq({3: gs.gps_ca_code(3)}, fs, n, [dict(prn=3, doppler=2100.0, code_phase_chips=400.0, cn0=48.0)], seed=8)
    raw = np.round(iq.view(np.float32) * 100).astype(np.int16)
    e = capi.Engine()
    e.iq_create(band, 8192)
    e.iq_push(band, iq)
    a = capi.PcpsAcquisition(e, fs_in=int(fs), samples_per_ms=float(n), samples_per_chip=4, doppler_max=5000, doppler_step=250, n_code_slots=2)
    a.set_local_code(0, gs.gps_ca_code_complex_sampled(3, int(fs)))
    a.set_local_code(1, gs.gps_ca_code_complex_sampled(4, int(fs)))
    a.set_step_two(2100.0, 125.0, 4)   # so that a step-two call is otherwise legal
    want = a.search(iq, [0, 1])
    res, slot = np.zeros(1, capi.ACQ_RESULT_DTYPE), np.zeros(1, np.uint32)

    def i16(name, *args):
        rc = getattr(capi.lib, name)(a.h, raw.ctypes.data, *args, res.ctypes.data)
        if rc:
            raise capi.B200Error(rc, name)

    calls = {
        "search": lambda: a.search(iq, [0]),
        "search_i16": lambda: i16("b200_acq_search_i16", slot.ctypes.data, 1, 1),
        "search_step_two": lambda: a.search_step_two(iq, 0, 1.0),
        "search_step_two_i16": lambda: i16("b200_acq_search_step_two_i16", 0, 1, C.c_float(1.0)),
        "search_submit": lambda: a.search_submit(iq, [0]),
        "search_band": lambda: a.search_band(band, 0, [0]),
        "search_band_submit": lambda: a.search_band_submit(band, 0, [0]),
        "search_step_two_band": lambda: a.search_step_two_band(band, 0, 0, 1.0),
    }
    a.search_submit(iq, [0, 1])
    with pytest.raises(capi.B200Error) as ei:
        calls[entry]()
    assert ei.value.code == -4
    assert a.search_wait().tobytes() == want.tobytes()
    a.close()
    e.close()
