"""The DLL/PLL loop oracle (oracle/port_loop.c) pinned against the reference's OWN library code
(oracle/_ref/liboracle_ref_loop.so = tracking_discriminators.cc, tracking_FLL_PLL_filter.cc,
tracking_loop_filter.cc, lock_detectors.cc, exponential_smoother.cc compiled where they lie), and the
closed loop over the reference's CPU correlator.  CPU only."""
import numpy as np
import pytest

from gnss_sdr_b200.abi import TrkLoopStatus
from oracle import loop as ol
import gnss_synth as gs
import loop_harness as lh


@pytest.fixture(scope="module")
def reflib():
    lib = ol.ref_lib()
    if lib is None:
        pytest.skip("oracle/_ref/liboracle_ref_loop.so not built (no reference sources here)")
    return lib


def test_library_functions_bit_exact(reflib):
    import ctypes as C
    port = ol.port_lib()
    rng = np.random.default_rng(11)
    fp = lambda a: a.ctypes.data_as(C.POINTER(C.c_float))
    for _ in range(4000):
        v = (rng.standard_normal(8) * 10 ** rng.uniform(-2, 4)).astype(np.float32)
        if rng.random() < 0.05:
            v[rng.integers(0, 8)] = 0.0
        a, b = port.port_disc_pll_cloop(v[0], v[1]), reflib.ref_disc_pll_cloop(v[0], v[1])
        assert a == b
        a = port.port_disc_fll_diff_atan(v[0], v[1], v[2], v[3], 0.0, 0.001)
        b = reflib.ref_disc_fll_diff_atan(v[0], v[1], v[2], v[3], 0.0, 0.001)
        assert a == b or (np.isnan(a) and np.isnan(b))
        a = port.port_disc_dll_e_minus_l(v[0], v[1], v[2], v[3], 0.5, 1.0, 1.0)
        b = reflib.ref_disc_dll_e_minus_l(v[0], v[1], v[2], v[3], 0.5, 1.0, 1.0)
        assert a == b
        assert port.port_disc_dll_vemlp(fp(v)) == reflib.ref_disc_dll_vemlp(fp(v))
    for _ in range(300):
        n = int(rng.integers(1, 40))
        buf = (rng.standard_normal(2 * n) * 300 + (2000 if rng.random() < 0.7 else 0)).astype(np.float32)
        a, b = port.port_cn0_m2m4(fp(buf), n, 0.001), reflib.ref_cn0_m2m4(fp(buf), n, 0.001)
        assert a == b or (np.isnan(a) and np.isnan(b))
        assert port.port_carrier_lock_detector(fp(buf), n) == reflib.ref_carrier_lock_detector(fp(buf), n)


CONFS = [
    dict(),
    dict(pll_filter_order=2, dll_filter_order=1),
    dict(pll_filter_order=3, dll_filter_order=3, enable_fll_pull_in=1, pull_in_time_s=1),
    dict(enable_fll_steady_state=1, carrier_aiding=0),
    dict(veml=1, code_samples_per_chip=2, early_late_space_chips=0.15, cn0_samples=10),
    dict(pull_in_time_s=0, max_code_lock_fail=5, cn0_min=40),     # loses lock on the weak stretch
    dict(bit_synchronization_time_limit_s=1, pull_in_time_s=0),     # fail-safe fires after 1 s
]


@pytest.mark.parametrize("kw", CONFS)
def test_cycle_port_vs_reference_classes_bit_exact(reflib, kw):
    """Same taps in, every item scalar and every dump-record byte equal, epoch by epoch."""
    conf = ol.default_conf(fs_in=4e6, **kw)
    P, R = ol.PortLoop(conf), ol.RefLoop(conf)
    for L in (P, R):
        L.start(524.3, 1680.0, 1000, 9000)
    taps_seq = lh.synthetic_taps(3000, 5 if conf.veml else 3, seed=5, weak_from=1500 if conf.cn0_min == 40 else None)
    lost = False
    for k in range(3000):
        a, b = P.prepare(), R.prepare()
        if a is None or b is None:
            assert a is None and b is None
            lost = True
            break
        assert a[0] == b[0] and a[1] == b[1]
        assert np.array_equal(a[2].view(np.uint32), b[2].view(np.uint32))
        la, ra = P.update(taps_seq[k])
        lb, rb = R.update(taps_seq[k])
        assert la == lb
        if la:
            assert ra.tobytes() == rb.tobytes(), (k, ra, rb)
    sa, sb = P.status(), R.status()
    for f, _ in TrkLoopStatus._fields_:
        assert getattr(sa, f) == getattr(sb, f), f
    if conf.cn0_min == 40 or conf.bit_synchronization_time_limit_s == 1:
        assert lost and sa.state == 0 and sa.loss_of_lock == 1
    else:
        assert not lost and sa.state == 2 and sa.epochs == 3000


def test_closed_loop_over_reference_correlator_locks(oracle, ref):
    """Oracle loop + the reference's Cpu_Multicorrelator_Real_Codes on a synthetic 4 Msps signal: pulls in from a
    coarse acquisition and reports the true Doppler, code rate and C/N0 (pins the sign conventions of the cycle)."""
    fs, prn, doppler, cn0 = 4e6, 7, 1234.0, 47.0
    code = oracle.port.gps_ca_code(prn)
    delay = 1337
    n = int(fs * 1.6)
    iq = gs.make_iq({prn: code}, fs, n, [dict(prn=prn, doppler=doppler, code_phase_chips=(-delay * 1.023e6 / fs) % 1023, cn0=cn0)], seed=21)
    conf = ol.default_conf(fs_in=fs, prn=prn, pull_in_time_s=1)
    corr = lh.RefCorrelator(ref, code, [-0.5, 0.0, 0.5], int(conf.vector_length))
    L = ol.PortLoop(conf)
    L.start(float(delay % 4000) + 0.4, doppler - 60.0, 0, 0)
    recs = lh.run_closed_loop(L, corr, iq, 1500)
    assert len(recs) == 1500
    tail = recs[-300:]
    assert abs(np.mean(tail["carrier_doppler_hz"]) - doppler) < 2.0
    assert abs(np.mean(tail["code_freq_chips"].astype(np.float64)) - 1.023e6 * (1 + doppler / 1575.42e6)) < 0.2  # float32 record: 0.0625 chips/s steps
    assert abs(np.mean(tail["CN0_SNV_dB_Hz"]) - cn0) < 1.5
    # alpha = 0.002 smoother: still climbing from its pull-in average after 1.5 s
    assert np.all(tail["carrier_lock_test"] > 0.5) and tail["carrier_lock_test"][-1] > tail["carrier_lock_test"][0]
    assert np.mean(tail["abs_P"]) > 1.8 * np.mean(tail["abs_E"]) * 0.9
    # PRN start stamps advance by ~4000 samples and follow the true code phase
    d = np.diff(recs["PRN_start_sample_count"].astype(np.int64))
    assert set(np.unique(d)) <= {3999, 4000, 4001}
    s = L.status()
    assert s.state == 2 and s.epochs == 1500


def test_dump_file_is_readable_by_the_reference_reader(reflib, tmp_path):
    """b200_trk_dump_write (host-only entry point of the product library) -> the reference's own
    Tracking_Dump_Reader (tests/unit-tests/signal-processing-blocks/libs/tracking_dump_reader.cc:22-50)."""
    from gnss_sdr_b200 import capi
    conf = ol.default_conf()
    L = ol.PortLoop(conf)
    L.start(100.0, 500.0, 0, 0)
    taps = lh.synthetic_taps(50, 3, seed=3)
    recs = []
    for k in range(50):
        L.prepare()
        ok, r = L.update(taps[k])
        recs.append(r)
    recs = np.array(recs, capi.TRK_DUMP_RECORD_DTYPE)
    fn = str(tmp_path / "trk_dump_ch0.dat")
    capi.trk_dump_write(fn, recs[:20])
    capi.trk_dump_write(fn, recs[20:], append=True)
    got = ol.ref_dump_read(fn)
    assert got.shape == (50, 24)
    for j, name in enumerate(capi.TRK_DUMP_RECORD_DTYPE.names):
        assert np.array_equal(got[:, j], recs[name].astype(np.float64)), name
