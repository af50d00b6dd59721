"""Free-running DLL/PLL loops on the device (b200_trk_loop_*) against the CPU oracle (oracle/port_loop.c, itself
pinned bit-exact on the reference's own loop libraries by tests/test_oracle_loop.py) and against the committed
reference fixture tests/golden/loop_ref_golden.npz.  Everything goes through the C ABI.

Parity contract (DESIGN.md section 4.5):
  * every integer the loop produces is exact: epoch length, sample stamps, state, counters;
  * the float32 NCO commands handed to the correlator and the float fields of the dump record agree to
    LOOP_RTOL: the cycle is evaluated with the reference's own float/double types and unfused IEEE operations;
    atanf and log10f are correctly rounded on the device and <= 1 ulp in glibc, which can move a discriminator
    by one float ulp and, through the loop filters' integrators, the commands by a few ulp.
"""
import os

import numpy as np
import pytest

import gnss_synth as gs
import loop_harness as lh
from oracle import loop as ol

pytestmark = pytest.mark.gpu

LOOP_RTOL = 2e-6
HERE = os.path.dirname(os.path.abspath(__file__))

EXACT_FIELDS = ("abs_VE", "abs_E", "abs_P", "abs_L", "abs_VL", "prompt_I", "prompt_Q", "PRN_start_sample_count", "aux2", "PRN", "TOW_ms", "WN")
# absolute floors for fields that hover around zero (discriminator outputs, error terms)
ATOL = dict(acc_carrier_phase_rad=2e-3, carrier_doppler_hz=1e-3, carrier_doppler_rate_hz_s=0.0, code_freq_chips=0.13,
            code_freq_rate_chips=0.0, carr_error_hz=1e-7, carr_error_filt_hz=1e-3, code_error_chips=1e-7,
            code_error_filt_chips=1e-5, CN0_SNV_dB_Hz=2e-4, carrier_lock_test=1e-6, aux1=1e-6)


def assert_records_match(got, want, what=""):
    assert got.dtype == want.dtype and got.shape == want.shape
    for f in EXACT_FIELDS:
        assert np.array_equal(got[f], want[f]), (what, f)
    for f, atol in ATOL.items():
        g, w = got[f].astype(np.float64), want[f].astype(np.float64)
        bad = np.abs(g - w) > atol + LOOP_RTOL * np.abs(w)
        assert not bad.any(), (what, f, int(np.argmax(bad)), g[bad][:3], w[bad][:3])


def make_engine_with_loops(capi, oracle, confs, fs, band_samples=None, prns=None, tables=None):
    e = capi.Engine()
    if band_samples is not None:
        e.iq_create(0, len(band_samples) + 16)
    else:
        e.iq_create(0, 1 << 16)
    ids = []
    for i, c in enumerate(confs):
        taps = 5 if c.veml else 3
        spc = c.code_samples_per_chip
        els, vels = c.early_late_space_chips, 0.5
        shifts = ([-vels * spc, -els * spc, 0.0, els * spc, vels * spc] if c.veml else [-els * spc, 0.0, els * spc])
        if tables is not None:
            code = tables[i]
        else:
            code = oracle.port.gps_ca_code(prns[i] if prns else 1 + i)
            if spc == 2:
                code = np.repeat(code, 2)
        ch = e.channel_create(0, taps)
        e.channel_set_code(ch, code, shifts)
        ids.append(e.loop_create(ch, c))
    return e, ids


CONFS = [
    dict(),
    dict(pll_filter_order=2, dll_filter_order=1),
    dict(pll_filter_order=3, dll_filter_order=3, enable_fll_pull_in=1, pull_in_time_s=1),
    dict(enable_fll_steady_state=1, carrier_aiding=0),
    dict(veml=1, code_samples_per_chip=2, early_late_space_chips=0.15, cn0_samples=10),
    dict(pull_in_time_s=0, max_code_lock_fail=5, cn0_min=40),
    dict(bit_synchronization_time_limit_s=1, pull_in_time_s=0),
]


def test_cycle_with_supplied_taps_matches_oracle(oracle):
    """All configurations side by side as loops of one engine, 3000 epochs, same correlator outputs as the oracle:
    item scalars bit-exact for the first epochs and within LOOP_RTOL throughout, records per the contract, the two
    loss-of-lock scenarios end in standby at the same epoch."""
    from gnss_sdr_b200 import capi
    confs = [ol.default_conf(fs_in=4e6, prn=1 + i, **kw) for i, kw in enumerate(CONFS)]
    e, ids = make_engine_with_loops(capi, oracle, confs, 4e6)
    orc = [ol.PortLoop(c) for c in confs]
    n_ep = 3000
    taps = [lh.synthetic_taps(n_ep, 5 if c.veml else 3, seed=40 + i, weak_from=1500 if c.cn0_min == 40 else None) for i, c in enumerate(confs)]
    for i, lid in enumerate(ids):
        e.loop_start(lid, 524.3 + 10 * i, 1680.0 - 100 * i, 1000, 9000)
        orc[i].start(524.3 + 10 * i, 1680.0 - 100 * i, 1000, 9000)
    got = [[] for _ in confs]
    want = [[] for _ in confs]
    lost_at = [None] * len(confs)
    for k in range(n_ep):
        items = e.loop_peek_items()
        t = np.zeros((len(confs), 8), np.complex64)
        for i, o in enumerate(orc):
            it = o.prepare()
            if it is None:
                assert items[i]["n"] == 0
                lost_at[i] = lost_at[i] if lost_at[i] is not None else k
                continue
            s, n, p6 = it
            assert items[i]["n"] == n and items[i]["sample_index"] == s, (k, i)
            dev = np.array([items[i][f] for f in ("rem_carrier_phase_rad", "phase_step_rad", "phase_rate_step_rad",
                                                  "rem_code_phase_chips", "code_phase_step_chips", "code_phase_rate_step_chips")], np.float32)
            if k < 2:
                assert np.array_equal(dev.view(np.uint32), p6.view(np.uint32)), (k, i, dev, p6)
            # rem_carrier_phase is a phase mod 2 pi: compare on the circle
            d0 = abs(float(dev[0]) - float(p6[0]))
            assert min(d0, abs(d0 - 2 * np.pi)) < 1e-4, (k, i, dev[0], p6[0])
            assert np.allclose(dev[1:], p6[1:], rtol=LOOP_RTOL, atol=1e-9), (k, i, dev, p6)
            t[i, :taps[i].shape[1]] = taps[i][k]
        rec, logged = e.loop_step_taps(t)
        for i, o in enumerate(orc):
            if lost_at[i] is not None:
                assert logged[i] == 0
                continue
            ok, r = o.update(taps[i][k])
            assert bool(logged[i]) == ok, (k, i)
            if ok:
                got[i].append(rec[i])
                want[i].append(r)
    for i, c in enumerate(confs):
        g, w = np.array(got[i], capi.TRK_DUMP_RECORD_DTYPE), np.array(want[i], capi.TRK_DUMP_RECORD_DTYPE)
        assert_records_match(g, w, what=f"conf {i}")
        sd, so = e.loop_status(ids[i]), orc[i].status()
        assert (sd.state, sd.loss_of_lock, sd.sample_counter, sd.epochs) == (so.state, so.loss_of_lock, so.sample_counter, so.epochs), i
    assert lost_at[5] is not None and lost_at[6] is not None and all(l is None for l in lost_at[:5])
    e.close()


def test_cycle_matches_reference_golden(oracle):
    """Same, against records the reference's own loop classes produced (committed fixture; no oracle in the loop)."""
    from gnss_sdr_b200 import capi
    sys_path_golden = os.path.join(HERE, "golden")
    import importlib.util
    spec = importlib.util.spec_from_file_location("make_golden", os.path.join(sys_path_golden, "make_golden.py"))
    mg = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mg)
    gold = np.load(os.path.join(sys_path_golden, "loop_ref_golden.npz"))
    confs = [ol.default_conf(fs_in=4e6, **kw) for _, kw, _ in mg.LOOP_CASES]
    e, ids = make_engine_with_loops(capi, oracle, confs, 4e6)
    for lid in ids:
        e.loop_start(lid, 524.3, 1680.0, 1000, 9000)
    n_ep = mg.LOOP_CASES[0][2]
    taps = [lh.synthetic_taps(n_ep, 5 if c.veml else 3, seed=mg.LOOP_SEED) for c in confs]
    recs = []
    for k in range(n_ep):
        items = e.loop_peek_items()
        for i, (name, _, _) in enumerate(mg.LOOP_CASES):
            g = gold[f"{name}/items"][k]
            assert items[i]["sample_index"] == g[0] and items[i]["n"] == g[1], (name, k)
        t = np.zeros((len(confs), 8), np.complex64)
        for i in range(len(confs)):
            t[i, :taps[i].shape[1]] = taps[i][k]
        r, logged = e.loop_step_taps(t)
        assert logged.all()
        recs.append(r)
    recs = np.array(recs, capi.TRK_DUMP_RECORD_DTYPE)
    for i, (name, _, _) in enumerate(mg.LOOP_CASES):
        want = np.frombuffer(gold[f"{name}/records"].tobytes(), capi.TRK_DUMP_RECORD_DTYPE)
        assert_records_match(recs[:, i], want, what=name)
    e.close()


def _closed_loop_case(oracle, fs=4e6, seconds=1.3, seed=31):
    svs = [dict(prn=3, doppler=2310.0, delay=777, cn0=46.0), dict(prn=11, doppler=-1875.0, delay=2345, cn0=44.0),
           dict(prn=22, doppler=640.0, delay=3901, cn0=48.0)]
    codes = {sv["prn"]: oracle.port.gps_ca_code(sv["prn"]) for sv in svs}
    n = int(fs * seconds)
    iq = gs.make_iq(codes, fs, n, [dict(prn=sv["prn"], doppler=sv["doppler"], code_phase_chips=(-sv["delay"] * 1.023e6 / fs) % 1023,
                                        cn0=sv["cn0"]) for sv in svs], seed=seed)
    return svs, codes, iq


@pytest.mark.parametrize("mode", [0, 2], ids=["persistent", "per_epoch_launches"])
def test_free_running_loops_track_and_follow_the_oracle_closed_loop(oracle, mode):
    """b200_trk_loop_run: correlator and loop alternate on the device for 1200 epochs, three satellites in one band
    (mode 0: one persistent CTA per loop; mode 2: a correlator launch and a loop launch per epoch).
    Integer epoch lengths equal the oracle's closed loop (oracle loop over the oracle correlator) except where the
    two correlators' float summation orders move K_blk across an integer; commands stay within the drift the
    reference's own generic-vs-AVX kernels show (tests/test_chain_gpu.py: 0.7 Hz, 5e-2 samples)."""
    from gnss_sdr_b200 import capi
    fs = 4e6
    svs, codes, iq = _closed_loop_case(oracle)
    confs = [ol.default_conf(fs_in=fs, prn=sv["prn"], pull_in_time_s=1) for sv in svs]
    e, ids = make_engine_with_loops(capi, oracle, confs, fs, band_samples=iq, prns=[sv["prn"] for sv in svs])
    e.iq_push(0, iq)
    e.loop_set_mode(mode)
    n_ep = 1200
    for lid, sv in zip(ids, svs):
        e.loop_start(lid, float(sv["delay"]) + 0.3, sv["doppler"] - 55.0, 0, 0)
    rec, cnt = e.loop_run(n_ep)
    assert (cnt == n_ep).all()
    for i, sv in enumerate(svs):
        o = ol.PortLoop(confs[i])
        o.start(float(sv["delay"]) + 0.3, sv["doppler"] - 55.0, 0, 0)
        want = lh.run_closed_loop(o, lh.PortCorrelator(oracle.port, codes[sv["prn"]], [-0.5, 0.0, 0.5]), iq, n_ep)
        got = rec[i]
        assert len(want) == n_ep
        tail = slice(n_ep - 300, n_ep)
        assert abs(np.mean(got["carrier_doppler_hz"][tail]) - sv["doppler"]) < 2.0
        assert abs(np.mean(got["CN0_SNV_dB_Hz"][tail]) - sv["cn0"]) < 1.5
        assert np.max(np.abs(got["carrier_doppler_hz"] - want["carrier_doppler_hz"])) < 0.7
        assert np.max(np.abs(got["aux1"] - want["aux1"])) < 5e-2
        stamp_diff = got["PRN_start_sample_count"].astype(np.int64) - want["PRN_start_sample_count"].astype(np.int64)
        assert np.max(np.abs(stamp_diff)) <= 1
        same = (stamp_diff == 0) & (np.roll(stamp_diff, 1) == 0)      # epochs that cover the very same samples
        assert same.mean() > 0.9
        # the two closed loops may sit up to 5e-2 samples (1.3e-2 chips) apart: |P| follows the correlation triangle
        assert np.max(np.abs(got["abs_P"][same] - want["abs_P"][same])) < 2e-2 * np.mean(want["abs_P"])
        sd = e.loop_status(ids[i])
        assert sd.state == 2 and sd.epochs == n_ep
    e.close()


def test_persistent_kernel_and_per_epoch_launches_agree(oracle):
    """Mode 0 (persistent CTA per loop; the correlator templates compiled in the --fmad=false unit) and mode 1
    (batch correlator kernel with slices = 1 + loop-update kernel per epoch): same per-item arithmetic, same loop
    arithmetic; the persistent CTA is wider than the batch kernel's (512 threads for a handful of loops vs 256), so the taps
    are summed in a different order - integers must be exact, floats agree to the closed-loop noise of a last-bit tap
    difference carried through 590 epochs of feedback."""
    from gnss_sdr_b200 import capi
    fs = 4e6
    svs, codes, iq = _closed_loop_case(oracle, seconds=0.6)
    confs = [ol.default_conf(fs_in=fs, prn=sv["prn"], pull_in_time_s=1) for sv in svs]
    # a 5-tap loop rides along on the first satellite
    confs.append(ol.default_conf(fs_in=fs, prn=svs[0]["prn"], veml=1, early_late_space_chips=0.25))
    prns = [sv["prn"] for sv in svs] + [svs[0]["prn"]]
    starts = [(float(sv["delay"]) + 0.3, sv["doppler"] - 40.0) for sv in svs] + [(float(svs[0]["delay"]), svs[0]["doppler"] + 30.0)]
    out = {}
    for mode in (0, 1):
        e, ids = make_engine_with_loops(capi, oracle, confs, fs, band_samples=iq, prns=prns)
        e.iq_push(0, iq)
        e.loop_set_mode(mode)
        for lid, (d, f) in zip(ids, starts):
            e.loop_start(lid, d, f, 0, 0)
        rec, cnt = e.loop_run(590)
        assert (cnt >= 585).all()
        out[mode] = (rec, cnt, [e.loop_status(l).sample_counter for l in ids])
        e.close()
    assert np.array_equal(out[0][1], out[1][1]) and out[0][2] == out[1][2]
    a, b = out[0][0], out[1][0]
    n = int(min(out[0][1].min(), out[1][1].min()))
    assert np.array_equal(a["PRN_start_sample_count"][:, :n], b["PRN_start_sample_count"][:, :n])
    assert np.array_equal(a["PRN"][:, :n], b["PRN"][:, :n])
    assert np.max(np.abs(a["carrier_doppler_hz"][:, :n] - b["carrier_doppler_hz"][:, :n])) < 0.5
    assert np.max(np.abs(a["abs_P"][:, :n] - b["abs_P"][:, :n]) / np.maximum(b["abs_P"][:, :n], 1.0)) < 2e-2
    assert np.median(np.abs(a["abs_P"][:, :n] - b["abs_P"][:, :n]) / np.maximum(b["abs_P"][:, :n], 1.0)) < 1e-4
    assert np.max(np.abs(a["CN0_SNV_dB_Hz"][:, :n] - b["CN0_SNV_dB_Hz"][:, :n])) < 0.2


def test_galileo_e1_like_veml_loop_with_4ms_epochs(oracle):
    """Galileo-E1-shaped loop: sinBOC(1,1) table with 2 samples per chip (8184 values), 4 ms code period
    (vector_length 16000 at 4 Msps), five taps VE,E,P,L,VL with the VEML discriminator, C/N0 smoother initialised
    over cn0_smoother_samples / 4 estimates.  Persistent kernel vs the oracle closed loop."""
    from gnss_sdr_b200 import capi
    fs, doppler, cn0 = 4e6, -1540.0, 45.0
    rng = np.random.default_rng(17)
    primary = (2 * rng.integers(0, 2, 4092) - 1).astype(np.int32)
    table = oracle.port.sinboc11(primary)
    L = len(table)
    rate = 1.023e6 * 2.0 * (1.0 + doppler / 1575.42e6)           # table entries per second
    cp = 2711.0                                                      # table entries at sample 0
    delay = ((L - cp) % L) / (rate / fs)
    n = int(fs * 2.0)
    iq = gs.make_iq({1: table}, fs, n, [dict(prn=1, doppler=doppler, code_phase_chips=cp, cn0=cn0)], seed=23, chips_per_table_chip=2.0)
    conf = ol.default_conf(fs_in=fs, prn=1, code_length_chips=4092, code_period=0.004, vector_length=16000, code_samples_per_chip=2,
                           veml=1, early_late_space_chips=0.15, pull_in_time_s=1)
    e, ids = make_engine_with_loops(capi, oracle, [conf], fs, band_samples=iq, tables=[table])
    e.iq_push(0, iq)
    e.loop_start(ids[0], delay + 0.2, doppler + 25.0, 0, 0)
    n_ep = 490
    rec, cnt = e.loop_run(n_ep)
    assert cnt[0] == n_ep
    o = ol.PortLoop(conf)
    o.start(delay + 0.2, doppler + 25.0, 0, 0)
    shifts = [-0.5 * 2, -0.15 * 2, 0.0, 0.15 * 2, 0.5 * 2]
    want = lh.run_closed_loop(o, lh.PortCorrelator(oracle.port, table, shifts), iq, n_ep)
    got = rec[0]
    assert len(want) == n_ep
    tail = slice(n_ep - 100, n_ep)
    assert abs(np.mean(got["carrier_doppler_hz"][tail]) - doppler) < 1.0
    assert abs(np.mean(got["CN0_SNV_dB_Hz"][tail]) - cn0) < 1.5
    assert np.all(got["abs_P"][tail] > got["abs_E"][tail]) and np.all(got["abs_P"][tail] > got["abs_L"][tail])
    assert np.max(np.abs(got["carrier_doppler_hz"] - want["carrier_doppler_hz"])) < 0.7
    assert np.max(np.abs(got["aux1"] - want["aux1"])) < 5e-2
    d = np.diff(got["PRN_start_sample_count"].astype(np.int64))
    assert set(np.unique(d)) <= {15999, 16000, 16001}
    assert np.max(np.abs(got["PRN_start_sample_count"].astype(np.int64) - want["PRN_start_sample_count"].astype(np.int64))) <= 1
    e.close()


def test_loops_stall_on_missing_samples_and_resume(oracle):
    """Pushing the band in three pieces and running after each gives byte-identical records to one push + one run:
    a loop whose next vector_length samples are not resident waits instead of correlating stale memory."""
    from gnss_sdr_b200 import capi
    fs = 4e6
    svs, codes, iq = _closed_loop_case(oracle, seconds=0.5)
    confs = [ol.default_conf(fs_in=fs, prn=sv["prn"], pull_in_time_s=1) for sv in svs]

    def run(pieces):
        e, ids = make_engine_with_loops(capi, oracle, confs, fs, band_samples=iq, prns=[sv["prn"] for sv in svs])
        for lid, sv in zip(ids, svs):
            e.loop_start(lid, float(sv["delay"]), sv["doppler"] - 20.0, 0, 0)
        out = [[] for _ in ids]
        pos = 0
        for p in pieces:
            e.iq_push(0, iq[pos:pos + p])
            pos += p
            rec, cnt = e.loop_run(600)
            for i in range(len(ids)):
                out[i].append(rec[i, :cnt[i]])
        res = [np.concatenate(o) for o in out]
        e.close()
        return res

    whole = run([len(iq)])
    parts = run([700_001, 512_345, len(iq) - 700_001 - 512_345])
    for a, b in zip(whole, parts):
        assert len(a) > 480 and len(a) == len(b)
        assert a.tobytes() == b.tobytes()


def test_streaming_through_a_small_ring_is_identical(oracle):
    """A receiver-like session: the band is a ring of 2^20 samples (0.26 s) fed 0.1 s at a time while the loops run;
    epochs straddle the wrap-around and old samples are overwritten behind the loops.  Records must equal those of
    one push into a band that holds everything."""
    from gnss_sdr_b200 import capi
    fs = 4e6
    svs, codes, iq = _closed_loop_case(oracle, seconds=1.0)
    confs = [ol.default_conf(fs_in=fs, prn=sv["prn"], pull_in_time_s=1) for sv in svs]

    def start_all(e, ids):
        for lid, sv in zip(ids, svs):
            e.loop_start(lid, float(sv["delay"]), sv["doppler"] + 15.0, 0, 0)

    e, ids = make_engine_with_loops(capi, oracle, confs, fs, band_samples=iq, prns=[sv["prn"] for sv in svs])
    e.iq_push(0, iq)
    start_all(e, ids)
    whole, wcnt = e.loop_run(1000)
    e.close()

    e = capi.Engine()
    e.iq_create(0, 1 << 20)
    ids = []
    for c, sv in zip(confs, svs):
        ch = e.channel_create(0, 3)
        e.channel_set_code(ch, codes[sv["prn"]], [-0.5, 0.0, 0.5])
        ids.append(e.loop_create(ch, c))
    start_all(e, ids)
    got = [[] for _ in ids]
    step = 400_000
    for pos in range(0, len(iq), step):
        e.iq_push(0, iq[pos:pos + step])
        rec, cnt = e.loop_run(150)
        for i in range(len(ids)):
            got[i].append(rec[i, :cnt[i]])
    e.close()
    for i in range(len(ids)):
        g = np.concatenate(got[i])
        assert len(g) == wcnt[i] and wcnt[i] > 980
        assert g.tobytes() == whole[i, :wcnt[i]].tobytes()


def test_noise_only_input_ends_in_loss_of_lock(oracle):
    """Noise only: once the pull-in transitory is over (:1910-1918, integer seconds since acquisition) the C/N0
    carrier lock test sits near 0 < carrier_lock_th and the carrier-lock counter runs out - same epoch as the oracle's
    closed loop.  (The M2M4 estimator reads ~26.7 dB-Hz on pure noise, above the default cn0_min = 25, so the code-lock
    counter alone would not fire; that is the reference's behaviour too.)"""
    from gnss_sdr_b200 import capi
    fs = 4e6
    rng = np.random.default_rng(9)
    n = int(fs * 1.3)
    iq = (rng.standard_normal(n) + 1j * rng.standard_normal(n)).astype(np.complex64)
    conf = ol.default_conf(fs_in=fs, pull_in_time_s=0, max_carrier_lock_fail=30)
    e, ids = make_engine_with_loops(capi, oracle, [conf], fs, band_samples=iq)
    e.iq_push(0, iq)
    e.loop_start(ids[0], 100.0, 0.0, 0, 0)
    rec, cnt = e.loop_run(1290)
    s = e.loop_status(ids[0])
    assert s.state == 0 and s.loss_of_lock == 1
    o = ol.PortLoop(conf)
    o.start(100.0, 0.0, 0, 0)
    want = lh.run_closed_loop(o, lh.PortCorrelator(oracle.port, oracle.port.gps_ca_code(1), [-0.5, 0.0, 0.5]), iq, 1290)
    assert o.status().state == 0 and 1000 < len(want) < 1100
    assert abs(int(cnt[0]) - len(want)) <= 2
    e.close()


def test_dump_file_round_trip(oracle, tmp_path):
    from gnss_sdr_b200 import capi
    fs = 4e6
    svs, codes, iq = _closed_loop_case(oracle, seconds=0.2)
    conf = ol.default_conf(fs_in=fs, prn=svs[0]["prn"])
    e, ids = make_engine_with_loops(capi, oracle, [conf], fs, band_samples=iq, prns=[svs[0]["prn"]])
    e.iq_push(0, iq)
    e.loop_start(ids[0], float(svs[0]["delay"]), svs[0]["doppler"], 0, 0)
    rec, cnt = e.loop_run(150)
    fn = str(tmp_path / "trk.dat")
    capi.trk_dump_write(fn, rec[0, :cnt[0]])
    back = np.fromfile(fn, capi.TRK_DUMP_RECORD_DTYPE)
    assert back.tobytes() == rec[0, :cnt[0]].tobytes() and os.path.getsize(fn) == 108 * cnt[0]
    if ol.ref_lib() is not None:
        got = ol.ref_dump_read(fn)
        assert np.array_equal(got[:, 7], rec[0, :cnt[0]]["PRN_start_sample_count"].astype(np.float64))
    e.close()


def test_loop_api_rejects_inconsistent_requests(oracle):
    """Error behaviour of the loop entry points: return codes, never exit() (SURVEY 8b: all functions return int)."""
    from gnss_sdr_b200 import capi
    e = capi.Engine()
    e.iq_create(0, 1 << 16)
    code = oracle.port.gps_ca_code(1)
    ch3 = e.channel_create(0, 3)
    e.channel_set_code(ch3, code, [-0.5, 0.0, 0.5])
    ch_hd = e.channel_create(0, 3)
    e.channel_set_code(ch_hd, code, [-0.5, 0.0, 0.5], high_dyn=True)
    ch_empty = e.channel_create(0, 3)
    good = ol.default_conf()
    with pytest.raises(capi.B200Error) as ei:
        e.loop_create(ch_empty, good)                      # no code table
    assert ei.value.code == -4
    with pytest.raises(capi.B200Error) as ei:
        e.loop_create(ch3, ol.default_conf(veml=1))   # five taps wanted, three registered
    assert ei.value.code == -1
    with pytest.raises(capi.B200Error) as ei:
        e.loop_create(ch_hd, good)                          # high-dynamics resampler: not in the device loop
    assert ei.value.code == -1
    for bad in (dict(cn0_samples=65), dict(cn0_samples=0), dict(pll_filter_order=4), dict(dll_filter_order=0), dict(slope=0.0),
                dict(code_period=0.0004)):
        with pytest.raises(capi.B200Error) as ei:
            e.loop_create(ch3, ol.default_conf(**bad))
        assert ei.value.code == -5, bad
    rec, cnt = e.loop_run(5)                                # no loops yet: nothing to do, no error
    assert rec.shape == (0, 5) and cnt.size == 0
    lid = e.loop_create(ch3, good)
    rec, cnt = e.loop_run(5)                                # created but never started: standby
    assert cnt[lid] == 0 and e.loop_status(lid).state == 0
    with pytest.raises(capi.B200Error):
        e.loop_start(lid + 7, 0.0, 0.0, 0, 0)
    with pytest.raises(capi.B200Error):
        e.loop_set_mode(3)
    e.close()
