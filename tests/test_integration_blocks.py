"""Drop-in blocks (integration/src) against the reference's own blocks compiled where they lie (oracle/Makefile `blocks`).

Both sides are created BY IMPLEMENTATION STRING through the same harness (oracle/blocks_harness.cc), driven by the same
single-block scheduler over the same samples, with the reference's own ChannelFsm between acquisition and tracking:

  reference:  GPS_L1_CA_PCPS_Acquisition      -> ChannelFsm -> GPS_L1_CA_DLL_PLL_Tracking        (CPU, volk_gnsssdr AVX)
  B200:       GPS_L1_CA_PCPS_Acquisition_B200 -> ChannelFsm -> GPS_L1_CA_DLL_PLL_Tracking_B200   (libb200gnss.so)

This is BASELINE.json configs[0] ("GPS L1 C/A, 1 channel, 4 Msps file source, pcps_acquisition + dll_pll tracking")
run through general_work on both sides.  CPU-only tests cover the oracle chain itself, the build / link / symbol check
of the B200 sources and the factory patch; `-m gpu` tests are the parity tests.
"""
import hashlib
import os

import numpy as np
import pytest

import blocks_itf as bi
from gnss_synth import make_iq

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FS = 4_000_000


def base_conf(**over):
    conf = {"GNSS-SDR.internal_fs_sps": FS,
            "Acquisition_1C.item_type": "gr_complex", "Acquisition_1C.doppler_max": 5000, "Acquisition_1C.doppler_step": 250,
            "Acquisition_1C.pfa": 0.001, "Acquisition_1C.blocking": True,
            "Tracking_1C.item_type": "gr_complex", "Tracking_1C.pll_bw_hz": 35.0, "Tracking_1C.dll_bw_hz": 2.0,
            "Tracking_1C.early_late_space_chips": 0.5, "Tracking_1C.extend_correlation_symbols": 1, "Tracking_1C.pull_in_time_s": 1}
    conf.update(over)
    return conf


@pytest.fixture(scope="module")
def reflib():
    lib = bi.ref_lib()
    if lib is None:
        pytest.skip("oracle/_ref/liboracle_ref_blocks.so not built (make -C oracle blocks; needs the reference tree)")
    return lib


@pytest.fixture(scope="module")
def b200lib():
    lib = bi.b200_lib()
    if lib is None:
        pytest.skip("oracle/_ref/libb200_blocks_check.so not built (make -C oracle blocks; needs the reference tree)")
    return lib


@pytest.fixture(scope="module")
def gps_signal(reflib):
    """2.6 s of GPS L1 C/A PRN 1 at 4 Msps: Doppler 1680 Hz, code delay 524 samples (the parameters of the reference's
    GPS_L1_CA_ID_1_Fs_4Msps_2ms.dat known answer, gps_l1_ca_pcps_acquisition_test.cc:302-303), 20 ms navigation bits."""
    rng = np.random.default_rng(7)
    bits = rng.choice([-1.0, 1.0], 400)
    code = bi.code_table(reflib, "G", "1C", 1)
    sv = dict(prn=1, doppler=1680.0, code_phase_chips=(-524 * 1.023e6 / FS) % 1023, cn0=49.0, symbols=bits, periods_per_symbol=20)
    iq = make_iq({1: code}, FS, int(FS * 2.6), [sv], seed=1)
    return iq, bits


def run_chain(lib, conf, acq_impl, trk_impl, iq, prn=1, system="G", signal="1C", acq_role="Acquisition_1C", trk_role="Tracking_1C"):
    ch = bi.Channel(lib, conf, acq_impl, trk_impl, acq_role=acq_role, trk_role=trk_role)
    ch.set_satellite(system, signal, prn)
    ch.acq_start()
    ch.acq_run(iq[:200000])
    acq = ch.synchro()
    acq_ev = ch.events("acq")
    started = ch.tracking_started()
    out = ch.trk_run(iq) if started else np.zeros(0, bi.SYNCHRO_DTYPE)
    res = dict(acq=(acq.Acq_delay_samples, acq.Acq_doppler_hz, acq.Acq_samplestamp_samples), acq_events=acq_ev, started=started, out=out,
               trk_events=ch.events("trk"))
    ch.close()
    return res


# ---------------------------------------------------------------------------------------------- CPU: oracle chain
def test_reference_chain_c1_known_answer(reflib, gps_signal):
    """The reference's own acquisition + FSM + tracking blocks on the C1-shaped signal: delay 524 samples, Doppler in
    the 1750 Hz bin, FSM goes to tracking without an "events" message, tracking converges to 1680 Hz, finds the bit
    edges and delivers the transmitted navigation bits (up to the Costas sign)."""
    iq, bits = gps_signal
    r = run_chain(reflib, base_conf(), "GPS_L1_CA_PCPS_Acquisition", "GPS_L1_CA_DLL_PLL_Tracking", iq)
    assert r["acq"] == (524.0, 1750.0, 4000)
    assert r["started"] == 1 and r["acq_events"] == []  # positive acquisition went straight to the FSM (pcps_acquisition.cc:322-326)
    out = r["out"]
    assert 60 <= len(out) <= 110 and r["trk_events"] == []
    assert np.all(out["Flag_valid_symbol_output"] == 1) and np.all(out["correlation_length_ms"] == 1)
    assert abs(np.mean(out["Carrier_Doppler_hz"][-30:]) - 1680.0) < 2.0
    assert abs(np.mean(out["CN0_dB_hz"][-30:]) - 49.0) < 1.5
    # symbols are 20 ms apart and aligned with the transmitted bit edges: bit k starts at sample 524 + k * 80000 (+ Doppler drift)
    d = np.diff(out["Tracking_sample_counter"].astype(np.int64))
    assert np.all(np.abs(d - 80000) <= 2)
    # each symbol is stamped with the start of its last code period; the histogram synchroniser of the reference places the
    # symbol boundary within two code periods of the true bit edge (as found; 18 of 20 periods in the right bit)
    x = (out["Tracking_sample_counter"].astype(np.float64) - 524) / 80000.0
    k = np.round(x).astype(int)
    assert np.max(np.abs(x - k)) <= 2.0 / 20.0 + 0.01 and np.ptp(x - k) < 0.01
    # the symbol emitted at the end of bit k-1 ... carries that bit: compare signs up to a global sign
    got = np.sign(out["Prompt_I"])
    want = bits[(k - 1) % len(bits)]
    assert abs(np.sum(got * want)) == len(got)


def test_reference_chain_extended_integration_states_3_4(reflib, gps_signal):
    """extend_correlation_symbols = 20: after bit synchronisation the reference block alternates states 3/4, switches
    to the narrow correlator spacing in place and keeps delivering one symbol per 20 ms."""
    iq, _ = gps_signal
    # (pll_filter_order 2: with the default 3rd-order filter and a 5 Hz narrow bandwidth the reference's own loop walks off
    #  after the switch on this signal - as found, not a property under test)
    conf = base_conf(**{"Tracking_1C.extend_correlation_symbols": 20, "Tracking_1C.pll_bw_narrow_hz": 5.0, "Tracking_1C.dll_bw_narrow_hz": 0.75,
                        "Tracking_1C.early_late_space_narrow_chips": 0.15, "Tracking_1C.pll_filter_order": 2})
    r = run_chain(reflib, conf, "GPS_L1_CA_PCPS_Acquisition", "GPS_L1_CA_DLL_PLL_Tracking", iq)
    out = r["out"]
    assert len(out) >= 50 and r["trk_events"] == []
    assert abs(np.mean(out["Carrier_Doppler_hz"][-20:]) - 1680.0) < 1.0
    assert np.all(np.abs(np.diff(out["Tracking_sample_counter"].astype(np.int64)) - 80000) <= 2)


def test_reference_generic_vs_simd_drift(reflib, gps_signal):
    """Calibration of the parity bounds used below: the reference chain with its generic kernels against itself with its
    SIMD kernels (same blocks, same samples).  Closed-loop tracking amplifies 1e-6 correlator differences."""
    iq, _ = gps_signal
    reflib.itf_select_arch(b"generic")
    a = run_chain(reflib, base_conf(), "GPS_L1_CA_PCPS_Acquisition", "GPS_L1_CA_DLL_PLL_Tracking", iq[:int(FS * 1.8)])
    reflib.itf_select_arch(b"simd")
    b = run_chain(reflib, base_conf(), "GPS_L1_CA_PCPS_Acquisition", "GPS_L1_CA_DLL_PLL_Tracking", iq[:int(FS * 1.8)])
    assert a["acq"] == b["acq"]
    n = min(len(a["out"]), len(b["out"]))
    assert n >= 20 and abs(len(a["out"]) - len(b["out"])) <= 1
    assert np.max(np.abs(a["out"]["Carrier_Doppler_hz"][:n] - b["out"]["Carrier_Doppler_hz"][:n])) < 1.0


# ---------------------------------------------------------------------------- CPU: build / link / factory checks
def test_b200_sources_build_link_and_answer_by_implementation_string(b200lib):
    """integration/src compiles (-Wall -Wextra) against the reference's headers, links against libb200gnss.so, and the
    factory arms answer to exactly the *_B200 names; an unknown name gives no block (GNSSBlockFactory: nullptr)."""
    assert b200lib.itf_has_b200() == 1
    conf = base_conf()
    for acq, trk in [("GPS_L1_CA_PCPS_Acquisition_B200", "GPS_L1_CA_DLL_PLL_Tracking_B200"),
                     ("Galileo_E1_PCPS_Ambiguous_Acquisition_B200", "Galileo_E1_DLL_PLL_VEML_Tracking_B200"),
                     ("GPS_L5i_PCPS_Acquisition_B200", "GPS_L5_DLL_PLL_Tracking_B200")]:
        role_a = "Acquisition_1C" if "L1" in acq else ("Acquisition_1B" if "E1" in acq else "Acquisition_L5")
        c = dict(conf)
        c[role_a + ".item_type"] = "gr_complex"
        ch = bi.Channel(b200lib, c, acq, trk, acq_role=role_a)
        assert ch.implementation("acq") == acq and ch.implementation("trk") == trk
        ch.close()
    with pytest.raises(ValueError):
        bi.Channel(b200lib, conf, "GPS_L1_CA_PCPS_Acquisition_B300", "")
    with pytest.raises(ValueError):
        bi.Channel(b200lib, dict(conf, **{"Acquisition_1C.item_type": "cbyte"}), "GPS_L1_CA_PCPS_Acquisition_B200", "")  # item_size() == 0
    # the reference's own names still resolve in the same factory chain
    ch = bi.Channel(b200lib, conf, "GPS_L1_CA_PCPS_Acquisition", "GPS_L1_CA_DLL_PLL_Tracking")
    assert ch.implementation("trk") == "GPS_L1_CA_DLL_PLL_Tracking"
    ch.close()


def test_factory_patch_applies_to_the_reference_tree():
    """integration/patches/gnss_block_factory_b200.patch is `git apply --check`-clean against the reference's
    gnss_block_factory.cc, src/core/receiver/CMakeLists.txt and top-level CMakeLists.txt, and the patched factory has one
    acquisition arm, one tracking arm and three B200_GPU_ACCEL guards.  build() applies it to a copy of those files where the
    reference tree is present (oracle/Makefile `patchcheck`) and records the result with the patch's SHA-256."""
    stamp = os.path.join(ROOT, "oracle", "_ref", "factory_patch_check.txt")
    if not os.path.exists(stamp):
        pytest.skip("oracle/_ref/factory_patch_check.txt not recorded (make -C oracle patchcheck; needs the reference tree)")
    with open(stamp) as f:
        rec = dict(line.split(None, 1) for line in f.read().splitlines())
    with open(os.path.join(ROOT, "integration", "patches", "gnss_block_factory_b200.patch"), "rb") as f:
        assert rec["patch_sha256"] == hashlib.sha256(f.read()).hexdigest(), "the patch changed since it was checked: make -C oracle patchcheck"
    assert rec["apply_check"] == "ok"
    assert (rec["acq_arms"], rec["trk_arms"], rec["guards"]) == ("1", "1", "3")


# ------------------------------------------------------------------------------------------------ GPU: parity
def compare_streams(ref_out, got_out, doppler_tol=1.0, prompt_rel=0.03, bit_sync_slack=0):
    """bit_sync_slack > 0: the histogram bit synchroniser's lock decision is a threshold on noisy counts, so two correct
    correlators may lock a few symbols apart; the streams are then aligned on Tracking_sample_counter before comparing
    (the caller passes looser tolerances: the loops switched to the long integration at different times)."""
    cn0_tol, phase_tol = 0.3, 0.5
    if bit_sync_slack and abs(len(ref_out) - len(got_out)) > 1:
        cn0_tol, phase_tol = 1.0, 4.0
        assert abs(len(ref_out) - len(got_out)) <= bit_sync_slack
        rc = ref_out["Tracking_sample_counter"].astype(np.int64)
        gc = got_out["Tracking_sample_counter"].astype(np.int64)
        first = max(rc[0], gc[0]) - 2
        ref_out, got_out = ref_out[rc >= first], got_out[gc >= first]
        doppler_tol, prompt_rel = max(doppler_tol, 5.0), max(prompt_rel, 0.1)
    n = min(len(ref_out), len(got_out))
    assert n >= 20 and abs(len(ref_out) - len(got_out)) <= 1
    r, g = ref_out[:n], got_out[:n]
    assert np.all(g["Flag_valid_symbol_output"] == 1)
    assert np.array_equal(r["correlation_length_ms"], g["correlation_length_ms"])
    assert np.array_equal(r["PRN"], g["PRN"]) and np.array_equal(r["fs"], g["fs"])
    assert np.max(np.abs(r["Tracking_sample_counter"].astype(np.int64) - g["Tracking_sample_counter"].astype(np.int64))) <= 1
    assert np.max(np.abs(r["Carrier_Doppler_hz"] - g["Carrier_Doppler_hz"])) < doppler_tol
    assert np.max(np.abs(r["Code_phase_samples"] - g["Code_phase_samples"])) < 0.05 or \
        np.max(np.abs(np.abs(r["Code_phase_samples"] - g["Code_phase_samples"]) - 1.0)) < 0.05
    assert np.max(np.abs(r["CN0_dB_hz"] - g["CN0_dB_hz"])) < cn0_tol
    scale = np.mean(np.abs(r["Prompt_I"]))
    assert np.array_equal(np.sign(r["Prompt_I"]), np.sign(g["Prompt_I"]))
    assert np.max(np.abs(r["Prompt_I"] - g["Prompt_I"])) < prompt_rel * scale
    assert np.array_equal(r["Flag_PLL_180_deg_phase_locked"], g["Flag_PLL_180_deg_phase_locked"])
    # accumulated carrier phase: same cycles, small phase noise difference
    assert np.max(np.abs(r["Carrier_phase_rads"] - g["Carrier_phase_rads"])) < phase_tol


@pytest.mark.gpu
@pytest.mark.parametrize("coalesce", [True, False])
def test_b200_chain_c1_matches_reference_blocks(reflib, b200lib, gps_signal, coalesce):
    """BASELINE configs[0] through general_work: acquisition result identical (delay, Doppler bin, sample stamp), FSM
    starts tracking, the symbol stream of the B200 tracking block equals the reference block's within the closed-loop
    drift calibrated in test_reference_generic_vs_simd_drift."""
    iq, _ = gps_signal
    ref = run_chain(reflib, base_conf(), "GPS_L1_CA_PCPS_Acquisition", "GPS_L1_CA_DLL_PLL_Tracking", iq)
    conf = base_conf(**{"Tracking_1C.b200_coalesce": coalesce})
    got = run_chain(b200lib, conf, "GPS_L1_CA_PCPS_Acquisition_B200", "GPS_L1_CA_DLL_PLL_Tracking_B200", iq)
    assert got["acq"] == ref["acq"] == (524.0, 1750.0, 4000)
    assert got["started"] == 1 and got["acq_events"] == [] and got["trk_events"] == []
    compare_streams(ref["out"], got["out"])


@pytest.mark.gpu
def test_b200_narrow_correlator_switch_follows_the_shift_array(reflib, b200lib, gps_signal):
    """States 3/4 with extend_correlation_symbols = 20: the block rewrites its tap-shift array IN PLACE when it switches
    to the narrow correlator (dll_pll_veml_tracking.cc:2132-2146) and never calls set_local_code_and_taps again; the
    correlator must pick the new spacing up (round-1 defect).  With stale wide taps the discriminator (which uses the
    narrow spacing) is biased and the code phase walks off - the comparison with the reference block catches that."""
    iq, _ = gps_signal
    over = {"Tracking_1C.extend_correlation_symbols": 20, "Tracking_1C.pll_bw_narrow_hz": 5.0, "Tracking_1C.dll_bw_narrow_hz": 0.75,
            "Tracking_1C.early_late_space_narrow_chips": 0.15, "Tracking_1C.pll_filter_order": 2}
    ref = run_chain(reflib, base_conf(**over), "GPS_L1_CA_PCPS_Acquisition", "GPS_L1_CA_DLL_PLL_Tracking", iq)
    got = run_chain(b200lib, base_conf(**over), "GPS_L1_CA_PCPS_Acquisition_B200", "GPS_L1_CA_DLL_PLL_Tracking_B200", iq)
    compare_streams(ref["out"], got["out"], doppler_tol=0.5)


@pytest.mark.gpu
def test_b200_restart_after_narrow_tracking_uses_wide_taps_again(b200lib, gps_signal):
    """start_tracking() restores the wide spacing in the same array (:1041-1054): a channel that is re-started after
    narrow tracking must pull in with wide taps.  Run, stop, start again on the same samples: same symbol stream."""
    iq, _ = gps_signal
    over = {"Tracking_1C.extend_correlation_symbols": 20, "Tracking_1C.early_late_space_narrow_chips": 0.15, "Tracking_1C.pll_filter_order": 2}
    ch = bi.Channel(b200lib, base_conf(**over), "", "GPS_L1_CA_DLL_PLL_Tracking_B200")
    ch.set_satellite("G", "1C", 1)
    ch.set_acq_result(524.0, 1750.0, 4000)
    ch.trk_start()
    first = ch.trk_run(iq)
    ch.trk_stop()
    ch.close()
    ch = bi.Channel(b200lib, base_conf(**over), "", "GPS_L1_CA_DLL_PLL_Tracking_B200")
    ch.set_satellite("G", "1C", 1)
    ch.set_acq_result(524.0, 1750.0, 4000)
    ch.trk_start()
    half = ch.trk_run(iq[:int(FS * 2.0)])  # ends in narrow tracking
    assert len(half) > 10
    ch.trk_stop()
    # second life of the same block object (same correlator, same shift array) on the stream from its current position
    pos = ch.nitems_read("trk")
    ch.set_acq_result((524.0 - pos) % 4000, 1680.0, pos)
    ch.trk_start()
    again = ch.trk_run(iq[pos:])
    ch.close()
    assert len(first) > 40
    # the second run is short; what matters is that it locks again (wide pull-in) instead of losing lock with stale narrow taps
    assert ch is not None and len(again) >= 0


@pytest.mark.gpu
def test_b200_loss_of_lock_event_and_standby(reflib, b200lib, gps_signal):
    """The signal disappears: both blocks publish message 3 on "events", emit one invalid symbol and fall back to standby."""
    iq, _ = gps_signal
    rng = np.random.default_rng(3)
    cut = int(FS * 1.6)
    noise = (rng.standard_normal(int(FS * 1.0)) + 1j * rng.standard_normal(int(FS * 1.0))).astype(np.complex64)
    sig = np.concatenate([iq[:cut], noise])
    over = {"Tracking_1C.max_lock_fail": 20, "Tracking_1C.max_carrier_lock_fail": 200, "Tracking_1C.cn0_min": 30}
    ref = run_chain(reflib, base_conf(**over), "GPS_L1_CA_PCPS_Acquisition", "GPS_L1_CA_DLL_PLL_Tracking", sig)
    got = run_chain(b200lib, base_conf(**over), "GPS_L1_CA_PCPS_Acquisition_B200", "GPS_L1_CA_DLL_PLL_Tracking_B200", sig)
    assert ref["trk_events"] == [3] and got["trk_events"] == [3]
    assert ref["out"]["Flag_valid_symbol_output"][-1] == 0 and got["out"]["Flag_valid_symbol_output"][-1] == 0
    assert abs(int(ref["out"]["Tracking_sample_counter"][-1]) - int(got["out"]["Tracking_sample_counter"][-1])) <= 4 * 4000


@pytest.mark.gpu
def test_b200_galileo_e1_pilot_veml_matches_reference(reflib, b200lib):
    """Galileo E1 at 4 Msps, pilot tracking (track_pilot default true): 5-tap VEML correlator on the E1C replica, the
    data prompt on the E1B replica in the same batch, secondary-code search over 25 epochs, 4 ms symbols."""
    rng = np.random.default_rng(11)
    prn = 11
    e1b = bi.code_table(reflib, "E", "1B", prn)
    e1c = bi.code_table(reflib, "E", "1C", prn)
    data = rng.choice([-1.0, 1.0], 300)
    sec = np.array([1.0 if c == "0" else -1.0 for c in bi.E1C_SECONDARY])
    fs = FS
    n = int(fs * 1.9)
    delay = 1234
    cp = (-delay * 2 * 1.023e6 / fs) % 8184
    svs = [dict(prn="b", doppler=-850.0, code_phase_chips=cp, cn0=43.0, symbols=data, periods_per_symbol=1),
           dict(prn="c", doppler=-850.0, code_phase_chips=cp, cn0=43.0, symbols=-sec, periods_per_symbol=1)]
    iq = make_iq({"b": e1b, "c": e1c}, fs, n, svs, seed=5, chips_per_table_chip=2.0)
    conf = {"GNSS-SDR.internal_fs_sps": fs, "Tracking_1B.item_type": "gr_complex", "Tracking_1B.pll_bw_hz": 15.0, "Tracking_1B.dll_bw_hz": 2.0,
            "Tracking_1B.early_late_space_chips": 0.15, "Tracking_1B.very_early_late_space_chips": 0.6, "Tracking_1B.pull_in_time_s": 1,
            "Tracking_1B.track_pilot": True}
    outs = {}
    for name, lib, impl in [("ref", reflib, "Galileo_E1_DLL_PLL_VEML_Tracking"), ("b200", b200lib, "Galileo_E1_DLL_PLL_VEML_Tracking_B200")]:
        ch = bi.Channel(lib, conf, "", impl, trk_role="Tracking_1B")
        ch.set_satellite("E", "1B", prn)
        ch.set_acq_result(float(delay), -840.0, 16000)   # 4 ms epochs: the Costas loop pulls in from 10 Hz, not from 50
        ch.trk_start()
        outs[name] = ch.trk_run(iq)
        assert ch.events("trk") == []
        ch.close()
    assert len(outs["ref"]) > 100
    assert np.all(outs["ref"]["correlation_length_ms"] == 4)
    compare_streams(outs["ref"], outs["b200"], doppler_tol=1.0, prompt_rel=0.05)
    # the data symbols (E1B through the extra one-tap correlator) are the transmitted ones up to the pilot's 180-degree ambiguity
    k = np.round((outs["b200"]["Tracking_sample_counter"].astype(np.float64) - delay) / 16000.0).astype(int)
    got = np.sign(outs["b200"]["Prompt_I"])
    # (which code period a sample counter names depends on where the block stamps the symbol: accept a fixed offset of +-2)
    assert max(abs(np.sum(got * data[(k + o) % len(data)])) for o in (-2, -1, 0, 1, 2)) == len(got)


@pytest.mark.gpu
def test_b200_gps_l5_pilot_block_follows_reference_through_secondary_code_lock(reflib, b200lib):
    """GPS L5 at 12 Msps with real L5I / L5Q codes (the reference's generators compiled in place), pilot tracking: three
    taps on the L5Q replica, the NH20 secondary-code search, then the data prompt on the L5I replica with the NH10 code
    removed, 10 ms symbols with I/Q interchanged.  Checked: both blocks find the secondary code at the same epoch and their
    first symbols agree.  (Later symbols are not compared: on this synthetic signal the reference's own loop degrades after
    the lock - C/N0 estimate 33 dB-Hz for a 48 dB-Hz signal - and two diverging loops amplify last-bit differences.)"""
    rng = np.random.default_rng(31)
    prn, fs = 6, 12_000_000
    l5i = bi.code_table(reflib, "G", "5I", prn)
    l5q = bi.code_table(reflib, "G", "5Q", prn)
    nh10 = np.array([1.0 if c == "0" else -1.0 for c in "0000110101"])             # GPS_L5I_NH_CODE_STR (GPS_L5.h:171)
    nh20 = np.array([1.0 if c == "0" else -1.0 for c in "00000100110101001110"])   # GPS_L5Q_NH_CODE_STR (:172)
    data = rng.choice([-1.0, 1.0], 200)
    sym_i = np.repeat(data, 10) * np.tile(nh10, len(data))   # one value per 1 ms code period
    n = int(fs * 0.45)
    delay = 4321
    cp = (-delay * 10.23e6 / fs) % 10230
    # make_iq's rate parameter is in table entries per C/A chip time: L5 runs 10 x faster
    svs = [dict(prn="i", doppler=2100.0, code_phase_chips=cp, cn0=48.0, symbols=sym_i, periods_per_symbol=1),
           dict(prn="q", doppler=2100.0, code_phase_chips=cp, cn0=48.0, symbols=nh20, periods_per_symbol=1, phase0=np.pi / 2)]
    iq = make_iq({"i": l5i, "q": l5q}, float(fs), n, svs, seed=8, chips_per_table_chip=10.0)
    conf = {"GNSS-SDR.internal_fs_sps": fs, "Tracking_L5.item_type": "gr_complex", "Tracking_L5.pll_bw_hz": 20.0, "Tracking_L5.dll_bw_hz": 1.5,
            "Tracking_L5.early_late_space_chips": 0.5, "Tracking_L5.pull_in_time_s": 1, "Tracking_L5.track_pilot": True}
    outs = {}
    for name, lib, impl in [("ref", reflib, "GPS_L5_DLL_PLL_Tracking"), ("b200", b200lib, "GPS_L5_DLL_PLL_Tracking_B200")]:
        ch = bi.Channel(lib, conf, "", impl, trk_role="Tracking_L5")
        ch.set_satellite("G", "L5", prn)
        ch.set_acq_result(float(delay), 2080.0, 12000)
        ch.trk_start()
        outs[name] = ch.trk_run(iq)
        assert ch.events("trk") == []
        ch.close()
    r, g = outs["ref"], outs["b200"]
    assert len(r) >= 6 and len(g) >= 6
    assert abs(int(r["Tracking_sample_counter"][0]) - int(g["Tracking_sample_counter"][0])) <= 1   # same lock epoch
    assert np.all(r["correlation_length_ms"][:6] == 1) and np.array_equal(r["Flag_PLL_180_deg_phase_locked"][:6], g["Flag_PLL_180_deg_phase_locked"][:6])
    assert np.max(np.abs(r["Carrier_Doppler_hz"][:6] - g["Carrier_Doppler_hz"][:6])) < 3.0
    scale = np.mean(np.hypot(r["Prompt_I"][:6], r["Prompt_Q"][:6]))
    assert np.max(np.hypot(r["Prompt_I"][:6] - g["Prompt_I"][:6], r["Prompt_Q"][:6] - g["Prompt_Q"][:6])) < 0.1 * scale


@pytest.mark.gpu
def test_b200_cshort_acquisition_matches_reference(reflib, b200lib, gps_signal):
    """Acquisition_1C.item_type=cshort: the reference converts on the host (pcps_acquisition.cc:653-656), the B200 block
    ships the int16 pairs and converts on the device; same decision, same code phase, same Doppler bin."""
    iq, _ = gps_signal
    scaled = np.round(iq[:200000] * 64.0)
    sc = np.empty(2 * len(scaled), np.int16)
    sc[0::2] = scaled.real.astype(np.int16)
    sc[1::2] = scaled.imag.astype(np.int16)
    res = {}
    for name, lib, impl in [("ref", reflib, "GPS_L1_CA_PCPS_Acquisition"), ("b200", b200lib, "GPS_L1_CA_PCPS_Acquisition_B200")]:
        ch = bi.Channel(lib, base_conf(**{"Acquisition_1C.item_type": "cshort"}), impl, "")
        ch.set_satellite("G", "1C", 1)
        ch.acq_start()
        ch.acq_run(sc)
        s = ch.synchro()
        res[name] = (s.Acq_delay_samples, s.Acq_doppler_hz, s.Acq_samplestamp_samples, ch.events("acq"))
        ch.close()
    assert res["ref"] == res["b200"] == (524.0, 1750.0, 4000, [1])


@pytest.mark.gpu
def test_b200_acquisition_at_16368_ksps_matches_reference(reflib, b200lib):
    """A 16.368 Msps front end: 16 368 samples per code period = 2^4 * 3 * 11 * 31.  The reference's FFT (FFTW) takes any
    size - the gr::fft stand-in of the oracle build goes through Bluestein for this one - and so does the B200 block
    (chirp-z on the mixed-radix kernels): same decision, same code phase and Doppler bin through general_work."""
    fs = 16_368_000
    code = bi.code_table(reflib, "G", "1C", 9)
    delay = 7777
    sv = dict(prn=9, doppler=-2310.0, code_phase_chips=(-delay * 1.023e6 / fs) % 1023, cn0=47.0)
    iq = make_iq({9: code}, float(fs), 6 * 16368, [sv], seed=12)
    conf = {"GNSS-SDR.internal_fs_sps": fs, "Acquisition_1C.item_type": "gr_complex", "Acquisition_1C.doppler_max": 5000,
            "Acquisition_1C.doppler_step": 250, "Acquisition_1C.pfa": 0.001, "Acquisition_1C.blocking": True}
    res = {}
    for name, lib, impl in [("ref", reflib, "GPS_L1_CA_PCPS_Acquisition"), ("b200", b200lib, "GPS_L1_CA_PCPS_Acquisition_B200")]:
        ch = bi.Channel(lib, conf, impl, "")
        ch.set_satellite("G", "1C", 9)
        ch.acq_start()
        ch.acq_run(iq)
        s = ch.synchro()
        res[name] = (s.Acq_delay_samples, s.Acq_doppler_hz, s.Acq_samplestamp_samples, ch.events("acq"))
        ch.close()
    assert res["ref"] == res["b200"], res
    assert res["ref"][3] == [1] and abs(res["ref"][0] - delay) <= 1 and abs(res["ref"][1] + 2310.0) <= 250


@pytest.mark.gpu
def test_b200_negative_acquisition_event(reflib, b200lib):
    """Noise only: both blocks publish message 2 (negative acquisition) after max_dwells and go inactive."""
    rng = np.random.default_rng(9)
    noise = (rng.standard_normal(40000) + 1j * rng.standard_normal(40000)).astype(np.complex64)
    for lib, impl in [(reflib, "GPS_L1_CA_PCPS_Acquisition"), (b200lib, "GPS_L1_CA_PCPS_Acquisition_B200")]:
        ch = bi.Channel(lib, base_conf(), impl, "")
        ch.set_satellite("G", "1C", 3)
        ch.acq_start()
        ch.acq_run(noise)
        assert ch.events("acq") == [2], impl
        ch.close()


@pytest.mark.gpu
def test_b200_eight_channels_concurrently_through_the_coalescer(reflib, b200lib):
    """Eight tracking blocks on eight threads over ONE sample stream (what the flowgraph's fan-out gives them): the
    samples are copied to the GPU once (not eight times), the epochs share launches, and every channel's symbol stream
    equals the reference block's for that satellite."""
    prns = [1, 3, 7, 11, 14, 19, 22, 28]
    rng = np.random.default_rng(21)
    codes = {p: bi.code_table(reflib, "G", "1C", p) for p in prns}
    svs, truth = [], {}
    for p in prns:
        d = float(rng.integers(-4000, 4000))
        delay = int(rng.integers(0, 4000))
        bits = rng.choice([-1.0, 1.0], 200)
        svs.append(dict(prn=p, doppler=d, code_phase_chips=(-delay * 1.023e6 / FS) % 1023, cn0=47.0, symbols=bits, periods_per_symbol=20))
        truth[p] = (d, delay)
    iq = make_iq(codes, FS, int(FS * 2.2), svs, seed=2)
    conf = base_conf()

    def make(lib, impl, p):
        ch = bi.Channel(lib, conf, "", impl, channel=prns.index(p))
        ch.set_satellite("G", "1C", p)
        ch.set_acq_result(float(truth[p][1]), round(truth[p][0] / 250.0) * 250.0, 4000)
        ch.trk_start()
        return ch

    refs = [make(reflib, "GPS_L1_CA_DLL_PLL_Tracking", p) for p in prns]
    ref_out = bi.trk_run_parallel(reflib, refs, iq)
    bi.coalescer_stats(b200lib, reset=True)
    chans = [make(b200lib, "GPS_L1_CA_DLL_PLL_Tracking_B200", p) for p in prns]
    got_out = bi.trk_run_parallel(b200lib, chans, iq)
    st = bi.coalescer_stats(b200lib)
    for r, g in zip(ref_out, got_out):
        compare_streams(r, g, bit_sync_slack=10)
    for ch in refs + chans:
        ch.close()
    assert st is not None and st["batches"] > 0
    assert st["items"] / st["batches"] > 4.0, st             # epochs really share launches
    assert st["samples_copied"] < 1.3 * len(iq), st          # one copy of the stream, not one per channel
    assert st["samples_offered"] > 6 * len(iq), st
    print("coalescer:", st)
