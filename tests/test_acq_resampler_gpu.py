"""Band searches through the acquisition resampler (b200_acq_set_band_resampler): the band holds the full rate, the search
decimates its span on the device and runs at the signal's acquisition rate, as the reference's
GNSS-SDR.use_acquisition_resampler does.

The decimated vector is the float32 loop of acq_resampler_np in the kernel's order, so a decimated band search gives, byte
for byte, the records and grids of b200_acq_search on that vector, on every plan family and band type; decimation 1 turns
it off again; spans outside the band and bad filters are refused before anything is launched; and one search costs one
launch more than b200_acq_search_dev.  The last two tests acquire at a real front-end rate: a cold start at 25 Msps into
the device loops on the same band, and a 4 ms search from a 100 Msps band that the full-rate plans refuse.
"""
import math

import numpy as np
import pytest

import acq_resampler_np as rnp
import acq_rig as ar
import gnss_synth as gs
from gpu_fixtures import capi, engine  # noqa: F401

pytestmark = pytest.mark.gpu


def _decimated_pair(capi, engine, rng, fs_full, opt, **kw):
    """(band object with the designed resampler, host-input object, codes, D, taps) at fs_full / D"""
    d, taps = capi.acq_resampler_design(fs_full, opt)
    assert d > 1
    acq, host, codes = ar.pair(capi, engine, rng, fs_full // d, **kw)
    acq.set_band_resampler(d, taps)
    return acq, host, codes, d, taps


def _full_rate_stream(rng, n_full, code, d, fs_full):
    """full-rate samples carrying the local code held for d samples per decimated sample: one clear peak after decimation"""
    return ar.stream(rng, n_full, np.repeat(code, d), fs_full)


def _push(engine, band, x, item_type, chunk):
    """x into a fresh band of item_type in chunks; returns the complex64 samples the band holds"""
    if item_type == "gr_complex":
        held = x.astype(np.complex64)
        for k in range(0, x.size, chunk):
            engine.iq_push(band, held[k:k + chunk])
        return held
    dt, lim = (np.int16, 32767) if item_type == "ishort" else (np.int8, 127)
    raw = ar.to_int(x, dt, 30.0 if item_type == "ishort" else 20.0, clip=(-lim, lim))
    for k in range(0, x.size, chunk):
        engine.iq_push_int(band, raw[2 * k:2 * (k + chunk)])
    return ar.from_int(raw)


# (id, full rate, optimal rate, band type, object keywords): one case per plan family, every band type, peaks and dwells
CASES = [
    ("single_d10_cfar", 25_000_000, 2_000_000, "gr_complex", dict()),
    ("single_d10_peaks_grid", 25_000_000, 2_000_000, "gr_complex", dict(use_CFAR_algorithm_flag=False, keep_grid=True)),
    ("single_d10_dwells_ishort", 25_000_000, 2_000_000, "ishort", dict(max_dwells=2)),
    ("single_d10_peaks_ibyte", 25_000_000, 2_000_000, "ibyte", dict(use_CFAR_algorithm_flag=False)),
    ("two_level_d5_4ms", 50_000_000, 10_000_000, "gr_complex", dict(sampled_ms=4, ms_per_code=4, keep_grid=True)),
    ("chirpz_d8_dwells", 16_368_000, 2_000_000, "ishort", dict(max_dwells=2)),
]


@pytest.mark.parametrize("fs,opt,item_type,kw", [c[1:] for c in CASES], ids=[c[0] for c in CASES])
def test_decimated_band_search_is_byte_identical_to_host_search(capi, engine, fs, opt, item_type, kw):
    """The span straddles the end of an owned ring; dwell k starts k * consumed * D further on."""
    rng = np.random.default_rng(fs // 1000 + len(kw))
    acq, host, codes, d, taps = _decimated_pair(capi, engine, rng, fs, opt, **kw)
    c = host.conf
    n, dwells, hist = c.consumed_samples, c.max_dwells, taps.size - 1
    span = hist + (n - 1) * d + 1
    cap = ar.pow2(3 * span)
    x = _full_rate_stream(rng, 2 * cap + 2 * n * d, codes[1][:n], d, fs)
    engine.iq_create(4, cap, item_type)
    held = _push(engine, 4, x, item_type, cap // 3 + 7)
    idx = 2 * cap - n * d // 3                           # the first span crosses ring offset 0
    lo, hi = engine.iq_window(4)
    assert lo <= idx - hist and idx + (dwells - 1) * n * d + (n - 1) * d < hi
    for k in range(dwells):
        s0 = idx + k * n * d
        y = rnp.decimate_f32(held, taps, d, s0, n)
        want = host.search(y, [1, 0], dwell_counter=k + 1)
        got = acq.search_band(4, s0, [1, 0], dwell_counter=k + 1)
        assert got.tobytes() == want.tobytes(), (k, got, want)
    assert got[0]["test_statistics"] > got[1]["test_statistics"]     # slot 1's code is in the stream
    assert ar.grids(acq) == ar.grids(host)
    acq.close()
    host.close()


def test_submit_wait_and_step_two_from_the_band(capi, engine):
    rng = np.random.default_rng(3)
    fs = 25_000_000
    acq, host, codes, d, taps = _decimated_pair(capi, engine, rng, fs, 2_000_000, n_code_slots=1)
    n = host.conf.consumed_samples
    x = _full_rate_stream(rng, 5 * n * d, codes[0], d, fs)
    engine.iq_create(5, ar.pow2(x.size))
    held = _push(engine, 5, x, "gr_complex", x.size)
    s0 = taps.size + 321
    acq.search_band_submit(5, s0, [0])
    got = acq.search_wait()
    first = host.search(rnp.decimate_f32(held, taps, d, s0, n), [0])
    assert got.tobytes() == first.tobytes()
    for a in (acq, host):
        a.set_step_two(float(first[0]["doppler"]), 125.0, 4)
    s1 = s0 + n * d
    want = host.search_step_two(rnp.decimate_f32(held, taps, d, s1, n), 0, float(first[0]["input_power"]))
    got = acq.search_step_two_band(5, s1, 0, float(first[0]["input_power"]))
    assert got.tobytes() == want.tobytes(), (got, want)
    # the host-input searches ignore the resampler
    y = rnp.decimate_f32(held, taps, d, s1, n)
    assert acq.search(y, [0]).tobytes() == host.search(y, [0]).tobytes()
    acq.close()
    host.close()


def test_decimation_one_turns_the_resampler_off(capi, engine):
    rng = np.random.default_rng(5)
    fs = 25_000_000
    acq, plain, codes, d, taps = _decimated_pair(capi, engine, rng, fs, 2_000_000)
    n = plain.conf.consumed_samples
    x = _full_rate_stream(rng, 3 * n * d, codes[0], d, fs)
    engine.iq_create(6, ar.pow2(x.size))
    _push(engine, 6, x, "gr_complex", x.size)
    acq.search_band(6, 1000, [0, 1])
    acq.set_band_resampler(1, taps)
    assert acq.search_band(6, 1000, [0, 1]).tobytes() == plain.search_band(6, 1000, [0, 1]).tobytes()
    acq.set_band_resampler(d, taps)
    acq.set_band_resampler(1, [])                         # what acq_resampler_design returns where no filter is needed
    assert acq.search_band(6, 7, [0, 1]).tobytes() == plain.search_band(6, 7, [0, 1]).tobytes()
    acq.close()
    plain.close()


def test_refusals_launch_nothing(capi, engine):
    rng = np.random.default_rng(7)
    fs = 25_000_000
    acq, _, codes, d, taps = _decimated_pair(capi, engine, rng, fs, 2_000_000)
    n, hist = acq.conf.consumed_samples, taps.size - 1
    engine.iq_create(7, 1 << 17)
    engine.iq_push(7, _full_rate_stream(rng, 60_000, codes[0], d, fs))
    lo, hi = engine.iq_window(7)
    gap = hi + 10_000
    engine.iq_push_at(7, gap, _full_rate_stream(rng, 3 * n * d, codes[0], d, fs))
    lo, hi = engine.iq_window(7)
    assert lo == gap

    def refused(call, code):
        k0 = engine.launch_count()
        with pytest.raises(capi.B200Error) as ei:
            call()
        assert ei.value.code == code, str(ei.value)
        assert engine.launch_count() == k0
        return str(ei.value)

    s0 = gap + hist - 1                                    # one sample of history before valid_from
    msg = refused(lambda: acq.search_band(7, s0, [0, 1]), ar.ERR_RANGE)
    assert f"[{s0 - hist}, {s0 + (n - 1) * d + 1})" in msg and f"[{lo}, {hi})" in msg, msg
    acq.search_band(7, s0 + 1, [0, 1])                     # the first span that fits
    s0 = hi - (n - 1) * d                                  # one sample past write_index
    msg = refused(lambda: acq.search_band(7, s0, [0, 1]), ar.ERR_RANGE)
    assert f"[{s0 - hist}, {hi + 1})" in msg, msg
    acq.search_band(7, s0 - 1, [0, 1])
    engine.iq_create(8, 1 << 17)
    engine.iq_push(8, _full_rate_stream(rng, 60_000, codes[0], d, fs))
    refused(lambda: acq.search_band(8, hist - 1, [0, 1]), ar.ERR_RANGE)    # history before the band's first sample
    acq.search_band(8, hist, [0, 1])
    # filters
    t = np.ascontiguousarray(taps, np.float32)
    set_ = capi.lib.b200_acq_set_band_resampler
    big = np.zeros(1025, np.float32)
    for dd, ptr, nt, code in ((0, t.ctypes.data, t.size, ar.ERR_ARG), (d, t.ctypes.data, 0, ar.ERR_ARG), (d, None, t.size, ar.ERR_ARG),
                              (d, big.ctypes.data, big.size, ar.ERR_RANGE)):
        k0 = engine.launch_count()
        assert set_(acq.h, dd, ptr, nt) == code, (dd, nt)
        assert engine.launch_count() == k0
    assert capi.B200_ACQ_MAX_RESAMPLER_TAPS == 1024
    # the refused calls left the resampler as it was
    y = acq.search_band(8, hist, [0, 1])
    # one sweep in flight
    acq.search_band_submit(8, hist, [0, 1])
    refused(lambda: acq.set_band_resampler(1, []), ar.ERR_STATE)
    assert acq.search_wait().tobytes() == y.tobytes()
    acq.close()


def test_decimated_band_search_launches_search_dev_plus_one(capi, engine):
    import torch
    rng = np.random.default_rng(9)
    fs = 25_000_000
    acq, _, codes, d, taps = _decimated_pair(capi, engine, rng, fs, 2_000_000)
    n = acq.conf.consumed_samples
    x = _full_rate_stream(rng, 2 * n * d, codes[0], d, fs)
    engine.iq_create(9, ar.pow2(x.size))
    held = _push(engine, 9, x, "gr_complex", x.size)
    y = rnp.decimate_f32(held, taps, d, 500, n)
    yt = torch.from_numpy(y.view(np.float32)).cuda()
    res = torch.zeros(2 * capi.ACQ_RESULT_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    k0 = engine.launch_count()
    acq.search_dev(yt.data_ptr(), [0, 1], res.data_ptr())
    k1 = engine.launch_count()
    got = acq.search_band(9, 500, [0, 1])
    k2 = engine.launch_count()
    assert k2 - k1 == k1 - k0 + 1 and k1 > k0
    engine.sync()
    torch.cuda.synchronize()
    assert got.tobytes() == res.cpu().numpy().tobytes()
    acq.close()


# ---- acquisition at real front-end rates -------------------------------------------------------------------------------
def _threshold(conf, pfa):
    from scipy.special import gammaincinv
    return 2.0 * gammaincinv(2.0, (1.0 - pfa) ** (1.0 / (conf.effective_fft_size * conf.num_doppler_bins)))


def test_cold_start_at_25_msps_through_the_resampler_into_device_loops(capi, tmp_path):
    """GPS L1 C/A at 25 Msps written as an ishort file and pushed into a band once; PRNs 1-32 swept from it at 2.5 Msps
    through the designed resampler (D = 10, 49 taps, latency 24) and judged against the reference's CFAR threshold for the
    decimated grid; device loops at 25 Msps on the same band, started from the delay, Doppler and sample stamp mapped back
    to the full rate as pcps_acquisition::update_synchro does, track their satellites."""
    from oracle import loop as ol
    fs, opt, n_ep, pfa, scale = 25_000_000, 2_000_000, 500, 0.001, 64.0
    spc_full = fs // 1000
    # 47-48 dB-Hz: the decimated sweep's threshold (pfa 1e-3 over 2 500 x 100 cells) is a statistic of 45; these satellites
    # peak at 74-118 and the strongest absent PRN of this seed at 30.  Their Doppler errors are at most 70 Hz, which the
    # loops pull in well within the 300 epochs before the tail that is judged.
    svs = [dict(prn=3, doppler=-2730.0, delay=3111, cn0=47.5), dict(prn=8, doppler=1330.0, delay=17_770, cn0=47.0),
           dict(prn=14, doppler=3125.0, delay=9_950, cn0=48.0), dict(prn=21, doppler=-620.0, delay=21_433, cn0=47.5),
           dict(prn=29, doppler=215.0, delay=6_095, cn0=48.0)]
    abs_index = 12_345
    total = abs_index + spc_full + (n_ep + 3) * spc_full
    codes = {sv["prn"]: gs.gps_ca_code(sv["prn"]) for sv in svs}
    iq = gs.make_iq(codes, fs, total, [dict(prn=sv["prn"], doppler=sv["doppler"], cn0=sv["cn0"],
                                            code_phase_chips=(-sv["delay"] * 1.023e6 / fs) % 1023) for sv in svs], seed=31)
    raw = ar.to_int(iq, np.int16, scale, clip=(-32767, 32767))
    path = tmp_path / "gps_l1_25msps.ishort"
    raw.tofile(path)
    del iq, raw

    e = capi.Engine(0)
    e.iq_create(0, total)                                              # the loops read gr_complex bands
    assert e.iq_push_file(0, str(path), "ishort") == (0, total)
    d, taps = capi.acq_resampler_design(fs, opt)
    assert (d, taps.size) == (10, 49)
    latency = (taps.size - 1) // 2
    acq = ar.make(capi, e, fs // d, doppler_max=5000, doppler_step=100, n_code_slots=32)
    ar.load_codes(acq, [ar.ca_code(gs, p, fs // d) for p in range(1, 33)])
    acq.set_band_resampler(d, taps)
    res = acq.search_band(0, abs_index, np.arange(32))
    c = acq.conf
    th = _threshold(c, pfa)
    detected = [p for p in range(1, 33) if res[p - 1]["test_statistics"] > th]
    assert detected == [sv["prn"] for sv in svs], (detected, th, res["test_statistics"])

    stamp = abs_index + c.consumed_samples * d                         # Acq_samplestamp_samples = rint(sample_count * D)
    ids = []
    for sv in svs:
        r = res[sv["prn"] - 1]
        delay = math.fmod(float(r["index_time"]), float(c.consumed_samples)) * d - latency   # Acq_delay_samples at the full rate
        err = (delay - (sv["delay"] - abs_index) + spc_full / 2) % spc_full - spc_full / 2
        assert abs(err) <= d, (sv, r, delay)
        assert abs(r["doppler"] - sv["doppler"]) <= 150
        ch = e.channel_create(0, 3)
        e.channel_set_code(ch, codes[sv["prn"]], [-0.5, 0.0, 0.5])
        lid = e.loop_create(ch, ol.default_conf(fs_in=fs, prn=sv["prn"], pull_in_time_s=1))
        e.loop_start(lid, delay, float(r["doppler"]), stamp, stamp)
        ids.append(lid)
    rec, cnt = e.loop_run(n_ep)
    for i, sv in enumerate(svs):
        assert cnt[ids[i]] == n_ep, (sv, cnt)
        got = rec[ids[i], :n_ep]
        tail = slice(n_ep - 200, n_ep)
        assert e.loop_status(ids[i]).state == 2, sv
        assert abs(np.mean(got["carrier_doppler_hz"][tail]) - sv["doppler"]) < 3.0, (sv, np.mean(got["carrier_doppler_hz"][tail]))
        assert abs(np.mean(got["CN0_SNV_dB_Hz"][tail]) - sv["cn0"]) < 2.0, (sv, np.mean(got["CN0_SNV_dB_Hz"][tail]))
    acq.close()
    e.close()


def test_four_ms_search_from_a_100_msps_band_past_the_full_rate_plan_limits(capi, engine):
    """400 000 points at 100 Msps exceed every plan, so b200_acq_create refuses the full-rate search; decimated by 50 to
    2 Msps (241 taps) the same 4 ms search is 8 000 points and finds its satellite."""
    fs, opt, prn = 100_000_000, 2_000_000, 11
    sv = dict(prn=prn, doppler=1875.0, delay=61_234, cn0=44.0)
    with pytest.raises(capi.B200Error) as ei:
        ar.make(capi, engine, fs, doppler_max=5000, doppler_step=250, sampled_ms=4, ms_per_code=4)
    assert ei.value.code == ar.ERR_RANGE
    d, taps = capi.acq_resampler_design(fs, opt)
    assert (d, taps.size) == (50, 241)
    acq = ar.make(capi, engine, fs // d, doppler_max=5000, doppler_step=125, sampled_ms=4, ms_per_code=4, n_code_slots=1)
    assert acq.conf.fft_size == 8000
    acq.set_local_code(0, ar.ca_code(gs, prn, fs // d, periods=4))
    acq.set_band_resampler(d, taps)
    abs_index = 1000
    total = abs_index + 4 * (fs // 1000) + 1000
    iq = gs.make_iq({prn: gs.gps_ca_code(prn)}, fs, total, [dict(prn=prn, doppler=sv["doppler"], cn0=sv["cn0"],
                                                                code_phase_chips=(-sv["delay"] * 1.023e6 / fs) % 1023)], seed=37)
    engine.iq_create(10, ar.pow2(total))
    engine.iq_push(10, iq)
    r = acq.search_band(10, abs_index, [0])[0]
    assert r["test_statistics"] > _threshold(acq.conf, 0.001), r
    assert abs(r["doppler"] - sv["doppler"]) <= 125, r
    spc_full = fs // 1000
    delay = math.fmod(float(r["index_time"]), float(acq.conf.consumed_samples)) * d - (taps.size - 1) // 2
    err = (delay - (sv["delay"] - abs_index) + spc_full / 2) % spc_full - spc_full / 2
    assert abs(err) <= d, (r, delay)
    acq.close()
