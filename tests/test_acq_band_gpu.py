"""Acquisition searched straight from a device IQ band (b200_acq_search_band, _band_submit, b200_acq_search_step_two_band).

The band search reads the window [abs_index, abs_index + consumed_samples) where it lies in the band, so its result records
and magnitude grids are byte for byte those of the host-input search on a host copy of the same samples, on every plan
family; it is ordered after the band's pushes without a host synchronisation; windows outside the band are refused before
anything is launched; and it issues exactly the kernels b200_acq_search_dev issues.  The last test is a cold start that
never leaves the device: a sample file pushed into a band once, one 32-PRN sweep from the band, and the device tracking
loops started from its results on the same band.
"""
import math

import numpy as np
import pytest

import gnss_synth as gs
from gpu_fixtures import capi, engine  # noqa: F401
import acq_rig as ar

pytestmark = pytest.mark.gpu

PEAKS, BITS = dict(use_CFAR_algorithm_flag=False), dict(bit_transition_flag=True)


def _push_chunks(engine, band, x, chunk):
    for k in range(0, x.size, chunk):
        engine.iq_push(band, x[k:k + chunk])


# (id, samples per ms, options): every plan family, with the search options each supports
CASES = [
    ("single4000_cfar", 4000, dict()),
    ("single4000_peaks", 4000, PEAKS),
    ("single4000_grid_dwells", 4000, dict(keep_grid=True, max_dwells=2)),
    ("single4000_bits", 4000, BITS),
    ("single4000_zero_padded", 4000, dict(ms_per_code=2)),
    ("single25000_cfar", 25000, dict()),
    ("single25000_peaks_grid", 25000, dict(PEAKS, keep_grid=True)),
    ("two50000_cfar_dwells", 50000, dict(max_dwells=2)),
    ("two50000_peaks", 50000, PEAKS),
    ("two50000_bits", 25000, dict(BITS, **PEAKS)),
    ("two50000_zero_padded", 25000, dict(ms_per_code=2)),
    ("two200000_cfar", 50000, dict(sampled_ms=4, ms_per_code=4)),
    ("two200000_peaks_grid", 50000, dict(PEAKS, sampled_ms=4, ms_per_code=4, keep_grid=True)),
    ("chirpz16368_cfar_dwells", 16368, dict(max_dwells=2)),
    ("chirpz16368_zero_padded", 16368, dict(ms_per_code=2)),
    ("chirpz5456_grid", 5456, dict(keep_grid=True)),
    ("chirpz5456_bits", 5456, BITS),
]


@pytest.mark.parametrize("spms,opts", [c[1:] for c in CASES], ids=[c[0] for c in CASES])
def test_band_search_is_byte_identical_to_host_search(capi, engine, spms, opts):
    """The window straddles the end of an owned ring; every dwell takes the next window."""
    rng = np.random.default_rng(spms + len(opts))
    host, acq, codes = ar.pair(capi, engine, rng, 1000 * spms, **opts)
    c = host.conf
    n, fs, dwells = c.consumed_samples, c.fs_in, c.max_dwells
    cap = ar.pow2(3 * n)
    total = 2 * cap + 2 * n
    x = ar.stream(rng, total, np.resize(codes[1], n), fs)
    engine.iq_create(4, cap)
    _push_chunks(engine, 4, x, cap // 3 + 7)
    idx = 2 * cap - n // 3                     # crosses ring offset 0
    lo, hi = engine.iq_window(4)
    assert lo <= idx and idx + dwells * n <= hi
    for d in range(1, dwells + 1):
        s0 = idx + (d - 1) * n
        want = host.search(x[s0:s0 + n], [1, 0], dwell_counter=d)
        got = acq.search_band(4, s0, [1, 0], dwell_counter=d)
        assert got.tobytes() == want.tobytes(), (d, got, want)
    assert ar.grids(acq) == ar.grids(host)
    host.close()
    acq.close()


def test_windows_at_the_band_edges(capi, engine):
    """A window that ends exactly at write_index, one that starts exactly at the oldest sample still held, one that starts
    exactly at valid_from after a gap push; one sample further is refused."""
    rng = np.random.default_rng(7)
    host, acq, codes = ar.pair(capi, engine, rng, 4e6)
    n = host.conf.consumed_samples
    cap = 16384
    x = ar.stream(rng, 3 * cap + 1000, np.resize(codes[0], n), 4e6)
    engine.iq_create(5, cap)
    _push_chunks(engine, 5, x, 5000)
    lo, hi = engine.iq_window(5)
    assert (lo, hi) == (x.size - cap, x.size)
    for s0 in (hi - n, lo):
        assert acq.search_band(5, s0, [0, 1]).tobytes() == host.search(x[s0:s0 + n], [0, 1]).tobytes(), s0
    for s0 in (hi - n + 1, lo - 1):
        with pytest.raises(capi.B200Error) as ei:
            acq.search_band(5, s0, [0, 1])
        assert ei.value.code == ar.ERR_RANGE
    gap = hi + 12345
    y = ar.stream(rng, 2 * n, np.resize(codes[1], n), 4e6)
    engine.iq_push_at(5, gap, y)
    assert engine.iq_window(5) == (gap, gap + y.size)
    assert acq.search_band(5, gap, [0, 1]).tobytes() == host.search(y[:n], [0, 1]).tobytes()
    host.close()
    acq.close()


@pytest.mark.parametrize("spms", [4000, 16368], ids=["mixed_radix", "chirp_z"])
def test_step_two_from_the_band(capi, engine, spms):
    """Step two on the window after step one's equals b200_acq_search_step_two on a host copy of it."""
    rng = np.random.default_rng(spms)
    host, acq, codes = ar.pair(capi, engine, rng, 1000 * spms, n_code_slots=1)
    c = host.conf
    n, fs = c.consumed_samples, c.fs_in
    cap = ar.pow2(3 * n)
    x = ar.stream(rng, cap + n, np.resize(codes[0], n), fs)
    engine.iq_create(6, cap)
    _push_chunks(engine, 6, x, n // 2 + 3)
    idx = cap - n // 2 - n                     # step one before the ring end, step two across it
    first = host.search(x[idx:idx + n], [0])[0]
    assert acq.search_band(6, idx, [0]).tobytes() == host.search(x[idx:idx + n], [0]).tobytes()
    for a in (host, acq):
        a.set_step_two(float(first["doppler"]), 125.0, 4)
    s1 = idx + n
    want = host.search_step_two(x[s1:s1 + n], 0, float(first["input_power"]))
    got = acq.search_step_two_band(6, s1, 0, float(first["input_power"]))
    assert got.tobytes() == want.tobytes(), (got, want)
    host.close()
    acq.close()


def test_search_is_ordered_after_pushes_without_host_synchronisation(capi, engine):
    """The ring holds PRN A's signal; PRN B's is pushed over the same ring slots (16-bit, 8-bit and float pushes) and searched
    right away, with no sync() in between: the result is B's, byte-equal to the host search of the converted samples."""
    rng = np.random.default_rng(11)
    host, acq, codes = ar.pair(capi, engine, rng, 25e6)
    n, fs = host.conf.consumed_samples, host.conf.fs_in
    cap = ar.pow2(2 * n)
    engine.iq_create(7, cap)
    for rep in range(3):
        for kind in ("i16", "i8", "f32"):
            engine.iq_push(7, 20.0 * ar.stream(rng, cap, np.resize(codes[0], n), fs))   # the ring is A's everywhere
            b = 20.0 * ar.stream(rng, n, codes[1], fs)
            if kind == "f32":
                conv = b.astype(np.complex64)
                first = engine.iq_push(7, conv)
            else:
                dt, lim = (np.int16, 32767) if kind == "i16" else (np.int8, 127)
                raw = ar.to_int(b, dt, clip=(-lim, lim))
                conv = ar.from_int(raw)
                first = engine.iq_push_int(7, raw)
            got = acq.search_band(7, first, [0, 1])
            assert got[1]["test_statistics"] > 3 * got[0]["test_statistics"], (rep, kind, got)   # found B, not A
            assert got.tobytes() == host.search(conv, [0, 1]).tobytes(), (rep, kind)
    host.close()
    acq.close()


def test_attached_band_then_refill(capi, engine):
    """A caller-owned device buffer attached with a non-zero first_index, then refilled from the host at another index."""
    import torch
    rng = np.random.default_rng(13)
    host, acq, codes = ar.pair(capi, engine, rng, 4e6)
    n = host.conf.consumed_samples
    m, first_index = 5 * n + 17, 10_000_000
    x = ar.stream(rng, m, np.resize(codes[0], n), 4e6)
    xt = torch.from_numpy(x.view(np.float32)).cuda()
    torch.cuda.synchronize()
    engine.iq_attach_dev(8, xt.data_ptr(), m, first_index)
    for off in (0, 2 * n + 5, m - n):
        got = acq.search_band(8, first_index + off, [0, 1])
        assert got.tobytes() == host.search(x[off:off + n], [0, 1]).tobytes(), off
    with pytest.raises(capi.B200Error) as ei:
        acq.search_band(8, first_index + m - n + 1, [0, 1])
    assert ei.value.code == ar.ERR_RANGE
    y = ar.stream(rng, 3 * n, np.resize(codes[1], n), 4e6)
    engine.iq_refill_ptr(8, y.ctypes.data, y.size, 77_000)
    assert engine.iq_window(8) == (77_000, 77_000 + y.size)
    for off in (0, 2 * n):
        got = acq.search_band(8, 77_000 + off, [0, 1])
        assert got.tobytes() == host.search(y[off:off + n], [0, 1]).tobytes(), off
    engine.sync()
    del xt
    host.close()
    acq.close()


def test_refusals_launch_nothing(capi, engine):
    rng = np.random.default_rng(17)
    acq = ar.pair(capi, engine, rng, 4e6)[1]
    n = acq.conf.consumed_samples
    cap = 16384
    engine.iq_create(9, cap)
    _push_chunks(engine, 9, ar.stream(rng, 2 * cap, np.zeros(n, np.complex64), 4e6), cap // 2)
    lo, hi = engine.iq_window(9)

    def refused(band, s0, code=ar.ERR_RANGE):
        k0 = engine.launch_count()
        with pytest.raises(capi.B200Error) as ei:
            acq.search_band(band, s0, [0, 1])
        assert ei.value.code == code, str(ei.value)
        assert engine.launch_count() == k0
        if code == ar.ERR_RANGE:
            assert f"[{s0}, {(s0 + n) % 2**64})" in str(ei.value) and f"band {band}" in str(ei.value), str(ei.value)
        return str(ei.value)

    msg = refused(9, hi - n + 1)                                   # past write_index
    assert f"[{lo}, {hi})" in msg
    idx = lo + 100
    acq.search_band(9, idx, [0, 1])                                # valid now ...
    engine.iq_push(9, np.zeros(200, np.complex64))
    refused(9, idx)                                                # ... lapped by a later push
    refused(9, 2**64 - 10)                                         # no wrap-around in the window arithmetic
    engine.iq_forget(9)
    refused(9, engine.iq_window(9)[0] - n)                         # everything before a forget
    w = engine.iq_window(9)[1]
    engine.iq_push_at(9, w + 50_000, np.zeros(2 * n, np.complex64))
    refused(9, w + 50_000 - 1)                                     # before valid_from after a gap
    acq.search_band(9, w + 50_000, [0, 1])
    refused(15, 0, ar.ERR_STATE)                                   # a band nobody created
    refused(16, 0, ar.ERR_ARG)                                     # no such band
    # one search in flight per object
    acq.search_band_submit(9, w + 50_000, [0, 1])
    with pytest.raises(capi.B200Error) as ei:
        acq.search_band_submit(9, w + 50_000, [0, 1])
    assert ei.value.code == ar.ERR_STATE
    with pytest.raises(capi.B200Error) as ei:
        acq.search_step_two_band(9, w + 50_000, 0, 1.0)
    assert ei.value.code == ar.ERR_STATE
    res = acq.search_wait()
    assert res.tobytes() == acq.search_band(9, w + 50_000, [0, 1]).tobytes()
    acq.close()


@pytest.mark.parametrize("spms,opts", [
    (4000, dict()), (4000, PEAKS),
    (50000, dict()), (50000, PEAKS), (50000, dict(PEAKS, keep_grid=True)),
    (16368, dict()),
], ids=["single_cfar", "single_peaks", "two_level_cfar", "two_level_peaks", "two_level_peaks_grid", "chirp_z_cfar"])
def test_band_search_launches_what_search_dev_launches(capi, engine, spms, opts):
    import torch
    rng = np.random.default_rng(19)
    acq = ar.pair(capi, engine, rng, 1000 * spms, **opts)[1]
    n = acq.conf.consumed_samples
    x = ar.stream(rng, n, np.zeros(n, np.complex64), acq.conf.fs_in)
    engine.iq_create(10, ar.pow2(n))
    engine.iq_push(10, x)
    xt = torch.from_numpy(x.view(np.float32)).cuda()
    res = torch.zeros(2 * capi.ACQ_RESULT_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    k0 = engine.launch_count()
    acq.search_dev(xt.data_ptr(), [0, 1], res.data_ptr())
    k1 = engine.launch_count()
    got = acq.search_band(10, 0, [0, 1])
    k2 = engine.launch_count()
    assert k2 - k1 == k1 - k0 > 0
    engine.sync()
    torch.cuda.synchronize()
    assert got.tobytes() == res.cpu().numpy().tobytes()
    acq.close()


# ---- cold start on the device ------------------------------------------------------------------------------------------
def test_cold_start_from_a_pushed_file_into_device_loops(capi, tmp_path):
    """GPS L1 C/A at 4 Msps written as an ishort file and pushed into a band once; PRNs 1-32 swept from the band in one call
    and judged against the reference's CFAR threshold; a device loop started for each detection from the acquisition result
    (code phase, Doppler, sample stamp abs_index + consumed_samples) tracks its satellite on the same band."""
    from scipy.special import gammaincinv
    from oracle import loop as ol
    fs, spms, n_ep, pfa, scale = 4e6, 4000, 1000, 0.001, 64.0
    # 46-48 dB-Hz: with one 1 ms dwell the reference's threshold (pfa 1e-3 over 4000 x 100 cells) is a statistic of 46; a
    # satellite at 46 dB-Hz peaks near 80 on average, the strongest absent PRN of this seed reaches 35
    svs = [dict(prn=2, doppler=-2730.0, delay=311, cn0=47.0), dict(prn=7, doppler=1410.0, delay=1777, cn0=46.0),
           dict(prn=13, doppler=3125.0, delay=2950, cn0=46.5), dict(prn=19, doppler=-620.0, delay=3433, cn0=47.0),
           dict(prn=24, doppler=215.0, delay=95, cn0=47.5), dict(prn=30, doppler=-4180.0, delay=2204, cn0=48.0)]
    abs_index = 1234
    total = abs_index + spms + (n_ep + 3) * spms
    codes = {sv["prn"]: gs.gps_ca_code(sv["prn"]) for sv in svs}
    iq = gs.make_iq(codes, fs, total, [dict(prn=sv["prn"], doppler=sv["doppler"], cn0=sv["cn0"],
                                            code_phase_chips=(-sv["delay"] * 1.023e6 / fs) % 1023) for sv in svs], seed=29)
    raw = ar.to_int(iq, np.int16, scale, clip=(-32767, 32767))
    path = tmp_path / "gps_l1_4msps.ishort"
    raw.tofile(path)
    del iq, raw

    e = capi.Engine(0)
    e.iq_create(0, total)
    first, pushed = e.iq_push_file(0, str(path), "ishort")
    assert (first, pushed) == (0, total)
    acq = ar.make(capi, e, fs, doppler_max=5000, doppler_step=100, n_code_slots=32)
    ar.load_codes(acq, [ar.ca_code(gs, p, fs) for p in range(1, 33)])
    res = acq.search_band(0, abs_index, np.arange(32))
    c = acq.conf
    th = 2.0 * gammaincinv(2.0, (1.0 - pfa) ** (1.0 / (c.effective_fft_size * c.num_doppler_bins)))
    detected = [p for p in range(1, 33) if res[p - 1]["test_statistics"] > th]
    assert detected == [sv["prn"] for sv in svs], (detected, th, res["test_statistics"])

    stamp = abs_index + c.consumed_samples                          # Acq_samplestamp_samples, also nitems_read
    ids = []
    for sv in svs:
        r = res[sv["prn"] - 1]
        ch = e.channel_create(0, 3)
        e.channel_set_code(ch, codes[sv["prn"]], [-0.5, 0.0, 0.5])
        lid = e.loop_create(ch, ol.default_conf(fs_in=fs, prn=sv["prn"], pull_in_time_s=1))
        e.loop_start(lid, math.fmod(float(r["index_time"]), float(spms)), float(r["doppler"]), stamp, stamp)
        assert abs(r["doppler"] - sv["doppler"]) <= 150            # a 1 ms peak spans several 100 Hz bins
        assert abs(int(r["index_time"]) - (sv["delay"] - abs_index) % spms) <= 1
        ids.append(lid)
    rec, cnt = e.loop_run(n_ep)
    items = e.loop_peek_items()
    for i, sv in enumerate(svs):
        assert cnt[ids[i]] == n_ep, (sv, cnt)
        got = rec[ids[i], :n_ep]
        tail = slice(n_ep - 300, n_ep)
        assert e.loop_status(ids[i]).state == 2, sv
        assert abs(np.mean(got["carrier_doppler_hz"][tail]) - sv["doppler"]) < 3.0, (sv, np.mean(got["carrier_doppler_hz"][tail]))
        assert abs(np.mean(got["CN0_SNV_dB_Hz"][tail]) - sv["cn0"]) < 2.0, (sv, np.mean(got["CN0_SNV_dB_Hz"][tail]))
        # code phase of the next epoch against the truth (the item carries minus the local code phase at its first sample)
        it = items[ids[i]]
        rate = gs.CA_RATE * (1.0 + sv["doppler"] / gs.GPS_L1_FREQ)
        truth = ((-sv["delay"] * 1.023e6 / fs) + float(it["sample_index"]) * rate / fs) % 1023.0
        err = (-float(it["rem_code_phase_chips"]) - truth + 511.5) % 1023.0 - 511.5
        assert abs(err) < 0.1, (sv, err)
    acq.close()
    e.close()
