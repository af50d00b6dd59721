"""The signal conditioner on the device (b200_iq_set_conditioner): every push into a source band fills a destination band with
the frequency-translating decimating FIR of gr::filter::freq_xlating_fir_filter_ccf, in absolute stream indices.

Read back with b200_iq_read, the destination is byte for byte the float32 restatement (iq_conditioner_np) at IF = 0 for every
source type, decimation and tap count, push by push across the ring's end; at IF != 0 it is within two float ulps of that
restatement and within the float32 loop's rounding bound of the float64 truth, at output indices past 2^32 and 2^40.  One
push and many give the same bytes; the destination's window follows the source's through stream start, a push_at gap, a
forget and a conditioner set mid-stream; a band search and a batch issued right after a push read the new outputs; a push
launches what it launched before plus one kernel per conditioner with new outputs, and every refusal launches nothing.  End
to end, a 25 Msps ibyte stream conditioned to 5 Msps is acquired and tracked by the device loops exactly as the same loops
track the restatement's output, and at an IF they follow the loops fed with the float64 truth."""
import math

import numpy as np
import pytest

import acq_rig as ar
import gnss_synth as gs
import iq_conditioner_np as cnp
from gpu_fixtures import capi, engine  # noqa: F401

pytestmark = pytest.mark.gpu

ERR_ARG, ERR_STATE, ERR_RANGE = -1, -4, -5
FS = 25e6


def _stream(rng, n, item_type):
    """n samples of item_type -> (what a push takes, the complex64 samples the band holds)"""
    if item_type == "gr_complex":
        x = (rng.normal(0, 300, n) + 1j * rng.normal(0, 300, n)).astype(np.complex64)
        return x, x
    dt, lim = (np.int16, 3000) if item_type == "ishort" else (np.int8, 127)
    raw = rng.integers(-lim, lim + 1, 2 * n).astype(dt)
    return raw, ar.from_int(raw)


def _push(e, band, raw, item_type, a, b):
    """samples [a, b) of raw into band"""
    if item_type == "gr_complex":
        return e.iq_push(band, raw[a:b])
    return e.iq_push_int(band, raw[2 * a:2 * b])


@pytest.mark.parametrize("t", [1, 17, 48, 301])
@pytest.mark.parametrize("d", [1, 2, 5, 10])
@pytest.mark.parametrize("item_type", ["gr_complex", "ishort", "ibyte"])
def test_if_zero_is_bit_exact_push_by_push(engine, item_type, d, t):
    """odd push sizes that are not multiples of D, three times around a 4096-sample source ring; 301 taps span more
    samples than a CTA's run of 128 outputs"""
    rng = np.random.default_rng(100 * d + t)
    cap = 1 << 12
    h = rng.normal(0, 0.1, t).astype(np.float32)
    engine.iq_create(0, cap, item_type)
    engine.iq_create(1, cnp.ceil_div(cap, d))
    engine.iq_set_conditioner(1, 0, d, h, 0.0, FS)
    total = 3 * cap + 123
    raw, held = _stream(rng, total, item_type)
    limit = cap - (t - 1)
    pos = 0
    while pos < total:
        n = min(int(rng.integers(1, limit // 2)) | 1, total - pos)
        if n % d == 0 and d > 1:
            n -= 1 if n > 1 else -1
        _push(engine, 0, raw, item_type, pos, pos + n)
        j0, j1 = cnp.ceil_div(pos, d), cnp.ceil_div(pos + n, d)
        pos += n
        lo, hi = engine.iq_window(1)
        assert hi == j1 and lo <= j0, (lo, hi, j0, j1)
        if j1 > j0:
            got = engine.iq_read(1, j0, j1 - j0)
            want = cnp.condition_f32(held, 0, h, d, 0.0, FS, j0, j1 - j0)
            assert got.tobytes() == want.tobytes(), (pos, np.flatnonzero(got != want)[:5])


def _ulps(got, want):
    """per component |got - want| in units of the float32 spacing at |want|"""
    sp = np.spacing(np.abs(want).astype(np.float32)).astype(np.float64)
    return np.maximum(np.abs(got.real - want.real), np.abs(got.imag - want.imag)) / sp


@pytest.mark.parametrize("j_start", [(1 << 32) + 777, (1 << 40) - 5000], ids=["past_2_32", "near_2_40"])
@pytest.mark.parametrize("if_hz", [2.1e6, -3.3e6])
def test_if_nonzero_past_2_32(capi, engine, if_hz, j_start):
    """the stream starts at a push_at far into the stream, so every output index is past 2^32 (the second case reaches
    2^40); error bound of the float64 truth: (T + 4) 2^-23 sum_k |c[k]| |x[jD - k]|, the float32 loop's rounding"""
    rng = np.random.default_rng(7)
    d = 5
    h = capi.iq_conditioner_lowpass(FS, d)
    t = h.size
    engine.iq_create(2, 1 << 16)
    engine.iq_create(3, 1 << 14)
    engine.iq_set_conditioner(3, 2, d, h, if_hz, FS)
    x0 = j_start * d - (t - 1) - 3
    x, _ = _stream(rng, 40_000, "gr_complex")
    assert engine.iq_push_at(2, x0, x[:10_001]) == 10_001
    engine.iq_push(2, x[10_001:])
    lo, hi = engine.iq_window(3)
    assert (lo, hi) == (cnp.ceil_div(x0 + t - 1, d), cnp.ceil_div(x0 + x.size, d)) and lo == j_start
    got = engine.iq_read(3, lo, hi - lo)
    want = cnp.condition_f32(x, x0, h, d, if_hz, FS, lo, hi - lo)
    assert np.max(_ulps(got, want)) <= 2.0
    truth, scale = cnp.condition_f64(x, x0, h, d, if_hz, FS, lo, hi - lo)
    assert np.all(np.abs(got - truth) <= (t + 4) * 2.0 ** -23 * scale)


@pytest.mark.parametrize("if_hz", [0.0, 1.7e6])
@pytest.mark.parametrize("item_type", ["gr_complex", "ibyte"])
def test_one_push_and_many_give_the_same_bytes(capi, engine, item_type, if_hz):
    rng = np.random.default_rng(11)
    d, cap = 5, 1 << 16
    h = capi.iq_conditioner_lowpass(FS, d)
    raw, _ = _stream(rng, cap - (h.size - 1), item_type)
    n = raw.size if item_type == "gr_complex" else raw.size // 2
    for src, dst in ((4, 5), (6, 7)):
        engine.iq_create(src, cap, item_type)
        engine.iq_create(dst, cap // d + 1)
        engine.iq_set_conditioner(dst, src, d, h, if_hz, FS)
    _push(engine, 4, raw, item_type, 0, n)
    pos = 0
    while pos < n:
        k = min(int(rng.integers(1, 700)), n - pos)
        _push(engine, 6, raw, item_type, pos, pos + k)
        pos += k
    assert engine.iq_window(5) == engine.iq_window(7) == (0, cnp.ceil_div(n, d))
    m = cnp.ceil_div(n, d)
    assert engine.iq_read(5, 0, m).tobytes() == engine.iq_read(7, 0, m).tobytes()


def test_destination_window_follows_the_source(capi, engine):
    e = engine
    rng = np.random.default_rng(13)
    d, t, cap = 4, 9, 1 << 12
    h = np.full(t, 1.0 / t, np.float32)
    x, _ = _stream(rng, 20_000, "gr_complex")
    e.iq_create(0, cap)
    e.iq_create(1, cap)
    e.iq_set_conditioner(1, 0, d, h, 0.0, FS)
    assert e.iq_window(1) == (0, 0)                                       # stream start

    def check_data(band, x0, a, b):
        lo, hi = e.iq_window(band)
        assert e.iq_read(band, lo, hi - lo).tobytes() == cnp.condition_f32(x[x0:b], x0, h, d, 0.0, FS, lo, hi - lo).tobytes()

    e.iq_push(0, x[:1001])
    assert e.iq_window(1) == (0, 251)
    check_data(1, 0, 0, 1001)
    g = 1501                                                               # push_at gap
    assert e.iq_push_at(0, g, x[g:g + 2001]) == 2001
    w = g + 2001
    assert e.iq_window(0) == (g, w)
    assert e.iq_window(1) == (cnp.ceil_div(g + t - 1, d), cnp.ceil_div(w, d))
    check_data(1, g, g, w)
    e.iq_forget(0)                                                         # forget on the source: empty until T - 1 more
    assert e.iq_window(1) == (cnp.ceil_div(w, d), cnp.ceil_div(w, d))
    e.iq_push(0, x[w:w + 1003])
    w2 = w + 1003
    assert e.iq_window(1) == (cnp.ceil_div(w + t - 1, d), cnp.ceil_div(w2, d))
    check_data(1, w, w, w2)
    e.iq_create(2, cap)                                                    # set mid-stream: starts empty at ceil(w / D)
    e.iq_set_conditioner(2, 0, d, h, 0.0, FS)
    assert e.iq_window(2) == (cnp.ceil_div(w2, d),) * 2
    e.iq_forget(1)                                                         # forget on a destination: a floor of its own
    f1 = cnp.ceil_div(w2, d)
    assert e.iq_window(1) == (f1, f1)
    k0 = e.launch_count()
    e.iq_push(0, x[w2:w2 + 777])
    w3 = w2 + 777
    e.sync()
    assert e.launch_count() - k0 == 2
    assert e.iq_window(2) == (cnp.ceil_div(w2, d), cnp.ceil_div(w3, d))
    assert e.iq_window(1) == (f1, cnp.ceil_div(w3, d))
    check_data(2, w, w2, w3)
    check_data(1, w, w2, w3)
    # removal, and re-creation of the destination: pushes launch nothing for them, their windows stay
    e.iq_remove_conditioner(2)
    e.iq_create(1, cap)
    wins = (e.iq_window(1), e.iq_window(2))
    k0 = e.launch_count()
    e.iq_push(0, x[w3:w3 + 500])
    e.sync()
    assert e.launch_count() == k0 and (e.iq_window(1), e.iq_window(2)) == wins == ((0, 0), (cnp.ceil_div(w2, d), cnp.ceil_div(w3, d)))
    e.iq_push(2, x[:10])                                                   # an ordinary band again
    # re-creating the source removes its conditioners
    e.iq_set_conditioner(1, 0, d, h, 0.0, FS)
    e.iq_create(0, cap)
    k0 = e.launch_count()
    e.iq_push(0, x[:100])
    e.sync()
    assert e.launch_count() == k0 and e.iq_window(1) == (cnp.ceil_div(w3 + 500, d),) * 2


def test_search_and_batch_right_after_a_push_read_the_new_outputs(capi, engine):
    """no host synchronisation between the push and the band search or the batch; then repeated pushes of the largest
    size into a conditioned source, read back only at the end: every output is intact"""
    rng = np.random.default_rng(17)
    e = engine
    d, fs = 5, 25_000_000
    h = capi.iq_conditioner_lowpass(fs, d)
    acq, host, codes = ar.pair(capi, e, rng, fs // d)
    n = host.conf.consumed_samples
    total = 4 * n * d
    x = ar.stream(rng, total, np.repeat(codes[1][:n], d), fs)
    e.iq_create(8, ar.pow2(total))
    e.iq_create(9, ar.pow2(total // d))
    e.iq_set_conditioner(9, 8, d, h, 0.0, fs)
    e.iq_push(8, x)
    got = acq.search_band(9, 1000, [1, 0])
    y = cnp.condition_f32(x, 0, h, d, 0.0, fs, 1000, n)
    want = host.search(y, [1, 0])
    assert got.tobytes() == want.tobytes()
    assert got[0]["test_statistics"] > got[1]["test_statistics"]
    # a batch on the conditioned band against the same batch on a band pushed with the restatement's output; the
    # channels are set up first (setting a code table synchronises), the batch follows the push that makes its samples
    m2 = total // d + 777
    yy = cnp.condition_f32(np.concatenate([x, x[:d * 777]]), 0, h, d, 0.0, fs, 0, m2)
    e.iq_create(10, ar.pow2(m2))
    e.iq_push(10, yy)
    items = {}
    for band in (9, 10):
        ch = e.channel_create(band, 3)
        e.channel_set_code(ch, gs.gps_ca_code(3), [-0.5, 0.0, 0.5])
        it = np.zeros(8, capi.TRK_ITEM_DTYPE)
        it["channel"] = ch
        it["n"] = 5000
        it["sample_index"] = m2 - 5000 - 97 * np.arange(8)
        it["phase_step_rad"] = 2 * np.pi * 1234.0 / (fs / d)
        it["code_phase_step_chips"] = 1.023e6 / (fs / d)
        items[band] = it
    e.iq_push(8, x[:d * 777])                                              # the outputs [m2 - 777, m2) the batch reads
    got = e.trk_batch(items[9], 3)
    assert got.tobytes() == e.trk_batch(items[10], 3).tobytes()
    # repeated pushes of the largest size: the next copy into the source waits for the launch that reads it
    cap = 1 << 14
    e.iq_create(11, cap)
    e.iq_create(12, 1 << 16)
    e.iq_set_conditioner(12, 11, d, h, 0.0, fs)
    big = cap - (h.size - 1)
    xs, _ = _stream(rng, 12 * big, "gr_complex")
    for k in range(12):
        e.iq_push(11, xs[k * big:(k + 1) * big])
    m = cnp.ceil_div(xs.size, d)
    assert e.iq_window(12) == (0, m)
    assert e.iq_read(12, 0, m).tobytes() == cnp.condition_f32(xs, 0, h, d, 0.0, fs, 0, m).tobytes()
    acq.close()
    host.close()


def test_push_launches_and_refusals(capi, engine, tmp_path):
    e = engine
    rng = np.random.default_rng(19)
    cap = 1 << 12
    h = np.full(9, 1.0 / 9, np.float32)
    x, _ = _stream(rng, 3 * cap, "gr_complex")
    raw16 = rng.integers(-100, 100, 2 * cap).astype(np.int16)
    raw8 = rng.integers(-100, 100, 2 * cap).astype(np.int8)
    for b in (0, 1, 2):
        e.iq_create(b, cap)
    e.iq_create(3, cap, "ibyte")
    e.iq_create(4, cap // 4)
    e.iq_create(5, cap // 4)

    def pushed(call):
        k0 = e.launch_count()
        call()
        e.sync()
        return e.launch_count() - k0

    assert pushed(lambda: e.iq_push(0, x[:100])) == 0                     # as before: a copy, no kernel
    assert pushed(lambda: e.iq_push_int(0, raw16[:200])) == 1              # as before: the conversion
    e.iq_set_conditioner(1, 0, 4, h, 0.0, FS)
    assert pushed(lambda: e.iq_push(0, x[:100])) == 1
    e.iq_set_conditioner(2, 0, 2, h, 1.0e6, FS)
    assert pushed(lambda: e.iq_push(0, x[:100])) == 2
    assert pushed(lambda: e.iq_push_int(0, raw16[:202])) == 3              # conversion + two conditioners
    w = e.iq_window(0)[1]
    assert w == 501                                                        # odd: one more sample completes no output
    assert pushed(lambda: e.iq_push(0, x[:1])) == 0
    assert pushed(lambda: e.iq_push_at(0, w + 1, x[:5])) == 2
    e.iq_set_conditioner(4, 3, 4, h, 0.0, FS)                             # an ibyte source
    assert pushed(lambda: e.iq_push_int(3, raw8[:200])) == 1

    def refused(call, code):
        wins = [e.iq_window(b) for b in range(6)]
        k0 = e.launch_count()
        with pytest.raises(capi.B200Error) as ei:
            call()
        assert ei.value.code == code, str(ei.value)
        e.sync()
        assert e.launch_count() == k0 and [e.iq_window(b) for b in range(6)] == wins
        return str(ei.value)

    t = np.ascontiguousarray(h)
    set_ = capi.lib.b200_iq_set_conditioner

    def raw_set(dst, src, dd, ptr, nt, if_hz, fs):
        return lambda: capi._chk(set_(e.h, dst, src, dd, ptr, nt, if_hz, fs), "b200_iq_set_conditioner")

    big = np.zeros(capi.B200_IQ_MAX_CONDITIONER_TAPS + 1, np.float32)
    refused(raw_set(5, 0, 0, t.ctypes.data, t.size, 0.0, FS), ERR_ARG)           # decimation < 1
    refused(raw_set(5, 0, 4, None, t.size, 0.0, FS), ERR_ARG)                    # no taps
    refused(raw_set(5, 0, 4, big.ctypes.data, big.size, 0.0, FS), ERR_RANGE)     # too many taps
    refused(raw_set(5, 0, capi.B200_IQ_MAX_CONDITIONER_DECIMATION + 1, t.ctypes.data, t.size, 0.0, FS), ERR_RANGE)
    for fs in (0.0, -FS, float("nan"), float("inf")):
        refused(raw_set(5, 0, 4, t.ctypes.data, t.size, 0.0, fs), ERR_ARG)       # fs <= 0 or not finite
    refused(raw_set(5, 0, 4, t.ctypes.data, t.size, float("inf"), FS), ERR_ARG)
    refused(raw_set(0, 0, 4, t.ctypes.data, t.size, 0.0, FS), ERR_ARG)           # dst == src
    refused(raw_set(3, 0, 4, t.ctypes.data, t.size, 0.0, FS), ERR_STATE)         # narrow destination
    refused(raw_set(5, 0, 2, t.ctypes.data, t.size, 0.0, FS), ERR_RANGE)         # 1024 x 2 < 4096: too small
    refused(raw_set(5, 1, 4, t.ctypes.data, t.size, 0.0, FS), ERR_STATE)         # a destination as source
    refused(raw_set(0, 5, 4, t.ctypes.data, t.size, 0.0, FS), ERR_STATE)         # a source as destination
    refused(raw_set(5, 13, 4, t.ctypes.data, t.size, 0.0, FS), ERR_STATE)        # an unused band
    import torch
    buf = torch.zeros(2 * cap, dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    e.iq_attach_dev(14, buf.data_ptr(), cap)
    refused(raw_set(5, 14, 4, t.ctypes.data, t.size, 0.0, FS), ERR_STATE)        # attached source
    refused(raw_set(14, 0, 1, t.ctypes.data, t.size, 0.0, FS), ERR_STATE)        # attached destination
    # while set: direct writes into a destination, and pushes into a source larger than capacity - (T - 1)
    refused(lambda: e.iq_push(1, x[:10]), ERR_STATE)
    refused(lambda: e.iq_push_int(1, raw16[:20]), ERR_STATE)
    refused(lambda: e.iq_push_at(1, e.iq_window(1)[1] + 5, x[:10]), ERR_STATE)
    path = tmp_path / "x.bin"
    x[:100].tofile(path)
    refused(lambda: e.iq_push_file(1, str(path), "gr_complex"), ERR_STATE)
    msg = refused(lambda: e.iq_push(0, x[:cap - 7]), ERR_RANGE)
    assert f"at most {cap - 8}" in msg, msg
    assert pushed(lambda: e.iq_push(0, x[:cap - 8])) == 2
    refused(lambda: e.iq_read(0, 0, 10), ERR_RANGE)                              # outside the window
    refused(lambda: e.iq_read(15, 0, 0), ERR_STATE)
    e.iq_create(14, cap)


def _ibyte_stream(svs, fs, total, seed, if_hz=0.0):
    """GPS L1 C/A satellites in unit noise at fs, moved to if_hz, as interleaved ibyte (x 20)"""
    codes = {sv["prn"]: gs.gps_ca_code(sv["prn"]) for sv in svs}
    iq = gs.make_iq(codes, fs, total, [dict(prn=sv["prn"], doppler=sv["doppler"], cn0=sv["cn0"],
                                            code_phase_chips=(-sv["delay"] * 1.023e6 / fs) % 1023) for sv in svs], seed=seed)
    if if_hz:
        iq = iq * np.exp(2j * np.pi * (if_hz / fs) * np.arange(total))
    return codes, ar.to_int(iq, np.int8, 20.0, clip=(-127, 127))


def _conditioned_and_plain(capi, fs, d, raw, h, if_hz, plain):
    """engine with the ibyte stream in band 0, conditioned into band 1, and `plain` (complex64 at fs / d) in band 2"""
    e = capi.Engine(0)
    n = raw.size // 2
    e.iq_create(0, 1 << 20, "ibyte")
    e.iq_create(1, ar.pow2(n // d + 1))
    e.iq_create(2, ar.pow2(n // d + 1))
    e.iq_set_conditioner(1, 0, d, h, if_hz, fs)
    chunk = 1 << 19
    for a in range(0, n, chunk):
        e.iq_push_int(0, raw[2 * a:2 * min(n, a + chunk)])
    e.iq_push(2, plain)
    assert e.iq_window(1) == e.iq_window(2) == (0, plain.size)
    return e


def _acquire_and_start(capi, e, sv, codes, fs_d, bands, conf):
    """acquire sv on each band (the records must agree) and start one loop per band from the result"""
    acq = ar.make(capi, e, fs_d, doppler_max=5000, doppler_step=100, n_code_slots=1)
    acq.set_local_code(0, ar.ca_code(gs, sv["prn"], fs_d))
    abs_index = 1000
    res = [acq.search_band(b, abs_index, [0])[0] for b in bands]
    assert all(r.tobytes() == res[0].tobytes() for r in res)
    r = res[0]
    spc = fs_d // 1000
    delay = math.fmod(float(r["index_time"]), float(acq.conf.consumed_samples))
    assert abs(r["doppler"] - sv["doppler"]) <= 100, r
    latency = sv["latency"]
    err = (delay - (sv["delay"] - abs_index) - latency + spc / 2) % spc - spc / 2
    assert abs(err) <= 2, (r, delay)
    stamp = abs_index + acq.conf.consumed_samples
    ids = []
    for b in bands:
        ch = e.channel_create(b, 3)
        e.channel_set_code(ch, codes[sv["prn"]], [-0.5, 0.0, 0.5])
        lid = e.loop_create(ch, conf)
        e.loop_start(lid, delay, float(r["doppler"]), stamp, stamp)
        ids.append(lid)
    acq.close()
    return ids


def test_ibyte_25_msps_conditioned_stream_is_acquired_and_tracked_as_its_restatement(capi):
    """a 25 Msps ibyte band conditioned into a gr_complex band at D = 5 (241-tap default low-pass); the band search finds
    the satellite, and the device loops on it write, in all three loop modes, the very dump records of the same loops on a
    band pushed with the restatement's output"""
    from oracle import loop as ol
    fs, d, n_ep = 25_000_000, 5, 500
    fs_d = fs // d
    h = capi.iq_conditioner_lowpass(fs, d)
    assert h.size == 241
    sv = dict(prn=7, doppler=1830.0, delay=2345, cn0=50.0, latency=(h.size - 1) // 2 / d)
    total = (1000 + (n_ep + 8) * (fs_d // 1000)) * d
    codes, raw = _ibyte_stream([dict(sv, delay=sv["delay"] * d)], fs, total, seed=41)
    y = cnp.condition_f32(ar.from_int(raw), 0, h, d, 0.0, fs, 0, cnp.ceil_div(total, d))
    for mode in (0, 1, 2):
        e = _conditioned_and_plain(capi, fs, d, raw, h, 0.0, y)
        e.loop_set_mode(mode)
        ids = _acquire_and_start(capi, e, sv, codes, fs_d, (1, 2), ol.default_conf(fs_in=fs_d, prn=sv["prn"], pull_in_time_s=1))
        rec, cnt = e.loop_run(n_ep)
        assert cnt[ids[0]] == cnt[ids[1]] >= n_ep - 2, (mode, cnt)
        k = cnt[ids[0]]
        assert rec[ids[0], :k].tobytes() == rec[ids[1], :k].tobytes(), mode
        assert e.loop_status(ids[0]).state == 2
        assert abs(np.mean(rec[ids[0], k - 100:k]["carrier_doppler_hz"]) - sv["doppler"]) < 5.0
        e.close()


def test_conditioned_stream_at_an_if_follows_the_float64_truth(capi):
    """the same satellite 1.2 MHz above baseband, moved down by the conditioner: the loops hold lock and follow the loops
    fed with the float64 truth within the closed-loop tolerance of the loop tests"""
    from oracle import loop as ol
    fs, d, n_ep, if_hz = 25_000_000, 5, 500, 1.2e6
    fs_d = fs // d
    h = capi.iq_conditioner_lowpass(fs, d)
    sv = dict(prn=7, doppler=1830.0, delay=2345, cn0=50.0, latency=(h.size - 1) // 2 / d)
    total = (1000 + (n_ep + 8) * (fs_d // 1000)) * d
    codes, raw = _ibyte_stream([dict(sv, delay=sv["delay"] * d)], fs, total, seed=43, if_hz=if_hz)
    truth, _ = cnp.condition_f64(ar.from_int(raw), 0, h, d, if_hz, fs, 0, cnp.ceil_div(total, d))
    e = _conditioned_and_plain(capi, fs, d, raw, h, if_hz, truth.astype(np.complex64))
    conf = ol.default_conf(fs_in=fs_d, prn=sv["prn"], pull_in_time_s=1)
    ids = _acquire_and_start_loose(capi, e, sv, codes, fs_d, conf)
    rec, cnt = e.loop_run(n_ep)
    assert cnt[ids[0]] >= n_ep - 2 and cnt[ids[1]] >= n_ep - 2, cnt
    k = min(cnt[ids[0]], cnt[ids[1]])
    got, want = rec[ids[0], :k], rec[ids[1], :k]
    for lid in ids:
        assert e.loop_status(lid).state == 2
    assert abs(np.mean(got["carrier_doppler_hz"][k - 100:]) - sv["doppler"]) < 5.0
    assert np.max(np.abs(got["carrier_doppler_hz"] - want["carrier_doppler_hz"])) < 0.7
    assert np.max(np.abs(got["aux1"] - want["aux1"])) < 5e-2
    stamp_diff = got["PRN_start_sample_count"].astype(np.int64) - want["PRN_start_sample_count"].astype(np.int64)
    assert np.max(np.abs(stamp_diff)) <= 1
    same = (stamp_diff == 0) & (np.roll(stamp_diff, 1) == 0)
    assert same.mean() > 0.9
    assert np.max(np.abs(got["abs_P"][same] - want["abs_P"][same])) < 2e-2 * np.mean(want["abs_P"])
    e.close()


def _acquire_and_start_loose(capi, e, sv, codes, fs_d, conf):
    """as _acquire_and_start, but the two bands differ in their last bits: each loop starts from its own band's search,
    which must agree on the cell"""
    acq = ar.make(capi, e, fs_d, doppler_max=5000, doppler_step=100, n_code_slots=1)
    acq.set_local_code(0, ar.ca_code(gs, sv["prn"], fs_d))
    abs_index = 1000
    ids = []
    cells = []
    for b in (1, 2):
        r = acq.search_band(b, abs_index, [0])[0]
        cells.append((int(r["index_time"]), int(r["index_doppler"])))
        assert abs(r["doppler"] - sv["doppler"]) <= 100, r
        delay = math.fmod(float(r["index_time"]), float(acq.conf.consumed_samples))
        ch = e.channel_create(b, 3)
        e.channel_set_code(ch, codes[sv["prn"]], [-0.5, 0.0, 0.5])
        lid = e.loop_create(ch, conf)
        stamp = abs_index + acq.conf.consumed_samples
        e.loop_start(lid, delay, float(r["doppler"]), stamp, stamp)
        ids.append(lid)
    assert cells[0] == cells[1]
    acq.close()
    return ids
