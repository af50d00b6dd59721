"""The pulse blanker on the device (b200_iq_set_pulse_blanking): every push into a source band fills a destination band with
pulse_blanking_cc's output, in absolute stream indices.

Read back with b200_iq_read, the destination is byte for byte the float32 restatement (pulse_blanking_np) for every source
type and segment length, push by push across the ring's end and through several estimation / detection / reset cycles, and
the compiled reference block on the prefix it publishes; the status is the restatement's state after every push.  One push
and many give the same bytes; the origin and window follow the stream start, a blanker set mid-stream, a push_at gap and a
forget on either band; a conditioner followed by a blanker is the restatement applied to the conditioner's output; a band
search right after a push reads the blanked samples; a push launches three kernels per blanker with new segments, and every
refusal launches nothing.  End to end, a GPS L1 C/A stream hit by strong pulse pairs is acquired better on the destination
than on the raw band, and tracked by the device loops exactly as on the restatement's output."""
import math

import numpy as np
import pytest

import acq_rig as ar
import gnss_synth as gs
import pulse_blanking_np as pnp
from gpu_fixtures import capi, engine  # noqa: F401

pytestmark = pytest.mark.gpu

ERR_ARG, ERR_STATE, ERR_RANGE = -1, -4, -5


def _pulsed(rng, n, item_type, pulse_every=1500):
    """n samples of complex noise with strong pulse pairs (12 us apart at 4 Msps, 40 samples each) about every
    pulse_every samples -> (what a push of item_type takes, the complex64 samples the band holds)"""
    sigma = 12.0 if item_type == "ibyte" else 300.0
    x = (rng.normal(0, sigma / math.sqrt(2), n) + 1j * rng.normal(0, sigma / math.sqrt(2), n)).astype(np.complex128)
    w = np.exp(-0.5 * ((np.arange(40) - 20) / 6.0) ** 2) * 8.0 * sigma
    for start in rng.integers(0, max(1, n - 100), max(1, n // pulse_every)):
        for off in (0, 48):
            seg = x[start + off:start + off + 40]
            seg += w[:seg.size] * np.exp(1j * rng.uniform(0, 2 * np.pi))
    if item_type == "gr_complex":
        x = x.astype(np.complex64)
        return x, x
    dt, lim = (np.int16, 32767) if item_type == "ishort" else (np.int8, 127)
    raw = ar.to_int(x, dt, 1.0, clip=(-lim, lim))
    return raw, ar.from_int(raw)


def _push(e, band, raw, item_type, a, b):
    """samples [a, b) of raw into band"""
    if item_type == "gr_complex":
        return e.iq_push(band, raw[a:b])
    return e.iq_push_int(band, raw[2 * a:2 * b])


def _check_status(e, band, ref, origin):
    st = e.iq_pulse_blanking_status(band)
    assert st["origin"] == origin
    assert np.float32(st["threshold"]) == ref.thres and st["length"] == ref.length
    for k, v in ref.state().items():
        if k == "noise_power":
            assert np.float32(st[k]).tobytes() == v.tobytes(), (k, st[k], v)
        else:
            assert st[k] == v, (k, st, ref.state())


@pytest.mark.parametrize("length", [1, 7, 32, 301])
@pytest.mark.parametrize("item_type", ["gr_complex", "ishort", "ibyte"])
def test_bit_exact_push_by_push(capi, engine, item_type, length):
    """odd push sizes three times around a 4096-sample source ring, with E and R small enough for several estimation,
    detection and reset cycles; the status after every push; and the compiled block on the prefix it publishes"""
    e = engine
    rng = np.random.default_rng(1000 * length + len(item_type))
    cap = 1 << 12
    total = 3 * cap + 123
    segs = total // length
    est, reset = segs // 20 + 1, segs // 8
    e.iq_create(0, cap, item_type)
    e.iq_create(1, cap)
    e.iq_set_pulse_blanking(1, 0, 0.04, length, est, reset)
    raw, held = _pulsed(rng, total, item_type)
    ref = pnp.Blanker(0.04, length, est, reset)
    _check_status(e, 1, ref, 0)
    limit = cap - (length - 1)
    pos, done, ends = 0, 0, []
    while pos < total:
        n = min(int(rng.integers(1, limit // 2)) | 1, total - pos)
        _push(e, 0, raw, item_type, pos, pos + n)
        want = ref.push(held[pos:pos + n])
        pos += n
        ends.append(pos)
        lo, hi = e.iq_window(1)
        assert hi == (pos // length) * length == done + want.size, (lo, hi, pos)
        assert lo == max(0, hi - cap)
        if want.size:
            got = e.iq_read(1, done, want.size)
            assert got.tobytes() == want.tobytes(), (pos, np.flatnonzero(got != want)[:5])
        done = hi
        _check_status(e, 1, ref, 0)
    assert 0 < ref.blanked < ref.segments
    assert (ref.segments - est) // (reset + 2) >= 2  # several reset cycles
    lib = pnp.reference_filter()
    if lib is not None:
        out, thres, (n_seg, lf, est_f) = pnp.reference_block(lib, held, 0.04, length, est, reset, ends)
        assert thres == ref.thres
        lo, hi = e.iq_window(1)
        assert out.size > lo
        assert e.iq_read(1, lo, out.size - lo).tobytes() == out[lo:].tobytes()


@pytest.mark.parametrize("item_type", ["gr_complex", "ibyte"])
def test_one_push_and_many_give_the_same_bytes(capi, engine, item_type):
    e = engine
    rng = np.random.default_rng(11)
    cap, length = 1 << 16, 32
    n = cap - (length - 1)
    raw, _ = _pulsed(rng, n, item_type)
    for src, dst in ((2, 3), (4, 5)):
        e.iq_create(src, cap, item_type)
        e.iq_create(dst, cap)
        e.iq_set_pulse_blanking(dst, src, 0.04, length, 100, 700)
    _push(e, 2, raw, item_type, 0, n)
    pos = 0
    while pos < n:
        k = min(int(rng.integers(1, 700)), n - pos)
        _push(e, 4, raw, item_type, pos, pos + k)
        pos += k
    m = (n // length) * length
    assert e.iq_window(3) == e.iq_window(5) == (0, m)
    assert e.iq_read(3, 0, m).tobytes() == e.iq_read(5, 0, m).tobytes()
    assert e.iq_pulse_blanking_status(3) == e.iq_pulse_blanking_status(5)


def test_origin_and_window_rules(capi, engine):
    e = engine
    rng = np.random.default_rng(13)
    L, E, R, cap = 32, 20, 100, 1 << 12
    x, _ = _pulsed(rng, 20_000, "gr_complex", pulse_every=400)
    e.iq_create(0, cap)
    e.iq_create(1, cap)
    e.iq_set_pulse_blanking(1, 0, 0.04, L, E, R)
    assert e.iq_window(1) == (0, 0)                                        # a fresh stream: origin 0

    def whole(o, w):
        return o + (w - o) // L * L

    e.iq_push(0, x[:1001])
    assert e.iq_window(1) == (0, whole(0, 1001))                           # only whole segments
    assert e.iq_read(1, 0, 992).tobytes() == pnp.blank(x[:1001], 0.04, L, E, R).tobytes()
    g = 1501                                                               # push_at gap: restart at g
    assert e.iq_push_at(0, g, x[g:g + 2001]) == 2001
    w = g + 2001
    assert e.iq_window(1) == (g, whole(g, w))
    assert e.iq_pulse_blanking_status(1)["origin"] == g
    assert e.iq_read(1, g, whole(g, w) - g).tobytes() == pnp.blank(x[g:w], 0.04, L, E, R).tobytes()
    e.iq_forget(0)                                                         # forget on the source: restart at its write index
    assert e.iq_window(1) == (w, w)
    st = e.iq_pulse_blanking_status(1)
    assert (st["origin"], st["segments"], st["n"], st["noise_power"]) == (w, 0, 0, 0.0)
    ref1 = pnp.Blanker(0.04, L, E, R)
    y1 = ref1.push(x[w:w + 1003])
    e.iq_push(0, x[w:w + 1003])
    w2 = w + 1003
    assert e.iq_window(1) == (w, w + y1.size)
    assert e.iq_read(1, w, y1.size).tobytes() == y1.tobytes()
    e.iq_create(2, cap)                                                    # set mid-stream: origin at the source's write index
    e.iq_set_pulse_blanking(2, 0, 0.04, L, E, R)
    assert e.iq_window(2) == (w2, w2)
    f1 = w + y1.size
    e.iq_forget(1)                                                         # forget on the destination: a floor, same state
    assert e.iq_window(1) == (f1, f1)
    k0 = e.launch_count()
    e.iq_push(0, x[w2:w2 + 777])
    w3 = w2 + 777
    e.sync()
    assert e.launch_count() - k0 == 6                                      # two blankers, three kernels each
    y1b = ref1.push(x[w2:w3])
    assert e.iq_window(1) == (f1, f1 + y1b.size)
    assert e.iq_read(1, f1, y1b.size).tobytes() == y1b.tobytes()
    _check_status(e, 1, ref1, w)
    y2 = pnp.blank(x[w2:w3], 0.04, L, E, R)
    assert e.iq_window(2) == (w2, w2 + y2.size)
    assert e.iq_read(2, w2, y2.size).tobytes() == y2.tobytes()
    # removal and re-creation of a destination: pushes launch nothing for them, their windows stay
    e.iq_remove_pulse_blanking(2)
    e.iq_create(1, cap)
    wins = (e.iq_window(1), e.iq_window(2))
    k0 = e.launch_count()
    e.iq_push(0, x[w3:w3 + 500])
    e.sync()
    assert e.launch_count() == k0 and (e.iq_window(1), e.iq_window(2)) == wins
    e.iq_push(2, x[:10])                                                   # an ordinary band again
    with pytest.raises(capi.B200Error):
        e.iq_pulse_blanking_status(2)
    # re-creating the source removes its blankers; setting one again replaces it
    e.iq_set_pulse_blanking(1, 0, 0.04, L, E, R)
    e.iq_set_pulse_blanking(1, 0, 0.1, 7, E, R)
    assert e.iq_pulse_blanking_status(1)["length"] == 7
    e.iq_create(0, cap)
    k0 = e.launch_count()
    e.iq_push(0, x[:100])
    e.sync()
    assert e.launch_count() == k0


def test_conditioner_then_blanker_is_the_restatement_of_the_conditioned_band(capi, engine):
    """the adapter's IF > 1 arm: freq_xlating_fir_filter_ccf(1, low_pass(1, fs, bw, tw), IF, fs), then the blanker; pushes
    wrap both rings, and a forget on the raw source restarts the blanker where the conditioned band's window restarts"""
    e = engine
    rng = np.random.default_rng(17)
    fs, if_hz, L, E, R = 8e6, 1.25e6, 32, 40, 300
    h = capi.iq_conditioner_lowpass(fs, 1, 2e6, 2e5)
    e.iq_create(6, 1 << 14)
    e.iq_create(7, 1 << 14)
    e.iq_create(8, 1 << 14)
    e.iq_set_conditioner(7, 6, 1, h, if_hz, fs)
    e.iq_set_pulse_blanking(8, 7, 0.04, L, E, R)
    x, _ = _pulsed(rng, 60_000, "gr_complex", pulse_every=700)
    ref = pnp.Blanker(0.04, L, E, R)
    pos, mid, done = 0, 0, 0
    k_first = None
    while pos < 50_000:
        n = int(rng.integers(1, 4000)) | 1
        k0 = e.launch_count()
        e.iq_push(6, x[pos:pos + n])
        pos += n
        _, hi = e.iq_window(7)
        y = e.iq_read(7, mid, hi - mid)                                    # what the conditioner wrote
        mid = hi
        want = ref.push(y)
        if k_first is None and want.size:
            k_first = e.launch_count() - k0
        lo, top = e.iq_window(8)
        assert top == done + want.size
        if want.size:
            assert e.iq_read(8, done, want.size).tobytes() == want.tobytes(), pos
        done = top
        _check_status(e, 8, ref, 0)
    assert k_first == 4                                                    # the conditioner, then the blanker's three
    assert ref.blanked > 0 and ref.segments > E
    e.iq_forget(6)
    e.iq_push(6, x[pos:pos + 3001])
    lo7, hi7 = e.iq_window(7)
    assert lo7 == pos + h.size - 1
    st = e.iq_pulse_blanking_status(8)
    assert st["origin"] == lo7
    y = e.iq_read(7, lo7, hi7 - lo7)
    want = pnp.blank(y, 0.04, L, E, R)
    assert e.iq_window(8) == (lo7, lo7 + want.size)
    assert e.iq_read(8, lo7, want.size).tobytes() == want.tobytes()


def test_search_right_after_a_push_reads_the_blanked_samples(capi, engine):
    """no host synchronisation between the push and the band search; then repeated pushes of the largest size, read back
    only at the end"""
    e = engine
    rng = np.random.default_rng(19)
    fs = 4_000_000
    acq, host, codes = ar.pair(capi, e, rng, fs)
    n = host.conf.consumed_samples
    total = 4 * n
    x = ar.stream(rng, total, codes[1][:n], fs)
    x[::997] += 40.0                                                       # isolated spikes for the blanker to find
    e.iq_create(9, ar.pow2(total))
    e.iq_create(10, ar.pow2(total))
    e.iq_set_pulse_blanking(10, 9, 0.04, 8, 50, 10_000)
    e.iq_push(9, x)
    got = acq.search_band(10, 1000, [1, 0])
    y = pnp.blank(x, 0.04, 8, 50, 10_000)
    assert not np.array_equal(y, x[:y.size])
    want = host.search(y[1000:1000 + n], [1, 0])
    assert got.tobytes() == want.tobytes()
    cap = 1 << 14
    e.iq_create(11, cap)
    e.iq_create(12, 1 << 18)
    e.iq_set_pulse_blanking(12, 11, 0.04, 32, 30, 200)
    big = cap - 31
    xs, _ = _pulsed(rng, 12 * big, "gr_complex")
    for k in range(12):
        e.iq_push(11, xs[k * big:(k + 1) * big])
    want = pnp.blank(xs, 0.04, 32, 30, 200)
    assert e.iq_window(12) == (0, want.size)
    assert e.iq_read(12, 0, want.size).tobytes() == want.tobytes()
    acq.close()
    host.close()


def test_push_launches_and_refusals(capi, engine, tmp_path):
    e = engine
    rng = np.random.default_rng(23)
    cap = 1 << 12
    x, _ = _pulsed(rng, 3 * cap, "gr_complex")
    raw16 = rng.integers(-100, 100, 2 * cap).astype(np.int16)
    raw8 = rng.integers(-100, 100, 2 * cap).astype(np.int8)
    for b in (0, 1, 2, 5, 6):
        e.iq_create(b, cap)
    e.iq_create(3, cap, "ibyte")
    e.iq_create(4, cap // 4)
    e.iq_create(7, cap // 2)
    e.iq_create(8, cap)

    def pushed(call):
        k0 = e.launch_count()
        call()
        e.sync()
        return e.launch_count() - k0

    assert pushed(lambda: e.iq_push(0, x[:100])) == 0                     # as before: a copy, no kernel
    assert pushed(lambda: e.iq_push_int(0, raw16[:200])) == 1              # as before: the conversion
    e.iq_set_pulse_blanking(1, 0, 0.04, 32, 5, 50)                         # origin 200
    assert pushed(lambda: e.iq_push(0, x[:100])) == 3                      # three whole segments
    assert pushed(lambda: e.iq_push(0, x[:10])) == 0                       # 110 samples: no new segment
    e.iq_set_pulse_blanking(2, 0, 0.04, 16, 5, 50)                         # origin 310
    assert pushed(lambda: e.iq_push(0, x[:64])) == 6
    assert pushed(lambda: e.iq_push_int(0, raw16[:202])) == 7              # conversion + two blankers
    e.iq_set_pulse_blanking(6, 3, 0.04, 32, 5, 50)                         # an ibyte source
    assert pushed(lambda: e.iq_push_int(3, raw8[:200])) == 3
    e.iq_set_conditioner(7, 5, 2, np.full(9, 1.0 / 9, np.float32), 0.0, 4e6)
    e.iq_set_pulse_blanking(8, 7, 0.04, 32, 5, 50)                         # chained through a D = 2 conditioner
    assert pushed(lambda: e.iq_push(5, x[:128])) == 4

    bands = range(10)

    def refused(call, code):
        wins = [e.iq_window(b) for b in bands]
        k0 = e.launch_count()
        with pytest.raises(capi.B200Error) as ei:
            call()
        assert ei.value.code == code, str(ei.value)
        e.sync()
        assert e.launch_count() == k0 and [e.iq_window(b) for b in bands] == wins
        return str(ei.value)

    def set_(dst, src, pfa=0.04, length=32, est=5, reset=50):
        return lambda: e.iq_set_pulse_blanking(dst, src, pfa, length, est, reset)

    e.iq_create(9, cap)
    refused(set_(9, 9), ERR_ARG)                                                  # dst == src
    refused(set_(9, 0, length=-1), ERR_ARG)
    refused(set_(9, 0, est=-1), ERR_ARG)
    refused(set_(9, 0, reset=-1), ERR_ARG)
    for pfa in (0.0, 1.0, -0.5, 2.0, float("nan")):
        refused(set_(9, 0, pfa=pfa), ERR_ARG)
    refused(set_(9, 0, length=capi.B200_IQ_MAX_BLANKING_LENGTH + 1), ERR_RANGE)
    refused(set_(3, 0), ERR_STATE)                                                # narrow destination
    refused(set_(4, 0), ERR_RANGE)                                                # smaller than the source
    refused(set_(9, 1), ERR_STATE)                                                # fed from a blanker
    refused(set_(0, 9), ERR_STATE)                                                # a destination that feeds blankers
    refused(set_(7, 9), ERR_STATE)                                                # a conditioner's destination
    refused(set_(9, 13), ERR_STATE)                                               # an unused band
    e.iq_create(15, 16)
    refused(set_(9, 15), ERR_RANGE)                                               # a source smaller than one segment
    h = np.full(9, 1.0 / 9, np.float32)
    refused(lambda: e.iq_set_conditioner(9, 1, 1, h, 0.0, 4e6), ERR_STATE)        # a conditioner fed from a blanker
    refused(lambda: e.iq_set_conditioner(1, 9, 1, h, 0.0, 4e6), ERR_STATE)        # a conditioner into a blanker's destination
    import torch
    buf = torch.zeros(2 * cap, dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    e.iq_attach_dev(14, buf.data_ptr(), cap)
    refused(set_(9, 14), ERR_STATE)                                               # attached source
    refused(set_(14, 0), ERR_STATE)                                               # attached destination
    # while set: direct writes into a destination, and pushes that would overwrite pending samples
    refused(lambda: e.iq_push(1, x[:10]), ERR_STATE)
    refused(lambda: e.iq_push_int(1, raw16[:20]), ERR_STATE)
    refused(lambda: e.iq_push_at(1, e.iq_window(1)[1] + 5, x[:10]), ERR_STATE)
    path = tmp_path / "x.bin"
    x[:100].tofile(path)
    refused(lambda: e.iq_push_file(1, str(path), "gr_complex"), ERR_STATE)
    msg = refused(lambda: e.iq_push(0, x[:cap - 30]), ERR_RANGE)
    assert f"at most {cap - 31}" in msg, msg
    assert pushed(lambda: e.iq_push(0, x[:cap - 31])) == 6                 # two blankers
    msg = refused(lambda: e.iq_push(5, x[:cap - 61]), ERR_RANGE)           # chained: D (capacity / 2 - 31)
    assert f"at most {cap - 62}" in msg, msg
    assert pushed(lambda: e.iq_push(5, x[:cap - 62])) == 4
    e.iq_remove_pulse_blanking(1)
    assert pushed(lambda: e.iq_push(0, x[:cap - 15])) == 3                 # only the 16-sample blanker is left
    e.iq_create(14, cap)


def _acquire(capi, e, band, prn, fs, abs_index):
    acq = ar.make(capi, e, fs, doppler_max=5000, doppler_step=100, n_code_slots=1)
    acq.set_local_code(0, ar.ca_code(gs, prn, fs))
    r = acq.search_band(band, abs_index, [0])[0]
    stamp = abs_index + acq.conf.consumed_samples
    period = acq.conf.consumed_samples
    acq.close()
    return r, stamp, period


def test_gps_l1_with_pulse_pairs_is_acquired_better_and_tracked_as_its_restatement(capi):
    """GPS L1 C/A at 4 Msps with DME-like pulse pairs 40 dB above the noise: the blanked band's test statistic is higher than
    the raw band's, the satellite is found at its Doppler and code phase, and the device loops in all three modes write
    the very dump records of the same loops on a band pushed with the restatement's output"""
    from oracle import loop as ol
    fs, n_ep, L, E, R, abs_index = 4_000_000, 400, 32, 100, 100_000, 4000   # the search starts past the estimation
    spc = fs // 1000
    sv = dict(prn=11, doppler=-1370.0, delay=1777, cn0=48.0)
    total = abs_index + (n_ep + 8) * spc
    codes = {sv["prn"]: gs.gps_ca_code(sv["prn"])}
    iq = gs.make_iq(codes, fs, total, [dict(prn=sv["prn"], doppler=sv["doppler"], cn0=sv["cn0"],
                                            code_phase_chips=(-sv["delay"] * 1.023e6 / fs) % 1023)], seed=29)
    rng = np.random.default_rng(31)
    sigma = float(np.std(iq))
    w = np.exp(-0.5 * ((np.arange(60) - 30) / 7.0) ** 2) * 100.0 * sigma
    for start in range(int(rng.integers(0, 1200)), total - 120, 1200):  # a pair every 300 us
        for off in (0, 48):
            iq[start + off:start + off + 60] += w * np.exp(1j * rng.uniform(0, 2 * np.pi))
    x = iq.astype(np.complex64)
    y = pnp.blank(x, 0.04, L, E, R)
    assert np.count_nonzero(y == 0) > 0.03 * y.size
    for mode in (0, 1, 2):
        e = capi.Engine(0)
        for b in (0, 1, 2):
            e.iq_create(b, ar.pow2(total))
        e.iq_set_pulse_blanking(1, 0, 0.04, L, E, R)
        for a in range(0, total, 1 << 18):
            e.iq_push(0, x[a:a + (1 << 18)])
        e.iq_push(2, y)
        assert e.iq_window(1) == e.iq_window(2) == (0, y.size)
        raw, _, _ = _acquire(capi, e, 0, sv["prn"], fs, abs_index)
        r1, stamp, period = _acquire(capi, e, 1, sv["prn"], fs, abs_index)
        r2, _, _ = _acquire(capi, e, 2, sv["prn"], fs, abs_index)
        assert r1.tobytes() == r2.tobytes()
        assert r1["test_statistics"] > 1.5 * raw["test_statistics"], (r1, raw)
        assert abs(r1["doppler"] - sv["doppler"]) <= 100, r1
        delay = math.fmod(float(r1["index_time"]), float(period))
        err = (delay - (sv["delay"] - abs_index) + spc / 2) % spc - spc / 2
        assert abs(err) <= 2, (r1, delay)
        e.loop_set_mode(mode)
        conf = ol.default_conf(fs_in=fs, prn=sv["prn"], pull_in_time_s=1)
        ids = []
        for b in (1, 2):
            ch = e.channel_create(b, 3)
            e.channel_set_code(ch, codes[sv["prn"]], [-0.5, 0.0, 0.5])
            lid = e.loop_create(ch, conf)
            e.loop_start(lid, delay, float(r1["doppler"]), stamp, stamp)
            ids.append(lid)
        rec, cnt = e.loop_run(n_ep)
        assert cnt[ids[0]] == cnt[ids[1]] >= n_ep - 2, (mode, cnt)
        k = cnt[ids[0]]
        assert rec[ids[0], :k].tobytes() == rec[ids[1], :k].tobytes(), mode
        assert e.loop_status(ids[0]).state == 2
        assert abs(np.mean(rec[ids[0], k - 100:k]["carrier_doppler_hz"]) - sv["doppler"]) < 5.0
        e.close()
