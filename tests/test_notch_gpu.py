"""The notch filters on the device (b200_iq_set_notch): every push into a source band fills a destination band with
Notch's or NotchLite's output, in absolute stream indices.

Read back with b200_iq_read, the destination is byte for byte the restatement (notch_np.run) for both variants, every
source type and segment length, push by push across the ring's end and through estimation, detection, reset and
coefficient-epoch cycles; the status matches the restatement after every push; filtered samples are within
notch_np.recursion_bound of the float64 truth.  One push and many give the same bytes; the origin follows the stream start
and a notch set mid-stream, with Lite's zero history item and Notch's one-sample look-ahead; a push launches six kernels
when it completes segments and none otherwise; the push limit is capacity - L; every refusal launches nothing.  A push_at
gap, a forget on either band and a replacement (notch by notch on a dirty state, blanker and notch by each other) restart
or keep the notch as the header states; a conditioner followed by a notch is the restatement of the conditioned band; a
band search right after a push reads the notched samples.  End to end, a GPS L1 C/A stream under a strong CW is acquired
only after the notch, and the device loops on the notched band follow loops fed the float64 truth."""
import math

import numpy as np
import pytest

import acq_rig as ar
import notch_np as nn
from gpu_fixtures import capi, engine  # noqa: F401

pytestmark = pytest.mark.gpu

ERR_ARG, ERR_STATE, ERR_RANGE = -1, -4, -5


def _cw_noise(rng, n, item_type, cw=6.0):
    """n samples of complex noise with a CW switched on and off every 3000 samples -> (what a push of item_type takes, the
    complex64 samples the band holds)"""
    sigma = 12.0 if item_type == "ibyte" else 300.0
    t = np.arange(n)
    x = (rng.normal(0, sigma / math.sqrt(2), n) + 1j * rng.normal(0, sigma / math.sqrt(2), n))
    x = x + ((t // 3000) % 2 == 1) * cw * sigma * np.exp(1j * (0.41 * t + 0.3))
    if item_type == "gr_complex":
        x = x.astype(np.complex64)
        return x, x
    dt, lim = (np.int16, 32767) if item_type == "ishort" else (np.int8, 127)
    raw = ar.to_int(x, dt, 1.0, clip=(-lim, lim))
    return raw, ar.from_int(raw)


def _push(e, band, raw, item_type, a, b):
    if item_type == "gr_complex":
        return e.iq_push(band, raw[a:b])
    return e.iq_push_int(band, raw[2 * a:2 * b])


def _f32(v):
    return np.float32(v).tobytes()


def _check_status(e, band, res, k, origin, variant, length):
    st = e.iq_notch_status(band)
    assert st["origin"] == origin and st["segments"] == k and st["length"] == length and st["variant"] == variant
    assert _f32(st["threshold"]) == _f32(res["thres"])
    if k == 0:
        return
    want = nn.state_after(res, k)
    for key in ("filtered", "n", "filter_state", "n_coeff"):
        assert st[key] == want[key], (key, st, want)
    assert _f32(st["noise_power"]) == _f32(want["noise_power"])
    assert _f32(st["z0"].real) == _f32(want["z0"][0]) and _f32(st["z0"].imag) == _f32(want["z0"][1]), (st["z0"], want["z0"])
    assert _f32(st["last_out"].real) == _f32(want["last_out"][0]) and _f32(st["last_out"].imag) == _f32(want["last_out"][1])


CASES = [(nn.NOTCH_LITE, 1, 1), (nn.NOTCH_LITE, 7, 3), (nn.NOTCH_LITE, 32, 1), (nn.NOTCH_LITE, 301, 3),
         (nn.NOTCH, 7, 1), (nn.NOTCH, 32, 1), (nn.NOTCH, 301, 1)]


@pytest.mark.parametrize("variant,length,n_coeff", CASES)
@pytest.mark.parametrize("item_type", ["gr_complex", "ishort", "ibyte"])
def test_bit_exact_push_by_push(capi, engine, item_type, variant, length, n_coeff):
    """odd push sizes three times around a 4096-sample source ring with small E and R; the status after every push;
    filtered samples within the stated bound of the float64 truth"""
    e = engine
    rng = np.random.default_rng(1000 * length + 10 * variant + len(item_type))
    cap = 1 << 12
    total = 3 * cap + 123
    segs = total // length
    est, reset = segs // 20 + 1, segs // 6
    p = 0.9 if length != 7 else -0.7
    e.iq_create(0, cap, item_type)
    e.iq_create(1, cap)
    e.iq_set_notch(1, 0, variant, 1e-3, p, length, est, reset, n_coeff)
    raw, held = _cw_noise(rng, total, item_type)
    res = nn.run(held, variant, 1e-3, p, length, est, reset, n_coeff)
    _check_status(e, 1, res, 0, 0, variant, length)
    limit = cap - length - (1 if (variant == nn.NOTCH_LITE and length == 1) else 0)
    pos, done = 0, 0
    lead = nn.lead(variant, length)
    while pos < total:
        n = min(int(rng.integers(1, limit // 2)) | 1, total - pos)
        _push(e, 0, raw, item_type, pos, pos + n)
        pos += n
        k = max(0, (pos - lead) // length)
        lo, hi = e.iq_window(1)
        assert hi == k * length, (lo, hi, pos)
        if hi > done:
            got = e.iq_read(1, done, hi - done)
            want = res["out"][done:hi]
            assert got.tobytes() == want.tobytes(), (pos, np.flatnonzero(got != want)[:5])
        done = hi
        _check_status(e, 1, res, k, 0, variant, length)
    flags = res["flags"]
    assert 0 < int((flags & 1).sum()) < flags.size and (flags & 2).sum() >= 2
    filt = res["filt"]
    err = np.max(np.abs(res["out"][filt].astype(np.complex128) - res["truth"][filt]))
    assert err <= nn.recursion_bound(res, p), (err, nn.recursion_bound(res, p))


@pytest.mark.parametrize("variant", [nn.NOTCH, nn.NOTCH_LITE])
def test_one_push_and_many_give_the_same_bytes(capi, engine, variant):
    """a clean stream where the filter is on for long runs that cross many grid blocks and pushes"""
    e = engine
    rng = np.random.default_rng(21 + variant)
    cap, length = 1 << 16, 32
    n = cap - length
    raw, held = _cw_noise(rng, n, "gr_complex", cw=0.0)
    for src, dst in ((2, 3), (4, 5)):
        e.iq_create(src, cap)
        e.iq_create(dst, cap)
        e.iq_set_notch(dst, src, variant, 1e-3, 0.9, length, 50, 100000, 1)
    e.iq_push(2, raw[:n])
    pos = 0
    while pos < n:
        m = min(int(rng.integers(1, 5000)), n - pos)
        e.iq_push(4, raw[pos:pos + m])
        pos += m
    lo, hi = e.iq_window(3)
    assert e.iq_window(5) == (lo, hi) and hi > 0.9 * n
    a, b = e.iq_read(3, lo, hi - lo), e.iq_read(5, lo, hi - lo)
    assert a.tobytes() == b.tobytes()
    res = nn.run(held, variant, 1e-3, 0.9, length, 50, 100000)
    assert a.tobytes() == res["out"][:hi].tobytes()
    assert res["filt"].mean() > 0.3  # the reference's estimator keeps the filter on for much of clean noise


def test_origin_mid_stream_and_lookahead(capi, engine):
    """set mid-stream, the origin is the source's write index: Lite reads a zero before it, Notch starts one sample later"""
    e = engine
    rng = np.random.default_rng(5)
    cap, length = 1 << 13, 16
    raw, held = _cw_noise(rng, 6000, "gr_complex")
    e.iq_create(0, cap)
    e.iq_create(1, cap)
    e.iq_create(2, cap)
    e.iq_push(0, raw[:1000])
    e.iq_set_notch(1, 0, nn.NOTCH_LITE, 1e-3, 0.9, length, 20, 300, 2)
    e.iq_set_notch(2, 0, nn.NOTCH, 1e-3, 0.9, length, 20, 300)
    assert e.iq_window(1) == (1000, 1000) and e.iq_window(2) == (1000, 1000)
    e.iq_push(0, raw[1000:1000 + length])
    assert e.iq_window(1)[1] == 1000 + length and e.iq_window(2)[1] == 1000  # Notch waits for the sample after the segment
    e.iq_push(0, raw[1000 + length:6000])
    for band, variant, n_coeff in ((1, nn.NOTCH_LITE, 2), (2, nn.NOTCH, 1)):
        res = nn.run(held[1000:6000], variant, 1e-3, 0.9, length, 20, 300, n_coeff)
        lo, hi = e.iq_window(band)
        assert lo == 1000 and hi == 1000 + res["segments"] * length
        assert e.iq_read(band, lo, hi - lo).tobytes() == res["out"].tobytes()
        assert e.iq_notch_status(band)["origin"] == 1000
    # removal: the destination keeps its window and takes pushes again
    e.iq_remove_notch(1)
    with pytest.raises(capi.B200Error):
        e.iq_notch_status(1)


def test_launch_counts_limit_and_refusals(capi, engine):
    e = engine
    cap, length = 1 << 12, 32
    e.iq_create(0, cap)
    e.iq_create(1, cap)
    e.iq_create(2, cap)
    x = (np.random.default_rng(3).normal(size=cap) * (1 + 1j)).astype(np.complex64)
    k0 = e.launch_count()
    e.iq_push(2, x[:100])
    assert e.launch_count() == k0  # a push into a band with no stage launches nothing
    e.iq_set_notch(1, 0, nn.NOTCH_LITE, 1e-3, 0.9, length, 10, 1000, 1)
    k0 = e.launch_count()
    e.iq_push(0, x[:length - 1])
    assert e.launch_count() == k0  # no complete segment
    e.iq_push(0, x[length - 1:3 * length])
    assert e.launch_count() - k0 == 6
    with pytest.raises(capi.B200Error) as r:
        e.iq_push(0, x[:cap - length + 1])
    assert r.value.code == ERR_RANGE
    e.iq_push(0, x[:cap - length])
    wins = (e.iq_window(0), e.iq_window(1))
    k0 = e.launch_count()
    bad = [
        dict(variant=7), dict(pfa=0.0), dict(pfa=1.0), dict(p_c_factor=1.0), dict(p_c_factor=float("nan")), dict(length=-1),
        dict(segments_est=-1), dict(segments_reset=-1), dict(segments_coeff=0),
    ]
    for b in bad:
        kw = dict(variant=nn.NOTCH_LITE, pfa=1e-3, p_c_factor=0.9, length=length, segments_est=10, segments_reset=1000, segments_coeff=1)
        kw.update(b)
        with pytest.raises(capi.B200Error) as r:
            e.iq_set_notch(1, 0, **kw)
        assert r.value.code == ERR_ARG, b
    for args, code in (((1, 0, nn.NOTCH, 1e-3, 0.9, 1025), ERR_RANGE), ((1, 1, nn.NOTCH, 1e-3, 0.9, 32), ERR_ARG),
                       ((0, 1, nn.NOTCH, 1e-3, 0.9, 32), ERR_STATE)):
        with pytest.raises(capi.B200Error) as r:
            e.iq_set_notch(*args)
        assert r.value.code == code, args
    with pytest.raises(capi.B200Error) as r:
        e.iq_push(1, x[:10])
    assert r.value.code == ERR_STATE
    assert e.launch_count() == k0 and (e.iq_window(0), e.iq_window(1)) == wins


def _whole(o, w, variant, length):
    """the destination's write index: o plus the whole segments that w source samples publish"""
    return o + max(0, w - o - nn.lead(variant, length)) // length * length


def test_origin_window_replacement_and_removal(capi, engine):
    """a push_at gap, a forget on either band, a notch set again with another variant and L on a dirty state, a blanker and
    a notch replacing each other on one destination, and removal of one kind leaving the other"""
    import pulse_blanking_np as pnp
    e = engine
    rng = np.random.default_rng(13)
    L, E, R, cap, LITE = 32, 20, 100, 1 << 12, nn.NOTCH_LITE
    x, _ = _cw_noise(rng, 20_000, "gr_complex")
    x[:] = np.roll(x, -2500)                                               # the CW is on from the first samples
    e.iq_create(0, cap)
    e.iq_create(1, cap)
    e.iq_set_notch(1, 0, LITE, 1e-3, 0.9, L, E, R, 2)
    assert e.iq_window(1) == (0, 0)

    def same(band, o, src, variant=LITE, length=L, n_coeff=2):
        res = nn.run(src, variant, 1e-3, 0.9, length, E, R, n_coeff)
        lo, hi = e.iq_window(band)
        assert hi == o + res["segments"] * length, (lo, hi, o)
        assert e.iq_read(band, lo, hi - lo).tobytes() == res["out"][lo - o:].tobytes()
        return res

    e.iq_push(0, x[:1001])
    same(1, 0, x[:1001])
    g = 1501                                                               # push_at gap: restart at g
    assert e.iq_push_at(0, g, x[g:g + 2001]) == 2001
    w = g + 2001
    assert e.iq_window(1)[0] == g and e.iq_notch_status(1)["origin"] == g
    same(1, g, x[g:w])
    e.iq_forget(0)                                                         # forget on the source: restart at its write index
    assert e.iq_window(1) == (w, w)
    st = e.iq_notch_status(1)
    assert (st["origin"], st["segments"], st["n"], st["filtered"]) == (w, 0, 0, 0)
    e.iq_push(0, x[w:w + 1003])
    w2 = w + 1003
    same(1, w, x[w:w2])
    f1 = e.iq_window(1)[1]
    e.iq_forget(1)                                                         # forget on the destination: a floor, same state
    assert e.iq_window(1) == (f1, f1)
    e.iq_push(0, x[w2:w2 + 2777])
    w3 = w2 + 2777
    res = same(1, w, x[w:w3])
    assert e.iq_window(1)[0] == f1
    assert e.iq_notch_status(1)["filtered"] == res["rec"]["filtered"][-1] > 0   # a dirty state: runs, z0, grid carry
    # replaced on a dirty state by a Notch with another L: it starts fresh at the source's write index
    e.iq_set_notch(1, 0, nn.NOTCH, 1e-3, 0.9, 7, E, R)
    assert e.iq_window(1) == (w3, w3)
    st = e.iq_notch_status(1)
    assert (st["origin"], st["variant"], st["length"], st["n"], st["z0"], st["last_out"]) == (w3, nn.NOTCH, 7, 0, 0j, 0j)
    e.iq_push(0, x[w3:w3 + 3001])
    w4 = w3 + 3001
    same(1, w3, x[w3:w4], nn.NOTCH, 7, 1)
    # a blanker replaces the notch, and a notch the blanker
    e.iq_set_pulse_blanking(1, 0, 0.04, 16, 5, 50)
    with pytest.raises(capi.B200Error):
        e.iq_notch_status(1)
    e.iq_push(0, x[w4:w4 + 1000])
    w5 = w4 + 1000
    assert e.iq_read(1, w4, 992).tobytes() == pnp.blank(x[w4:w5], 0.04, 16, 5, 50).tobytes()
    e.iq_remove_notch(1)                                                   # removes only a notch: the blanker stays
    assert e.iq_pulse_blanking_status(1)["origin"] == w4
    e.iq_set_notch(1, 0, LITE, 1e-3, 0.9, L, E, R, 2)
    e.iq_remove_pulse_blanking(1)                                          # removes only a blanker: the notch stays
    e.iq_push(0, x[w5:w5 + 2000])
    same(1, w5, x[w5:w5 + 2000])
    e.iq_remove_notch(1)
    wins = (e.iq_window(0), e.iq_window(1))
    k0 = e.launch_count()
    e.iq_push(0, x[:500])
    e.sync()
    assert e.launch_count() == k0 and e.iq_window(1) == wins[1]
    e.iq_push(1, x[:10])                                                   # an ordinary band again


def test_conditioner_then_notch_is_the_restatement_of_the_conditioned_band(capi, engine):
    """a conditioner at an IF followed by a Lite notch; pushes wrap both rings, and a forget on the raw source restarts the
    notch where the conditioned band's window restarts"""
    e = engine
    rng = np.random.default_rng(17)
    fs, if_hz, L, E, R = 8e6, 1.25e6, 32, 40, 300
    h = capi.iq_conditioner_lowpass(fs, 1, 2e6, 2e5)
    e.iq_create(6, 1 << 14)
    e.iq_create(7, 1 << 14)
    e.iq_create(8, 1 << 14)
    e.iq_set_conditioner(7, 6, 1, h, if_hz, fs)
    e.iq_set_notch(8, 7, nn.NOTCH_LITE, 1e-3, 0.9, L, E, R, 1)
    x, _ = _cw_noise(rng, 60_000, "gr_complex")
    pos, mid, k_first, ys = 0, 0, None, []
    while pos < 50_000:
        n = int(rng.integers(1, 4000)) | 1
        k0 = e.launch_count()
        e.iq_push(6, x[pos:pos + n])
        pos += n
        if k_first is None and e.iq_window(8)[1] > 0:
            k_first = e.launch_count() - k0
        _, hi = e.iq_window(7)
        ys.append(e.iq_read(7, mid, hi - mid))                             # what the conditioner wrote
        mid = hi
    assert k_first == 7                                                    # the conditioner, then the notch's six
    res = nn.run(np.concatenate(ys), nn.NOTCH_LITE, 1e-3, 0.9, L, E, R)
    lo, hi = e.iq_window(8)
    assert hi == res["segments"] * L and lo == hi - (1 << 14)
    assert e.iq_read(8, lo, hi - lo).tobytes() == res["out"][lo:hi].tobytes()
    _check_status(e, 8, res, res["segments"], 0, nn.NOTCH_LITE, L)
    assert 0 < res["rec"]["filtered"][-1] < res["segments"]
    e.iq_forget(6)
    e.iq_push(6, x[pos:pos + 3001])
    lo7, hi7 = e.iq_window(7)
    assert lo7 == pos + h.size - 1 and e.iq_notch_status(8)["origin"] == lo7
    res = nn.run(e.iq_read(7, lo7, hi7 - lo7), nn.NOTCH_LITE, 1e-3, 0.9, L, E, R)
    assert e.iq_window(8) == (lo7, lo7 + res["segments"] * L)
    assert e.iq_read(8, lo7, res["segments"] * L).tobytes() == res["out"].tobytes()


def test_search_right_after_a_push_reads_the_notched_samples(capi, engine):
    """no host synchronisation between the push and the band search; then repeated pushes of the largest size"""
    e = engine
    rng = np.random.default_rng(19)
    fs = 4_000_000
    acq, host, codes = ar.pair(capi, e, rng, fs)
    n = host.conf.consumed_samples
    total = 4 * n
    x = ar.stream(rng, total, codes[1][:n], fs)
    x = (x + 30.0 * np.exp(2j * np.pi * 0.11 * np.arange(total))).astype(np.complex64)
    e.iq_create(9, ar.pow2(total))
    e.iq_create(10, ar.pow2(total))
    e.iq_set_notch(10, 9, nn.NOTCH_LITE, 1e-3, 0.9, 8, 50, 10_000, 1)
    e.iq_push(9, x)
    got = acq.search_band(10, 1000, [1, 0])
    y = nn.run(x, nn.NOTCH_LITE, 1e-3, 0.9, 8, 50, 10_000)["out"]
    assert not np.array_equal(y, x[:y.size])
    want = host.search(y[1000:1000 + n], [1, 0])
    assert got.tobytes() == want.tobytes()
    cap = 1 << 14
    e.iq_create(11, cap)
    e.iq_create(12, 1 << 18)
    e.iq_set_notch(12, 11, nn.NOTCH, 1e-3, 0.9, 32, 30, 200)
    big = cap - 32
    xs, _ = _cw_noise(rng, 12 * big, "gr_complex")
    for k in range(12):
        e.iq_push(11, xs[k * big:(k + 1) * big])
    res = nn.run(xs, nn.NOTCH, 1e-3, 0.9, 32, 30, 200)
    assert e.iq_window(12) == (0, res["segments"] * 32)
    assert e.iq_read(12, 0, res["segments"] * 32).tobytes() == res["out"].tobytes()
    acq.close()
    host.close()


def test_stage_band_refusals(capi, engine):
    """the band rules a notch shares with the blanker: each refusal launches nothing and leaves every window unchanged"""
    e = engine
    cap = 1 << 12
    x = (np.random.default_rng(29).normal(size=cap) * (1 + 1j)).astype(np.complex64)
    for b in (0, 1, 2, 5, 9):
        e.iq_create(b, cap)
    e.iq_create(3, cap, "ibyte")
    e.iq_create(4, cap // 4)
    e.iq_create(7, cap // 2)
    e.iq_create(8, cap)
    e.iq_create(15, 32)
    e.iq_create(13, 2)
    e.iq_set_pulse_blanking(1, 0, 0.04, 32, 5, 50)
    e.iq_set_notch(2, 0, nn.NOTCH, 1e-3, 0.9, 32, 5, 50)
    e.iq_set_conditioner(7, 5, 2, np.full(9, 1.0 / 9, np.float32), 0.0, 4e6)
    e.iq_set_notch(8, 7, nn.NOTCH_LITE, 1e-3, 0.9, 32, 5, 50, 1)
    bands = range(16)

    def refused(call, code):
        wins = [e.iq_window(b) for b in bands if b not in (6, 10, 11, 12, 14)]
        k0 = e.launch_count()
        with pytest.raises(capi.B200Error) as ei:
            call()
        assert ei.value.code == code, str(ei.value)
        e.sync()
        assert e.launch_count() == k0 and [e.iq_window(b) for b in bands if b not in (6, 10, 11, 12, 14)] == wins
        return str(ei.value)

    def set_(dst, src, variant=nn.NOTCH, length=32):
        return lambda: e.iq_set_notch(dst, src, variant, 1e-3, 0.9, length, 5, 50, 1)

    refused(set_(9, 15), ERR_RANGE)                                        # a source smaller than L + 1
    e.iq_set_notch(9, 15, nn.NOTCH, 1e-3, 0.9, 31, 5, 50, 1)               # L + 1 = 32 samples: accepted
    e.iq_remove_notch(9)
    refused(set_(9, 13, nn.NOTCH_LITE, 1), ERR_RANGE)                      # Lite at L = 1 needs 3 samples
    refused(set_(4, 0), ERR_RANGE)                                         # a destination smaller than the source
    refused(set_(3, 0), ERR_STATE)                                         # a narrow destination
    import torch
    buf = torch.zeros(2 * cap, dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    e.iq_attach_dev(14, buf.data_ptr(), cap)
    refused(set_(9, 14), ERR_STATE)                                        # an attached source (not an owned ring)
    refused(set_(14, 0), ERR_STATE)                                        # an attached destination
    refused(set_(9, 1), ERR_STATE)                                         # blanker -> notch
    refused(set_(9, 2), ERR_STATE)                                         # notch -> notch
    refused(lambda: e.iq_set_pulse_blanking(9, 2, 0.04, 32, 5, 50), ERR_STATE)   # notch -> blanker
    refused(set_(0, 9), ERR_STATE)                                         # a destination that feeds stages
    refused(set_(7, 9), ERR_STATE)                                         # a conditioner's destination
    h = np.full(9, 1.0 / 9, np.float32)
    refused(lambda: e.iq_set_conditioner(9, 2, 1, h, 0.0, 4e6), ERR_STATE)        # a conditioner fed from a notch
    refused(lambda: e.iq_set_conditioner(2, 9, 1, h, 0.0, 4e6), ERR_STATE)        # a conditioner into a notch's band
    refused(lambda: e.iq_push(2, x[:10]), ERR_STATE)                       # a direct push into a notch's destination
    msg = refused(lambda: e.iq_push(5, x[:cap - 63]), ERR_RANGE)           # chained: D (capacity / 2 - L)
    assert f"at most {cap - 64}" in msg, msg
    k0 = e.launch_count()
    e.iq_push(5, x[:cap - 64])
    e.sync()
    assert e.launch_count() - k0 == 7
    e.iq_create(14, cap)


def test_gps_l1_with_a_strong_cw_is_acquired_after_the_notch_and_tracked_as_its_truth(capi):
    """GPS L1 C/A at 4 Msps (C/N0 48 dB-Hz, Doppler -1370 Hz) with a CW at +700 kHz whose power is 35 dB above the noise
    per sample.  The raw band's search lands on the wrong Doppler and code phase; after a Lite notch (p_c_factor 0.5, pfa
    0.001, L = 32) it finds the satellite within one Doppler bin of the bin nearest the truth and one sample of code phase.  The device loops on
    the notched band hold lock and follow loops fed the float64-truth output pushed as a band: Doppler within 2 Hz, mean
    prompt magnitude within 5 %, mean C/N0 within 1 dB over the last 100 epochs.  (Both still carry the notch's own
    distortion of the signal next to the CW's band; the test compares the device with the truth, not with the clean signal.)

    Why p_c_factor 0.5 and not the adapter's 0.9: Lite estimates z0 from two sample products per coefficient period, so
    its angle error is about the noise-to-CW amplitude ratio, and the residual CW amplitude, A eps / (1 - p), is about
    noise / (1 - p) whatever the CW's power.  At p = 0.9 that residual is some 16 dB above the noise and the search fails on
    the notched band too; at p = 0.5 it is within 4 dB of the noise."""
    from oracle import loop as ol
    import gnss_synth as gs
    fs, n_ep, L, E, R, p, abs_index = 4_000_000, 300, 32, 100, 100_000, 0.5, 4000
    spc = fs // 1000
    sv = dict(prn=11, doppler=-1370.0, delay=1777, cn0=48.0)
    total = abs_index + (n_ep + 8) * spc
    codes = {sv["prn"]: gs.gps_ca_code(sv["prn"])}
    iq = gs.make_iq(codes, fs, total, [dict(prn=sv["prn"], doppler=sv["doppler"], cn0=sv["cn0"],
                                            code_phase_chips=(-sv["delay"] * 1.023e6 / fs) % 1023)], seed=29)
    sigma = float(np.std(iq))
    t = np.arange(total)
    x = (iq + sigma * 10 ** (35 / 20) * np.exp(2j * np.pi * 700e3 / fs * t + 0.4j)).astype(np.complex64)
    res = nn.run(x, nn.NOTCH_LITE, 1e-3, p, L, E, R)
    y = res["out"]
    truth = y.astype(np.complex128)
    truth[res["filt"]] = res["truth"][res["filt"]]
    truth = truth.astype(np.complex64)
    e = capi.Engine(0)
    for b in (0, 1, 2):
        e.iq_create(b, ar.pow2(total))
    e.iq_set_notch(1, 0, nn.NOTCH_LITE, 1e-3, p, L, E, R, 1)
    for a in range(0, total, 1 << 18):
        e.iq_push(0, x[a:a + (1 << 18)])
    e.iq_push(2, truth)
    assert e.iq_window(1) == e.iq_window(2) == (0, y.size)
    assert e.iq_read(1, 0, y.size).tobytes() == y.tobytes()

    def acquire(band):
        acq = ar.make(capi, e, fs, doppler_max=5000, doppler_step=100, n_code_slots=1)
        acq.set_local_code(0, ar.ca_code(gs, sv["prn"], fs))
        r = acq.search_band(band, abs_index, [0])[0]
        period = acq.conf.consumed_samples
        acq.close()
        delay = math.fmod(float(r["index_time"]), float(period))
        err = (delay - (sv["delay"] - abs_index) + spc / 2) % spc - spc / 2
        return r, delay, err, abs_index + period

    raw, _, raw_err, _ = acquire(0)
    assert abs(raw["doppler"] - round(sv["doppler"] / 100) * 100) > 100 or abs(raw_err) > 1, raw
    r1, delay, err, stamp = acquire(1)
    nearest = round(sv["doppler"] / 100) * 100                              # the grid bin nearest the true Doppler
    assert abs(r1["doppler"] - nearest) <= 100 and abs(err) <= 1, (r1, delay)
    conf = ol.default_conf(fs_in=fs, prn=sv["prn"], pull_in_time_s=1)
    ids = []
    for b in (1, 2):
        ch = e.channel_create(b, 3)
        e.channel_set_code(ch, codes[sv["prn"]], [-0.5, 0.0, 0.5])
        lid = e.loop_create(ch, conf)
        e.loop_start(lid, delay, float(r1["doppler"]), stamp, stamp)
        ids.append(lid)
    rec, cnt = e.loop_run(n_ep)
    k = min(cnt[ids[0]], cnt[ids[1]])
    assert k >= n_ep - 2, cnt
    for lid in ids:
        assert e.loop_status(lid).state == 2
    a, b = rec[ids[0], k - 100:k], rec[ids[1], k - 100:k]
    assert abs(np.mean(a["carrier_doppler_hz"]) - np.mean(b["carrier_doppler_hz"])) < 2.0
    pa, pb = np.mean(np.hypot(a["prompt_I"], a["prompt_Q"])), np.mean(np.hypot(b["prompt_I"], b["prompt_Q"]))
    assert abs(pa / pb - 1) < 0.05, (pa, pb)
    assert abs(np.mean(a["CN0_SNV_dB_Hz"]) - np.mean(b["CN0_SNV_dB_Hz"])) < 1.0
    e.close()
