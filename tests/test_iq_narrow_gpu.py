"""16-bit and 8-bit IQ bands (b200_iq_create_typed "ishort" / "ibyte"): samples kept at their own width on the device.

The equality rule: the same integers pushed into a gr_complex band (widened on the device by b200_iq_push_i16 / _i8) and
into an ishort / ibyte band give byte-identical taps and acquisition records, because the narrow readers widen each sample
exactly right after its load and then run the float readers' arithmetic.  Also: narrow pushes are plain copies (no launch),
every push of another type into a narrow band is refused without writing anything, the shared-window kernel never reads a
narrow band, and the device loops refuse narrow bands.
"""
import numpy as np
import pytest

from acq_rig import ERR_ARG, ERR_STATE
import acq_rig as ar
from gpu_fixtures import capi, engine, torch  # noqa: F401
import trk_rig as tr
from trk_ref import exact_taps, int_code

pytestmark = pytest.mark.gpu

WIDTHS = {"ishort": np.int16, "ibyte": np.int8}


def _ints(rng, n, item_type):
    """2n interleaved I, Q integers of the item type's full range"""
    info = np.iinfo(WIDTHS[item_type])
    return rng.integers(info.min, info.max + 1, 2 * n).astype(WIDTHS[item_type])


class Pair:
    """Band 0 a gr_complex ring, band 1 a ring of item_type, both fed the same integer pushes; every channel is made on
    both bands alike, so item k on band 1 must give exactly what item k on band 0 gives."""

    def __init__(self, capi, item_type, cap, kernel=0):
        self.e = capi.Engine(0)
        self.e.trk_kernel_choice(kernel)
        self.e.iq_create(0, cap)
        self.e.iq_create(1, cap, item_type)
        self.item_type = item_type
        self.ch = ([], [])

    def push(self, iq):
        for b in (0, 1):
            self.e.iq_push_int(b, iq)
        assert self.e.iq_window(0) == self.e.iq_window(1)

    def channel(self, code, shifts, hd=False):
        for b in (0, 1):
            self.ch[b].append(tr.channel(self.e, b, code, shifts, hd))
        return len(self.ch[0]) - 1

    def items(self, specs):
        """specs: (channel index, start, n, rem_carr, dphi, rem_code, step[, rate]) -> (items on band 0, items on band 1)"""
        return [tr.items((self.ch[b][c], n, s0, rc, dp, 0.0, rem, step, *rate) for c, s0, n, rc, dp, rem, step, *rate in specs)
                for b in (0, 1)]

    def close(self):
        self.e.close()


def _item_specs(rng, lo, hi, cap, chans, count):
    """items at odd and even starts, across the ring's end, near the write index, whole and partial tiles"""
    lengths = [4096, 4097, 4000, 3999, 517, 511, 7, 12345]
    ends = hi - np.arange(count) * 997
    specs = []
    for k in range(count):
        n = lengths[k % len(lengths)]
        if k % 3 == 0:
            wrap = (hi // cap) * cap                    # a ring offset 0 inside the window
            s0 = wrap - n // 2 - (k % 2)
        else:
            s0 = int(ends[k]) - n - (k % 2)
        s0 = max(lo, min(s0, hi - n))
        specs.append((chans[k % len(chans)], int(s0), n, float(rng.uniform(-3, 3)), float(rng.uniform(-0.3, 0.3)),
                      float(rng.uniform(0, 0.9)), float(rng.uniform(0.2, 0.5))))
    return specs


@pytest.mark.parametrize("item_type", list(WIDTHS))
@pytest.mark.parametrize("taps", range(1, 9))
def test_taps_equal_the_float_band(capi, torch, item_type, taps):
    """1-8 taps on the per-item kernel, fast and modulo paths, high-dynamics channels, large absolute indices and
    windows across the ring's end, through b200_trk_batch (small and large batches) and b200_trk_batch_dev at 1, 2, 7
    and 64 slices."""
    rng = np.random.default_rng(100 * taps + len(item_type))
    cap = 1 << 16
    p = Pair(capi, item_type, cap)
    for _ in range(300):                                    # write index past 2^24
        p.push(_ints(rng, cap, item_type))
    lo, hi = p.e.iq_window(0)
    assert hi > 1 << 24
    code = np.sign(rng.standard_normal(1023)).astype(np.float32)
    c_fast = p.channel(code, tr.shifts(taps))
    c_mod = p.channel(code, [float(s) for s in np.linspace(-700.25, 1500.5, taps)] if taps > 1 else [900.5])
    c_hd = p.channel(code, tr.shifts(taps), hd=True)
    specs = _item_specs(rng, lo, hi, cap, [c_fast, c_mod], 24)
    specs += [(c_hd, s0, n, rc, dp, rem, step, 1e-7) for (_, s0, n, rc, dp, rem, step) in specs[:6]]
    a, b = p.items(specs)
    assert p.e.trk_batch(b, 8).tobytes() == p.e.trk_batch(a, 8).tobytes()
    many_a, many_b = np.tile(a, 50), np.tile(b, 50)         # > 1024 items: the copy-stream submit path
    assert p.e.trk_batch(many_b, 8).tobytes() == p.e.trk_batch(many_a, 8).tobytes()
    for slices in (1, 2, 7, 64):
        assert tr.run_dev(torch, p.e, b, 8, slices).tobytes() == tr.run_dev(torch, p.e, a, 8, slices).tobytes(), slices
    p.close()


@pytest.mark.parametrize("item_type", list(WIDTHS))
def test_integer_exact_against_the_oracle(capi, oracle, item_type):
    """Zero carrier, small-integer code: the narrow band's taps equal the exact integer correlation on their own."""
    rng = np.random.default_rng(5)
    e = capi.Engine(0)
    e.iq_create(0, 1 << 15, item_type)
    n, L, shifts, rem, step = 7001, 1023, [-0.5, -0.25, 0.0, 0.25, 0.5], 0.3, 0.341
    iq = rng.integers(-100, 101, 2 * (1 << 14)).astype(WIDTHS[item_type])
    e.iq_push_int(0, iq)
    code_int = int_code(L, nonzero=True)
    c = tr.channel(e, 0, code_int, shifts)
    for s0 in (0, 1, 9000):
        x = iq[2 * s0:2 * (s0 + n)].astype(np.int64)
        got = e.trk_batch(tr.items([(c, n, s0, 0.0, 0.0, 0.0, rem, step)]), len(shifts))[0]
        assert np.array_equal(got.real.astype(np.int64), exact_taps(oracle, x[0::2], code_int, rem, step, shifts, n)), s0
        assert np.array_equal(got.imag.astype(np.int64), exact_taps(oracle, x[1::2], code_int, rem, step, shifts, n)), s0
    e.close()


def test_mixed_band_types_and_tap_counts_in_one_batch(capi, torch):
    """Channels with 5, 1 and 3 taps on a gr_complex, an ishort and an ibyte band holding the same int8-range integers:
    one launch per (tap count, band type) present, and every item equals its twins on the other two bands."""
    rng = np.random.default_rng(21)
    e = capi.Engine(0)
    e.trk_kernel_choice(0)
    cap = 1 << 16
    for b, t in enumerate(("gr_complex", "ishort", "ibyte")):
        e.iq_create(b, cap, t)
    for _ in range(5):
        iq8 = _ints(rng, cap // 2, "ibyte")
        e.iq_push_int(0, iq8)
        e.iq_push_int(1, iq8.astype(np.int16))
        e.iq_push_int(2, iq8)
    lo, hi = e.iq_window(0)
    code = np.sign(rng.standard_normal(1023)).astype(np.float32)
    chans = {(b, taps): tr.channel(e, b, code, tr.shifts(taps)) for b in range(3) for taps in (5, 1, 3)}
    base = _item_specs(rng, lo, hi, cap, [5, 1, 3], 18)
    items = np.stack([tr.items((chans[(b, taps)], n, s0, rc, dp, 0.0, rem, step) for taps, s0, n, rc, dp, rem, step in base)
                      for b in range(3)])
    order = rng.permutation(3 * len(base))
    flat = items.reshape(-1)[order]
    k0 = e.launch_count()
    for slices in (1, 4):
        out = tr.run_dev(torch, e, flat, 8, slices)
        back = np.empty_like(out)
        back[order] = out
        back = back.reshape(3, len(base), 8, 2)
        assert back[1].tobytes() == back[0].tobytes() and back[2].tobytes() == back[0].tobytes(), slices
    assert e.launch_count() - k0 == 2 * 9                   # 3 tap counts x 3 band types, twice
    a = e.trk_submit(flat, 8)
    got = e.trk_wait(a)
    assert got.tobytes() == e.trk_batch(flat, 8).tobytes()
    e.close()


@pytest.mark.parametrize("mode", [1, 2])
def test_shared_kernel_never_reads_a_narrow_band(capi, mode):
    """1024 overlapping C/A items on an ishort band under kernel choice 1 and 2: per-item launches only, and the taps
    equal the gr_complex band's on the per-item kernel."""
    rng = np.random.default_rng(mode)
    p = Pair(capi, "ishort", 1 << 20, kernel=0)
    p.push(_ints(rng, 1 << 19, "ishort"))
    code = np.sign(rng.standard_normal(1023)).astype(np.float32)
    chans = [p.channel(code, [-0.5, 0.0, 0.5]) for _ in range(8)]
    specs = [(chans[k % 8], 1000 + 4000 * (k // 8) + 37 * (k % 8), 4000, 0.5, 0.01 * (k % 8), 0.25, 0.25575)
             for k in range(1024)]
    a, b = p.items(specs)
    want = p.e.trk_batch(a, 3)
    k0 = p.e.launch_count()
    p.e.trk_batch(b, 3)
    per_item = p.e.launch_count() - k0                      # one launch per band type
    assert per_item == 2
    p.e.trk_kernel_choice(mode)
    # the gr_complex band's channels alone would take the shared-window kernel: a narrow channel with a code table keeps
    # every batch off it
    for items in (b, a):
        k0 = p.e.launch_count()
        assert p.e.trk_batch(items, 3).tobytes() == want.tobytes()
        assert p.e.launch_count() - k0 == per_item
    p.close()


@pytest.mark.parametrize("item_type", list(WIDTHS))
def test_narrow_pushes_launch_nothing_and_files_match_arrays(capi, tmp_path, item_type):
    rng = np.random.default_rng(3)
    n = 5000
    iq = _ints(rng, n, item_type)
    e = capi.Engine(0)
    e.iq_create(0, 1 << 12, item_type)                     # 4096: the pushes wrap
    e.iq_create(1, 1 << 12, item_type)
    k0 = e.launch_count()
    e.iq_push_int(0, iq[:2 * 3000])
    e.iq_push_int(0, iq[2 * 3000:])
    e.sync()
    assert e.launch_count() == k0
    path = tmp_path / "iq.bin"
    iq.tofile(path)
    assert e.iq_push_file(1, str(path), item_type, chunk_samples=1000) == (0, n)
    e.sync()
    assert e.launch_count() == k0
    assert e.iq_window(0) == e.iq_window(1) == (n - 4096, n)
    code = np.sign(rng.standard_normal(1023)).astype(np.float32)
    ch = [tr.channel(e, b, code, [-0.5, 0.0, 0.5]) for b in (0, 1)]
    out = e.trk_batch(tr.items((c, 3000, n - 3500, 0.3, 0.02, 0.0, 0.1, 0.3) for c in ch), 3)
    assert out[0].tobytes() == out[1].tobytes()
    e.close()


@pytest.mark.parametrize("item_type", list(WIDTHS))
def test_refused_pushes_write_nothing(capi, torch, tmp_path, item_type):
    rng = np.random.default_rng(4)
    e = capi.Engine(0)
    with pytest.raises(capi.B200Error) as ei:
        e.iq_create(0, 1024, "cshort")
    assert ei.value.code == ERR_ARG
    e.iq_create(0, 1 << 12, item_type)
    iq = _ints(rng, 1000, item_type)
    e.iq_push_int(0, iq)
    e.sync()
    win, k0 = e.iq_window(0), e.launch_count()
    other = np.int8 if item_type == "ishort" else np.int16
    f_other = tmp_path / "other.bin"
    iq.astype(other).tofile(f_other)
    f_float = tmp_path / "float.bin"
    np.zeros(100, np.complex64).tofile(f_float)
    x = np.ones(100, np.complex64)
    buf = torch.zeros(200, dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    attempts = [
        lambda: e.iq_push(0, x),
        lambda: e.iq_push_at(0, win[1], x),
        lambda: e.iq_push_at(0, win[1] + 50000, x),        # a gap push would move the window before writing
        lambda: e.iq_refill_ptr(0, x.ctypes.data, 100, 0),
        lambda: e.iq_push_int(0, iq.astype(other)),
        lambda: e.iq_push_int(0, iq[:0].astype(other)),
        lambda: e.iq_push_file(0, str(f_other), "ishort" if other == np.int16 else "ibyte"),
        lambda: e.iq_push_file(0, str(f_float), "gr_complex"),
    ]
    for k, f in enumerate(attempts):
        with pytest.raises(capi.B200Error) as ei:
            f()
        assert ei.value.code == ERR_STATE, k
        assert item_type in capi.lib.b200_last_error().decode(), k
        assert e.iq_window(0) == win, k
    e.sync()
    assert e.launch_count() == k0
    del buf
    e.close()


def test_device_loops_refuse_narrow_bands(capi):
    """loop_create on a channel of a narrow band; then a loop made and started on a gr_complex band whose band is re-created
    narrow: set_data_channel and every run refuse it, in every loop mode, and launch nothing."""
    from oracle import loop as ol
    e = capi.Engine(0)
    e.iq_create(0, 1 << 16)
    e.iq_create(1, 1 << 16, "ishort")
    conf = ol.default_conf(fs_in=4e6, prn=1)
    code = np.sign(np.random.default_rng(1).standard_normal(1023)).astype(np.float32)
    chans = {}
    for b in (0, 1):
        chans[b] = e.channel_create(b, 3)
        e.channel_set_code(chans[b], code, [-0.5, 0.0, 0.5])
    data = e.channel_create(0, 1)
    e.channel_set_code(data, code, [0.0])
    with pytest.raises(capi.B200Error) as ei:
        e.loop_create(chans[1], conf)
    assert ei.value.code == ERR_STATE
    lid = e.loop_create(chans[0], conf)
    e.iq_push_int(0, np.zeros(2 * 40000, np.int16))
    e.loop_start(lid, 100.3, 1000.0, 0, 0)
    e.iq_create(0, 1 << 16, "ibyte")                       # the started loop's band re-created narrow
    e.iq_push_int(0, np.zeros(2 * 40000, np.int8))
    with pytest.raises(capi.B200Error) as ei:
        e.loop_set_data_channel(lid, data)
    assert ei.value.code == ERR_STATE
    for mode in (0, 1, 2):
        e.loop_set_mode(mode)
        k0 = e.launch_count()
        with pytest.raises(capi.B200Error) as ei:
            e.loop_run(4)
        assert ei.value.code == ERR_STATE
        with pytest.raises(capi.B200Error) as ei:
            e.loop_run_prompts(4)
        assert ei.value.code == ERR_STATE
        assert e.launch_count() == k0
    e.close()


@pytest.mark.parametrize("item_type", list(WIDTHS))
def test_retyped_band_takes_the_narrow_path(capi, item_type):
    """A band created gr_complex, then re-created narrow: its channels run the narrow path on their next batch."""
    rng = np.random.default_rng(8)
    cap = 1 << 14
    e = capi.Engine(0)
    e.trk_kernel_choice(0)
    e.iq_create(0, cap)
    e.iq_create(1, cap)
    code = np.sign(rng.standard_normal(1023)).astype(np.float32)
    ch = [tr.channel(e, b, code, [-0.5, 0.0, 0.5]) for b in (0, 1)]
    iq = _ints(rng, 3 * cap // 2, item_type)
    for b in (0, 1):
        for half in (iq[:cap], iq[cap:]):
            e.iq_push_int(b, half)
    items = tr.items((c, 4000, 3 * cap // 2 - 4100, 0.4, 0.03, 0.0, 0.2, 0.25) for c in ch)
    first = e.trk_batch(items, 3)
    assert first[0].tobytes() == first[1].tobytes()
    e.iq_create(1, cap, item_type)
    for half in (iq[:cap], iq[cap:]):
        e.iq_push_int(1, half)
    k0 = e.launch_count()
    out = e.trk_batch(items, 3)
    assert e.launch_count() - k0 == 2                      # one launch per band type
    assert out[1].tobytes() == out[0].tobytes() == first[0].tobytes()
    e.close()


# ---- acquisition band search --------------------------------------------------------------------------------------------
ACQ_CASES = [
    ("single4000_cfar", 4000, dict()),
    ("single25000_peaks", 25000, dict(use_CFAR_algorithm_flag=False)),
    ("two50000_cfar_dwells", 50000, dict(max_dwells=2)),
    ("chirpz16368_cfar_dwells", 16368, dict(max_dwells=2)),
    ("chirpz5456_bits_grid", 5456, dict(bit_transition_flag=True, keep_grid=True)),
]


@pytest.mark.parametrize("item_type", list(WIDTHS))
@pytest.mark.parametrize("spms,opts", [c[1:] for c in ACQ_CASES], ids=[c[0] for c in ACQ_CASES])
def test_band_search_equals_the_float_band(capi, engine, item_type, spms, opts):
    """The window straddles the ring's end and every dwell takes the next window; then b200_acq_search_band_submit and
    b200_acq_search_step_two_band on the same windows."""
    rng = np.random.default_rng(spms + len(opts) + len(item_type))
    *acqs, codes = ar.pair(capi, engine, rng, 1000 * spms, **opts)
    c = acqs[0].conf
    n, dwells = c.consumed_samples, c.max_dwells
    cap = ar.pow2(3 * n)
    info = np.iinfo(WIDTHS[item_type])
    x = ar.stream(rng, 2 * cap + 2 * n, np.resize(codes[1], n), c.fs_in, np.complex128)
    iq = ar.to_int(x, WIDTHS[item_type], 3000.0 if item_type == "ishort" else 30.0, clip=(info.min, info.max))
    engine.iq_create(6, cap)
    engine.iq_create(7, cap, item_type)
    for k in range(0, iq.size, 2 * (cap // 3 + 7)):
        for b in (6, 7):
            engine.iq_push_int(b, iq[k:k + 2 * (cap // 3 + 7)])
    idx = 2 * cap - n // 3
    for d in range(1, dwells + 1):
        s0 = idx + (d - 1) * n
        want = acqs[0].search_band(6, s0, [1, 0], dwell_counter=d)
        got = acqs[1].search_band(7, s0, [1, 0], dwell_counter=d)
        assert got.tobytes() == want.tobytes(), (d, got, want)
    assert ar.grids(acqs[1]) == ar.grids(acqs[0])
    acqs[0].search_band_submit(6, idx, [0, 1])
    want = acqs[0].search_wait()
    acqs[1].search_band_submit(7, idx, [0, 1])
    assert acqs[1].search_wait().tobytes() == want.tobytes()
    if not opts.get("bit_transition_flag"):
        for a in acqs:
            a.set_step_two(100.0, 125.0, 4)
        want = acqs[0].search_step_two_band(6, idx, 1, 1.0)
        assert acqs[1].search_step_two_band(7, idx, 1, 1.0).tobytes() == want.tobytes()
    for a in acqs:
        a.close()
