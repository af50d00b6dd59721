"""The correlator inside the free-running DLL/PLL loops (b200_trk_loop_run), epoch by epoch against exact references.

In the tracking state b200_trk_loop_peek_items is a pure function of the loop state, and loop_run(1) correlates exactly
that item and logs one record carrying the P tap's bits (prompt_I, prompt_Q) and hypotf of every tap (abs_*).  So
peek -> run(1) -> compare checks every epoch a loop actually produced, in each way the loops can run:

  * mode 0, the persistent CTA per loop, at both widths (512 threads while the engine holds no more loops than the device
    has SMs, else 256: the narrow case adds loops that are never started);
  * mode 1, the batch correlator with one slice per item and a loop-update launch per epoch;
  * mode 2, the same with each epoch split over several CTAs (batch_slices).

Integer samples with a zero imaginary part and loops at 0 Hz keep every tap an exactly representable integer (the PLL
error is exactly 0, so the carrier stays at phase 0 with step 0): those runs must EQUAL the integer oracle built from the
reference's chip indices.  Float data with a rotating carrier stays within the batch-kernel contract (DESIGN a2),
1e-5 |P| of the float64 truth.  One launch of N epochs must equal N launches of one epoch byte for byte (in mode 0 only
the chip-table window cache differs), and the persistent kernel's split loop update must equal the sequential update
(b200_trk_loop_step_taps) byte for byte.  Finally the loops stall outside [valid_from, write_index), the window
b200_iq_window reports: after a gap, a restart or b200_iq_forget they never correlate what the ring held before."""
import numpy as np
import pytest

from gpu_fixtures import capi  # noqa: F401
from loop_rig import (CA_RATE, DELAY, FS, MODES, PERSISTENT, RING_BASE, RING_CAP, TRUTH_RTOL, LoopSpec, RingFeeder, Stream,
                      capacities_for, check_int_epoch, check_loop, f64_taps, gps_stream, int_configs, int_taps,
                      lock_loss_case, make_engine, ol_port, other_band, push_all, rebuilt_taps, rec_mags, run_per_epoch,
                      set_mode, start_all, veml_int_case, window_engine)
from oracle import loop as ol

pytestmark = pytest.mark.gpu


# ---------------------------------------------------------------------------------------------------------------------
# configurations with integer data

def run_config(capi, specs, caps, ring, mode, n_ep):
    """-> per-epoch results (run_per_epoch), records of the multi-epoch twin, final status of both"""
    caps = capacities_for(specs, caps)
    e, ids = make_engine(capi, specs, caps)
    set_mode(e, mode, specs[0])
    if ring:
        assert len(specs) == 1
        feeder = RingFeeder(e, 0, specs[0].stream)
        start_all(e, ids, specs)
        per = run_per_epoch(e, ids, n_ep, feed=lambda items: feeder.until(int(items[0]["sample_index"]) + int(items[0]["n"])))
    else:
        push_all(e, specs)
        start_all(e, ids, specs)
        per = run_per_epoch(e, ids, n_ep)
    st = [e.loop_status(l) for l in ids]
    e.close()

    # the twin: the same loops in launches of many epochs
    e, ids = make_engine(capi, specs, caps)
    set_mode(e, mode, specs[0])
    if ring:
        feeder = RingFeeder(e, 0, specs[0].stream)
        start_all(e, ids, specs)
        got = [[] for _ in ids]
        while sum(len(g) for g in got) < n_ep:
            if not feeder.push_block():
                break
            rec, cnt = e.loop_run(16)
            got[0].append(rec[0, :cnt[0]])
        multi = [np.concatenate(g)[:n_ep] for g in got]
    else:
        push_all(e, specs)
        start_all(e, ids, specs)
        rec, cnt = e.loop_run(n_ep)
        multi = [rec[i, :cnt[i]] for i in range(len(ids))]
    st2 = [e.loop_status(l) for l in ids]
    e.close()
    return per, multi, st, st2


N_EP = 300


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("config", ["gps_ring", "veml_2spc", "galileo_like", "two_bands"])
def test_integer_epochs_equal_the_integer_oracle(capi, config, mode):
    """(a) every epoch's taps equal the integer oracle exactly, and (c) one launch of many epochs gives the same records,
    byte for byte, as one launch per epoch."""
    specs, caps, ring = int_configs(N_EP)[config]
    per, multi, st, st2 = run_config(capi, specs, caps, ring, mode, N_EP)
    for i, sp in enumerate(specs):
        items, recs = per[i]
        assert len(recs) == N_EP, (config, i, len(recs))
        for k in range(len(recs)):
            check_int_epoch(sp, items[k], recs[k], (config, mode, i, k))
        # the DLL moves the code phase every epoch, and the code step now and then
        assert len(np.unique(items["rem_code_phase_chips"])) > len(items) // 2
        assert len(np.unique(items["code_phase_step_chips"])) > 1
        if config == "gps_ring":
            d = np.diff(items["sample_index"].astype(np.int64))
            assert set(np.unique(d)) == {3999, 4000, 4001}, np.unique(d, return_counts=True)
            assert items["sample_index"][0] < (1 << 32) < items["sample_index"][-1]
            assert int(items["sample_index"][-1]) - RING_BASE > 20 * RING_CAP
        assert len(multi[i]) == N_EP and multi[i].tobytes() == recs.tobytes(), (config, mode, i)
    if not ring:
        for a, b in zip(st, st2):
            assert (a.state, a.sample_counter, a.epochs) == (b.state, b.sample_counter, b.epochs)


# ---------------------------------------------------------------------------------------------------------------------
# float data, rotating carrier

def check_float_epoch(sp, item, r, what):
    truth = f64_taps(sp, item)
    p = sp.taps // 2
    scale = TRUTH_RTOL * abs(truth[p])
    assert abs(complex(float(r["prompt_I"]), float(r["prompt_Q"])) - truth[p]) <= scale, (what, r["prompt_I"], r["prompt_Q"], truth[p])
    err = np.abs(rec_mags(sp, r) - np.abs(truth))
    assert np.all(err <= scale), (what, err / abs(truth[p]))


def float_configs(n_ep):
    from gnss_synth import make_iq
    port = ol_port()
    out = {}
    for name, prn, doppler, delay, veml in (("gps_3taps", 4, 1234.0, 1777, 0), ("veml_5taps", 12, -2710.0, 909, 1)):
        code = port.gps_ca_code(prn)
        spc = 2 if veml else 1
        table = np.repeat(code, spc)
        n = 4000 * (n_ep + 2) + delay
        iq = make_iq({prn: table}, FS, n, [dict(prn=prn, doppler=doppler, code_phase_chips=(-delay * spc * CA_RATE / FS) % len(table),
                                                cn0=60.0, phase0=0.7)], seed=prn, chips_per_table_chip=spc)
        kw = dict(veml=1, code_samples_per_chip=2, early_late_space_chips=0.15) if veml else {}
        conf = ol.default_conf(fs_in=FS, prn=prn, pull_in_time_s=1, **kw)
        out[name] = LoopSpec(0, table, conf, (delay + 0.2, doppler - 6.0, 0, 0), Stream(iq, 0))
    return out


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("config", ["gps_3taps", "veml_5taps"])
def test_float_epochs_within_the_float64_truth(capi, config, mode):
    """(b) complex samples with a real Doppler: every epoch's P and |tap| within 1e-5 |P| of the float64 correlation of the
    peeked item, and (c) one launch of many epochs equals one launch per epoch byte for byte."""
    sp = float_configs(N_EP)[config]
    per, multi, st, st2 = run_config(capi, [sp], None, False, mode, N_EP)
    items, recs = per[0]
    assert len(recs) == N_EP
    assert np.all(items["phase_step_rad"] != 0.0)
    for k in range(N_EP):
        check_float_epoch(sp, items[k], recs[k], (config, mode, k))
    assert abs(np.mean(recs["carrier_doppler_hz"][-100:]) - (1234.0 if config == "gps_3taps" else -2710.0)) < 2.0
    assert len(multi[0]) == N_EP and multi[0].tobytes() == recs.tobytes(), (config, mode)
    assert (st[0].sample_counter, st[0].epochs) == (st2[0].sample_counter, st2[0].epochs)


def test_loop_width_only_from_the_loop_count(capi, monkeypatch):
    """B200_LOOP_WIDTH in the environment selects nothing: with B200_LOOP_WIDTH=256 one loop still runs on 512-thread CTAs,
    so its records on float data, where a 256-thread CTA sums the taps in another order, are the same bytes."""
    sp = float_configs(N_EP)["gps_3taps"]

    def run():
        e, ids = make_engine(capi, [sp], capacities_for([sp], None))
        push_all(e, [sp])
        start_all(e, ids, [sp])
        rec, cnt = e.loop_run(N_EP)
        e.close()
        assert cnt[0] == N_EP
        return rec[0].tobytes()

    want = run()
    monkeypatch.setenv("B200_LOOP_WIDTH", "256")
    assert run() == want


# ---------------------------------------------------------------------------------------------------------------------
# the persistent kernel's split loop update against the sequential one

def split_configs():
    rng = np.random.default_rng(77)
    return {
        "gps_float_3taps": (float_configs(N_EP)["gps_3taps"], N_EP),
        "veml_int_5taps": (veml_int_case(rng, N_EP), N_EP),
        "gps_int_lock_loss": (lock_loss_case(rng), 120),
    }


@pytest.mark.parametrize("mode", PERSISTENT)
@pytest.mark.parametrize("config", ["gps_float_3taps", "veml_int_5taps", "gps_int_lock_loss"])
def test_split_update_equals_the_sequential_update(capi, config, mode):
    """(d) The persistent kernel updates the loop on three warps at once and, on a lost-lock verdict, restores its backup
    and replays the update.  Feeding its taps to b200_trk_loop_step_taps (the sequential update) on a twin started
    identically must reproduce every peeked item and every record byte for byte; the lock-loss configuration also
    takes the restore-and-replay branch."""
    sp, n_ep = split_configs()[config]
    caps = {0: len(sp.stream.x) + 16}
    e, ids = make_engine(capi, [sp], caps)
    set_mode(e, mode, sp)
    push_all(e, [sp])
    start_all(e, ids, [sp])
    items, recs = run_per_epoch(e, ids, n_ep)[0]
    st = e.loop_status(ids[0])
    e.close()
    lost = config == "gps_int_lock_loss"
    if lost:
        assert 40 < len(recs) < n_ep - 10 and st.state == 0 and st.loss_of_lock == 1, (len(recs), st.state, st.loss_of_lock)
        for k in range(len(recs)):
            check_int_epoch(sp, items[k], recs[k], (config, mode, k))
    else:
        assert len(recs) == n_ep and st.state == 2 and st.loss_of_lock == 0

    t, tids = make_engine(capi, [sp], caps)
    push_all(t, [sp])
    start_all(t, tids, [sp])
    for k in range(len(recs)):
        it = t.loop_peek_items()
        assert it[0].tobytes() == items[k].tobytes(), (config, mode, k)
        r, logged = t.loop_step_taps(rebuilt_taps(sp, recs[k])[None, :])
        assert logged[0] == 1 and r[0].tobytes() == recs[k].tobytes(), (config, mode, k)
    if lost:
        # the epoch that lost lock logged no record: its taps come from the integer oracle
        it = t.loop_peek_items()
        r, logged = t.loop_step_taps(int_taps(sp, it[0]).astype(np.complex64)[None, :])
        assert logged[0] == 0
    s2 = t.loop_status(tids[0])
    t.close()
    assert bytes(st) == bytes(s2), (config, mode)


# ---------------------------------------------------------------------------------------------------------------------
# the loops' sample window is [valid_from, write_index)

@pytest.mark.parametrize("mode", list(MODES))
def test_loops_below_valid_from_stall_after_a_gap(capi, mode):
    """iq_push_at(0, A[:60000]) then iq_push_at(1_000_000, B[:30000]) into a 2^16 ring: ring slots below valid_from still
    hold A.  A loop whose epochs lie below 1_000_000 must stall (no record, sample counter frozen after its first
    prepare); a loop started at 1_000_000 tracks B exactly; a loop on another band is unaffected."""
    rng = np.random.default_rng(5)
    code, a = gps_stream(rng, 3, 0, 60_000)
    _, b = gps_stream(rng, 3, 1_000_000, 30_000)
    low = LoopSpec(0, code, ol.default_conf(fs_in=FS, prn=3), (DELAY + 0.3, 0.0, 990_000, 990_000), None)
    high = LoopSpec(0, code, ol.default_conf(fs_in=FS, prn=3), (DELAY + 0.3, 0.0, 1_000_000, 1_000_000), b)
    oth = other_band(rng, 12)
    e, ids = window_engine(capi, mode, [low, high, oth], {0: 1 << 16, 1: len(oth.stream.x) + 16})
    e.iq_push_at(0, 0, a.x.astype(np.complex64))
    e.iq_push_at(0, 1_000_000, b.x.astype(np.complex64))
    push_all(e, [oth])
    assert e.iq_window(0) == (1_000_000, 1_030_000)
    start_all(e, ids, [low, high, oth])
    e.loop_peek_items()
    frozen = e.loop_status(ids[0]).sample_counter
    assert 990_000 < frozen < 1_000_000
    res = run_per_epoch(e, ids, 12)
    s = e.loop_status(ids[0])
    assert len(res[0][1]) == 0 and s.sample_counter == frozen and s.state == 2 and s.epochs == 0, (len(res[0][1]), s.sample_counter)
    check_loop(high, res[1], 6, "after the gap")
    check_loop(oth, res[2], 12, "other band")
    e.close()


@pytest.mark.parametrize("mode", list(MODES))
def test_loops_stall_after_iq_forget(capi, mode):
    """After b200_iq_forget every sample in the band is history: both of its loops stall, although the ring still holds
    those samples and more arrive behind them; the loop on the other band keeps running."""
    rng = np.random.default_rng(6)
    code, s = gps_stream(rng, 8, 0, 100_000)
    l0 = LoopSpec(0, code, ol.default_conf(fs_in=FS, prn=8), (DELAY + 0.3, 0.0, 0, 0), s)
    l1 = LoopSpec(0, code, ol.default_conf(fs_in=FS, prn=8, early_late_space_chips=0.25), (DELAY - 0.2, 0.0, 0, 0), s)
    oth = other_band(rng, 10)
    e, ids = window_engine(capi, mode, [l0, l1, oth], {0: 1 << 17, 1: len(oth.stream.x) + 16})
    e.iq_push_at(0, 0, s.x[:60_000].astype(np.complex64))
    push_all(e, [oth])
    start_all(e, ids, [l0, l1, oth])
    before = run_per_epoch(e, ids, 5)
    check_loop(l0, before[0], 5, "before forget")
    check_loop(l1, before[1], 5, "before forget")
    e.iq_forget(0)
    e.iq_push_at(0, 60_000, s.x[60_000:].astype(np.complex64))     # contiguous: valid_from stays at 60_000
    assert e.iq_window(0) == (60_000, 100_000)
    counters = [e.loop_status(l).sample_counter for l in ids[:2]]
    after = run_per_epoch(e, ids, 5)
    assert len(after[0][1]) == 0 and len(after[1][1]) == 0
    assert [e.loop_status(l).sample_counter for l in ids[:2]] == counters
    check_loop(oth, (np.concatenate([before[2][0], after[2][0]]), np.concatenate([before[2][1], after[2][1]])), 10, "other band")
    e.close()


@pytest.mark.parametrize("mode", list(MODES))
def test_loops_follow_a_restarted_stream(capi, mode):
    """A stream at 1_000_000 into a 2^16 ring, then a restart iq_push_at at the older index 500_000.  The loop on the old
    stream stalls, a loop started at 500_000 runs on the new samples exactly, and one started at 480_000 (below the new
    valid_from, yet inside what the ring's slots span) stalls instead of correlating the old stream."""
    rng = np.random.default_rng(7)
    code, s1 = gps_stream(rng, 30, 1_000_000, 60_000)
    _, s2 = gps_stream(rng, 30, 500_000, 40_000)
    conf = ol.default_conf(fs_in=FS, prn=30)
    old = LoopSpec(0, code, conf, (DELAY + 0.3, 0.0, 1_000_000, 1_000_000), s1)
    new = LoopSpec(0, code, conf, (DELAY + 0.3, 0.0, 500_000, 500_000), s2)
    below = LoopSpec(0, code, conf, (DELAY + 0.3, 0.0, 480_000, 480_000), None)
    oth = other_band(rng, 12)
    specs = [old, new, below, oth]
    e, ids = window_engine(capi, mode, specs, {0: 1 << 16, 1: len(oth.stream.x) + 16})
    e.iq_push_at(0, 1_000_000, s1.x.astype(np.complex64))
    push_all(e, [oth])
    e.loop_start(ids[0], *old.start)
    e.loop_start(ids[3], *oth.start)
    first = run_per_epoch(e, ids, 4)
    check_loop(old, first[0], 4, "old stream")
    e.iq_push_at(0, 500_000, s2.x.astype(np.complex64))
    assert e.iq_window(0) == (500_000, 540_000)
    e.loop_start(ids[1], *new.start)
    e.loop_start(ids[2], *below.start)
    e.loop_peek_items()
    frozen = [e.loop_status(ids[i]).sample_counter for i in (0, 2)]
    assert 480_000 < frozen[1] < 500_000
    second = run_per_epoch(e, ids, 8)
    assert len(second[0][1]) == 0 and len(second[2][1]) == 0
    assert [e.loop_status(ids[i]).sample_counter for i in (0, 2)] == frozen
    check_loop(new, second[1], 8, "new stream")
    check_loop(oth, (np.concatenate([first[3][0], second[3][0]]), np.concatenate([first[3][1], second[3][1]])), 12, "other band")
    e.close()
