"""The data correlator of a device loop that tracks a pilot (b200_trk_loop_set_data_channel, b200_trk_loop_run_prompts).

A loop with a data channel correlates each epoch's item against the data code too, with the pilot's NCO values; its record
carries the data prompt as prompt_I / prompt_Q (log_data, dll_pll_veml_tracking.cc:1614-1617), every other field comes from
the pilot taps, and run_prompts hands back the pilot prompt of every record.  The checks follow
tests/test_loop_correlator_gpu.py on its rig, tests/loop_rig.py (peek -> run(1) -> compare, in mode 0 at both CTA widths,
mode 1 and mode 2):

  * integer samples with a zero carrier: the data prompt equals the integer oracle of the data table, every abs_* and the
    returned pilot prompt equal the oracle of the pilot taps;
  * float samples with a rotating carrier: the data prompt within 1e-5 |P_data| of the float64 correlation;
  * a twin without the data channel logs the same records byte for byte except prompt_I / prompt_Q, and its prompts are
    the pilot prompts the data-carrying run returned (also through a loss of lock);
  * the persistent kernel's taps, data tap in its slot, replayed through b200_trk_loop_step_taps reproduce it byte for byte;
  * a synthetic pilot + data signal: the recorded data prompts carry the transmitted symbols, the pilot prompts do not."""
import numpy as np
import pytest

from gpu_fixtures import capi  # noqa: F401
import loop_rig as tl

pytestmark = pytest.mark.gpu

MODES = list(tl.MODES)
N_EP = 150


def run_per_epoch(e, ids, n_ep, feed=None):
    """peek -> run_prompts(1), n_ep times -> per loop: (items, records, pilot prompts) of the epochs that logged a record"""
    out = [([], [], []) for _ in ids]
    for _ in range(n_ep):
        items = e.loop_peek_items()
        if feed is not None:
            feed(items)
        rec, cnt, prm = e.loop_run_prompts(1)
        for i in range(len(ids)):
            if cnt[i]:
                out[i][0].append(items[i])
                out[i][1].append(rec[i, 0])
                out[i][2].append(prm[i, 0])
    return [(np.array(a, items.dtype), np.array(b, rec.dtype), np.array(c, np.complex64)) for a, b, c in out]


def check_int_epoch(sp, dt, item, r, pilot, what):
    """exact: prompt = the data table's integer oracle (or the pilot's without a data channel), abs_* and the returned pilot
    prompt = the pilot taps' oracle"""
    want = tl.int_taps(sp, item)
    p = sp.taps // 2
    assert pilot == np.complex64(want[p]), (what, pilot, want[p])
    if dt is None:
        tl.check_int_epoch(sp, item, r, what)
        return
    want_d = tl.int_taps(tl.data_view(sp, dt), item)[0]
    assert r["prompt_I"] == want_d and r["prompt_Q"] == 0.0, (what, r["prompt_I"], r["prompt_Q"], want_d)
    assert np.array_equal(tl.rec_mags(sp, r), np.abs(want).astype(np.float64)), (what, tl.rec_mags(sp, r), want)
    if sp.taps == 3:
        assert r["abs_VE"] == 0.0 and r["abs_VL"] == 0.0, what


# ---------------------------------------------------------------------------------------------------------------------
# integer data

def int_configs(n_ep):
    """name -> (specs, data tables (None: no data channel), band capacities, ring-fed?)"""
    specs = tl.int_configs(n_ep)
    port = tl.ol_port()
    rng = np.random.default_rng(99)

    def boc():
        return port.sinboc11((2 * rng.integers(0, 2, 4092) - 1).astype(np.int32))

    ring, caps, _ = specs["gps_ring"]
    gal, _, _ = specs["galileo_like"]
    two, _, _ = specs["two_bands"]
    return {
        "epl_1023_ring": (ring, [port.gps_ca_code(31)], caps, True),
        "veml_sinboc_8184": (gal, [boc()], None, False),
        "two_bands_one_data": (two, [None, boc()], None, False),
    }


def run_config(capi, specs, data, caps, ring, mode, n_ep):
    caps = tl.capacities_for(specs, caps)
    e, ids, _ = tl.make_engine_with_data(capi, specs, data, caps)
    tl.set_mode(e, mode, specs[0])
    if ring:
        feeder = tl.RingFeeder(e, 0, specs[0].stream)
        tl.start_all(e, ids, specs)
        per = run_per_epoch(e, ids, n_ep, feed=lambda items: feeder.until(int(items[0]["sample_index"]) + int(items[0]["n"])))
    else:
        tl.push_all(e, specs)
        tl.start_all(e, ids, specs)
        per = run_per_epoch(e, ids, n_ep)
    e.close()
    return per


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("config", ["epl_1023_ring", "veml_sinboc_8184", "two_bands_one_data"])
def test_integer_data_prompt_equals_the_integer_oracle(capi, config, mode):
    specs, data, caps, ring = int_configs(N_EP)[config]
    per = run_config(capi, specs, data, caps, ring, mode, N_EP)
    for i, (sp, dt) in enumerate(zip(specs, data)):
        items, recs, pilots = per[i]
        assert len(recs) == N_EP, (config, i, len(recs))
        for k in range(N_EP):
            check_int_epoch(sp, dt, items[k], recs[k], pilots[k], (config, mode, i, k))
        assert len(np.unique(items["rem_code_phase_chips"])) > len(items) // 2
        if dt is not None:
            # the data prompt is not the pilot prompt
            assert np.any(recs["prompt_I"] != pilots.real)
        if config == "epl_1023_ring":
            assert items["sample_index"][0] < (1 << 32) < items["sample_index"][-1]


# ---------------------------------------------------------------------------------------------------------------------
# float data: a pilot and a data component on one carrier

@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("veml", [0, 1])
def test_float_data_prompt_within_the_float64_truth(capi, veml, mode):
    sp, dt = tl.pilot_data_spec(5, 25, 1234.0 if not veml else -2710.0, 1777, N_EP, veml=veml)
    e, ids, _ = tl.make_engine_with_data(capi, [sp], [dt], {0: len(sp.stream.x) + 16})
    tl.set_mode(e, mode, sp)
    tl.push_all(e, [sp])
    tl.start_all(e, ids, [sp])
    items, recs, pilots = run_per_epoch(e, ids, N_EP)[0]
    e.close()
    assert len(recs) == N_EP and np.all(items["phase_step_rad"] != 0.0)
    p = sp.taps // 2
    for k in range(N_EP):
        truth_d = tl.f64_taps(tl.data_view(sp, dt), items[k])[0]
        got = complex(float(recs[k]["prompt_I"]), float(recs[k]["prompt_Q"]))
        assert abs(got - truth_d) <= tl.TRUTH_RTOL * abs(truth_d), (mode, k, got, truth_d)
        truth = tl.f64_taps(sp, items[k])
        assert abs(complex(pilots[k]) - truth[p]) <= tl.TRUTH_RTOL * abs(truth[p]), (mode, k, pilots[k], truth[p])


# ---------------------------------------------------------------------------------------------------------------------
# nothing but the record's prompt moves

def twin_configs():
    rng = np.random.default_rng(77)
    port = tl.ol_port()
    lost = tl.lock_loss_case(rng)
    gal = tl.int_configs(N_EP)["galileo_like"][0][0]
    sp, dt = tl.pilot_data_spec(14, 29, 2222.0, 909, 300)
    return {
        "gps_float_3taps": (sp, dt, 300),
        "veml_sinboc_int": (gal, port.sinboc11((2 * rng.integers(0, 2, 4092) - 1).astype(np.int32)), N_EP),
        "gps_int_lock_loss": (lost, port.gps_ca_code(18), 120),
    }


PROMPT_FIELDS = ("prompt_I", "prompt_Q")   # zeroed on copies: a multi-field view would still carry their bytes


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("config", ["gps_float_3taps", "veml_sinboc_int", "gps_int_lock_loss"])
def test_a_data_channel_changes_nothing_but_the_record_prompt(capi, config, mode):
    sp, dt, n_ep = twin_configs()[config]
    caps = {0: len(sp.stream.x) + 16}
    out = []
    for data in ([dt], [None]):
        e, ids, _ = tl.make_engine_with_data(capi, [sp], data, caps)
        tl.set_mode(e, mode, sp)
        tl.push_all(e, [sp])
        tl.start_all(e, ids, [sp])
        rec, cnt, prm = e.loop_run_prompts(n_ep)
        out.append((rec[0, :cnt[0]], prm[0, :cnt[0]], bytes(e.loop_status(ids[0]))))
        e.close()
    (rd, pd, sd), (rt, pt, st) = out
    assert len(rd) == len(rt) and sd == st, (config, mode, len(rd), len(rt))
    if config == "gps_int_lock_loss":
        assert 40 < len(rd) < n_ep - 10
    else:
        assert len(rd) == n_ep
    a, b = rd.copy(), rt.copy()
    for f in PROMPT_FIELDS:
        a[f] = b[f] = 0.0
    assert a.tobytes() == b.tobytes(), (config, mode)
    twin_prompts = (rt["prompt_I"] + 1j * rt["prompt_Q"]).astype(np.complex64)
    assert pd.tobytes() == twin_prompts.tobytes(), (config, mode)
    assert pt.tobytes() == twin_prompts.tobytes(), (config, mode)
    assert np.any(rd["prompt_I"] != rt["prompt_I"])


@pytest.mark.parametrize("mode", tl.PERSISTENT)
@pytest.mark.parametrize("config", ["gps_float_3taps", "veml_sinboc_int", "gps_int_lock_loss"])
def test_persistent_taps_replay_through_step_taps(capi, config, mode):
    """the persistent kernel's pilot taps (rebuilt from the record and the returned pilot prompt) and its data tap, in the
    slot after the pilot taps, fed to the sequential update of a twin reproduce every item, record and the final status"""
    sp, dt, n_ep = twin_configs()[config]
    caps = {0: len(sp.stream.x) + 16}
    e, ids, _ = tl.make_engine_with_data(capi, [sp], [dt], caps)
    tl.set_mode(e, mode, sp)
    tl.push_all(e, [sp])
    tl.start_all(e, ids, [sp])
    items, recs, pilots = run_per_epoch(e, ids, n_ep)[0]
    st = e.loop_status(ids[0])
    e.close()
    lost = config == "gps_int_lock_loss"
    assert (st.state == 0 and st.loss_of_lock == 1) if lost else len(recs) == n_ep

    t, tids, _ = tl.make_engine_with_data(capi, [sp], [dt], caps)
    tl.push_all(t, [sp])
    tl.start_all(t, tids, [sp])
    for k in range(len(recs)):
        it = t.loop_peek_items()
        assert it[0].tobytes() == items[k].tobytes(), (config, mode, k)
        r = recs[k].copy()
        r["prompt_I"], r["prompt_Q"] = pilots[k].real, pilots[k].imag
        taps = np.zeros(8, np.complex64)
        taps[:sp.taps] = tl.rebuilt_taps(sp, r)
        taps[sp.taps] = complex(float(recs[k]["prompt_I"]), float(recs[k]["prompt_Q"]))
        got, logged = t.loop_step_taps(taps[None, :])
        assert logged[0] == 1 and got[0].tobytes() == recs[k].tobytes(), (config, mode, k)
    if lost:
        it = t.loop_peek_items()
        taps = np.zeros(8, np.complex64)
        taps[:sp.taps] = tl.int_taps(sp, it[0])
        _, logged = t.loop_step_taps(taps[None, :])
        assert logged[0] == 0
    s2 = t.loop_status(tids[0])
    t.close()
    assert bytes(st) == bytes(s2), (config, mode)


# ---------------------------------------------------------------------------------------------------------------------
# navigation symbols come out of the records

@pytest.mark.parametrize("mode", MODES)
def test_data_prompts_carry_the_symbols(capi, mode):
    n_ep, settle = 400, 100
    rng = np.random.default_rng(3)
    sym = (2 * rng.integers(0, 2, n_ep + 8) - 1).astype(np.float64)
    sp, dt = tl.pilot_data_spec(7, 22, 1500.0, 1234, n_ep, symbols=sym, cn0=50.0, pull_in_now=True)
    e, ids, _ = tl.make_engine_with_data(capi, [sp], [dt], {0: len(sp.stream.x) + 16})
    tl.set_mode(e, mode, sp)
    tl.push_all(e, [sp])
    tl.start_all(e, ids, [sp])
    rec, cnt, prm = e.loop_run_prompts(n_ep)
    e.close()
    assert cnt[0] == n_ep
    r, p = rec[0, settle:], prm[0, settle:]
    # the code period each record integrated over, as make_iq numbers them: the one under the middle of the epoch, which
    # ends about at PRN_start_sample_count
    mid = r["PRN_start_sample_count"].astype(np.float64) - sp.stream.x0 - 2000.0
    rate = tl.CA_RATE * (1.0 + 1500.0 / 1575.42e6) / tl.FS
    cp = (-1234 * tl.CA_RATE / tl.FS) % 1023
    period = np.floor((cp + mid * rate) / 1023).astype(np.int64)
    want = sym[period % len(sym)]
    got = np.sign(r["prompt_I"])
    assert np.all(got == want) or np.all(got == -want), (mode, np.count_nonzero(got != want))
    assert len(np.unique(np.sign(p.real))) == 1, mode
    assert np.all(np.abs(p.real) > np.abs(p.imag)), mode       # the PLL holds the pilot on the real axis


# ---------------------------------------------------------------------------------------------------------------------
# the call's rules, and replacing the data channel

def rule_engine(capi):
    sp = tl.gps_int_case(np.random.default_rng(1), 40)
    e, ids = tl.make_engine(capi, [sp], {0: len(sp.stream.x) + 16, 1: 1 << 16})
    return e, ids[0], sp


@pytest.mark.parametrize("rule", ["no_loop", "no_table", "three_taps", "other_band", "high_dynamics"])
def test_set_data_channel_refuses_each_broken_rule(capi, rule):
    e, lid, sp = rule_engine(capi)
    code = tl.ol_port().gps_ca_code(3)
    if rule == "no_loop":
        ch, bad_loop, msg = e.channel_create(0, 1), lid + 1, "no loop"
        e.channel_set_code(ch, code, [0.0])
    elif rule == "no_table":
        ch, bad_loop, msg = e.channel_create(0, 1), lid, "no code table"
    elif rule == "three_taps":
        ch, bad_loop, msg = e.channel_create(0, 3), lid, "has 3 correlators, the data channel needs 1"
        e.channel_set_code(ch, code, [-0.5, 0.0, 0.5])
    elif rule == "other_band":
        ch, bad_loop, msg = e.channel_create(1, 1), lid, "is on band 1, loop 0 on band 0"
        e.channel_set_code(ch, code, [0.0])
    else:
        ch, bad_loop, msg = e.channel_create(0, 1), lid, "high-dynamics"
        e.channel_set_code(ch, code, [0.0], high_dyn=True)
    with pytest.raises(capi.B200Error) as ei:
        e.loop_set_data_channel(bad_loop, ch)
    assert ei.value.code == -1 and msg in str(ei.value), str(ei.value)
    e.close()


@pytest.mark.parametrize("mode", MODES)
def test_replacing_the_data_channel_between_runs(capi, mode):
    n_ep = 40
    rng = np.random.default_rng(12)
    sp = tl.gps_int_case(rng, 2 * n_ep)
    port = tl.ol_port()
    tables = [port.gps_ca_code(11), port.gps_ca_code(12)]
    e, ids, dids = tl.make_engine_with_data(capi, [sp], [tables[0]], {0: len(sp.stream.x) + 16})
    second = e.channel_create(0, 1)
    e.channel_set_code(second, tables[1], [0.0])
    tl.set_mode(e, mode, sp)
    tl.push_all(e, [sp])
    tl.start_all(e, ids, [sp])
    for table in tables:
        items, recs, pilots = run_per_epoch(e, ids, n_ep)[0]
        assert len(recs) == n_ep
        for k in range(n_ep):
            check_int_epoch(sp, table, items[k], recs[k], pilots[k], (mode, k))
        e.loop_set_data_channel(ids[0], second)
    e.close()
