"""The rig of the device-loop tests (b200_trk_loop_*): loop specifications with the stream their band carries, engines
built from them in each loop mode, ring feeding, the integer cases and configurations, the exact references of a peeked
item (integer taps, float64 taps) and the per-epoch runner peek -> run(1).  The pilot + data helpers at the end give a
loop a 1-tap data channel beside its pilot."""
import types

import numpy as np

from oracle import loop as ol

FS = 4e6
CA_RATE = 1.023e6
TRUTH_RTOL = 1e-5
# name -> (loop mode, standby loops?).  Mode 0 runs 512-thread CTAs up to one loop per SM and 256-thread CTAs beyond.
MODES = {"persistent256": (0, True), "persistent512": (0, False), "per_epoch": (1, False), "sliced": (2, False)}
PERSISTENT = ["persistent256", "persistent512"]


def set_mode(e, name, sp):
    """loop mode `name` of MODES on engine e, whose channel 0 is sp's pilot channel (make_engine creates it first).
    persistent256 adds one standby loop per SM there, never started: in state 0 it leaves the persistent kernel at its first
    prepare, so the started loops' taps and records do not change.  Standby rows follow the started loops' in every
    per-loop array and hold nothing defined."""
    import torch
    mode, standby = MODES[name]
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    for _ in range(sms if standby else 0):
        e.loop_create(0, sp.conf)
    if mode == 0:
        n_loops = len(e.loop_run(0)[1])          # a run of no epochs launches nothing and returns one count per loop
        assert (n_loops > sms) == standby, (name, n_loops, sms)
    e.loop_set_mode(mode)


def shifts_of(conf):
    spc, els = conf.code_samples_per_chip, conf.early_late_space_chips
    if conf.veml:
        return [-0.5 * spc, -els * spc, 0.0, els * spc, 0.5 * spc]
    return [-els * spc, 0.0, els * spc]


def int_signal(rng, table, n, amp, code_phase, rate, noise=2):
    """round(amp * code(t - tau)) + uniform integer noise in [-noise, noise]: real integers (int64[n])"""
    t = np.arange(n, dtype=np.float64)
    idx = np.floor(code_phase + t * rate).astype(np.int64) % len(table)
    return np.rint(amp * table[idx]).astype(np.int64) + rng.integers(-noise, noise + 1, n)


class Stream:
    """The samples of one band: host copy x (int64 or complex64) starting at absolute index x0."""

    def __init__(self, x, x0):
        self.x, self.x0 = x, x0

    def seg(self, s, n):
        a = int(s) - self.x0
        assert 0 <= a and a + n <= len(self.x), (s, n, self.x0, len(self.x))
        return self.x[a:a + n]


class LoopSpec:
    """One loop: band, code table, configuration, start (acq delay, acq Doppler, acq stamp, nitems_read) and the
    stream its band carries (for the reference)."""

    def __init__(self, band, table, conf, start, stream):
        self.band, self.table, self.conf, self.start, self.stream = band, np.asarray(table, np.float32), conf, start, stream
        self.shifts = shifts_of(conf)
        self.taps = len(self.shifts)


def make_engine(capi, specs, capacities):
    e = capi.Engine()
    for band, cap in capacities.items():
        e.iq_create(band, cap)
    ids = []
    for sp in specs:
        ch = e.channel_create(sp.band, sp.taps)
        e.channel_set_code(ch, sp.table, sp.shifts)
        ids.append(e.loop_create(ch, sp.conf))
    return e, ids


def start_all(e, ids, specs):
    for lid, sp in zip(ids, specs):
        e.loop_start(lid, *sp.start)


def int_taps(sp, item):
    """exact integer taps of one peeked item on integer data"""
    n = int(item["n"])
    _, idx = ol_port().resampler(1, sp.table, float(item["rem_code_phase_chips"]), float(item["code_phase_step_chips"]), sp.shifts, n,
                                 return_idx=True)
    x = sp.stream.seg(item["sample_index"], n)
    return (x[None, :] * sp.table.astype(np.int64)[idx]).sum(axis=1)


def f64_taps(sp, item):
    n = int(item["n"])
    return ol_port().multicorrelator_f64(1, sp.stream.seg(item["sample_index"], n), sp.table, sp.shifts, float(item["rem_carrier_phase_rad"]),
                                         float(item["phase_step_rad"]), float(item["rem_code_phase_chips"]),
                                         float(item["code_phase_step_chips"]), n)


def ol_port():
    import oracle
    return oracle.port


def rec_mags(sp, r):
    return np.array([r["abs_VE"], r["abs_E"], r["abs_P"], r["abs_L"], r["abs_VL"]] if sp.taps == 5 else [r["abs_E"], r["abs_P"], r["abs_L"]],
                    np.float64)


def check_int_epoch(sp, item, r, what):
    assert item["rem_carrier_phase_rad"] == 0.0 and item["phase_step_rad"] == 0.0 and item["phase_rate_step_rad"] == 0.0, (what, item)
    want = int_taps(sp, item)
    p = sp.taps // 2
    assert r["prompt_I"] == want[p] and r["prompt_Q"] == 0.0, (what, r["prompt_I"], r["prompt_Q"], want)
    assert np.array_equal(rec_mags(sp, r), np.abs(want).astype(np.float64)), (what, rec_mags(sp, r), want)
    if sp.taps == 3:
        assert r["abs_VE"] == 0.0 and r["abs_VL"] == 0.0, what

def run_per_epoch(e, ids, n_ep, feed=None):
    """peek -> run(1), n_ep times.  feed(items) pushes what the peeked items need first.
    -> per loop: (items, records) of the epochs that logged a record"""
    items_out = [[] for _ in ids]
    recs_out = [[] for _ in ids]
    for _ in range(n_ep):
        items = e.loop_peek_items()
        if feed is not None:
            feed(items)
        rec, cnt = e.loop_run(1)
        for i in range(len(ids)):
            if cnt[i]:
                items_out[i].append(items[i])
                recs_out[i].append(rec[i, 0])
    return [(np.array(a, items.dtype), np.array(b, rec.dtype)) for a, b in zip(items_out, recs_out)]


# ---------------------------------------------------------------------------------------------------------------------
# configurations with integer data

RING_BASE = (1 << 32) - 50_000          # absolute indices cross 2^32 inside the run
RING_CAP = 1 << 15


def gps_int_case(rng, n_ep, base=0, delay=1234, amp=3.0, code_ppm=0.0, conf_kw=None, prn=1, extra=8000):
    code = ol_port().gps_ca_code(prn)
    rate = CA_RATE * (1 + code_ppm * 1e-6) / FS
    x = int_signal(rng, code, 4000 * n_ep + delay + extra, amp, (-delay * rate) % 1023, rate)
    conf = ol.default_conf(fs_in=FS, prn=prn, **(conf_kw or {}))
    return LoopSpec(0, code, conf, (delay + 0.3, 0.0, base, base), Stream(x, base))


def galileo_int_case(rng, n_ep, band=0, base=0):
    primary = (2 * rng.integers(0, 2, 4092) - 1).astype(np.int32)
    table = ol_port().sinboc11(primary)
    L = len(table)
    rate = CA_RATE * 2.0 / FS                                          # table entries per sample
    cp = 2711.0
    delay = ((L - cp) % L) / rate
    x = int_signal(rng, table, 16000 * (n_ep + 4), 4.0, cp, rate)
    conf = ol.default_conf(fs_in=FS, prn=1, code_length_chips=4092, code_period=0.004, vector_length=16000, code_samples_per_chip=2,
                           veml=1, early_late_space_chips=0.15)
    return LoopSpec(band, table, conf, (delay + 0.2, 0.0, base, base), Stream(x, base))


def veml_int_case(rng, n_ep):
    code = np.repeat(ol_port().gps_ca_code(7), 2)
    delay = 2222
    rate = 2 * CA_RATE / FS
    x = int_signal(rng, code, 4000 * (n_ep + 2), 3.0, (-delay * rate) % len(code), rate)
    conf = ol.default_conf(fs_in=FS, prn=7, veml=1, code_samples_per_chip=2, early_late_space_chips=0.15, cn0_samples=10)
    return LoopSpec(0, code, conf, (delay - 0.4, 0.0, 0, 0), Stream(x, 0))


def int_configs(n_ep):
    """name -> (specs, band capacities, ring-fed?)"""
    rng = np.random.default_rng(2024)
    ring = gps_int_case(rng, n_ep, base=RING_BASE, amp=1.0)
    two_a = gps_int_case(rng, n_ep, delay=3001, prn=9)
    two_b = galileo_int_case(rng, n_ep, band=1, base=5_000_000)
    return {
        "gps_ring": ([ring], {0: RING_CAP}, True),
        "veml_2spc": ([veml_int_case(rng, n_ep)], None, False),
        "galileo_like": ([galileo_int_case(rng, n_ep)], None, False),
        "two_bands": ([two_a, two_b], None, False),
    }


class RingFeeder:
    """Pushes a band's stream into a small ring block by block, never ahead of what the ring can hold behind the loop."""

    def __init__(self, e, band, stream, block=8192):
        self.e, self.band, self.s, self.block = e, band, stream, block
        self.pos = 0
        e.iq_push_at(band, stream.x0, stream.x[:0].astype(np.complex64))

    def push_block(self):
        blk = self.s.x[self.pos:self.pos + self.block]
        if len(blk):
            self.e.iq_push_at(self.band, self.s.x0 + self.pos, blk.astype(np.complex64))
            self.pos += len(blk)
        return len(blk)

    def until(self, end):
        while self.s.x0 + self.pos < end and self.push_block():
            pass


def push_all(e, specs):
    seen = set()
    for sp in specs:
        if sp.band not in seen:
            seen.add(sp.band)
            e.iq_push_at(sp.band, sp.stream.x0, sp.stream.x.astype(np.complex64))


def capacities_for(specs, caps):
    if caps is not None:
        return caps
    return {sp.band: len(sp.stream.x) + 16 for sp in specs}


# ---------------------------------------------------------------------------------------------------------------------
# a loop that loses lock, and the taps a record carries

def lock_loss_case(rng):
    """integer data; cn0_min above the signal's C/N0 (about 70 dB-Hz), no pull-in time and the acquisition stamp a
    second before the first sample: the code-lock counter runs out after about 85 epochs"""
    base = 4_000_000
    sp = gps_int_case(rng, 120, conf_kw=dict(pull_in_time_s=0, max_code_lock_fail=60, cn0_min=80), prn=17)
    sp.start = (sp.start[0], 0.0, 0, base)
    sp.stream = Stream(sp.stream.x, base)      # 4e6 samples are exactly 1000 code periods: same code phase
    return sp


def rebuilt_taps(sp, r):
    """the taps of a record, exact for 3-tap loops and for integer data: P = (prompt_I, prompt_Q), the others (|tap|, 0)"""
    p = complex(float(r["prompt_I"]), float(r["prompt_Q"]))
    if sp.taps == 3:
        return np.array([r["abs_E"], p, r["abs_L"]], np.complex64)
    return np.array([r["abs_VE"], r["abs_E"], p, r["abs_L"], r["abs_VL"]], np.complex64)


# ---------------------------------------------------------------------------------------------------------------------
# the loops' sample window is [valid_from, write_index)

DELAY = 1234


def gps_stream(rng, prn, x0, n):
    """integer GPS C/A samples from absolute index x0 whose code starts DELAY samples after x0 (and every 4000 after)"""
    code = ol_port().gps_ca_code(prn)
    rate = CA_RATE / FS
    return code, Stream(int_signal(rng, code, n, 3.0, (-DELAY * rate) % 1023, rate), x0)


def window_engine(capi, mode, specs, caps):
    e, ids = make_engine(capi, specs, caps)
    set_mode(e, mode, specs[0])
    return e, ids


def other_band(rng, n_ep):
    """a loop on band 1 that must run undisturbed through whatever happens on band 0"""
    code, s = gps_stream(rng, 21, 0, 4000 * n_ep + 12000)
    return LoopSpec(1, code, ol.default_conf(fs_in=FS, prn=21), (DELAY + 0.3, 0.0, 0, 0), s)


def check_loop(sp, res, n, what):
    items, recs = res
    assert len(recs) == n, (what, len(recs), n)
    for k in range(n):
        check_int_epoch(sp, items[k], recs[k], (what, k))


# ---------------------------------------------------------------------------------------------------------------------
# a pilot loop with a data channel (b200_trk_loop_set_data_channel)

def data_view(sp, table):
    """the data correlator as the oracle sees it: one tap at the prompt's shift (0), the loop's stream"""
    return types.SimpleNamespace(table=np.asarray(table, np.float32), shifts=[0.0], taps=1, stream=sp.stream)


def make_engine_with_data(capi, specs, data_tables, caps):
    """make_engine plus a 1-tap data channel for every spec whose data table is not None -> (engine, loop ids, data ids)"""
    e, ids = make_engine(capi, specs, caps)
    dids = []
    for lid, sp, dt in zip(ids, specs, data_tables):
        if dt is None:
            dids.append(None)
            continue
        dch = e.channel_create(sp.band, 1)
        e.channel_set_code(dch, dt, [0.0])
        e.loop_set_data_channel(lid, dch)
        dids.append(dch)
    return e, ids, dids


def pilot_data_spec(prn, data_prn, doppler, delay, n_ep, veml=0, symbols=None, cn0=55.0, pull_in_now=False):
    """GPS-like pilot (code prn) + data (code data_prn) with the same Doppler and code phase; symbols (+-1, one per code
    period) modulate the data.  pull_in_now: the acquisition stamp lies a second before the first sample, so the loop
    leaves its pull-in transitory at once and the PLL (not the FLL alone) steers from the first epoch."""
    from gnss_synth import make_iq
    port = ol_port()
    spc = 2 if veml else 1
    pilot = np.repeat(port.gps_ca_code(prn), spc)
    data = np.repeat(port.gps_ca_code(data_prn), spc)
    n = 4000 * (n_ep + 2) + delay
    cp = (-delay * spc * CA_RATE / FS) % len(pilot)
    common = dict(doppler=doppler, code_phase_chips=cp, cn0=cn0, phase0=0.7)
    iq = make_iq({prn: pilot, data_prn: data}, FS, n, [dict(prn=prn, **common), dict(prn=data_prn, symbols=symbols, **common)],
                 seed=prn, chips_per_table_chip=spc)
    kw = dict(veml=1, code_samples_per_chip=2, early_late_space_chips=0.15) if veml else {}
    base = 4_000_000 if pull_in_now else 0       # 4e6 samples are exactly 1000 code periods: same code phase
    conf = ol.default_conf(fs_in=FS, prn=prn, pull_in_time_s=0 if pull_in_now else 1, cloop=0, **kw)
    sp = LoopSpec(0, pilot, conf, (delay + 0.2, doppler - (0.0 if pull_in_now else 6.0), 0, base), Stream(iq, base))
    return sp, data
