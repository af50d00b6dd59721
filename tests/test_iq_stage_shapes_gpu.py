"""The device input filters (conditioner, pulse blanker, notch) at the shapes where their launchers change path, against
the same restatements as their own test modules (iq_conditioner_np, pulse_blanking_np, notch_np), read back with
b200_iq_read after every push.

  - conditioner CTA widths: per_cta = min(128, (12672 - 2 T) / D + 1) from 2 to 128, T and D up to 4096, partial last
    CTAs, destinations as small as the band rule allows, and a source ring of exactly T samples pushed one at a time;
  - blanker energy staging at L > 2048 (one segment per CTA) and L = 4096, and a push long enough that the apply kernel's
    grid-stride loop goes round;
  - multi-step scans (more than 1024 segments in one push) for the blanker and both notch variants, with resets in later
    steps, estimation resumed mid-step, Lite epochs that cross steps and pushes, and a push of exactly 2048 segments;
  - the notch's compose / apply grid over 2 to 9 CTAs with pushes that start and end mid grid block, and its floor kernel
    at L = 1023 and 1024;
  - stage origins past 2^32 and near 2^40 after a push_at gap, direct and behind a conditioner, with Lite's zero history item;
  - one source feeding a conditioner, a blanker and a notch, the conditioner feeding two more stages: the push limit is
    the least of theirs, a push one longer is refused, and every accepted push launches what its completed segments need;
  - full-scale integer samples (-32768, -128) through every stage at its largest length."""
import math

import numpy as np
import pytest

import acq_rig as ar
import iq_conditioner_np as cnp
import notch_np as nn
import pulse_blanking_np as pnp
from gpu_fixtures import capi, engine  # noqa: F401

pytestmark = pytest.mark.gpu

ERR_RANGE = -5
FS = 25e6
COND_SMEM_FLOAT2 = 99 * 1024 // 8          # the conditioner's shared-memory budget in float2
LIMITS = {"ishort": (-32768, 32767), "ibyte": (-128, 127)}


# ---- streams -------------------------------------------------------------------------------------------------------

def _as_item(x, item_type):
    """complex samples -> (what a push of item_type takes, the complex64 samples the band holds)"""
    if item_type == "gr_complex":
        x = np.asarray(x, np.complex64)
        return x, x
    raw = ar.to_int(x, np.int16 if item_type == "ishort" else np.int8, 1.0, clip=LIMITS[item_type])
    return raw, ar.from_int(raw)


def _cw_bursts(rng, n, item_type, on, cw=6.0):
    """n samples of complex noise with a CW switched on over the sample ranges `on`"""
    sigma = 12.0 if item_type == "ibyte" else 300.0
    x = rng.normal(0, sigma / math.sqrt(2), n) + 1j * rng.normal(0, sigma / math.sqrt(2), n)
    t = np.arange(n)
    gate = np.zeros(n, bool)
    for a, b in on:
        gate[a:b] = True
    x = x + gate * cw * sigma * np.exp(1j * (0.41 * t + 0.3))
    return _as_item(x, item_type)


def _periodic(n, period, width, offset=0):
    return [(a, a + width) for a in range(offset, n, period)]


def _push(e, band, raw, item_type, a, b):
    """samples [a, b) of raw into band"""
    if item_type == "gr_complex":
        return e.iq_push(band, raw[a:b])
    return e.iq_push_int(band, raw[2 * a:2 * b])


def _odd_sizes(rng, total, lo, hi, first=()):
    """push sizes summing to total: `first`, then odd sizes in [lo, hi]"""
    sizes, pos = list(first), sum(first)
    while pos < total:
        n = min(int(rng.integers(lo, hi + 1)) | 1, hi, total - pos)
        sizes.append(n)
        pos += n
    return sizes


# ---- segment stages: set, restate, check ---------------------------------------------------------------------------

def _blanker(length, est, reset, pfa=0.04):
    return dict(kind="blanker", L=length, E=est, R=reset, pfa=pfa)


def _notch(variant, length, est, reset, n_coeff=1, p=0.9, pfa=1e-3):
    return dict(kind="notch", variant=variant, L=length, E=est, R=reset, nc=n_coeff, p=p, pfa=pfa)


def _set(e, dst, src, s):
    if s["kind"] == "blanker":
        e.iq_set_pulse_blanking(dst, src, s["pfa"], s["L"], s["E"], s["R"])
    else:
        e.iq_set_notch(dst, src, s["variant"], s["pfa"], s["p"], s["L"], s["E"], s["R"], s["nc"])


def _reach(s):
    """source samples beyond the published segments the stage may still read (engine.cu, stage_reach)"""
    if s["kind"] == "blanker":
        return s["L"] - 1
    return s["L"] + (1 if s["variant"] == nn.NOTCH_LITE and s["L"] == 1 else 0)


def _lead(s):
    return 0 if s["kind"] == "blanker" else nn.lead(s["variant"], s["L"])


def _f32(v):
    return np.float32(v).tobytes()


class _Restated:
    """The restatement of one segment stage over a stream that starts at its origin, pushed in pieces: check() compares
    the destination's window, its new samples and the stage's status after every push."""

    def __init__(self, s, held, origin=0):
        self.s, self.origin, self.done = s, origin, origin
        if s["kind"] == "blanker":
            self.ref = pnp.Blanker(s["pfa"], s["L"], s["E"], s["R"])
            self.fed = 0
            self.held = held
        else:
            self.res = nn.run(held, s["variant"], s["pfa"], s["p"], s["L"], s["E"], s["R"], s["nc"])

    def segments(self, pushed):
        """segments published once `pushed` samples from the origin are in the source"""
        return max(0, pushed - _lead(self.s)) // self.s["L"]

    def check(self, e, band, pushed):
        s, L = self.s, self.s["L"]
        if s["kind"] == "blanker":
            want = self.ref.push(self.held[self.fed:pushed])
            self.fed = pushed
            k = self.ref.segments
        else:
            k = self.segments(pushed)
            want = self.res["out"][self.done - self.origin:k * L]
        hi = self.origin + k * L
        assert e.iq_window(band)[1] == hi == self.done + want.size, (e.iq_window(band), hi, self.done)
        if want.size:
            got = e.iq_read(band, self.done, want.size)
            assert got.tobytes() == want.tobytes(), (band, pushed, self.done + np.flatnonzero(got != want)[:5])
        self.done = hi
        self.check_status(e, band, k)
        return k

    def check_status(self, e, band, k):
        s = self.s
        if s["kind"] == "blanker":
            st = e.iq_pulse_blanking_status(band)
            assert st["origin"] == self.origin and st["length"] == s["L"]
            assert _f32(st["threshold"]) == _f32(self.ref.thres)
            for key, v in self.ref.state().items():
                if key == "noise_power":
                    assert _f32(st[key]) == _f32(v), (key, st[key], v)
                else:
                    assert st[key] == v, (key, st, self.ref.state())
            return
        st = e.iq_notch_status(band)
        assert (st["origin"], st["segments"], st["length"], st["variant"]) == (self.origin, k, s["L"], s["variant"])
        assert _f32(st["threshold"]) == _f32(self.res["thres"])
        if k == 0:
            return
        want = nn.state_after(self.res, k)
        for key in ("filtered", "n", "filter_state", "n_coeff"):
            assert st[key] == want[key], (key, st, want)
        assert _f32(st["noise_power"]) == _f32(want["noise_power"])
        assert _f32(st["z0"].real) == _f32(want["z0"][0]) and _f32(st["z0"].imag) == _f32(want["z0"][1]), (st["z0"], want["z0"])
        assert _f32(st["last_out"].real) == _f32(want["last_out"][0]) and _f32(st["last_out"].imag) == _f32(want["last_out"][1])

    def check_bound(self):
        """notch: filtered samples within the float32 recursion's bound of the float64 truth"""
        if self.s["kind"] != "notch":
            return
        res, filt = self.res, self.res["filt"]
        if filt.any():
            err = np.max(np.abs(res["out"][filt].astype(np.complex128) - res["truth"][filt]))
            assert err <= nn.recursion_bound(res, self.s["p"]), (err, nn.recursion_bound(res, self.s["p"]))


def _run_stage(e, s, item_type, raw, held, sizes, src_cap, src=0, dst=1):
    """s reading a fresh source band of src_cap samples of item_type; the pieces `sizes` of raw pushed one by one, each
    checked; -> the restatement"""
    e.iq_create(src, src_cap, item_type)
    e.iq_create(dst, src_cap)
    _set(e, dst, src, s)
    ref = _Restated(s, held)
    ref.check_status(e, dst, 0)
    pos = 0
    for n in sizes:
        _push(e, src, raw, item_type, pos, pos + n)
        pos += n
        ref.check(e, dst, pos)
    ref.check_bound()
    return ref


# ---- 1. conditioner CTA widths -------------------------------------------------------------------------------------

def _cond_per_cta(t, d):
    """outputs per CTA of launch_iq_condition"""
    return min(128, max(1, (COND_SMEM_FLOAT2 - 2 * t) // d + 1))


def _ulps(got, want):
    sp = np.spacing(np.abs(want).astype(np.float32)).astype(np.float64)
    return np.maximum(np.abs(got.real - want.real), np.abs(got.imag - want.imag)) / sp


# (T, D, per_cta, source capacity)
COND_SHAPES = [(1, 100, 127, 1 << 14), (1, 4096, 4, 1 << 17), (4096, 1, 128, 1 << 13), (4096, 36, 125, 1 << 16),
               (4096, 4096, 2, 1 << 17), (241, 127, 96, 1 << 14)]


@pytest.mark.parametrize("if_hz", [0.0, 1.7e6])
@pytest.mark.parametrize("item_type", ["gr_complex", "ibyte"])
@pytest.mark.parametrize("t,d,per_cta,src_cap", COND_SHAPES)
def test_conditioner_cta_widths(engine, t, d, per_cta, src_cap, item_type, if_hz):
    """two and a bit times around the source ring in pushes of up to capacity - (T - 1) samples, the first of exactly that
    size; the destination ring is the smallest power of two whose capacity times D holds the source"""
    e = engine
    assert _cond_per_cta(t, d) == per_cta
    rng = np.random.default_rng(7 * t + d)
    h = rng.normal(0, 1.0 / math.sqrt(t), t).astype(np.float32)
    dst_cap = ar.pow2(cnp.ceil_div(src_cap, d))
    assert dst_cap * d >= src_cap > dst_cap // 2 * d
    e.iq_create(0, src_cap, item_type)
    e.iq_create(1, dst_cap)
    e.iq_set_conditioner(1, 0, d, h, if_hz, FS)
    total = 2 * src_cap + 123
    raw, held = _as_item(rng.normal(0, 40, total) + 1j * rng.normal(0, 40, total), item_type)
    m = cnp.ceil_div(total, d)
    want = cnp.condition_f32(held, 0, h, d, if_hz, FS, 0, m)
    if if_hz:
        truth, scale = cnp.condition_f64(held, 0, h, d, if_hz, FS, 0, m)
    limit = src_cap - (t - 1)
    pos, partial = 0, 0
    for n in _odd_sizes(rng, total, limit // 3, limit, first=(limit,)):
        _push(e, 0, raw, item_type, pos, pos + n)
        j0, j1 = cnp.ceil_div(pos, d), cnp.ceil_div(pos + n, d)
        pos += n
        assert e.iq_window(1)[1] == j1
        partial += (j1 - j0) % per_cta != 0
        if j1 == j0:
            continue
        got = e.iq_read(1, j0, j1 - j0)
        if not if_hz:
            assert got.tobytes() == want[j0:j1].tobytes(), (pos, j0 + np.flatnonzero(got != want[j0:j1])[:5])
        else:
            assert np.max(_ulps(got, want[j0:j1])) <= 2.0, pos
            assert np.all(np.abs(got - truth[j0:j1]) <= (t + 4) * 2.0 ** -23 * scale[j0:j1]), pos
    assert partial > 0 and pos > src_cap + limit


def test_conditioner_source_of_exactly_t_samples(capi, engine):
    """a source ring of T samples takes one sample per push: three times around it, each output checked"""
    e = engine
    rng = np.random.default_rng(3)
    t, d = 8, 3
    h = rng.normal(0, 0.3, t).astype(np.float32)
    e.iq_create(2, t)
    e.iq_create(3, 4)
    e.iq_set_conditioner(3, 2, d, h, 0.0, FS)
    x = (rng.normal(0, 100, 3 * t + 5) + 1j * rng.normal(0, 100, 3 * t + 5)).astype(np.complex64)
    want = cnp.condition_f32(x, 0, h, d, 0.0, FS, 0, cnp.ceil_div(x.size, d))
    with pytest.raises(capi.B200Error) as r:
        e.iq_push(2, x[:2])
    assert r.value.code == ERR_RANGE
    for i in range(x.size):
        e.iq_push(2, x[i:i + 1])
        j1 = cnp.ceil_div(i + 1, d)
        assert e.iq_window(3)[1] == j1
        if i % d == 0:                                                     # this sample completed output j1 - 1
            assert e.iq_read(3, j1 - 1, 1).tobytes() == want[j1 - 1:j1].tobytes(), i
    lo, hi = e.iq_window(3)
    assert hi == want.size and e.iq_read(3, lo, hi - lo).tobytes() == want[lo:].tobytes()


# ---- 2. blanker lengths and grid -----------------------------------------------------------------------------------

@pytest.mark.parametrize("length", [33, 2048, 2049, 4096])
@pytest.mark.parametrize("item_type", ["gr_complex", "ishort", "ibyte"])
def test_blanker_long_segments(engine, item_type, length):
    """energy staging at 124, 2 and 1 segments per CTA: twice around a 2^14 ring, CW bursts on some segments; the
    compiled block too on the prefix it publishes"""
    rng = np.random.default_rng(length + len(item_type))
    cap = 1 << 14
    total = 2 * cap + 123
    segs = total // length
    s = _blanker(length, segs // 20 + 1, max(1, segs // 8))
    raw, held = _cw_bursts(rng, total, item_type, _periodic(total, max(1500, 5 * length), max(200, 2 * length), 700))
    limit = cap - (length - 1)
    sizes = _odd_sizes(rng, total, limit // 4, limit, first=(limit,))
    ref = _run_stage(engine, s, item_type, raw, held, sizes, cap)
    assert 0 < ref.ref.blanked < ref.ref.segments
    lib = pnp.reference_filter()
    if lib is not None:
        out, thres, _ = pnp.reference_block(lib, held, s["pfa"], length, s["E"], s["R"], np.cumsum(sizes))
        assert thres == ref.ref.thres
        lo, hi = engine.iq_window(1)
        assert out.size > lo
        assert engine.iq_read(1, lo, out.size - lo).tobytes() == out[lo:].tobytes()


def test_blanker_apply_grid_strides(engine):
    """one push of 2^22 - 31 samples: more than the 132 x 64 CTAs x 256 threads of the apply grid, so its loop strides"""
    rng = np.random.default_rng(22)
    cap, length = 1 << 22, 32
    n = cap - (length - 1)
    assert n > 132 * 64 * 256
    s = _blanker(length, 50, 20_000)
    raw, held = _cw_bursts(rng, n + 4000, "gr_complex", _periodic(n + 4000, 9000, 700, 100))
    ref = _run_stage(engine, s, "gr_complex", raw, held, [n, 4000], cap, src=4, dst=5)
    assert ref.ref.blanked > 100 and ref.ref.segments == (n + 4000) // length


# ---- 3. multi-step scans -------------------------------------------------------------------------------------------

STEP = 1024
MULTI_L = 4
MULTI_SEGS = 4 * STEP + 1                    # the first push: four and a bit scan steps
# CW runs in segments: across the step boundaries 1024, 2048 and 3072; one covering the whole fourth step and the end of
# the first push (segment 4097); one across the end of the second push (6145, after exactly 2048 segments)
MULTI_RUNS = [(300, 340), (1000, 1060), (2030, 2080), (3069, 4200), (6100, 6150), (7000, 7040), (7600, 7700)]


def _resets(s, held, n_seg):
    """segments k > 0 at which the state machine resets (n becomes 1) among the first n_seg"""
    L = s["L"]
    if s["kind"] == "notch":
        ns = nn.run(held[:n_seg * L + 1], s["variant"], s["pfa"], s["p"], L, s["E"], s["R"], s["nc"])["rec"]["n"][:n_seg]
    else:
        b, ns = pnp.Blanker(s["pfa"], L, s["E"], s["R"]), []
        for k in range(n_seg):
            b.push(held[k * L:(k + 1) * L])
            ns.append(b.n)
    return [k for k in range(1, n_seg) if ns[k] == 1]


MULTI = [("blanker", _blanker(MULTI_L, 20, 300)),
         ("notch", _notch(nn.NOTCH, MULTI_L, 20, 300)),
         ("lite_nc3", _notch(nn.NOTCH_LITE, MULTI_L, 20, 300, 3)),
         ("lite_nc1031", _notch(nn.NOTCH_LITE, MULTI_L, 20, 300, 1031))]


@pytest.mark.parametrize("s", [m[1] for m in MULTI], ids=[m[0] for m in MULTI])
def test_multi_step_scans(engine, s):
    """a push of 4097 segments, one of exactly 2048, then odd pushes; resets fall in the second and third steps of the
    first push, estimation resumes inside them, and filtered runs cross steps and pushes (Lite's 1031-segment epoch from
    segment 3069 covers the fourth step and ends in the second push)"""
    rng = np.random.default_rng(31 + s.get("nc", 0))
    L, lead = s["L"], _lead(s)
    total = 40_000
    raw, held = _cw_bursts(rng, total, "gr_complex", [(a * L, b * L) for a, b in MULTI_RUNS])
    resets = _resets(s, held, MULTI_SEGS)
    assert any(STEP <= k < 2 * STEP for k in resets) and any(2 * STEP <= k < 3 * STEP for k in resets), resets
    first = (MULTI_SEGS * L + lead, 2 * STEP * L)
    cap = 1 << 15
    sizes = _odd_sizes(rng, total, 1, 3001, first=first)
    ref = _run_stage(engine, s, "gr_complex", raw, held, sizes, cap)
    k = ref.segments(total)
    if s["kind"] == "notch":
        flags = ref.res["flags"]
        assert flags[MULTI_SEGS - 1] & 1 and flags[MULTI_SEGS] & 1              # a run across the end of the first push
        assert flags[STEP - 1] & 1 and flags[STEP] & 1 and flags[2 * STEP - 1] & 1 and flags[2 * STEP] & 1
        if s["nc"] == 1031:
            assert (flags[3069:4200] & 1).all() and (flags[3068] & 1) == 0       # one epoch: the whole fourth step and 4097
    else:
        assert 0 < ref.ref.blanked < k


# ---- 4. notch grid and lengths -------------------------------------------------------------------------------------

@pytest.mark.parametrize("variant", [nn.NOTCH, nn.NOTCH_LITE])
def test_notch_grid_ctas(capi, engine, variant):
    """pushes of 2^18 - L and 2^20 - L samples (the second at the push limit capacity - L: 1025 grid blocks, 9 CTAs),
    then pushes that start and end mid grid block; the CW is on across every push boundary"""
    e = engine
    rng = np.random.default_rng(40 + variant)
    L, cap = 32, 1 << 20
    s = _notch(variant, L, 10, 100_000)
    sizes = [(1 << 18) - L, cap - L, 3001, 40_013, 77_777]
    total = sum(sizes)
    ends = np.cumsum(sizes)
    on = [(100_000, 300_000), (700_000, 900_000)] + [(int(b) - 20_000, int(b) + 20_000) for b in ends[1:-1]]
    raw, held = _cw_bursts(rng, total, "gr_complex", on)
    e.iq_create(6, cap)
    e.iq_create(7, cap)
    _set(e, 7, 6, s)
    ref = _Restated(s, held)
    pos = 0
    for n in sizes:
        r0 = ref.segments(pos) * L
        e.iq_push(6, raw[pos:pos + n])
        pos += n
        r1 = ref.segments(pos) * L
        assert r0 % nn.GRID or pos == sizes[0]                                  # pushes after the first start mid block
        ref.check(e, 7, pos)
        nb = (r1 - 1) // nn.GRID - r0 // nn.GRID + 1
        if n >= (1 << 18) - L:
            assert cnp.ceil_div(nb, 128) >= 2
    with pytest.raises(capi.B200Error) as r:
        e.iq_push(6, raw[:cap - L + 1])
    assert r.value.code == ERR_RANGE
    ref.check_bound()
    filt = ref.res["filt"]
    assert all(filt[int(b) - 100] and filt[int(b) + 100] for b in ends[:-1])  # filtered on either side of each push end


@pytest.mark.parametrize("length", [1023, 1024])
@pytest.mark.parametrize("variant", [nn.NOTCH, nn.NOTCH_LITE])
def test_notch_longest_segments(engine, variant, length):
    """the floor kernel at 1023 and 1024 threads: twice around a 2^14 ring with small E and R"""
    rng = np.random.default_rng(length + variant)
    cap = 1 << 14
    total = 2 * cap + 123
    segs = total // length
    s = _notch(variant, length, segs // 10 + 1, segs // 4, 2)
    raw, held = _cw_bursts(rng, total, "gr_complex", _periodic(total, 6 * length, 3 * length, length))
    limit = cap - _reach(s)
    ref = _run_stage(engine, s, "gr_complex", raw, held, _odd_sizes(rng, total, limit // 4, limit, first=(limit,)), cap)
    flags = ref.res["flags"]
    assert 0 < int((flags & 1).sum()) < flags.size


# ---- 5. far origins ------------------------------------------------------------------------------------------------

FAR = [("blanker", _blanker(32, 5, 40), None),
       ("notch", _notch(nn.NOTCH, 32, 0, 40), None),
       ("lite", _notch(nn.NOTCH_LITE, 32, 0, 40, 2), None),
       ("lite_l1", _notch(nn.NOTCH_LITE, 1, 0, 40, 2), None),
       ("cond_blanker", _blanker(32, 5, 40), (5, 9)),
       ("cond_lite", _notch(nn.NOTCH_LITE, 16, 0, 40, 2), (5, 9))]




@pytest.mark.parametrize("g", [(1 << 32) + 777, (1 << 40) - 4999], ids=["past_2_32", "near_2_40"])
@pytest.mark.parametrize("s,cond", [f[1:] for f in FAR], ids=[f[0] for f in FAR])
def test_far_origins(engine, s, cond, g):
    """a stage (or a conditioner (D, T) then a stage) that has run from 0 restarts at a push_at gap at g: its origin is g,
    or ceil((g + T - 1) / D) behind the conditioner, and its destination is the restatement of the stream after the gap.
    The 12 000 samples pushed before the gap leave an old sample in the source slot of g - 1; the notches run with E = 0,
    so they filter from their first segment and Lite reads its zero history item there instead"""
    e = engine
    rng = np.random.default_rng(g % 1000 + s["L"])
    cap = 1 << 14
    x, _ = _cw_bursts(rng, 30_000, "gr_complex", [(0, 3000), (8000, 9000), (15_000, 17_000), (25_000, 26_000)])
    e.iq_create(8, cap)
    e.iq_create(10, cap)
    src = 8
    if cond is not None:
        d, t = cond
        h = rng.normal(0, 0.4, t).astype(np.float32)
        e.iq_create(9, cap)
        e.iq_set_conditioner(9, 8, d, h, 0.0, FS)
        src = 9
    _set(e, 10, src, s)
    e.iq_push(8, x[15_000:27_000])                                         # a dirty state before the gap
    assert (g - 1) % cap < 12_000
    assert e.iq_push_at(8, g, x[:6001]) == 6001
    if cond is None:
        origin, y = g, x
    else:
        origin = cnp.ceil_div(g + t - 1, d)
        y = cnp.condition_f32(x, g, h, d, 0.0, FS, origin, cnp.ceil_div(g + 14_000, d) - origin)
    st = e.iq_pulse_blanking_status(10) if s["kind"] == "blanker" else e.iq_notch_status(10)
    assert st["origin"] == origin == e.iq_window(10)[0]
    ref = _Restated(s, y, origin)
    pos = 0
    for n in (6001, 3001, 4998):
        if pos:
            e.iq_push(8, x[pos:pos + n])
        pos += n
        if cond is None:
            pushed = pos
        else:
            lo, hi = e.iq_window(9)
            assert lo == origin and hi == cnp.ceil_div(g + pos, d)
            assert e.iq_read(9, lo, hi - lo).tobytes() == y[:hi - lo].tobytes()
            pushed = hi - origin
        ref.check(e, 10, pushed)
    assert ref.done > origin
    if s["kind"] == "notch":
        assert ref.res["flags"][0] & 1                                     # the first segment filtered
    ref.check_bound()


# ---- 6. fan-out ----------------------------------------------------------------------------------------------------

def test_fan_out_push_limit_and_launches(capi, engine):
    """band 0 feeds a D = 2 conditioner (band 1), a blanker (L = 32, band 2) and a Lite notch (L = 16, band 3); band 1
    feeds a blanker (L = 64, band 4) and a Notch (L = 48, band 5).  The push limit is the least of 2^14 - 31 (band 0's
    stages), 2 (2^13 - 63) (band 1's) and 2^14 - 8 (the conditioner's history): a push of exactly it is accepted, one more
    sample is refused; small pushes complete segments of some stages and not others"""
    e = engine
    rng = np.random.default_rng(61)
    cap, d, t = 1 << 14, 2, 9
    h = rng.normal(0, 0.4, t).astype(np.float32)
    for b in (0, 2, 3):
        e.iq_create(b, cap)
    for b in (1, 4, 5):
        e.iq_create(b, cap // d)
    e.iq_set_conditioner(1, 0, d, h, 0.0, FS)
    stages = {2: (0, _blanker(32, 20, 200)), 3: (0, _notch(nn.NOTCH_LITE, 16, 20, 200, 3)),
              4: (1, _blanker(64, 10, 100)), 5: (1, _notch(nn.NOTCH, 48, 10, 100))}
    for dst, (src, s) in stages.items():
        _set(e, dst, src, s)
    limit = min(cap - max(_reach(stages[2][1]), _reach(stages[3][1])), d * (cap // d - max(_reach(stages[4][1]), _reach(stages[5][1]))),
                cap - (t - 1))
    assert limit == 2 * (8192 - 63)
    sizes = [limit, 5, 17, 1, 31, 16, 47, 3001, limit, 64, 9999, limit]
    total = sum(sizes)
    x, _ = _cw_bursts(rng, total + 1, "gr_complex", _periodic(total, 5000, 1500, 2000))  # + 1: the refused push
    y = cnp.condition_f32(x, 0, h, d, 0.0, FS, 0, cnp.ceil_div(total, d))
    refs = {dst: _Restated(s, x if src == 0 else y) for dst, (src, s) in stages.items()}
    bands = range(6)

    def pushed_of(dst, pos):
        return pos if stages[dst][0] == 0 else cnp.ceil_div(pos, d)

    pos, mixed = 0, 0
    for i, n in enumerate(sizes):
        if n == limit and i:                                               # one sample more than the limit: refused
            wins = [e.iq_window(b) for b in bands]
            k0 = e.launch_count()
            with pytest.raises(capi.B200Error) as r:
                e.iq_push(0, x[pos:pos + n + 1])
            assert r.value.code == ERR_RANGE and f"at most {limit}" in str(r.value), str(r.value)
            e.sync()
            assert e.launch_count() == k0 and [e.iq_window(b) for b in bands] == wins
        before = {dst: refs[dst].segments(pushed_of(dst, pos)) for dst in stages}
        j0 = cnp.ceil_div(pos, d)
        k0 = e.launch_count()
        e.iq_push(0, x[pos:pos + n])
        e.sync()
        pos += n
        j1 = cnp.ceil_div(pos, d)
        new = {dst: refs[dst].segments(pushed_of(dst, pos)) > before[dst] for dst in stages}
        mixed += len(set(new.values())) == 2
        want = (j1 > j0) + 3 * (new[2] + new[4]) + 6 * (new[3] + new[5])
        assert e.launch_count() - k0 == want, (i, n, new)
        assert e.iq_window(1)[1] == j1
        lo = e.iq_window(1)[0]
        assert e.iq_read(1, lo, j1 - lo).tobytes() == y[lo:j1].tobytes()
        for dst, ref in refs.items():
            ref.check(e, dst, pushed_of(dst, pos))
    assert mixed >= 3
    for ref in refs.values():
        ref.check_bound()


# ---- 7. full-scale integers ----------------------------------------------------------------------------------------

def _full_scale(rng, n, item_type):
    """CW bursts in noise at a quarter of full scale, with runs where I and Q, or I alone, sit at the type's minimum"""
    lo, hi = LIMITS[item_type]
    sigma = hi / 4
    t = np.arange(n)
    x = rng.normal(0, sigma / math.sqrt(2), n) + 1j * rng.normal(0, sigma / math.sqrt(2), n)
    x = x + ((t // 9000) % 2 == 1) * 2 * sigma * np.exp(1j * 0.37 * t)
    raw = ar.to_int(x, np.int16 if item_type == "ishort" else np.int8, 1.0, clip=(lo, hi))
    for a in rng.integers(0, n - 600, n // 3000):
        m = int(rng.integers(1, 500))
        raw[2 * a:2 * (a + m)] = lo
        raw[2 * (a + m):2 * (a + m + 50):2] = lo
    return raw, ar.from_int(raw)


FULL = [("conditioner", None), ("blanker", _blanker(4096, 2, 3)), ("notch", _notch(nn.NOTCH, 1024, 2, 6)),
        ("lite", _notch(nn.NOTCH_LITE, 1024, 2, 6, 2))]


@pytest.mark.parametrize("s", [f[1] for f in FULL], ids=[f[0] for f in FULL])
@pytest.mark.parametrize("item_type", ["ishort", "ibyte"])
def test_full_scale_integers(engine, item_type, s):
    """a narrow source band holding runs of -32768 / -128 through the conditioner (T = 4096, D = 36), a blanker at L =
    4096 and both notches at L = 1024, byte for byte"""
    e = engine
    rng = np.random.default_rng(71 + len(item_type))
    cap = 1 << 15
    total = 2 * cap + 321
    raw, held = _full_scale(rng, total, item_type)
    lo = LIMITS[item_type][0]
    assert np.count_nonzero(held == complex(lo, lo)) > 1000 and np.count_nonzero(held.real == lo) > 1000
    if s is None:
        t, d = 4096, 36
        h = rng.normal(0, 1.0 / 64, t).astype(np.float32)
        e.iq_create(0, cap, item_type)
        e.iq_create(1, ar.pow2(cnp.ceil_div(cap, d)))
        e.iq_set_conditioner(1, 0, d, h, 0.0, FS)
        want = cnp.condition_f32(held, 0, h, d, 0.0, FS, 0, cnp.ceil_div(total, d))
        limit, pos = cap - (t - 1), 0
        for n in _odd_sizes(rng, total, limit // 3, limit, first=(limit,)):
            _push(e, 0, raw, item_type, pos, pos + n)
            j0, j1 = cnp.ceil_div(pos, d), cnp.ceil_div(pos + n, d)
            pos += n
            got = e.iq_read(1, j0, j1 - j0)
            assert got.tobytes() == want[j0:j1].tobytes(), (pos, j0 + np.flatnonzero(got != want[j0:j1])[:5])
        return
    limit = cap - _reach(s)
    ref = _run_stage(e, s, item_type, raw, held, _odd_sizes(rng, total, limit // 3, limit, first=(limit,)), cap)
    if s["kind"] == "blanker":
        assert 0 < ref.ref.blanked < ref.ref.segments
    else:
        assert 0 < int((ref.res["flags"] & 1).sum()) < ref.res["segments"]
