"""Every code path of the tracking correlators against exact references, at every tap count, through the C ABI.

The per-item kernel (trk_kernels.cu, process_item in trk_item.cuh) has one instantiation per tap count 1..8 and, per item,
picks one of these paths:

  * fast: extended table in shared memory, sample pairs, the floor trick; with and without a ring wrap inside the epoch,
    at both sample parities;
  * large index: the scalar loop over the extended table, when a chip index reaches 4e6;
  * modulo: integer modulo lookup, the table in shared memory (multi-period epochs, far-apart taps) or, when the code is
    longer than the shared table, in global memory;
  * high dynamics: quadratic code phase and a carrier phase rate, table in shared or global memory.

The shared-window kernel (trk_shared_kernel.cu) has its chunk path, the whole-table and sliding-window table paths
through warp_tile, the no-share path and the off-table fallback, and reads attached linear bands up to their last sample.

References:
  * integer-exact: small-integer samples and code values with a zero carrier make every partial sum an exact integer,
    so the taps must EQUAL the integer correlation with the reference's chip indices (oracle.port.resampler with the
    a_avx association, hd_resampler_avx for high dynamics).  One wrong chip on one sample changes a tap.
  * float64 truth: oracle.port.multicorrelator_f64 (same float32 chip indices, carrier and sums in double), and for
    high dynamics a numpy float64 restatement of the reference's phase law.  Signal epochs must be within 1e-5 |P|,
    noise-only epochs within 1e-4 sigma_t per tap, sigma_t = sqrt(sum |x_n|^2 c_t(n)^2): one wrong chip on one sample
    moves a tap by about 2 |x_n|, far above that bound.
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from gnss_synth import make_iq, trk_params_for  # noqa: E402
from gpu_fixtures import capi, torch  # noqa: E402,F401
import trk_rig as tr  # noqa: E402
from trk_ref import exact_taps, int_code  # noqa: E402

RING = 1 << 18          # ring bands of the per-item tests: 262 144 samples ...
WRAP_AT = 60000         # ... whose end falls between data samples WRAP_AT - 1 and WRAP_AT
N_DATA = RING - 4096
ST25 = 1.023e6 * (1 + 3000 / 1575.42e6) / 25e6   # C/A chips per sample at 25 Msps, +3 kHz
EDGE_NS = [0, 1, 7, 8, 9, 511, 512, 513, 1023, 1024, 1025, 8192 + 9, 16384 + 8]
SLICES = [1, 2, 3, 7, 64]

WORST = {}   # group -> worst measured error ratio (printed at the end of the module)


def _record(group, ratio):
    WORST[group] = max(WORST.get(group, 0.0), float(ratio))


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    for k in sorted(WORST):
        print(f"\nworst error ratio, {k}: {WORST[k]:.3g}", end="")
    print()


def _hd_phase(n, rem_carr, dphi, drate):
    """the reference's high-dynamics carrier phase in float64: the rate term lags one sample and its exponent is
    float32((n-1)^2 mod 2^32) (the rotator squares an unsigned int)"""
    k = np.arange(n, dtype=np.uint64)
    e = np.zeros(n)
    km1 = k[1:] - np.uint64(1)
    e[1:] = ((km1 * km1) % np.uint64(1 << 32)).astype(np.float32).astype(np.float64)
    return -(float(np.float32(rem_carr)) + k.astype(np.float64) * float(np.float32(dphi)) + e * float(np.float32(drate)))


class Rig:
    """One engine with two ring bands: band 0 holds small-integer samples, band 1 complex Gaussian noise.  Each case
    gets a channel on each band; its integer item has a zero carrier, its float item a rotating one."""

    def __init__(self, capi, oracle, seed):
        self.oracle = oracle
        self.e = capi.Engine(0)
        self.e.trk_kernel_choice(0)           # the per-item kernel
        rng = np.random.default_rng(seed)
        self.xi = rng.integers(-7, 8, N_DATA)
        self.xi[self.xi == 0] = 1
        self.xf = (rng.standard_normal(N_DATA) + 1j * rng.standard_normal(N_DATA)).astype(np.complex64)
        lead = np.zeros(RING - WRAP_AT, np.complex64)
        self.first = [tr.ring(self.e, band, data, RING, lead) for band, data in ((0, self.xi.astype(np.complex64)),
                                                                                  (1, self.xf))]
        self.rows = []
        self.cases = []

    def add(self, group, code, shifts, n, start, rem, step, hd=False, rate=0.0, carrier=(1.1, 0.21, 0.0)):
        """start: index of the epoch's first sample in the data (the ring's end lies before data sample WRAP_AT)"""
        assert start + n <= N_DATA
        for band in (0, 1):
            cid = tr.channel(self.e, band, code, shifts, hd)
            rc, dp, dr = carrier if band == 1 else (0, 0, 0)
            self.rows.append((cid, n, self.first[band] + start, rc, dp, dr, rem, step, rate))
            self.cases.append((group, band, code, shifts, n, start, rem, step, hd, rate, (rc, dp, dr)))

    def items(self):
        return tr.items(self.rows)

    def expected(self, k):
        """integer item: exact taps (int64); float item: (float64 truth, sigma per tap)"""
        group, band, code, shifts, n, start, rem, step, hd, rate, (rc, dp, dr) = self.cases[k]
        port = self.oracle.port
        if band == 0 and not hd:
            return exact_taps(self.oracle, self.xi[start:start + n], code, rem, step, shifts, n)
        if hd:
            codes = port.hd_resampler_avx(code.astype(np.float32), rem, step, rate, shifts, n).astype(np.float64)
        else:
            codes = port.resampler(1, code.astype(np.float32), rem, step, shifts, n)
        if band == 0:
            return (codes.astype(np.int64) * self.xi[start:start + n][None, :]).sum(axis=1)
        x = self.xf[start:start + n]
        if hd:
            xr = x.astype(np.complex128) * np.exp(1j * _hd_phase(n, rc, dp, dr))
            truth = (codes * xr[None, :]).sum(axis=1)
        else:
            truth = port.multicorrelator_f64(1, x, code, shifts, rc, dp, rem, step)
        sigma = np.sqrt((np.abs(x.astype(np.complex128)) ** 2 * codes.astype(np.float64) ** 2).sum(axis=1))
        return truth, sigma

    def check(self, out, k, label):
        group, band, _, shifts, n = self.cases[k][:5]
        taps = len(shifts)
        got = out[k]
        assert np.all(got[taps:] == tr.SENTINEL), (label, group, "wrote past its taps")
        want = self.expected(k)
        if band == 0:
            assert np.array_equal(got[:taps, 0].astype(np.int64), want), (label, group, got[:taps, 0], want)
            assert np.all(got[:taps, 1] == 0), (label, group)
            return
        truth, sigma = want
        g = got[:taps, 0].astype(np.float64) + 1j * got[:taps, 1]
        if n == 0:
            assert np.all(g == 0), (label, group)
            return
        ratio = np.max(np.abs(g - truth) / sigma)
        _record(f"noise epochs, {label}" + (", high dynamics" if self.cases[k][8] else ""), ratio / 1e-4)
        assert ratio <= 1e-4, (label, group, ratio)

    def close(self):
        self.e.close()


# ---- 1. every tap count on every per-item path ------------------------------------------------------------------------
@pytest.mark.parametrize("taps", range(1, 9))
def test_every_per_item_path_at_every_tap_count(capi, torch, oracle, taps):
    """One engine per table size, so that the shared-memory table capacity (the longest code + 64) selects the path:
    with 1023-entry tables, every case but the modulo ones fits the extended table; with a 60 000-entry table (longer
    than the 50 944 entries shared memory holds) an epoch spanning 70 000 chips reads the table from global memory."""
    near = tr.shifts(taps, 0.6)
    carrier = (1.1, 0.2 + 0.013 * taps, 0.0)
    small = Rig(capi, oracle, 100 + taps)
    code = int_code(1023, taps, nonzero=True)
    small.add("fast", code, near, 25000, 1000, 0.37, ST25, carrier=carrier)
    small.add("fast, ring wrap, even start", code, near, 25000, WRAP_AT - 10000, -0.81, ST25, carrier=carrier)
    small.add("fast, ring wrap, odd start", code, near, 25001, WRAP_AT - 9999, 1.93, ST25, carrier=carrier)
    small.add("fast, odd start", code, near, 25000, 2001, 0.37, ST25, carrier=carrier)
    small.add("large index", code, near, 25000, 3000, -5.0e6 + 0.37, ST25, carrier=carrier)
    small.add("modulo, smem, 4 periods", code, near, 100000, 4001, 0.37, 0.0409, carrier=carrier)
    if taps > 1:
        far = [float(s) for s in np.linspace(-700.25, 500.5, taps).astype(np.float32)]
        small.add("modulo, smem, far taps", code, far, 6000, 7001, 3.3, 0.7, carrier=carrier)
    small.add("high dynamics, smem", code, tr.shifts(taps), 100000, 9000, 0.37, 0.04092, hd=True, rate=3e-12,
              carrier=(0.7, 1.1e-3, 2e-9))
    big = Rig(capi, oracle, 200 + taps)
    code_b = int_code(60000, taps, nonzero=True)
    big.add("modulo, gmem", code_b, near, 100000, 1000, 0.37, 0.7, carrier=carrier)
    big.add("high dynamics, gmem", code_b, tr.shifts(taps), 70001, 2001, 0.37, 0.7, hd=True, rate=1e-11,
            carrier=(0.7, -1.3e-3, -3e-9))
    for rig in (small, big):
        out = tr.run_dev(torch, rig.e, rig.items(), 8)
        for k in range(len(rig.cases)):
            rig.check(out, k, "per-item paths")
        rig.close()


@pytest.mark.parametrize("n,L,shifts,rem,step", [
    (25001, 1023, [-0.6, -0.3, -0.1, 0.1, 0.3, 0.6], 0.81, 0.0409),                   # 6 taps
    (5003, 2046, [-0.75, -0.5, -0.25, 0.0, 0.25, 0.5, 0.75], -1.27, 0.341),          # 7 taps
])
def test_single_correlator_six_and_seven_taps_integer_exact(capi, oracle, n, L, shifts, rem, step):
    """Multicorrelator (b200_trk_correlate, automatic slices) at the two tap counts no other single-correlator test
    uses: integer-exact against the reference's chip indices."""
    rng = np.random.default_rng(n + L)
    x_int = rng.integers(-7, 8, n)
    x_int[x_int == 0] = 1
    code_int = int_code(L, 0, nonzero=True)
    e = capi.Engine(0)
    mc = capi.Multicorrelator(e, n, len(shifts))
    mc.set_high_dynamics_resampler(False)
    mc.set_local_code_and_taps(code_int.astype(np.float32), shifts)
    got = mc.Carrier_wipeoff_multicorrelator_resampler(x_int.astype(np.complex64), 0.0, 0.0, 0.0, rem, step, 0.0)
    mc.free()
    e.close()
    assert np.array_equal(got.real.astype(np.int64), exact_taps(oracle, x_int, code_int, rem, step, shifts, n))
    assert np.all(got.imag == 0)


# ---- 2. edge lengths --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("taps", range(1, 9))
def test_edge_lengths_at_every_tap_count(capi, torch, oracle, taps):
    """No main tile (n < 512 + head), one tile plus remainder, the tails of the generic association and the ends of the
    16-tile re-seed groups, at both sample parities; an empty epoch gives zeros."""
    rig = Rig(capi, oracle, 300 + taps)
    code = int_code(1023, taps + 8, nonzero=True)
    shifts = tr.shifts(taps)
    for n in EDGE_NS:
        for parity in (0, 1):
            rig.add(f"n={n} parity={parity}", code, shifts, n, 20000 + parity, 0.41 - 0.1 * parity, ST25 * 1.5,
                    carrier=(2.3, -0.31, 0.0))
    out = tr.run_dev(torch, rig.e, rig.items(), 8)
    for k in range(len(rig.cases)):
        rig.check(out, k, "edge lengths")
    rig.close()


# ---- 3. slices --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("taps", range(1, 9))
def test_slices_at_every_tap_count(capi, torch, oracle, taps):
    """An epoch split over 1..64 CTAs: tile counts that the slice count does not divide (48 tiles over 7 slices), more
    slices than tiles (64 over 7), the modulo and high-dynamics paths.  Integer items stay exact, float items stay within
    2e-5 of the one-slice result and of the truth, and three launches give the same bits."""
    rig = Rig(capi, oracle, 400 + taps)
    code = int_code(1023, taps + 16, nonzero=True)
    shifts = tr.shifts(taps)
    rig.add("48 tiles", code, shifts, 25000, 1000, 0.2, ST25)
    rig.add("7 tiles", code, shifts, 7 * 512 + 5, 30000, 0.7, ST25 * 2)
    rig.add("odd start", code, shifts, 25001, 40001, -0.3, ST25)
    rig.add("ring wrap", code, shifts, 20000, WRAP_AT - 7001, 0.9, ST25)
    rig.add("modulo", code, shifts, 100000, 70000, 0.37, 0.0409)
    rig.add("high dynamics", code, shifts, 30001, 180000, 0.37, 0.04092, hd=True, rate=2e-12, carrier=(0.4, 2e-3, 1e-9))
    items = rig.items()
    outs = {}
    for slices in SLICES:
        reps = [tr.run_dev(torch, rig.e, items, 8, slices) for _ in range(3)]
        assert np.array_equal(reps[0], reps[1]) and np.array_equal(reps[0], reps[2]), slices
        outs[slices] = reps[0]
        for k in range(len(items)):
            rig.check(reps[0], k, "slices")
    for k in range(1, len(items), 2):      # float items
        truth, _ = rig.expected(k)
        one = outs[1][k, :taps, 0] + 1j * outs[1][k, :taps, 1].astype(np.float64)
        for slices in SLICES:
            v = outs[slices][k, :taps, 0] + 1j * outs[slices][k, :taps, 1].astype(np.float64)
            assert np.max(np.abs(v - one)) <= 2e-5 * np.max(np.abs(one)), (slices, rig.cases[k][0])
            assert np.max(np.abs(v - truth)) <= 2e-5 * np.max(np.abs(truth)), (slices, rig.cases[k][0])
    rig.close()


# ---- 4. mixed tap counts ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("slices", [1, 3])
def test_mixed_tap_counts_with_slices(capi, torch, oracle, slices):
    """Channels with 1, 2, 5 and 8 taps in one engine and one batch: one launch per tap count, each serving only its own
    items (and, with slices, only its own partials and arrival counters).  out_stride 8: every item is checked against
    its own reference, and the columns past its taps must stay untouched."""
    rig = Rig(capi, oracle, 500 + slices)
    for taps in (1, 2, 5, 8):
        code = int_code(1023 if taps != 5 else 2046, taps + 24, nonzero=True)
        shifts = tr.shifts(taps, 0.6)
        rig.add(f"{taps} taps", code, shifts, 25000 + taps, 1000 * taps, 0.3, ST25)
        rig.add(f"{taps} taps, ring wrap", code, shifts, 9000 + taps, WRAP_AT - 3001, -1.3, ST25)
        rig.add(f"{taps} taps, empty", code, shifts, 0, 0, 0.0, ST25)
        rig.add(f"{taps} taps, high dynamics", code, shifts, 8111, 100000 + 9000 * taps, 0.37, 0.04092, hd=True,
                rate=1e-10, carrier=(0.2, 1e-3, 1e-8))
    launches = rig.e.launch_count()
    out = tr.run_dev(torch, rig.e, rig.items(), 8, slices)
    assert rig.e.launch_count() - launches == 4
    out2 = tr.run_dev(torch, rig.e, rig.items(), 8, slices)
    assert np.array_equal(out, out2)
    for k in range(len(rig.cases)):
        rig.check(out, k, "mixed tap counts")
    rig.close()


# ---- 5. long epochs ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("taps", [1, 3, 5])
@pytest.mark.parametrize("fs", [25e6, 50e6, 100e6])
def test_long_epochs_against_float64(capi, torch, oracle, fs, taps):
    """GPS L2 CM-like: a +-1 table of 10 230 chips at 511.5 kchip/s, 20 ms epochs (500 000 to 2 000 000 samples), Doppler
    of +-4 kHz, one signal epoch with an fs/4 IF offset in phase_step_rad, and a noise-only epoch.  Through the per-item
    kernel with one slice (the longest run of the carrier recurrence), through Multicorrelator (automatic slices) and
    through the shared-window kernel (its sliding code window)."""
    n = int(round(0.02 * fs))
    rng = np.random.default_rng(int(fs / 1e6) + taps)
    code = np.where(rng.integers(0, 2, 10230) > 0, 1.0, -1.0).astype(np.float32)
    shifts = [float(s) for s in (np.arange(taps) * 0.5 - 0.5 * (taps // 2))]
    prompt = taps // 2
    cases = [   # (label, doppler, IF offset, signal)
        ("+4 kHz", 4000.0, False, True),
        ("-4 kHz, fs/4 IF", -4000.0, True, True),
        ("noise, +4 kHz, fs/4 IF", 4000.0, True, False),
    ]
    segs, params = [], []
    for k, (label, dop, if_off, sig) in enumerate(cases):
        sv = dict(prn=1, doppler=dop, code_phase_chips=1234.5 + 1000 * k, cn0=45.0, phase0=0.3 + k)
        x = make_iq({1: code}, fs, n, [sv] if sig else [], seed=k + taps, chips_per_table_chip=0.5)
        _, rc, dp, rcode, st = trk_params_for(sv, fs, n, 1, table_chips_per_chip=0.5, L=10230)
        dphi = float(dp[0])
        if if_off:
            x = (x * np.exp(0.5j * np.pi * np.arange(n))).astype(np.complex64)
            dphi = float(np.float32(dphi + 0.5 * np.pi))
        segs.append(x)
        params.append((float(rc[0]), dphi, float(rcode[0]), float(st[0])))
    truths = [oracle.port.multicorrelator_f64(1, segs[k], code, shifts, *params[k]) for k in range(len(cases))]
    sigmas = [np.sqrt(np.sum(np.abs(s.astype(np.complex128)) ** 2)) for s in segs]   # |c| = 1

    def check(got, k, path):
        label, _, _, sig = cases[k]
        err = np.abs(got - truths[k])
        if sig:
            p = np.abs(truths[k][prompt])
            assert p > 5 * np.sqrt(n)
            ratio = np.max(err) / p
            _record(f"long signal epochs, {fs / 1e6:.0f} Msps, {path}", ratio / 1e-5)
            assert ratio <= 1e-5, (path, label, ratio)
        else:
            ratio = np.max(err) / sigmas[k]
            _record(f"long noise epochs, {fs / 1e6:.0f} Msps, {path}", ratio / 1e-4)
            assert ratio <= 1e-4, (path, label, ratio)

    e = capi.Engine(0)
    first = tr.ring(e, 0, np.concatenate(segs))
    rows = []
    for k in range(len(cases)):
        rc, dphi, rcode, st = params[k]
        rows.append((tr.channel(e, 0, code, shifts), n, first + k * n, rc, dphi, 0.0, rcode, st))
    items = tr.items(rows)
    for mode, path in ((0, "per-item kernel"), (1, "shared kernel")):
        e.trk_kernel_choice(mode)
        out = tr.run_dev(torch, e, items, 8)
        for k in range(len(cases)):
            check(out[k, :taps, 0] + 1j * out[k, :taps, 1].astype(np.float64), k, path)
    mc = capi.Multicorrelator(e, n, taps)
    mc.set_high_dynamics_resampler(False)
    mc.set_local_code_and_taps(code, shifts)
    for k in range(len(cases)):
        rc, dphi, rcode, st = params[k]
        got = mc.Carrier_wipeoff_multicorrelator_resampler(segs[k], rc, dphi, 0.0, rcode, st, 0.0)
        check(got.astype(np.complex128), k, "Multicorrelator")
    mc.free()
    e.close()


# ---- 6. shared-window kernel ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("taps", [1, 5])
def test_shared_kernel_paths_integer_exact(capi, torch, oracle, taps):
    """The shared-window kernel forced on, one homogeneous group of 8 items per path: the chunk path (C/A at 25 Msps),
    the whole-epoch table through warp_tile (C/A at 4 Msps), the sliding code window (8184-entry table), groups whose
    epochs lie too far apart to share (each warp streams its own tiles) and the off-table fallback (rem = 2e6)."""
    rng = np.random.default_rng(600 + taps)
    shifts = tr.shifts(taps, 0.6)
    blocks = [   # (path, L, n, step, rem base, spacing of the 8 starts)
        ("chunk", 1023, 25000, ST25, 0.0, 37),
        ("chunk", 1023, 25001, ST25, 0.0, 53),
        ("whole table", 1023, 4000, 0.25575, 0.0, 41),
        ("sliding window", 8184, 20000, 0.08184, 0.0, 111),
        ("no share", 1023, 6000, 0.1705, 0.0, 12001),
        ("off table", 1023, 6000, 0.1705, 2.0e6, 29),
    ]
    total = sum(7 * sp + n + 2 for (_, _, n, _, _, sp) in blocks) + 64
    x = rng.integers(-7, 8, total)
    e = capi.Engine(0)
    e.trk_kernel_choice(1)
    first = tr.ring(e, 0, x.astype(np.complex64))
    rows, want = [], []
    pos = 1
    for b, (path, L, n, step, rem0, sp) in enumerate(blocks):
        for j in range(8):
            code = int_code(L, 8 * b + j, nonzero=True)
            cid = tr.channel(e, 0, code, shifts)
            s0 = pos + j * sp
            rem = float(np.float32(rem0 + float(rng.uniform(-3, 3)) if rem0 == 0.0 else rem0 + 0.25 * j))
            rows.append((cid, n, first + s0, 0.0, 0.0, 0.0, rem, step))
            want.append((path, exact_taps(oracle, x[s0:s0 + n], code, rem, step, shifts, n)))
        pos += 7 * sp + n + 2
    launches = e.launch_count()
    out = tr.run_dev(torch, e, tr.items(rows), taps)
    assert e.launch_count() - launches == 1
    e.close()
    for i, (path, w) in enumerate(want):
        assert np.array_equal(out[i, :, 0].astype(np.int64), w), (path, i)
        assert np.all(out[i, :, 1] == 0), (path, i)


# ---- 7. attached linear bands -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("total", [60000, 60001])
def test_shared_kernel_linear_band_to_its_last_sample(capi, torch, oracle, total):
    """A torch buffer attached as a linear band (b200_iq_attach_dev), read by the shared-window kernel: the last tiles of
    the band are clipped, and two items of each group end exactly at the band's end, one with a length that is a
    multiple of 8 (so that its last sample is a main-loop sample) and one with a tail.  Shared groups on the chunk and
    whole-table paths, and a group whose items are too far apart to share.  Integer-exact."""
    rng = np.random.default_rng(total)
    x = rng.integers(-7, 8, total)
    xt = torch.zeros(total, 2, dtype=torch.float32, device="cuda")
    xt[:, 0] = torch.from_numpy(x.astype(np.float32)).cuda()
    shifts = [-0.5, 0.0, 0.5]
    e = capi.Engine(0)
    e.trk_kernel_choice(1)
    e.iq_attach_dev(0, xt.data_ptr(), total, 0)
    groups = [   # (path, step, lengths of the 8 items, gap between consecutive ends)
        ("chunk", ST25, [5003, 4096] * 4, 31),
        ("whole table", 0.25575, [4001, 4000] * 4, 17),
        ("no share", 0.1705, [4003, 4096] * 4, 7001),
    ]
    rows, want = [], []
    for g, (path, step, ns, gap) in enumerate(groups):
        for j in range(8):
            n = ns[j]
            s0 = total - n - gap * max(6 - j, 0)   # items 6 and 7 end at the band's last sample
            code = int_code(1023, 8 * g + j, nonzero=True)
            cid = tr.channel(e, 0, code, shifts)
            rem = float(np.float32(rng.uniform(-3, 3)))
            rows.append((cid, n, s0, 0.0, 0.0, 0.0, rem, step))
            want.append((path, n, exact_taps(oracle, x[s0:s0 + n], code, rem, step, shifts, n)))
    out = tr.run_dev(torch, e, tr.items(rows), 3)
    e.close()
    for i, (path, n, w) in enumerate(want):
        assert np.array_equal(out[i, :, 0].astype(np.int64), w), (path, n, i)
        assert np.all(out[i, :, 1] == 0), (path, n, i)
