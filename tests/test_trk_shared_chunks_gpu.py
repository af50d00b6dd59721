"""The chunk path of the shared-window tracking kernel (trk_shared_kernel.cu, warp_tile_chunks): each lane correlates a
contiguous 16-sample chunk and splits it at the one exact chip boundary per tap.  All through the C ABI with the shared
kernel forced on.  Integer samples and codes with a zero carrier keep every sum exact, so these runs must EQUAL the
integer oracle built from the reference's chip indices; float data stays within the bounds of test_trk_gpu.py."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from gnss_sdr_b200.build import LIB, build_variant  # noqa: E402
from gnss_synth import make_iq, trk_params_for  # noqa: E402
from gpu_fixtures import capi  # noqa: E402,F401
from ring_worker import run_worker  # noqa: E402
import trk_rig as tr  # noqa: E402
from trk_ref import chip_indices, exact_taps, ref_or_port_avx  # noqa: E402

SHIFTS = [-0.5, 0.0, 0.5]
CA_16368 = 1023.0 / 16368
CA_25 = 1.023e6 * (1 + 3000 / 1575.42e6) / 25e6
CA_50 = 1.023e6 * (1 - 4500 / 1575.42e6) / 50e6


def run_shared(capi, x_int, chans, epochs, filler=0, capacity=None):
    """chans: list of (code, rem, step, n, start).  epochs of every channel back to back from `start`, items sorted by
    start sample as the host API groups them.  filler: samples pushed before x_int (to make a ring wrap inside x_int).
    Returns {(channel, epoch): taps}."""
    e = capi.Engine(0)
    try:
        e.trk_kernel_choice(1)
        first = tr.ring(e, 0, x_int.astype(np.complex64), capacity, np.ones(filler, np.complex64) if filler else None)
        cids = [tr.channel(e, 0, code, SHIFTS) for code, *_ in chans]
        keys, rows = [], []
        for c, (code, rem, step, n, start) in enumerate(chans):
            for k in range(epochs):
                keys.append((c, k))
                rows.append((cids[c], n, first + start + k * n, 0.0, 0.0, 0.0, rem, step))
        items = tr.items(rows)
        order = np.argsort(items["sample_index"], kind="stable")
        got = e.trk_batch(items[order], len(SHIFTS))
    finally:
        e.close()
    return {keys[o]: got[i] for i, o in enumerate(order)}


def check_exact(oracle, x_int, chans, epochs, got):
    for c, (code, rem, step, n, start) in enumerate(chans):
        for k in range(epochs):
            s0 = start + k * n
            want = exact_taps(oracle, x_int[s0:s0 + n], code, float(np.float32(rem)), step, SHIFTS, n)
            assert np.array_equal(got[(c, k)].real.astype(np.int64), want), (c, k, step, n, rem)
            assert np.all(got[(c, k)].imag == 0), (c, k)


def random_code(rng, L=1023):
    """a table of L integers drawn uniformly from [-15, 15]"""
    return rng.integers(-15, 16, L)


def test_chip_boundary_at_every_chunk_position(capi, oracle):
    """16 channels whose rem puts the first chip boundary of the epoch at sample 0..15 of the first chunk; over the epoch
    the boundaries also fall on every position of every later chunk.  Epochs start on the tile grid (a_i = 0)."""
    rng = np.random.default_rng(11)
    n, step, epochs = 25000, CA_25, 2
    x = rng.integers(-7, 8, n * epochs + 1024)
    chans = [(random_code(rng), float(np.float32(-(j + 0.5) * step)), step, n, 0) for j in range(16)]
    # the rises of the prompt tap inside 16-sample chunks cover every position
    pos = set()
    for code, rem, *_ in chans:
        d = np.flatnonzero(np.diff(chip_indices(oracle, code, rem, step, SHIFTS, n)[1])) + 1
        pos |= set((d % 16).tolist())
    assert pos == set(range(16))
    check_exact(oracle, x, chans, epochs, run_shared(capi, x, chans, epochs))


@pytest.mark.parametrize("step,n", [
    (CA_16368, 16368),         # GPS L1 C/A at 16.368 Msps
    (CA_25, 25000),            # ... 25 Msps
    (CA_50, 50000),            # ... 50 Msps
    (CA_25, 24999),            # n neither a multiple of 16 nor of 512
    (0.0666, 15001),           # just inside the chunk path's step limit (15 step + margin < 1)
    (0.0668, 15001),           # just outside it: warp_tile
    (0.17, 6000),              # well outside (4-6 Msps front ends)
])
def test_staggered_groups_integer_exact(capi, oracle, step, n):
    """11 channels with odd and unaligned epoch starts and random code phases, 3 epochs each: groups of 8 items span
    several extra tiles and items start at any sample of a tile and of a chunk."""
    rng = np.random.default_rng(int(n + step * 1e6))
    epochs, n_ch = 3, 11
    starts = np.sort(rng.integers(0, n, n_ch))
    starts[1] |= 1
    x = rng.integers(-7, 8, n * (epochs + 1) + 1024)
    chans = [(random_code(rng), float(rng.uniform(-3, 3)), step, n, int(starts[c])) for c in range(n_ch)]
    check_exact(oracle, x, chans, epochs, run_shared(capi, x, chans, epochs))


def test_one_cta_holds_items_on_both_paths(capi, oracle):
    """Channels alternate between a chunk-path step and a warp_tile step, so every group of 8 items mixes the two paths
    on the same ring of tiles."""
    rng = np.random.default_rng(5)
    n, epochs, n_ch = 6000, 3, 12
    starts = np.sort(rng.integers(0, 700, n_ch))
    x = rng.integers(-7, 8, n * (epochs + 1) + 1024)
    chans = [(random_code(rng), float(rng.uniform(-2, 2)), CA_25 if c % 2 else 0.1705, n, int(starts[c])) for c in range(n_ch)]
    check_exact(oracle, x, chans, epochs, run_shared(capi, x, chans, epochs))


def test_ring_band_wraps_inside_a_tile(capi, oracle):
    """The band is a 64 Ki-sample ring and the epochs cross its end in the middle of a tile and of a chunk: the producer
    splits that chunk's copy in two."""
    rng = np.random.default_rng(8)
    n, epochs, n_ch, cap = 25000, 2, 8, 1 << 16
    filler = cap - 9000 - 206     # the wrap falls 9206 samples into x, not on a 16-sample boundary of any group
    x = rng.integers(-7, 8, n * epochs + 3000)
    starts = np.sort(rng.integers(0, 2000, n_ch))
    assert (cap - filler - (int(starts[0]) & ~1)) % 16 != 0     # not on a chunk boundary of the first group's tiles
    chans = [(random_code(rng), float(rng.uniform(-2, 2)), CA_25, n, int(starts[c])) for c in range(n_ch)]
    check_exact(oracle, x, chans, epochs, run_shared(capi, x, chans, epochs, filler=filler, capacity=cap))


def test_float_signal_full_epochs_within_bounds(capi, oracle):
    """C2-shaped float data (32 GPS L1 C/A channels at 25 Msps, Doppler and carrier phase) over full 1 ms epochs: within
    1e-3 of the AVX oracle and 1e-5 |prompt| of the float64 truth."""
    fs, n, nch, nep = 25e6, 25000, 32, 3
    rng = np.random.default_rng(21)
    codes = {p: oracle.port.gps_ca_code(p) for p in range(1, nch + 1)}
    svs = [dict(prn=p, doppler=float(rng.uniform(-5000, 5000)), code_phase_chips=float(rng.uniform(0, 1023)),
                cn0=45.0, phase0=float(rng.uniform(0, 6.28))) for p in range(1, nch + 1)]
    iq = make_iq(codes, fs, n * nep + 64, svs, seed=21)
    e = capi.Engine(0)
    e.trk_kernel_choice(1)
    first = tr.ring(e, 0, iq)
    rows = [None] * (nch * nep)
    for c, sv in enumerate(svs):
        cid = tr.channel(e, 0, codes[sv["prn"]], SHIFTS)
        s, rc, dp, rcode, st = trk_params_for(sv, fs, n, nep)
        for k in range(nep):
            rows[k * nch + c] = (cid, n, first + int(s[k]), rc[k], dp[k], 0.0, rcode[k], st[k])
    items = tr.items(rows)
    order = np.argsort(items["sample_index"], kind="stable")
    got = np.empty((len(items), 3), np.complex64)
    got[order] = e.trk_batch(items[order], 3)
    e.close()
    worst_ref, worst_truth = 0.0, 0.0
    for i in range(0, len(items), 3):
        it = items[i]
        sv = svs[i % nch]
        seg = iq[int(it["sample_index"]) - first: int(it["sample_index"]) - first + n]
        a = (float(it["rem_carrier_phase_rad"]), float(it["phase_step_rad"]), float(it["rem_code_phase_chips"]),
             float(it["code_phase_step_chips"]))
        want = ref_or_port_avx(oracle, seg, codes[sv["prn"]], SHIFTS, *a)
        truth = oracle.port.multicorrelator_f64(1, seg, codes[sv["prn"]], SHIFTS, *a)
        assert np.abs(truth[1]) > 3 * np.sqrt(n)
        worst_ref = max(worst_ref, float(np.max(np.abs(got[i] - want) / np.abs(want))))
        worst_truth = max(worst_truth, float(np.max(np.abs(got[i] - truth)) / np.abs(truth[1])))
    assert worst_ref < 1e-3
    assert worst_truth < 1e-5


@pytest.mark.parametrize("stages", [2, 4, 8])
def test_ring_under_injected_delays_chunk_path(stages):
    """The -DSH_STRESS=1 builds (delays injected into producer and consumers) at a chunk-path step: 500 launches bitwise
    stable and equal to the production build on integer-exact inputs.  test_ring_stress_gpu.py runs the same worker at
    its own step (about 0.17, warp_tile only); this one at a C2-like step, 25 Msps."""
    step = 1.023e6 / 25e6
    prod = run_worker(LIB, 3, step)
    got = run_worker(build_variant(stages, stress=True), 500, step)
    assert got["bad"] == 0, got
    assert got["sha"] == prod["sha"], (got, prod)
