"""The chunk path's shared running-sum pick (warp_tile_chunks in csrc/trk_shared_kernel.cu): when the first and the
last tap of a channel are a whole number of chips apart and every lane of a warp finds the same boundary sample for
both, the last tap reuses the first tap's select.  Integer samples and codes with a zero carrier keep every sum exact,
so each run must EQUAL the integer oracle built from the reference's chip indices, whether the pick was shared, never
shared, or shared in some tiles and not in others."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from gpu_fixtures import capi  # noqa: E402,F401
import trk_rig as tr  # noqa: E402
from trk_ref import exact_taps  # noqa: E402
from test_chunk_tap_pair_cpu import CA_25, find_split_items, pair_disagreements  # noqa: E402

N = 25000


def run_shared(capi, x_int, chans, epochs):
    """chans: list of (code, shifts, rem, start); 3 taps, N-sample epochs back to back from `start`, items sorted by start
    sample.  Returns {(channel, epoch): taps}."""
    e = capi.Engine(0)
    try:
        e.trk_kernel_choice(1)
        first = tr.ring(e, 0, x_int.astype(np.complex64))
        cids = [tr.channel(e, 0, code, shifts) for code, shifts, *_ in chans]
        keys, rows = [], []
        for c, (code, shifts, rem, start) in enumerate(chans):
            for k in range(epochs):
                keys.append((c, k))
                rows.append((cids[c], N, first + start + k * N, 0.0, 0.0, 0.0, rem, CA_25))
        items = tr.items(rows)
        order = np.argsort(items["sample_index"], kind="stable")
        got = e.trk_batch(items[order], 3)
    finally:
        e.close()
    return {keys[o]: got[i] for i, o in enumerate(order)}


def check_exact(oracle, x_int, chans, epochs, got):
    for c, (code, shifts, rem, start) in enumerate(chans):
        for k in range(epochs):
            s0 = start + k * N
            want = exact_taps(oracle, x_int[s0:s0 + N], code, float(np.float32(rem)), CA_25, shifts, N)
            assert np.array_equal(got[(c, k)].real.astype(np.int64), want), (c, k, shifts, rem)
            assert np.all(got[(c, k)].imag == 0), (c, k)


def chans_for(rng, shifts_of, rems, starts):
    return [(rng.integers(-15, 16, 1023), shifts_of(c), float(np.float32(rem)), int(s)) for c, (rem, s) in enumerate(zip(rems, starts))]


@pytest.mark.parametrize("shifts", [[-0.5, 0.0, 0.5], [-1.0, 0.0, 1.0], [-0.4, 0.0, 0.45]])
def test_tap_spacings_integer_exact(capi, oracle, shifts):
    """E/P/L half a chip and a whole chip from P (the pick is shared), and -0.4 / +0.45 (never shared); 16 channels with
    random code phases over two epochs, groups starting anywhere in a tile"""
    rng = np.random.default_rng(int(100 * shifts[-1]) + 7)
    epochs = 2
    x = rng.integers(-7, 8, N * (epochs + 1))
    chans = chans_for(rng, lambda c: shifts, -rng.uniform(0, 1023, 16), np.sort(rng.integers(0, 900, 16)))
    check_exact(oracle, x, chans, epochs, run_shared(capi, x, chans, epochs))


def test_one_cta_mixes_sharing_and_non_sharing_warps(capi, oracle):
    """Channels alternate between -0.5/0/+0.5 and -0.4/0/+0.45, so every group of 8 items holds both kinds"""
    rng = np.random.default_rng(12)
    epochs = 2
    x = rng.integers(-7, 8, N * (epochs + 1))
    chans = chans_for(rng, lambda c: [-0.5, 0.0, 0.5] if c % 2 else [-0.4, 0.0, 0.45], -rng.uniform(0, 1023, 16),
                      np.sort(rng.integers(0, 300, 16)))
    check_exact(oracle, x, chans, epochs, run_shared(capi, x, chans, epochs))


def test_split_pairs_fall_back_to_their_own_pick(capi, oracle):
    """Code phases for which, in some chunk, the -0.5 and +0.5 taps keep their index to different samples (found by the
    float32 restatement of the index formula): those tiles fail the vote and take the last tap's own select tree"""
    # The prediction holds only if the kernel sees the same float32 rem and step as the CPU restatement: the item
    # stores both as float32, and the restatement rounds them the same way.
    dt = capi.TRK_ITEM_DTYPE
    assert dt["rem_code_phase_chips"] == np.float32 and dt["code_phase_step_chips"] == np.float32
    rng = np.random.default_rng(13)
    rems = find_split_items(CA_25, N, 8, seed=13)
    for rem in rems:
        assert pair_disagreements(CA_25, rem, N)[0].size > 0
    x = rng.integers(-7, 8, N + 1024)
    # epochs on the tile grid, as the CPU search assumes: each group's hull starts at its first item
    chans = chans_for(rng, lambda c: [-0.5, 0.0, 0.5], rems, [0] * len(rems))
    check_exact(oracle, x, chans, 1, run_shared(capi, x, chans, 1))
