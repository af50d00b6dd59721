"""When the chunk path of the shared-window kernel (warp_tile_chunks in csrc/trk_shared_kernel.cu) may let the last tap
reuse the first tap's running-sum pick, restated in numpy float32.  No GPU.

For a channel whose first and last shifts are a whole number of chips apart (E and L at -0.5 and +0.5), the two taps
usually rise at the same sample of a 16-sample chunk, and a warp whose 32 lanes all find the same last-kept sample m
for both takes one select tree instead of two.  The indices are i(n) = floor(fl(fl(step n) + aux)), aux = fl(shift -
rem), so the two can still floor differently where a power of two lies between the two taps' sums.  This
module finds such items (tests/test_trk_shared_tap_classes_gpu.py correlates them on the GPU) and counts how often the
vote fails on bench.py's C2 items."""
import numpy as np

F32 = np.float32
CHUNK, TILE = 16, 512
CA_25 = 1.023e6 * (1 + 3000 / 1575.42e6) / 25e6


def chip_index(step, n, aux):
    """floor(fl(fl(step n) + aux)) in float32, as the kernel computes it (its round-down add of 1.5 * 2^23 is a floor)"""
    return np.floor((F32(step) * n.astype(F32)).astype(F32) + F32(aux)).astype(np.int64)


def chunk_m(step, aux, n_chunks):
    """m of every 16-sample chunk of an epoch that starts on the tile grid: the last sample that keeps the chunk's first
    index (the chunk path's precondition lets the index rise at most once inside a chunk)"""
    i = chip_index(step, np.arange(n_chunks * CHUNK + 1), aux)
    i = i[: n_chunks * CHUNK].reshape(n_chunks, CHUNK)
    return np.sum(i == i[:, :1], axis=1) - 1


def pair_disagreements(step, rem, n, shifts=(-0.5, 0.5)):
    """(chunks, tiles) of an n-sample epoch where the first and the last tap keep their index to different samples; a
    tile's vote fails when any of its 32 chunks does"""
    rem = F32(rem)
    n_chunks = (n + CHUNK - 1) // CHUNK
    m0 = chunk_m(step, F32(F32(shifts[0]) - rem), n_chunks)
    m1 = chunk_m(step, F32(F32(shifts[-1]) - rem), n_chunks)
    bad = np.flatnonzero(m0 != m1)
    return bad, np.unique(bad // (TILE // CHUNK))


def find_split_items(step, n, count, seed=0, shifts=(-0.5, 0.5)):
    """`count` code phases rem in (-512, 0] for which some chunk of an n-sample epoch splits the pair (the taps' sums
    then cross 256, 512 or 1024 inside the epoch)"""
    rng = np.random.default_rng(seed)
    found = []
    while len(found) < count:
        rem = float(F32(-rng.uniform(0.0, 512.0)))
        if pair_disagreements(step, rem, n, shifts)[0].size:
            found.append(rem)
    return found


def test_integer_spaced_taps_split_only_at_binade_edges():
    """A pair splits only where a power of two lies between the two taps' sums: either aux and aux + 1 fall in different
    binades (so fl(0.5 - rem) is not fl(-0.5 - rem) + 1), or the split chunk's index sits next to a power of two"""
    rems = find_split_items(CA_25, 25000, 6, seed=3)
    for rem in rems:
        bad, _ = pair_disagreements(CA_25, rem, 25000)
        aux0, aux2 = F32(F32(-0.5) - F32(rem)), F32(F32(0.5) - F32(rem))
        if np.float64(aux2) - np.float64(aux0) != 1.0:
            continue
        idx = chip_index(CA_25, bad * CHUNK + CHUNK // 2, aux2)
        near = np.min(np.abs(idx[:, None] - np.array([2 ** k for k in range(1, 12)])[None, :]), axis=1)
        assert np.all(near <= 1), (rem, bad, idx)


def test_non_integer_spacing_almost_never_agrees():
    """-0.4 / +0.45 chips: the two taps rise about 3.6 samples apart, so most tiles have some lane that disagrees"""
    _, tiles = pair_disagreements(CA_25, -123.25, 25000, shifts=(-0.4, 0.45))
    assert tiles.size > 0.9 * ((25000 + TILE - 1) // TILE)


def test_vote_failure_rate_on_c2_items():
    """Items that approximate bench.py's C2 shape (test_vote_failure_rate_on_bench_c2_items takes its own items): 32 GPS
    L1 C/A channels at 25 Msps, 1 ms epochs on the tile grid, E/L at -0.5 / +0.5 chips, random code phase and Doppler
    within +-5 kHz.  Reports how many warp-tiles fall back to their own select tree (expected: rarely)."""
    rng = np.random.default_rng(3)
    n, tiles_per_epoch = 25000, (25000 + TILE - 1) // TILE
    total, failed, split_chunks = 0, 0, 0
    for _ in range(32):
        step = 1.023e6 * (1 + rng.uniform(-5000, 5000) / 1575.42e6) / 25e6
        u = rng.uniform(0, 1023)
        for k in range(8):
            rem = -np.mod(u + step * k * n, 1023.0)
            bad, tiles = pair_disagreements(step, rem, n)
            total += tiles_per_epoch
            failed += tiles.size
            split_chunks += bad.size
    print(f"C2 items: {failed} of {total} warp-tiles ({failed / total:.2e}) fail the vote, {split_chunks} split chunks")
    assert failed < 0.01 * total


def chunk_m_at(index, lo, lo_off):
    """m of chunks whose first valid sample is lo (lo_off samples into the chunk), from the exact indices `index` of the
    epoch's samples: the last chunk sample that keeps index[lo], clamped to the chunk as the kernel's masked tiles do"""
    i0 = index[lo]
    rise = index[lo[:, None] + np.arange(1, CHUNK + 1)[None, :]] > i0[:, None]
    j = np.where(rise.any(axis=1), rise.argmax(axis=1) + 1, CHUNK + 1)
    return np.clip(lo_off + j - 1, 0, CHUNK - 1)


def item_vote_failures(step, rem, n, a_i, shifts=(-0.5, 0.5)):
    """(tiles, tiles whose vote fails) of one item in a shared-window group whose first sample lies a_i samples after
    the group's first tile: the tiles, chunks, masking and lo of trk_shared_kernel's chunk path"""
    body = 8 * (n // 8)
    step, rem = F32(step), F32(rem)
    samples = np.arange(body + CHUNK + 1)
    idx = [chip_index(step, samples, F32(F32(s) - rem)) for s in (shifts[0], shifts[-1])]
    t_first, t_last = a_i // TILE, (a_i + body + TILE - 1) // TILE
    n_tile0 = np.arange(t_first, t_last) * TILE - a_i
    n0 = (n_tile0[:, None] + CHUNK * np.arange(TILE // CHUNK)[None, :]).ravel()
    vlo = np.repeat(np.maximum(n_tile0, 0), TILE // CHUNK)
    vhi = np.repeat(np.minimum(n_tile0 + TILE, body) - 1, TILE // CHUNK)
    lo = np.clip(n0, vlo, vhi)
    m0, m1 = (chunk_m_at(i, lo, lo - n0) for i in idx)
    tiles = t_last - t_first
    return tiles, np.unique(np.flatnonzero(m0 != m1) // (TILE // CHUNK)).size


def test_vote_failure_rate_on_bench_c2_items():
    """The items of bench.py's headline C2 step (32 GPS L1 C/A channels at 25 Msps, E/P/L at -0.5 / 0 / +0.5 chips),
    built by bench.py's own svs_for_rank and build_items, for the first 20 of its 1000 epochs; grouped in eights as the
    kernel groups them.  Reports how many warp-tiles fall back to the last tap's own select tree."""
    import importlib
    import os
    import sys
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    bench = importlib.import_module("bench")
    from gnss_sdr_b200.abi import TRK_ITEM_DTYPE

    class Capi:
        pass

    capi = Capi()
    capi.TRK_ITEM_DTYPE = TRK_ITEM_DTYPE
    assert bench.SHIFTS == [-0.5, 0.0, 0.5] and bench.FS == 25e6
    items = bench.build_items(capi, bench.svs_for_rank(0), list(range(bench.N_CH)), 0)[: 20 * bench.N_CH]
    total, failed = 0, 0
    for g in range(0, len(items), 8):
        group = items[g:g + 8]
        hull = int(group["sample_index"].min()) & ~1
        for it in group:
            t, f = item_vote_failures(it["code_phase_step_chips"], it["rem_code_phase_chips"], int(it["n"]),
                                      int(it["sample_index"]) - hull)
            total, failed = total + t, failed + f
    print(f"bench.py C2 items: {failed} of {total} warp-tiles ({failed / total:.2e}) fail the vote")
    assert total >= 20 * bench.N_CH * (bench.EPOCH // TILE)
    assert failed <= 0.001 * total
