"""The chip-boundary estimate of the shared-window kernel's chunk path (warp_tile_chunks in csrc/trk_shared_kernel.cu),
restated in numpy float32 and checked against a scan of the exact index formula.  No GPU.

The kernel finds, for every tap and 16-sample chunk, the last sample m that keeps the chip index i0 of the chunk's first
sample.  The index of sample n is floor(a(n)), a(n) = fl(fl(step n) + aux), with floor taken by the kFloorMagic
round-down.  The kernel estimates the first sample past the boundary from a per-item fl(1 / step), evaluates the exact
formula at the estimate and selects.  Here the same float32 operations (round-to-nearest products and sums, one fused
multiply-add, round-down additions of kFloorMagic) run on hundreds of thousands of (step, aux, n0) inside the chunk
path's precondition, at C/A chipping rates for 16.368, 25 and 50 Msps and at random steps up to its limit, with n0 up to
2 000 000."""
import numpy as np

F32 = np.float32
MAGIC = F32(12582912.0)   # kFloorMagic, 1.5 * 2^23
CHUNK = 16


def add_rd(x, y):
    """fl_rd(x + y) for float32 arrays: the round-to-nearest sum, moved one ulp down where it lies above the exact sum"""
    s = (x + y).astype(F32)
    above = (s.astype(np.float64) - y.astype(np.float64)) > x.astype(np.float64)   # exact: s - y is an integer here
    return np.where(above, np.nextafter(s, F32(-np.inf)), s).astype(F32)


def fma_rn(a, b, c):
    """fl(a b + c) for float32 arrays, rounded once: the exact product in float64, the sum rounded to odd, then to float32"""
    p = a.astype(np.float64) * b.astype(np.float64)   # 24 x 24 bits: exact
    c64 = c.astype(np.float64)
    s = p + c64
    bv = s - p
    err = (p - (s - bv)) + (c64 - bv)                 # TwoSum: p + c = s + err exactly
    even = (s.view(np.int64) & 1) == 0
    s = np.where((err != 0) & even, np.nextafter(s, np.where(err > 0, np.inf, -np.inf)), s)
    return s.astype(F32)


def index_magic(step, n, aux):
    """kFloorMagic + floor(fl(fl(step n) + aux)), as the kernel computes it"""
    return add_rd((step * n).astype(F32) + aux, np.full_like(step, MAGIC))


def boundary_estimate(step, inv_step, aux, lo):
    """warp_tile_chunks: the last sample (relative to lo) that keeps the index of sample lo, clamped to the chunk"""
    magic = np.full_like(step, MAGIC)
    g = ((step * lo).astype(F32) + aux).astype(F32)
    t0 = add_rd(g, magic)
    e = ((t0 - (MAGIC - F32(1.0))).astype(F32) - g).astype(F32)
    c = np.minimum(fma_rn(e, inv_step, np.full_like(step, F32(0.5))), F32(16.5))
    tk = add_rd(c, magic)
    nk = (tk + (lo - MAGIC).astype(F32)).astype(F32)
    tb = index_magic(step, nk, aux)
    k = (tk.view(np.int32) - MAGIC.view(np.int32)).astype(np.int64)
    return np.minimum(k - (tb != t0), CHUNK - 1), t0


def boundary_scan(step, aux, lo):
    """the same from the exact formula at every sample of the chunk"""
    i = np.stack([np.floor((step * (lo + F32(j))).astype(F32) + aux).astype(np.float64) for j in range(CHUNK + 1)])
    assert np.all(i[1:] >= i[:-1])
    assert np.all(i[CHUNK - 1] - i[0] <= 1)   # at most one rise inside a chunk: the precondition's first half
    return np.sum(i[:CHUNK] == i[0], axis=0) - 1, i[0]


def chunk_precondition(step, aux, n_last):
    """the kernel's test at the item set-up, for an epoch whose last sample is n_last, in float64"""
    s = step.astype(np.float64)
    i_first = np.floor((step * F32(0)).astype(F32) + aux)
    i_last = np.floor((step * n_last.astype(F32)).astype(F32) + aux)
    M = s * (n_last + 16.0) + np.maximum(np.abs(i_first), np.abs(i_last)) + 3.0
    return (s > 0) & (15 * s + M * 2.0 ** -22 < 1.0) & ((M + 1.0) * 2.0 ** -22 < s * (1.0 - 2.0 ** -18))


def draw(rng, n):
    aux = rng.uniform(-1100.0, 1100.0, n).astype(F32)
    n0 = rng.integers(0, 2_000_001, n)
    n0[: n // 4] = rng.integers(0, 30_000, n // 4)   # a quarter inside a 1 ms epoch at 25 Msps
    return aux, n0.astype(F32)


def check(step, aux, n0):
    keep = chunk_precondition(step, aux, n0.astype(np.float64) + 15.0)
    step, aux, n0 = step[keep], aux[keep], n0[keep]
    inv_step = (F32(1.0) / step).astype(F32)
    got, t0 = boundary_estimate(step, inv_step, aux, n0)
    want, i0 = boundary_scan(step, aux, n0)
    assert np.array_equal(t0.astype(np.float64) - float(MAGIC), i0)
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, [(float(step[k]), float(aux[k]), float(n0[k]), int(got[k]), int(want[k])) for k in bad[:5]]
    return int(keep.sum()), np.bincount(want, minlength=CHUNK)


def test_fma_and_round_down_restatements():
    rng = np.random.default_rng(1)
    a = rng.uniform(-2, 2, 100000).astype(F32)
    b = rng.uniform(-2, 2, 100000).astype(F32)
    c = rng.uniform(-2, 2, 100000).astype(F32)
    from fractions import Fraction
    for k in range(0, 100000, 997):
        exact = Fraction(float(a[k])) * Fraction(float(b[k])) + Fraction(float(c[k]))
        got = fma_rn(a[k:k + 1], b[k:k + 1], c[k:k + 1])[0]
        lo, hi = np.nextafter(got, F32(-np.inf)), np.nextafter(got, F32(np.inf))
        assert abs(Fraction(float(got)) - exact) <= abs(Fraction(float(lo)) - exact)
        assert abs(Fraction(float(got)) - exact) <= abs(Fraction(float(hi)) - exact)
    x = rng.uniform(-4e6, 4e6, 100000).astype(F32)
    x[:1000] = rng.uniform(-1e-3, 1e-3, 1000).astype(F32)
    assert np.array_equal(add_rd(x, np.full_like(x, MAGIC)).astype(np.float64) - float(MAGIC), np.floor(x.astype(np.float64)))


def test_boundary_estimate_matches_exact_scan():
    rng = np.random.default_rng(20261018)
    n = 200_000
    total, hist = 0, np.zeros(CHUNK, dtype=np.int64)
    for fs in (16.368e6, 25e6, 50e6):
        dop = rng.uniform(-10e3, 10e3, n)
        step = (1.023e6 * (1.0 + dop / 1575.42e6) / fs).astype(F32)
        step[: n // 8] = F32(1.023e6 / fs)
        kept, h = check(step, *draw(rng, n))
        assert kept > 0.9 * n
        total, hist = total + kept, hist + h
    # steps anywhere up to the 15 step + margin < 1 limit
    step = rng.uniform(0.004, 1.0 / 15.0, n).astype(F32)
    kept, h = check(step, *draw(rng, n))
    total, hist = total + kept, hist + h
    assert total > 600_000
    assert np.all(hist > 0)   # the boundary fell on every position of a chunk, and on none (15)


def test_boundary_estimate_at_boundaries_placed_on_every_sample():
    """aux chosen so that the index rises exactly at, or one float step around, sample j of the chunk"""
    rng = np.random.default_rng(7)
    n = 50_000
    for fs in (16.368e6, 25e6, 50e6):
        step = np.full(n, 1.023e6 / fs, dtype=F32)
        n0 = rng.integers(0, 2_000_001, n).astype(F32)
        j = rng.integers(1, CHUNK + 1, n)
        chip = rng.integers(-1000, 1000, n)
        prod = (step * (n0 + j.astype(F32))).astype(F32).astype(np.float64)
        aux = (chip - prod).astype(F32)
        aux = np.where(rng.integers(0, 3, n) == 0, np.nextafter(aux, F32(-np.inf)), aux)
        aux = np.where(rng.integers(0, 3, n) == 0, np.nextafter(aux, F32(np.inf)), aux).astype(F32)
        check(step, aux, n0)
