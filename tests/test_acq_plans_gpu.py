"""The PCPS acquisition search at every FFT plan shape, on the recomputed second peak and through the device entry points,
against a float64 correlation.

Reference: the object's own wipe-off rows (read_wipeoffs, pinned bit-exact by test_wipeoff_grid_bitexact), then in
complex128 X = FFT(x . wipe), C = conj(FFT(placed code)), |IFFT_unnormalised(X . C)|^2 over columns [off, off + ne),
summed over dwells.  The statistics come from that grid through PcpsAcquisitionOracle's own rules.  Contract (the one
the float32 parity tests hold):
  * the magnitude grid within 2e-5 of the grid peak, element-wise;
  * grid_maximum, input_power, second_peak and test_statistics within 1e-4 relative;
  * index_time, index_doppler and doppler equal to the float64 arg-max.  Every input is built so that the arg-max is
    unique and beats the runner-up by at least 1e-3 (asserted on the float64 grid), so this equality is not a near-tie.
Inputs are random +-1 (I and Q) codes at one sample per symbol on carriers at the bin frequencies, plus Gaussian noise.
"""
import numpy as np
import pytest

from gpu_fixtures import capi, engine  # noqa: F401
import acq_rig as ar

pytestmark = pytest.mark.gpu

MARGIN = 1e-3
BINS4 = dict(doppler_max=1000, doppler_step=500)   # 4 Doppler bins: -1000, -500, 0, +500 Hz


def _params(n, **kw):
    """PcpsAcquisition keywords for a 1 ms code of n samples (fs = n kHz) and 4 Doppler bins."""
    return ar.params(n * 1000, **BINS4, **kw)


def _codes(rng, slots, n):
    return [(rng.choice([-1.0, 1.0], n) + 1j * rng.choice([-1.0, 1.0], n)).astype(np.complex64) for _ in range(slots)]


def _tone(f, fs, n):
    """the carrier that the wipe-off row of Doppler f removes"""
    return np.exp(2j * np.pi * f * np.arange(n) / fs)


def _signal(rng, codes, conf, fs, placements, noise=0.5, n=None):
    """sum of amp * roll(tile(code), k) * carrier(f) over placements (slot, amp, k, f), plus noise; n samples (consumed)"""
    n = conf.consumed_samples if n is None else n
    x = rng.normal(0, noise, n) + 1j * rng.normal(0, noise, n)
    for s, amp, k, f in placements:
        x += amp * np.roll(np.resize(codes[s], n), k) * _tone(f, fs, n)
    return x.astype(np.complex64)


def _ref_grid(conf, wipe, x, code):
    """float64 |IFFT_unnormalised(FFT(x . wipe) . conj(FFT(placed code)))|^2, columns [off, off + ne)"""
    n, ne, consumed, layout = conf.fft_size, conf.effective_fft_size, conf.consumed_samples, conf.code_layout
    sig = np.zeros(n, np.complex128)
    sig[:consumed] = x[:consumed]
    X = np.fft.fft(sig[None, :] * wipe.astype(np.complex128), axis=1)
    buf = np.zeros(n, np.complex128)
    place = n // 2 if layout == 1 else (n - consumed if layout == 2 else 0)   # acq_code_offset
    need = n // 2 if layout == 1 else consumed
    buf[place:place + need] = code[:need]
    y = np.fft.ifft(X * np.conj(np.fft.fft(buf))[None, :], axis=1) * n
    off = ne if conf.bit_transition_flag else 0
    return np.abs(y[:, off:off + ne]) ** 2


def _ref_stats(o, grid, dwells=1):
    o.magnitude_grid = grid
    o.num_noncoherent_integrations_counter = dwells
    return o.max_to_input_power_statistic() if o.c.use_CFAR_algorithm_flag else o.first_vs_second_peak_statistic()


def _assert_unique_peak(grid):
    top = np.partition(grid.ravel(), -2)[-2:]
    assert top[1] >= (1.0 + MARGIN) * top[0], f"input has no unique arg-max: {top[1]:.6g} vs runner-up {top[0]:.6g}"


def _search_all_slots(capi, engine, p, codes, iq, dwell_inputs=()):
    """Search every other slot in descending order ([2, 0] of three), then all of them in order (and again on each further
    dwell input); check every slot's record against the float64 reference, and that both searches give it the same bytes.
    Returns (acq, records of the last search, reference grids)."""
    acq = capi.PcpsAcquisition(engine, **p)
    conf = acq.conf
    ar.load_codes(acq, codes)
    wipe = acq.read_wipeoffs()
    o = ar.oracle(p)
    stats = ar.CFAR_STATS if o.c.use_CFAR_algorithm_flag else ar.PEAK_STATS
    assert (o.c.fft_size, o.c.effective_fft_size, o.c.num_doppler_bins) == (conf.fft_size, conf.effective_fft_size, conf.num_doppler_bins)
    refs = [_ref_grid(conf, wipe, iq, c) for c in codes]
    every = list(range(len(codes)))
    some = every[::-2]   # [2, 0] of three slots
    part = acq.search(iq, some)
    res = acq.search(iq, every)
    for i, s in enumerate(some):
        assert part[i].tobytes() == res[s].tobytes(), (some, s)
    for d, x in enumerate(dwell_inputs, start=2):   # further dwells accumulate into the grid
        refs = [g + _ref_grid(conf, wipe, x, c) for g, c in zip(refs, codes)]
        res = acq.search(x, every, dwell_counter=d)
    for s, g in enumerate(refs):
        _assert_unique_peak(g)
        ar.check(res[s], _ref_stats(o, g, 1 + len(dwell_inputs)), stats, f"slot {s}")
    return acq, res, refs


def _plan_case(capi, engine, n, cfar, keep_grid, seed, slots=3, **kw):
    p = _params(n, use_CFAR_algorithm_flag=cfar, keep_grid=keep_grid, n_code_slots=slots, **kw)
    rng = np.random.default_rng(seed)
    probe = ar.oracle(p).c
    need = ar.code_len(probe)
    codes = _codes(rng, slots, need)
    # slot s: amplitude 1 - 0.2 s, its own delay and Doppler bin (bins are -1000, -500, 0, +500 Hz)
    # zero-padded layout: a delay k splits the correlation into peaks of k and consumed - k samples; keep them far apart
    kmax = need // 4 if kw.get("ms_per_code", 1) != kw.get("sampled_ms", 1) else need
    placements = [(s, 1.0 - 0.2 * s, int(rng.integers(0, kmax)), (500.0, -1000.0, -500.0)[s]) for s in range(slots)]
    iq = _signal(rng, codes, probe, p["fs_in"], placements)
    acq, res, refs = _search_all_slots(capi, engine, p, codes, iq)
    errs = [ar.check_grid(acq.read_grid(s), refs[s]) for s in range(slots)] if keep_grid else []
    fft_size, layout = acq.conf.fft_size, acq.conf.code_layout
    acq.close()
    if errs:
        print(f"grid error vs float64, fft_size {fft_size}, code layout {layout}: {max(errs):.3e} of the peak")


# two-level sizes: expected plan n1 x [in-shared-memory radices] in the comment.  (56 000 points in test_acq_gpu.py plans as
# 4 x 14 000, since 56 000 / 2 = 28 000 exceeds 27 648: global radix 7 runs here first.)
@pytest.mark.parametrize("n", [
    75000,    # 3 x [8, 5, 5, 5, 5, 5]: global radix 3
    125000,   # 5 x [8, 5, 5, 5, 5, 5]: global radix 5
    175000,   # 7 x [8, 5, 5, 5, 5, 5]: global radix 7
    147000,   # 7 x [8, 3, 7, 5, 5, 5]: radix 7 over blocks with radix-3 and radix-7 stages
    250000,   # 10 x [8, 5, 5, 5, 5, 5]: global radix 10
    276480,   # 10 x [8, 8, 8, 2, 3, 3, 3]: the largest size the planner accepts
])
@pytest.mark.parametrize("cfar,keep_grid", [(True, True), (True, False), (False, True), (False, False)])
def test_two_level_radices_against_float64(capi, engine, n, cfar, keep_grid):
    """Without a grid and without CFAR the second-peak pass recomputes the winning row through the block kernel, the
    final radix-n1 stage and the row reduction."""
    _plan_case(capi, engine, n, cfar, keep_grid, seed=n)


@pytest.mark.parametrize("n", [
    25000,    # [8, 25, 25, 5] on 512 threads
    3125,     # [25, 25, 5] on 512 threads
    15625,    # [5, 5, 5, 5, 5, 5] on 1024 threads: six radix-5 stages
    27648,    # [8, 8, 8, 2, 3, 3, 3]: seven stages, the single-CTA maximum
    4802,     # [2, 7, 7, 7, 7]
    210,      # [2, 3, 7, 5]
])
def test_single_cta_plans_against_float64(capi, engine, n):
    for cfar, keep_grid in ((True, True), (False, True), (False, False)):
        _plan_case(capi, engine, n, cfar, keep_grid, seed=n + 1)


def test_fft_plan_only_from_the_size(capi, engine, monkeypatch):
    """B200_ACQ_RADIX25 in the environment selects nothing: with B200_ACQ_RADIX25=0 a 25 000-point search still plans
    [8, 25, 25, 5], so its records and grids, which [8, 5, 5, 5, 5, 5] would sum in another order, are the same bytes."""
    p = _params(25000, keep_grid=True, n_code_slots=3)
    rng = np.random.default_rng(25)
    codes = _codes(rng, 3, 25000)
    iq = _signal(rng, codes, ar.oracle(p).c, p["fs_in"], [(0, 1.0, 777, 500.0), (1, 0.8, 12345, -1000.0)])

    def search():
        acq = capi.PcpsAcquisition(engine, **p)
        ar.load_codes(acq, codes)
        out = acq.search(iq, [0, 1, 2]).tobytes() + b"".join(acq.read_grid(s).tobytes() for s in range(3))
        acq.close()
        return out

    want = search()
    monkeypatch.setenv("B200_ACQ_RADIX25", "0")
    assert search() == want


@pytest.mark.parametrize("n", [7, 8, 25])   # one stage of 7, one of 8, two of 5
def test_smallest_sizes_search_right_or_refuse(capi, engine, n):
    try:
        capi.PcpsAcquisition(engine, **_params(n)).close()
    except capi.B200Error:
        return   # refusing a size is allowed; a wrong answer is not
    rng = np.random.default_rng(n)
    for cfar, keep_grid in ((True, True), (False, False)):
        p = _params(n, use_CFAR_algorithm_flag=cfar, keep_grid=keep_grid)
        code = _codes(rng, 1, n)
        iq = np.roll(code[0], 3).astype(np.complex64)   # zero Doppler: exact wipe-off row, no noise
        acq = capi.PcpsAcquisition(engine, **p)
        acq.set_local_code(0, code[0])
        ref = _ref_grid(acq.conf, acq.read_wipeoffs(), iq, code[0])
        _assert_unique_peak(ref)
        ar.check(acq.search(iq, [0])[0], _ref_stats(ar.oracle(p), ref), ar.CFAR_STATS if cfar else ar.PEAK_STATS, f"N = {n}")
        if keep_grid:
            ar.check_grid(acq.read_grid(0), ref)
        acq.close()


def test_two_level_dwells_accumulate_against_float64(capi, engine):
    """max_dwells = 2 at 125 000 points (5 x [8, 5, 5, 5, 5, 5]): the grid and the CFAR input power (divided by the dwell
    counter) of two accumulated dwells."""
    p = _params(125000, max_dwells=2, n_code_slots=3)
    rng = np.random.default_rng(2)
    codes = _codes(rng, 3, 125000)
    placements = [(0, 1.0, 4321, 500.0), (1, 0.8, 99999, -1000.0), (2, 0.6, 7, -500.0)]
    conf = ar.oracle(p).c
    iq1, iq2 = (_signal(rng, codes, conf, p["fs_in"], placements, noise=2.0) for _ in range(2))
    acq, _, refs = _search_all_slots(capi, engine, p, codes, iq1, dwell_inputs=[iq2])
    errs = [ar.check_grid(acq.read_grid(s), refs[s]) for s in range(3)]
    print(f"grid error vs float64, N = 125000, two dwells: {max(errs):.3e} of the peak")
    acq.close()


@pytest.mark.parametrize("cfar,keep_grid", [(True, True), (False, False)])
def test_two_level_bit_transition_layout(capi, engine, cfar, keep_grid):
    """bit_transition_flag at 37.5 MHz: fft_size 75 000 = 3 x [8, 5, 5, 5, 5, 5], code in the second half, magnitudes
    from the second half (code layout 1)."""
    _plan_case(capi, engine, 37500, cfar, keep_grid, seed=375, bit_transition_flag=True)


@pytest.mark.parametrize("cfar,keep_grid", [(True, True), (False, False)])
def test_two_level_zero_padded_layout(capi, engine, cfar, keep_grid):
    """62 500 consumed samples of a 2 ms code: fft_size 125 000 = 5 x [8, 5, 5, 5, 5, 5], code zero-padded at the front
    (code layout 2)."""
    _plan_case(capi, engine, 62500, cfar, keep_grid, seed=625, ms_per_code=2)


def test_two_level_step_two_against_float64(capi, engine):
    """Step two at 175 000 points (7 x [8, 5, 5, 5, 5, 5]): 4 bins of 125 Hz around the step-one Doppler, the wipe-off rows
    of update_grid_doppler_wipeoffs_step2, the float Doppler formula and the step-one input power."""
    p = _params(175000, keep_grid=True)
    rng = np.random.default_rng(175)
    code = _codes(rng, 1, 175000)
    conf = ar.oracle(p).c
    iq1 = _signal(rng, code, conf, p["fs_in"], [(0, 1.0, 123456, 500.0)])
    acq, res, _ = _search_all_slots(capi, engine, p, code, iq1)
    first = res[0]
    o = ar.oracle(p, num_doppler_bins_step2=4, doppler_step2=125.0)
    o.doppler_center_step_two = np.float32(first["doppler"])
    o.update_grid_doppler_wipeoffs_step2()
    iq2 = _signal(rng, code, conf, p["fs_in"], [(0, 1.0, 123456, float(first["doppler"]) - 125.0)])
    acq.set_step_two(float(first["doppler"]), 125.0, 4)
    got = acq.search_step_two(iq2, 0, float(first["input_power"]))
    ref = _ref_grid(acq.conf, o.grid_doppler_wipeoffs_step_two, iq2, code[0])
    _assert_unique_peak(ref)
    o.step_two = True
    o.input_power = np.float32(first["input_power"])
    ar.check(got, _ref_stats(o, ref), what="step two")
    assert int(got["doppler"]) == int(first["doppler"]) - 125
    ar.check_grid(acq.read_grid(0), ref)   # as many step-two bins as step-one bins: the whole grid of the slot
    acq.close()


@pytest.fixture(scope="module")
def window_refs():
    return {}


@pytest.mark.parametrize("n,spc", [
    (4000, 4),      # single CTA: the pass runs in acq_corr_kernel
    (75000, 73),    # 3 x [8, 5, 5, 5, 5, 5]: block kernel -> final radix-3 stage -> row reduction
])
@pytest.mark.parametrize("keep_grid", [True, False])   # with a grid the pass reads the stored row, without it recomputes it
def test_second_peak_exclusion_window(capi, engine, window_refs, n, spc, keep_grid):
    """first_vs_second_peak_statistic zeroes [t - spc, t + spc) around the peak t, wrapping at both ends
    (pcps_acquisition.cc:485-509), before its second arg-max.  Input: the code rolled by k plus half of it rolled by
    k + lag.  lag = -spc and spc - 1 fall inside the window, -spc - 1 and spc do not, so an off-by-one at either end moves
    second_peak from a sidelobe to a quarter of the peak or back."""
    p = _params(n, samples_per_chip=spc, use_CFAR_algorithm_flag=False, keep_grid=keep_grid)
    rng = np.random.default_rng(n + spc)
    code = _codes(rng, 1, n)[0]
    acq = capi.PcpsAcquisition(engine, **p)
    acq.set_local_code(0, code)
    wipe = acq.read_wipeoffs()
    o = ar.oracle(p)
    for k in (0, 1, spc - 1, spc, n - spc - 1, n - spc, n - 1):
        for lag in (-spc - 1, -spc, spc - 1, spc):
            key = (n, spc, k, lag)
            if key not in window_refs:
                iq = (np.roll(code, k) + 0.5 * np.roll(code, k + lag)).astype(np.complex64)   # zero Doppler (bin 2)
                ref = _ref_grid(acq.conf, wipe, iq, code)
                _assert_unique_peak(ref)
                window_refs[key] = (iq, ref, _ref_stats(o, ref))
            iq, ref, want = window_refs[key]
            assert (want["index_time"], want["index_doppler"]) == (k, 2)
            inside = lag in (-spc, spc - 1)
            ratio = want["second_peak"] / want["grid_maximum"]
            assert (ratio < 0.01) if inside else (0.15 < ratio < 0.4), (k, lag, ratio)
            got = acq.search(iq, [0])[0]
            ar.check(got, want, ar.PEAK_STATS, f"k = {k}, lag = {lag}")
            if keep_grid:
                ar.check_grid(acq.read_grid(0), ref)
    acq.close()


# ---- chirp-z (Bluestein) sizes: N-point transforms as M-point circular convolutions, M >= 2N - 1 ----------------------
@pytest.mark.parametrize("n", [
    5456,     # M = 10 935 = 3 x [3, 3, 3, 3, 3, 3, 5]
    13000,    # M = 26 244 = 2 x [2, 3, 3, 3, 3, 3, 3, 3, 3]
    16368,    # M = 32 768 = 2 x [8, 8, 8, 8, 4]
    32736,    # M = 65 536 = 4 x [8, 8, 8, 8, 4]
    122760,   # M = 245 760 = 10 x [8, 8, 8, 8, 2, 3]
])
def test_chirp_z_selftest_dft_against_float64(capi, engine, n):
    acq = capi.PcpsAcquisition(engine, **_params(n))
    rng = np.random.default_rng(n)
    x = (rng.normal(size=n) + 1j * rng.normal(size=n)).astype(np.complex64)
    want = np.fft.fft(x.astype(np.complex128))
    got = acq.selftest_dft(x)
    acq.close()
    rel = float(np.sqrt(np.mean(np.abs(got - want) ** 2) / np.mean(np.abs(want) ** 2)))
    print(f"chirp-z DFT RMS error vs float64, N = {n}: {rel:.3e} of the RMS of X")
    assert rel < 1e-5


@pytest.mark.parametrize("keep_grid", [True, False])
def test_chirp_z_largest_radix_search_against_float64(capi, engine, keep_grid):
    """N = 122 760 = 2^3 * 3 * 5 * 11 * 31: M = 245 760 = 10 x 24 576, the radix-10 global stage under the chirp-z search."""
    _plan_case(capi, engine, 122760, True, keep_grid, seed=12276)


# ---- device entry points ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [4000, 75000, 16368])   # single CTA, 3 x [8, 5, 5, 5, 5, 5], chirp-z
def test_search_dev_leaves_what_search_returns(capi, engine, n):
    import torch
    p = _params(n, n_code_slots=3)
    acq = capi.PcpsAcquisition(engine, **p)
    rng = np.random.default_rng(n)
    codes = _codes(rng, 3, n)
    ar.load_codes(acq, codes)
    iq = _signal(rng, codes, acq.conf, p["fs_in"], [(1, 1.0, 77, 500.0), (0, 0.7, n // 3, 0.0)])
    want = acq.search(iq, [1, 2, 0])
    x = torch.from_numpy(iq.view(np.float32)).cuda()
    res = torch.full((3 * capi.ACQ_RESULT_DTYPE.itemsize,), 0xAB, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()   # the acquisition object works on its own stream
    acq.search_dev(x.data_ptr(), [1, 2, 0], res.data_ptr())
    torch.cuda.synchronize()
    assert res.cpu().numpy().tobytes() == want.tobytes()
    acq.close()


@pytest.mark.parametrize("n", [4000, 75000])   # single CTA, 3 x [8, 5, 5, 5, 5, 5]
def test_search_i16_equals_search_on_widened_samples(capi, engine, n):
    p = _params(n, n_code_slots=2)
    acq = capi.PcpsAcquisition(engine, **p)
    rng = np.random.default_rng(n + 16)
    codes = _codes(rng, 2, n)
    ar.load_codes(acq, codes)
    raw = ar.to_int(_signal(rng, codes, acq.conf, p["fs_in"], [(0, 1.0, 1234, -500.0)], noise=1.0), np.int16, 300)
    got = ar.search_i16(acq, raw, [1, 0])
    assert got.tobytes() == acq.search(ar.from_int(raw), [1, 0]).tobytes()
    acq.close()


@pytest.mark.parametrize("n", [0, 1, 31, 32, 33, 100])
@pytest.mark.parametrize("prns", ["descending", "shuffled", "repeated"])
def test_sweep_best_dev_breaks_ties_like_best_peak(capi, engine, n, prns):
    """The record b200_acq_sweep_best_dev leaves equals dist.best_peak of the same records: the largest statistic, ties to
    the lowest PRN, then the lowest Doppler bin, then the lowest code phase, whatever order the results come in."""
    import torch
    from gnss_sdr_b200 import dist as bd
    acq = capi.PcpsAcquisition(engine, **_params(4000))
    rng = np.random.default_rng(1000 * n + len(prns))
    res = np.zeros(max(n, 1), capi.ACQ_RESULT_DTYPE)
    res["test_statistics"] = rng.choice(np.float32([0.0, 2.5, 7.25]), res.size)
    res["test_statistics"][rng.permutation(res.size)[:3]] = 9.5     # up to three records share the best statistic
    res["index_doppler"] = rng.integers(0, 3, res.size)
    res["index_time"] = rng.integers(0, 200000, res.size)
    if prns == "descending":
        prn = np.arange(res.size, 0, -1)
    elif prns == "shuffled":
        prn = rng.permutation(res.size) + 1
    else:   # the same PRN more than once: bin and code phase decide
        prn = rng.integers(1, 3, res.size)
    prn = prn.astype(np.uint32)
    peaks = np.zeros(n, bd.PEAK_DTYPE)
    for f in ("test_statistics", "index_doppler", "index_time"):
        peaks[f] = res[f][:n]
    peaks["prn"] = prn[:n]
    want = np.array([bd.best_peak(peaks)], bd.PEAK_DTYPE)
    res_dev = torch.from_numpy(res.view(np.uint8).copy()).cuda()
    prn_dev = torch.from_numpy(prn.view(np.int32).copy()).cuda()
    out = torch.full((16,), 0xAB, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()   # the acquisition object works on its own stream
    acq.sweep_best_dev(res_dev.data_ptr(), prn_dev.data_ptr(), n, out.data_ptr())
    torch.cuda.synchronize()
    got = out.cpu().numpy().view(bd.PEAK_DTYPE)
    assert got.tobytes() == want.tobytes(), (got, want)
    acq.close()
