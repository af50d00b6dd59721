"""BASELINE.json's full sizes (C2: 32 channels x 1000 epochs x 25 000 samples; C4: 32 PRNs x 80-81 Doppler bins x 25 000 points)
checked through size-independent properties - the CPU oracle cannot cover 8e8 channel-samples in seconds, the properties can:
  tracking     exact linearity on integer-valued samples, batch-splitting invariance, the two kernels agreeing bit for bit,
               the oracle on a random handful of the 32 000 work items;
  acquisition  one 32-PRN sweep == 32 single-PRN searches, a circular shift of the input moves the peak by that many samples
               and nothing else, a frequency shift by one Doppler step moves it one bin."""
import numpy as np
import pytest

from gnss_synth import make_iq, trk_params_for
import acq_rig as ar
from gpu_fixtures import capi  # noqa: F401
import trk_rig as tr

pytestmark = pytest.mark.gpu

FS, N, NCH, NEP = 25e6, 25000, 32, 1000


@pytest.fixture(scope="module")
def c2(capi, oracle):
    """The C2 workload with integer-valued samples (|re|, |im| <= 6) on two independent streams x1, x2 and their combination
    3*x1 - 2*x2; zero carrier so that every tap is an exact integer sum (< 2^24: exact in float32 whatever the order)."""
    rng = np.random.default_rng(20)
    n_iq = N * NEP + 64
    x1 = (rng.integers(-6, 7, n_iq) + 1j * rng.integers(-6, 7, n_iq)).astype(np.complex64)
    x2 = (rng.integers(-6, 7, n_iq) + 1j * rng.integers(-6, 7, n_iq)).astype(np.complex64)
    eng = capi.Engine(0)
    bands = {b: tr.ring(eng, b, x) for b, x in enumerate((x1, x2, 3 * x1 - 2 * x2))}
    codes = [oracle.port.gps_ca_code(p) for p in range(1, NCH + 1)]
    shifts = [-0.5, 0.0, 0.5]
    items = {}
    steps = 1.023e6 * (1 + rng.uniform(-4000, 4000, NCH) / 1575.42e6) / FS
    phase0 = rng.uniform(0, 1023, NCH)
    k = np.arange(NEP)
    rems = [-np.mod(phase0[c] + steps[c] * k * N, 1023.0) for c in range(NCH)]
    for b in bands:
        cids = [tr.channel(eng, b, codes[c], shifts) for c in range(NCH)]
        # epoch-major: the channels of one epoch are neighbours; staggered epoch starts, as real channels have
        items[b] = tr.items((cids[c], N, bands[b] + j * N + (c % 7), 0.0, 0.0, 0.0, rems[c][j], steps[c])
                            for j in range(NEP) for c in range(NCH))
    yield eng, items, (x1, x2), codes, shifts
    eng.close()


def test_c2_full_size_linearity_is_exact(c2):
    """taps(3 x1 - 2 x2) == 3 taps(x1) - 2 taps(x2), all 96 000 complex taps, exactly."""
    eng, items, _, _, _ = c2
    t1, t2, t3 = (eng.trk_batch(items[b], 3) for b in (0, 1, 2))
    assert t1.shape == (NCH * NEP, 3)
    assert np.array_equal(t3, 3 * t1 - 2 * t2)
    assert np.all(t1.real == np.round(t1.real)) and np.count_nonzero(t1) > 0.99 * t1.size


def test_c2_full_size_batch_splitting_and_kernel_choice(c2):
    """The 32 000-item batch in one launch, in eight launches of 4000, through the shared-window kernel and through the
    per-item kernel: the same bits."""
    eng, items, _, _, _ = c2
    it = items[0]
    eng.trk_kernel_choice(1)
    whole = eng.trk_batch(it, 3)
    parts = np.concatenate([eng.trk_batch(it[i:i + 4000], 3) for i in range(0, len(it), 4000)])
    eng.trk_kernel_choice(0)
    per_item = eng.trk_batch(it, 3)
    eng.trk_kernel_choice(-1)
    assert np.array_equal(whole, parts)
    assert np.array_equal(whole, per_item)


def test_c2_full_size_random_items_against_the_oracle(c2, oracle):
    eng, items, (x1, _), codes, shifts = c2
    it = items[0]
    got = eng.trk_batch(it, 3)
    rng = np.random.default_rng(3)
    for i in rng.choice(len(it), 24, replace=False):
        c = i % NCH
        s0 = int(it[i]["sample_index"])
        want = oracle.port.multicorrelator(1, x1[s0:s0 + N], codes[c], shifts, 0.0, 0.0, float(it[i]["rem_code_phase_chips"]),
                                           float(it[i]["code_phase_step_chips"]))
        assert np.array_equal(got[i], want), i


def test_c2_full_size_signal_prompt_dominates(capi, oracle):
    """A real C2 stretch: 32 satellites at 45 dB-Hz, perfectly steered replicas.  Per channel, averaged over its epochs, the
    prompt carries the full signal amplitude (N A) and the early / late taps half of it - i.e. no work item read the wrong
    samples, the wrong code or the wrong NCO parameters."""
    from gnss_synth import ca_amplitude
    rng = np.random.default_rng(5)
    codes = {p: oracle.port.gps_ca_code(p) for p in range(1, NCH + 1)}
    svs = [dict(prn=p, doppler=float(rng.uniform(-5000, 5000)), code_phase_chips=float(rng.uniform(0, 1023)), cn0=45.0,
                phase0=float(rng.uniform(0, 6.28))) for p in range(1, NCH + 1)]
    n_ep = 200                                       # 0.2 s of the stream is enough for this property (5 M samples)
    iq = make_iq(codes, FS, N * n_ep + 64, svs, seed=6)
    eng = capi.Engine(0)
    first = tr.ring(eng, 0, iq)
    rows = [None] * (NCH * n_ep)
    for c, sv in enumerate(svs):
        cid = tr.channel(eng, 0, codes[sv["prn"]], [-0.5, 0.0, 0.5])
        s, rc, dp, rcode, st = trk_params_for(sv, FS, N, n_ep)
        rows[c::NCH] = [(cid, N, first + int(s[k]), rc[k], dp[k], 0.0, rcode[k], st[k]) for k in range(n_ep)]
    taps = eng.trk_batch(tr.items(rows), 3)
    eng.close()
    full = N * ca_amplitude(45.0, FS)
    for c in range(NCH):
        t = taps[c::NCH]
        # coherent mean over the epochs: the replica is steered to the signal's phase, the signal adds up, the noise does not
        assert abs(np.mean(t[:, 1]).real - full) < 0.1 * full, c
        assert abs(abs(np.mean(t[:, 0])) - 0.5 * full) < 0.1 * full and abs(abs(np.mean(t[:, 2])) - 0.5 * full) < 0.1 * full, c


# ---------------------------------------------------------------------------------------------------------------- acquisition
ACQ_FS, ACQ_N, DMAX, DSTEP = 25_000_000, 25000, 10000, 250     # C4's grid moved by half a bin: whole-kHz carriers sit ON a bin (80 bins)


@pytest.fixture(scope="module")
def c4(capi, oracle):
    eng = capi.Engine(0)
    acq = ar.make(capi, eng, ACQ_FS, doppler_max=DMAX, doppler_step=DSTEP, n_code_slots=32)
    ar.load_codes(acq, [ar.ca_code(oracle.port, p, ACQ_FS) for p in range(1, 33)])
    present = [2, 5, 9, 13, 17, 21, 26, 30]
    rng = np.random.default_rng(8)
    codes = {p: oracle.port.gps_ca_code(p) for p in present}
    # Dopplers on whole kHz: the carrier is then periodic in the 1 ms block, which makes a rotation of the block an exact symmetry
    svs = [dict(prn=p, doppler=1000.0 * float(rng.integers(-8, 9)), code_phase_chips=float(rng.uniform(0, 1023)), cn0=47.0,
                phase0=float(rng.uniform(0, 6.28))) for p in present]
    iq = make_iq(codes, float(ACQ_FS), ACQ_N, svs, seed=9)
    yield acq, iq, present
    acq.close()
    eng.close()


def test_c4_sweep_equals_single_prn_searches(c4):
    acq, iq, present = c4
    assert acq.conf.num_doppler_bins == 80
    sweep = acq.search(iq, np.arange(32))
    for p in range(32):
        assert acq.search(iq, [p])[0] == sweep[p], p
    from oracle.acq_np import compute_threshold
    th = compute_threshold(0.001, ACQ_N, 80, 1)
    # (whole-kHz Dopplers are the worst case for C/A cross-correlation - the code's spectral lines sit 1 kHz apart - so a
    # satellite or two may stay under the threshold; nothing that is not there may cross it)
    detected = {p + 1 for p in range(32) if sweep[p]["test_statistics"] > th}
    assert detected <= set(present) and len(detected) >= len(present) - 2


def test_c4_circular_shift_moves_the_peak_only(c4):
    """PCPS is a circular correlation over the 1 ms block: with carriers that are periodic in the block (fixture), rotating the
    block by s samples moves every code phase by s and leaves the rest alone."""
    acq, iq, present = c4
    base = acq.search(iq, np.arange(32))
    strong = [p for p in present if base[p - 1]["test_statistics"] > 40.0]     # the noise floor's maximum is not a symmetry of anything
    assert len(strong) >= len(present) - 2
    for s in (1, 777, 12500, 24999):
        got = acq.search(np.roll(iq, s), np.arange(32))
        for p in strong:
            b, g = base[p - 1], got[p - 1]
            # +-3 samples: at 24.4 samples per chip the correlation of two sampled chip sequences has a flat top a few samples
            # wide, and which of its equal values wins is rounding
            assert (int(g["index_time"]) - int(b["index_time"]) - s + 3) % ACQ_N <= 6, (p, s)
            # (the neighbouring bins are only 0.9 dB down and NOT symmetric under the rotation: with noise one of them may win)
            assert abs(int(g["index_doppler"]) - int(b["index_doppler"])) <= 1
            assert abs(g["test_statistics"] - b["test_statistics"]) / b["test_statistics"] < 0.15


def test_c4_frequency_shift_moves_one_doppler_bin(c4):
    acq, iq, present = c4
    base = acq.search(iq, np.arange(32))
    n = np.arange(ACQ_N, dtype=np.float64)
    shifted = (iq.astype(np.complex128) * np.exp(2j * np.pi * DSTEP * n / ACQ_FS)).astype(np.complex64)
    got = acq.search(shifted, np.arange(32))
    for p in [q for q in present if base[q - 1]["test_statistics"] > 40.0]:
        b, g = base[p - 1], got[p - 1]
        assert int(g["index_doppler"]) == int(b["index_doppler"]) + 1, p
        assert int(g["doppler"]) == int(b["doppler"]) + DSTEP
        assert abs(int(g["index_time"]) - int(b["index_time"])) <= 3
        assert abs(g["test_statistics"] - b["test_statistics"]) / b["test_statistics"] < 5e-3
