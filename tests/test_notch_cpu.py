"""The notch restatement (notch_np) against the reference's Notch and NotchLite blocks compiled in place
(oracle/_ref/liboracle_ref_notch.so), with no GPU.

With the block's own est and z0 injected segment by segment, the restatement's serial float32 recursion reproduces the block
byte for byte: decisions, resets, runs, coefficient epochs, copied, estimation and filtered samples.  Without injection, the
restatement's est stays within EST_ULPS of the block's and each z0 component within Z0_ULPS units of 2^-24: the block takes its spectrum from a float
FFT and its transcendentals from float libm functions, the restatement (and the device) from float64 rounded once.  The
device's split-invariant recursion stays within notch_np.recursion_bound of the float64 truth.  The status struct matches
the header's layout, and the argument refusals that need no engine are covered."""
import ctypes

import numpy as np
import pytest

import notch_np as nn

EST_ULPS = 16   # largest seen over these streams: 11 (L = 301)
Z0_ULPS = 8     # of 1 (2^-24 each), on each component: z0 is a unit vector, so its error is the angle's, up to 2^-22

LIB = nn.reference_lib()
needs_ref = pytest.mark.skipif(LIB is None, reason="the reference notch blocks are not built (oracle/notch.mk)")


def _stream(seed, n, kind):
    rng = np.random.default_rng(seed)
    if kind == "zeros":
        return np.zeros(n, np.complex64)
    x = (rng.standard_normal(n) + 1j * rng.standard_normal(n)) * 0.7
    if kind == "cw":
        t = np.arange(n)
        x = x + ((t // 2500) % 2 == 1) * 5.0 * np.exp(1j * (0.37 * t + 0.2))
    return x.astype(np.complex64)


def _ulps(a, b):
    return abs(int(np.float32(a).view(np.int32)) - int(np.float32(b).view(np.int32)))


PARAMS = [(v, L, nc) for v, Ls in ((nn.NOTCH_LITE, (1, 7, 32, 301)), (nn.NOTCH, (7, 32, 301))) for L in Ls
          for nc in ((1, 3) if v == nn.NOTCH_LITE else (1,))]


@needs_ref
@pytest.mark.parametrize("kind", ["noise", "cw", "zeros"])
@pytest.mark.parametrize("p", [0.9, 0.5, -0.7])
@pytest.mark.parametrize("pfa", [1e-3, 0.04])
@pytest.mark.parametrize("variant,length,n_coeff", PARAMS)
def test_injected_restatement_is_the_block(variant, length, n_coeff, pfa, p, kind):
    n = max(30 * length, 6000)
    x = _stream(7 * length + n_coeff, n, kind)
    E, R = 6, 45
    out, st, f, est, z0 = nn.reference_block(LIB, x, variant, pfa, p, length, E, R, n_coeff)
    res = nn.run(x, variant, pfa, p, length, E, R, n_coeff, inject={"est": est, "z0": z0}, block=True)
    m = out.size
    assert m > 0 and res["block"].size >= m
    assert out.tobytes() == res["block"][:m].tobytes(), np.flatnonzero(out != res["block"][:m])[:5]
    k = m // length
    if k:
        want = nn.state_after(res, k)
        assert (st[0], st[1], st[2]) == (want["n"], want["filter_state"], want["n_coeff"])
        assert _ulps(f[1], res["thres"]) == 0
    if kind != "zeros":
        # without injection: est and z0 within the stated ulps of the block's, over the segments the block published
        for s, own in res["own_est"].items():
            if s >= k:
                continue  # a segment the block has not published
            assert _ulps(own, est[s]) <= EST_ULPS, (s, own, est[s])
        if variant == nn.NOTCH_LITE:
            for s, (zr, zi) in res["own_z0"].items():
                if s >= k:
                    continue
                assert max(abs(float(zr) - float(z0[s * length, 0])), abs(float(zi) - float(z0[s * length, 1]))) <= Z0_ULPS * 2.0 ** -24
        else:
            filt = res["filt"].copy()
            filt[k * length:] = False
            for a, b in ((res["own_z0"]["r"], z0[:filt.size, 0]), (res["own_z0"]["i"], z0[:filt.size, 1])):
                d = np.abs(a[filt].astype(np.float64) - b[filt].astype(np.float64))
                assert d.size == 0 or float(d.max()) <= Z0_ULPS * 2.0 ** -24


@needs_ref
@pytest.mark.parametrize("variant", [nn.NOTCH, nn.NOTCH_LITE])
def test_chunking_does_not_change_the_block(variant):
    """the block itself, chunked unevenly, equals its one-segment-per-call run: both alignments are chunking-invariant"""
    x = _stream(3, 9000, "cw")
    a = nn.reference_block(LIB, x, variant, 1e-3, 0.9, 32, 6, 45, 2)[0]
    ends = np.cumsum(np.random.default_rng(4).integers(1, 700, 40))
    b = nn.reference_block(LIB, x, variant, 1e-3, 0.9, 32, 6, 45, 2, chunk_ends=ends)[0]
    m = min(a.size, b.size)
    assert m > 0.5 * min(ends[-1], x.size) and a[:m].tobytes() == b[:m].tobytes()


@pytest.mark.parametrize("p", [0.9, 0.5, -0.7])
@pytest.mark.parametrize("variant", [nn.NOTCH, nn.NOTCH_LITE])
def test_split_invariant_recursion_within_bound_of_truth(variant, p):
    x = _stream(11, 40000, "noise")
    res = nn.run(x, variant, 1e-3, p, 32, 20, 100000)
    filt = res["filt"]
    assert filt.mean() > 0.3
    err = np.max(np.abs(res["out"][filt].astype(np.complex128) - res["truth"][filt]))
    assert 0 < err <= nn.recursion_bound(res, p)


def test_threshold_is_the_blankers():
    import pulse_blanking_np as pnp
    for L in (1, 32, 301):
        assert nn.threshold(1e-3, L) == pnp.threshold(1e-3, L)


def test_status_layout():
    from gnss_sdr_b200.abi import NotchStatus
    assert ctypes.sizeof(NotchStatus) == 72
    assert NotchStatus.n.offset == 24 and NotchStatus.z0_re.offset == 40 and NotchStatus.filter_state.offset == 56
    assert NotchStatus.variant.offset == 68


def test_refusals_that_need_no_engine():
    """no engine, or a threshold that cannot be formed: B200_ERR_ARG before anything else"""
    from gnss_sdr_b200 import capi
    assert capi.lib.b200_iq_set_notch(None, 1, 0, nn.NOTCH_LITE, 1e-3, 0.9, 32, 10, 100, 1) == -1
    assert capi.lib.b200_iq_notch_status(None, 1, None) == -1
    t = ctypes.c_float(0)
    for pfa, length in ((0.0, 32), (1.0, 32), (1e-3, 0), (1e-3, capi.B200_IQ_MAX_BLANKING_LENGTH + 1)):
        assert capi.lib.b200_iq_pulse_blanking_threshold(pfa, length, ctypes.byref(t)) == -1
