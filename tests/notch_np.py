"""numpy restatement of the notch filters (b200_iq_set_notch): Notch(pfa, p, L, E, R) and NotchLite(p, pfa, L, E, R, Nc) in
float32, segment by segment from the notch's origin, as include/b200gnss.h states them.

run() gives, for a stream x that starts at the origin:
  - the device's output: copied and estimation segments verbatim, filtered samples by the split-invariant recursion (grid
    blocks of GRID samples, each block's affine map composed in float64, y carried from grid point to grid point in
    float64, the float32 recursion inside each block started from float32(y));
  - the block's output (block=True): the same segments, filtered samples by one serial float32 recursion per run, which is
    what notch_cc / notch_lite_cc compute;
  - the float64 truth of the filtered samples: the same recursion with the same z0 and inputs in complex128;
  - the state after every segment.
inject={"est": ..., "z0": ...} replaces est after each estimation segment and the z0 of each filtered sample with the
reference block's own (ref_notch's per-segment mode), so that the logic and the serial recursion can be compared with the
block byte for byte; own_est / own_z0 then hold the values the restatement computed in their place.

Every float32 operation is one numpy float32 operation (rounded on its own); complex products are written out by
component.  atan2, log10, pow, cos and sin are taken in float64 and rounded once to float32."""
import ctypes as C
import math
import os

import numpy as np

from pulse_blanking_np import threshold  # noqa: F401  (the same chi-squared quantile)

NOTCH, NOTCH_LITE = 0, 1
GRID = 1024
NOTCH_SO = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "liboracle_ref_notch.so")
F = np.float32


def cmul(ar, ai, br, bi):
    """the block's gr_complex product, float32 components"""
    return ar * br - ai * bi, ar * bi + ai * br


def lead(variant: int, length: int) -> int:
    """source samples past a segment's end that must exist before it is published"""
    return 1 if (variant == NOTCH or length == 1) else 0


def twiddles(length: int):
    """W[m] = exp(-2 pi i m / L) in float64, from libm's cos and sin like the host code"""
    w = [complex(math.cos(-2.0 * math.pi * m / length), math.sin(-2.0 * math.pi * m / length)) for m in range(length)]
    return np.array([v.real for v in w]), np.array([v.imag for v in w])


def energies(seg: np.ndarray) -> np.ndarray:
    """Re(volk_32fc_x2_conjugate_dot_prod_32fc(in, in, L)) of each row, in the generic kernel's order"""
    re, im = seg.real.astype(F), seg.imag.astype(F)
    mag = re * re + im * im
    K, L = seg.shape
    s0, s1 = np.zeros(K, F), np.zeros(K, F)
    for i in range(0, L - 1, 2):
        s0 = s0 + mag[:, i]
        s1 = s1 + mag[:, i + 1]
    e = s0 + s1
    if L % 2:
        e = e + mag[:, L - 1]
    return e


def sig2lin(seg: np.ndarray, wr: np.ndarray, wi: np.ndarray) -> np.float32:
    """the noise-floor term of one segment: direct DFT in float64, dB per bin, the VOLK noise floor in float32"""
    L = seg.size
    xr, xi = seg.real.astype(np.float64), seg.imag.astype(np.float64)
    q = np.arange(L)
    ar, ai = np.zeros(L), np.zeros(L)
    for m in range(L):
        idx = (m * q) % L
        pr, pi = xr[m] * wr[idx] - xi[m] * wi[idx], xr[m] * wi[idx] + xi[m] * wr[idx]
        ar, ai = ar + pr, ai + pi
    pw = ar * ar + ai * ai
    db = (10.0 * np.log10(pw + 1e-20)).astype(F)
    s = F(0)
    for v in db:
        s = F(s + v)
    mean = F(F(s / F(L)) + F(15.0))
    s, cnt = F(0), L
    for v in db:
        if v <= mean:
            s = F(s + v)
        else:
            cnt -= 1
    floor = mean if cnt == 0 else F(s / F(cnt))
    return F(F(10.0 ** float(F(floor / F(10.0)))) / F(2 * L))


def angle(ar, ai, br, bi):
    """float32 atan2 of a conj(b), in float64 rounded once"""
    cr, ci = cmul(F(ar), F(ai), F(br), -F(bi))
    return np.arctan2(np.float64(ci), np.float64(cr)).astype(F)


def unit(a):
    a = np.float64(a)
    return np.cos(a).astype(F), np.sin(a).astype(F)


def run(x, variant, pfa, p, length, n_est, n_reset, n_coeff=1, thres=None, inject=None, block=False):
    """the notch over the stream x from its origin (all whole segments x publishes); returns a dict of arrays"""
    x = np.asarray(x, np.complex64)
    L = int(length)
    lite = variant == NOTCH_LITE
    nc_mod = int(n_coeff) if lite else 1
    thres = threshold(pfa, L) if thres is None else F(thres)
    p = F(p)
    u = np.concatenate([np.zeros(1, np.complex64), x]) if lite else x
    K = max(0, (x.size - lead(variant, L)) // L)
    seg_in = u[1:1 + K * L].reshape(K, L)
    seg_prev = u[0:K * L].reshape(K, L)
    e = energies(seg_in) if K else np.zeros(0, F)
    wr, wi = twiddles(L)
    n, est, fs, nc, filtered = 0, F(0), False, 0, 0
    z0 = (F(0), F(0))
    flags = np.zeros(K, np.uint8)                      # bit 0 filtered, bit 1 run start
    zseg = np.zeros((K, 2), F)
    rec = {k: [] for k in ("n", "noise_power", "filter_state", "n_coeff", "filtered", "z0")}
    own_est, own_z0 = {}, {}
    sig_all = {}
    with np.errstate(divide="ignore", invalid="ignore"):
        for k in range(K):
            if n < n_est and not fs:
                s = sig2lin(seg_in[k], wr, wi)
                sig_all[k] = s
                new = F(F(F(n) * est + s) / F(n + 1))
                if inject is not None:
                    own_est[k] = new
                    new = F(inject["est"][k])
                est = new
            elif F(e[k] / est) > thres:
                if not fs:
                    fs, nc = True, 0
                    flags[k] |= 2
                flags[k] |= 1
                filtered += 1
                if lite and nc == 0:
                    a1 = angle(seg_in[k, 1].real if L > 1 else u[k * L + 2].real, seg_in[k, 1].imag if L > 1 else u[k * L + 2].imag,
                               seg_in[k, 0].real, seg_in[k, 0].imag)
                    s2a, s2b = (seg_in[k, L - 1], seg_in[k, L - 2]) if L > 1 else (seg_in[k, 0], seg_prev[k, 0])
                    a2 = angle(s2a.real, s2a.imag, s2b.real, s2b.imag)
                    z0 = unit(F(F(a1 + a2) / F(2.0)))
                    if inject is not None:
                        own_z0[k] = z0
                        z0 = (F(inject["z0"][k * L, 0]), F(inject["z0"][k * L, 1]))
                if lite:
                    nc = (nc + 1) % nc_mod
                zseg[k] = z0
            else:
                if n > n_reset:
                    n = 0
                fs = False
            n += 1
            rec["n"].append(n)
            rec["noise_power"].append(est)
            rec["filter_state"].append(int(fs))
            rec["n_coeff"].append(nc)
            rec["filtered"].append(filtered)
            rec["z0"].append(z0)
    # per-sample terms
    N = K * L
    xin, xp = seg_in.reshape(-1), seg_prev.reshape(-1)
    filt = np.repeat(flags & 1, L).astype(bool)
    start = np.zeros(N, bool)
    start[::L] = (flags & 2).astype(bool) if K else start[::L]
    if lite:
        zr, zi = np.repeat(zseg[:, 0], L), np.repeat(zseg[:, 1], L)
    else:
        ang = np.zeros(N, F)
        ang[filt] = angle(xin.real[filt], xin.imag[filt], xp.real[filt], xp.imag[filt])
        zr, zi = np.zeros(N, F), np.zeros(N, F)
        zr[filt], zi[filt] = unit(ang[filt])
        if inject is not None:
            own_z0 = {"r": zr.copy(), "i": zi.copy()}
            zr = np.where(filt, inject["z0"][:N, 0], zr).astype(F)
            zi = np.where(filt, inject["z0"][:N, 1], zi).astype(F)
        for k in range(K):
            if flags[k] & 1:
                z0 = (zr[k * L + L - 1], zi[k * L + L - 1])
            rec["z0"][k] = z0 if flags[k] & 1 else (rec["z0"][k - 1] if k else (F(0), F(0)))
    xr, xi = xin.real.astype(F), xin.imag.astype(F)
    tr, ti = cmul(zr, zi, xp.real.astype(F), xp.imag.astype(F))
    br, bi = xr - tr, xi - ti
    ar, ai = cmul(np.full(N, p, F), np.zeros(N, F), zr, zi)
    out = xin.copy()
    # the device's split-invariant recursion: grid blocks of GRID samples
    nb = (N + GRID - 1) // GRID
    pad = nb * GRID - N

    def padded(v, fill=0):
        return np.concatenate([v, np.full(pad, fill, v.dtype)]).reshape(nb, GRID)
    P = {k: padded(v) for k, v in dict(filt=filt, start=start, ar=ar, ai=ai, br=br, bi=bi, xr=xr, xi=xi).items()}
    Ar, Ai, Br, Bi = np.ones(nb), np.zeros(nb), np.zeros(nb), np.zeros(nb)
    for c in range(GRID):
        f, s = P["filt"][:, c], P["start"][:, c]
        a_r, a_i = P["ar"][:, c].astype(np.float64), P["ai"][:, c].astype(np.float64)
        b_r, b_i = P["br"][:, c].astype(np.float64), P["bi"][:, c].astype(np.float64)
        nAr, nAi = a_r * Ar - a_i * Ai, a_r * Ai + a_i * Ar
        nBr, nBi = (a_r * Br - a_i * Bi) + b_r, (a_r * Bi + a_i * Br) + b_i
        valid = np.arange(nb) * GRID + c < N
        Ar = np.where(valid, np.where(f, np.where(s, 0.0, nAr), 0.0), Ar)
        Ai = np.where(valid, np.where(f, np.where(s, 0.0, nAi), 0.0), Ai)
        Br = np.where(valid, np.where(f, np.where(s, b_r, nBr), 0.0), Br)
        Bi = np.where(valid, np.where(f, np.where(s, b_i, nBi), 0.0), Bi)
    yr, yi = np.zeros(nb), np.zeros(nb)
    cr, ci = 0.0, 0.0
    for g in range(nb):
        yr[g], yi[g] = cr, ci
        cr, ci = (Ar[g] * cr - Ai[g] * ci) + Br[g], (Ar[g] * ci + Ai[g] * cr) + Bi[g]
    lr, li = yr.astype(F), yi.astype(F)
    dev = np.zeros((nb, GRID), np.complex64)
    for c in range(GRID):
        f, s = P["filt"][:, c], P["start"][:, c]
        lr, li = np.where(s, F(0), lr), np.where(s, F(0), li)
        ur, ui = cmul(P["ar"][:, c], P["ai"][:, c], lr, li)
        vr, vi = P["br"][:, c] + ur, P["bi"][:, c] + ui
        lr, li = np.where(f, vr, lr), np.where(f, vi, li)
        dev[:, c].real, dev[:, c].imag = vr, vi
    dev = dev.reshape(-1)[:N]
    out[filt] = dev[filt]
    # float64 truth and (optionally) the block's serial float32 recursion, per filtered sample
    truth = np.zeros(N, np.complex128)
    ser = xin.copy()
    idx = np.nonzero(filt)[0]
    z64 = zr.astype(np.float64) + 1j * zi.astype(np.float64)
    a64 = ar.astype(np.float64) + 1j * ai.astype(np.float64)
    bt = xin.astype(np.complex128) - z64 * xp.astype(np.complex128)
    y = 0j
    for r in idx:
        y = bt[r] + (0j if start[r] else a64[r] * y)
        truth[r] = y
    if block:
        lr, li = F(0), F(0)
        for r in idx:
            if start[r]:
                lr, li = F(0), F(0)
            ur, ui = cmul(ar[r], ai[r], lr, li)
            lr, li = F(br[r] + ur), F(bi[r] + ui)
            ser[r] = complex(lr, li)
    # last_out_ after each segment: the device's value at the last filtered sample so far
    last = np.zeros((K, 2), F)
    lo = (F(0), F(0))
    for k in range(K):
        if flags[k] & 1:
            v = out[k * L + L - 1]
            lo = (F(v.real), F(v.imag))
        last[k] = lo
    return {"out": out, "block": ser if block else None, "truth": truth, "filt": filt, "flags": flags, "energy": e, "sig2lin": sig_all,
            "b": br + 1j * bi.astype(np.complex64), "a": ar + 1j * ai.astype(np.complex64), "bt": bt, "segments": K, "rec": rec,
            "last_out": last, "thres": thres, "own_est": own_est, "own_z0": own_z0, "z0": zr + 1j * zi.astype(np.complex64)}


def state_after(res, k):
    """the status fields of the notch after its first k segments (k >= 1)"""
    r = res["rec"]
    return {"segments": k, "filtered": r["filtered"][k - 1], "n": r["n"][k - 1], "noise_power": F(r["noise_power"][k - 1]),
            "filter_state": r["filter_state"][k - 1], "n_coeff": r["n_coeff"][k - 1], "z0": r["z0"][k - 1],
            "last_out": tuple(res["last_out"][k - 1])}


def recursion_bound(res, p):
    """|device - truth| bound on filtered samples: the float32 roundings of each step (b's two, the product's three, the
    sum's one, relative to u = 2^-24, on magnitudes up to M = max |x| + |x_prev| and Y = max |y|) accumulate geometrically
    by |p z0| <= |p| (1 + 2u), so the error stays below 8 u (M + |p| Y) / (1 - |p|) plus the start's rounding of y
    (u Y); the float64 composition and carry add about GRID 2^-52 relative, negligible.  GRID does not enter: each grid
    block restarts the float32 recursion from a float64-accurate value."""
    filt = res["filt"]
    if not filt.any():
        return 0.0
    u = 2.0 ** -24
    M = float(np.max(np.abs(res["bt"][filt]))) * 2.0 + 1e-30
    Y = float(np.max(np.abs(res["truth"][filt])))
    return 8 * u * (M + abs(p) * Y) / (1 - abs(p)) + 2 * u * Y


def reference_lib():
    """the reference's notch blocks compiled in place (oracle/_ref/liboracle_ref_notch.so), or None where not built"""
    if not os.path.exists(NOTCH_SO):
        return None
    lib = C.CDLL(NOTCH_SO)
    lib.ref_notch.argtypes = [C.c_int, C.c_float, C.c_float, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_uint64, C.c_void_p,
                              C.c_int, C.c_int, C.c_void_p, C.POINTER(C.c_uint64), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.ref_notch.restype = C.c_int
    return lib


def reference_block(lib, x, variant, pfa, p, length, n_est, n_reset, n_coeff=1, chunk_ends=None):
    """the block over x: fed in chunks ending at chunk_ends, or one segment per call when chunk_ends is None (then also est
    after each segment and the z0 of each sample).  Returns (out, state (n, filter_state, n_coeff), floats (est, thres, z0,
    last_out), est per segment, z0 per sample)."""
    x = np.ascontiguousarray(x, np.complex64)
    per_seg = chunk_ends is None
    ends = np.ascontiguousarray([x.size] if per_seg else chunk_ends, np.uint64)
    out = np.zeros(x.size + 1, np.complex64)
    n_out = C.c_uint64(0)
    state = np.zeros(3, np.int64)
    f = np.zeros(6, np.float32)
    K = x.size // max(1, length) + 1
    est = np.zeros(K, np.float32)
    z0 = np.zeros((K * length, 2), np.float32)
    assert lib.ref_notch(variant, pfa, p, length, n_est, n_reset, n_coeff, x.ctypes.data, x.size, ends.ctypes.data, ends.size, int(per_seg),
                         out.ctypes.data, C.byref(n_out), state.ctypes.data, f.ctypes.data, est.ctypes.data, z0.ctypes.data) == 0
    return out[:n_out.value], state, f, est, z0
