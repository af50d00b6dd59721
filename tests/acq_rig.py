"""The rig of the acquisition tests (b200_acq_*): objects and their oracles from one set of keywords, local codes, band
streams, int16 / int8 samples, the raw int16 entry points, and the parity checks on result records and grids."""
import numpy as np

ERR_ARG, ERR_STATE, ERR_RANGE = -1, -4, -5
STAT_TOL = 1e-4         # relative, on the statistics: float32 FFTs summed in another order than the reference's
GRID_TOL = 2e-5         # of the reference grid's peak, element-wise
CFAR_STATS = ("grid_maximum", "test_statistics", "input_power")
PEAK_STATS = ("grid_maximum", "test_statistics", "second_peak")
# the PcpsAcquisition keywords that are also AcqConf fields of the oracle
SHARED = ("fs_in", "samples_per_ms", "samples_per_chip", "doppler_max", "doppler_step", "sampled_ms", "ms_per_code",
          "max_dwells", "bit_transition_flag", "use_CFAR_algorithm_flag")


def params(fs, **kw):
    """PcpsAcquisition keywords at fs samples per second: fs_in = int(fs), samples_per_ms = fs / 1000 and
    samples_per_chip = int(fs / 1.023 MHz), at least 1.  kw adds the Doppler bounds and the flags, and may override any
    of the three."""
    return {"fs_in": int(fs), "samples_per_ms": fs / 1000.0, "samples_per_chip": max(1, int(fs / 1.023e6)), **kw}


def make(capi, engine, fs, **kw):
    """a PcpsAcquisition on engine with the keywords params(fs, **kw)"""
    return capi.PcpsAcquisition(engine, **params(fs, **kw))


def oracle(p, code=None, *, samples_per_code=None, center=0, **extra):
    """PcpsAcquisitionOracle configured as PcpsAcquisition(**p) is: the fields the two share come from p, the oracle's own
    (samples_per_code, by default samples_per_ms; pfa; step-two fields) from the keywords, which may also override a
    shared one.  Then the Doppler centre, unless 0, and the local code, if given."""
    from oracle.acq_np import AcqConf, PcpsAcquisitionOracle
    fields = {k: p[k] for k in SHARED if k in p}
    fields["samples_per_code"] = p["samples_per_ms"] if samples_per_code is None else samples_per_code
    o = PcpsAcquisitionOracle(AcqConf(**{**fields, **extra}))
    if center:
        o.set_doppler_center(center)
    if code is not None:
        o.set_local_code(code)
    return o


def code_len(conf):
    """samples of local code an object (or oracle) of this configuration takes: half the FFT with bit transition, else
    the consumed samples"""
    return conf.fft_size // 2 if conf.bit_transition_flag else conf.consumed_samples


def ca_code(gen, prn, fs, periods=1):
    """GPS C/A code of prn sampled at fs by gen (oracle.port or gnss_synth), as a complex64 local code of periods code
    periods"""
    return np.tile(gen.gps_ca_code_complex_sampled(prn, int(fs)), periods)


def load_codes(acq, codes):
    """codes[s] into slot s, in slot order"""
    for s, code in enumerate(codes):
        acq.set_local_code(s, code)


def pair(capi, engine, rng, fs, **kw):
    """Two objects of one configuration (two code slots, +-1000 Hz in 500 Hz steps, unless kw says otherwise) holding the
    same random +-1 codes: one searches a band, the other the same samples another way.  Returns (a, b, codes)."""
    kw = {"doppler_max": 1000, "doppler_step": 500, "n_code_slots": 2, **kw}
    a, b = make(capi, engine, fs, **kw), make(capi, engine, fs, **kw)
    codes = [rng.choice([-1.0, 1.0], code_len(a.conf)).astype(np.complex64) for _ in range(a.conf.n_code_slots)]
    for acq in (a, b):
        load_codes(acq, codes)
    return a, b, codes


def check(got, want, stats=CFAR_STATS, what="", period=None):
    """got's index_time, index_doppler and doppler exactly want's, and each field in stats within STAT_TOL of want's.
    With period, index_time only modulo period: a buffer of several code periods has that many equal peaks."""
    t, w = int(got["index_time"]), int(want["index_time"])
    if period:
        t, w = t % period, w % period
    assert (t, int(got["index_doppler"]), int(got["doppler"])) == (w, want["index_doppler"], want["doppler"]), \
        (what, got, want)
    for k in stats:
        g, w = float(got[k]), float(want[k])
        assert abs(g - w) < STAT_TOL * abs(w), (what, k, g, w)


def check_grid(got, ref, rows=None, cols=None):
    """got[:rows, :cols] within GRID_TOL of the peak of ref[:rows, :cols], element-wise; returns the largest error as a
    fraction of that peak"""
    ref = ref[:rows, :cols]
    err = float(np.max(np.abs(got[:rows, :cols] - ref)) / ref.max())
    assert err < GRID_TOL, err
    return err


def grids(acq):
    """the bytes of every slot's magnitude grid, or b"" when the object keeps none"""
    c = acq.conf
    if not (c.keep_grid or c.max_dwells > 1):
        return b""
    return b"".join(acq.read_grid(s).tobytes() for s in range(c.n_code_slots))


def pow2(n):
    """the smallest power of two >= n"""
    return 1 << (int(n) - 1).bit_length()


def stream(rng, n, code, fs, dtype=np.complex64):
    """n samples of unit complex noise plus half of code, rolled by a random delay and repeated, on a carrier within
    +-900 Hz: one clear peak for the statistics"""
    t = np.arange(n)
    x = np.resize(np.roll(code, int(rng.integers(0, code.size))), n) * np.exp(2j * np.pi * rng.uniform(-900, 900) / fs * t)
    return (0.5 * x + rng.normal(0, 1.0, n) + 1j * rng.normal(0, 1.0, n)).astype(dtype)


def to_int(x, dtype, scale=1.0, clip=None):
    """complex samples -> interleaved I, Q integers of dtype: round(scale * x), clipped to clip = (lo, hi) if given"""
    v = np.round(np.stack([x.real, x.imag], 1).ravel() * scale)
    if clip is not None:
        v = np.clip(v, *clip)
    return v.astype(dtype)


def from_int(raw):
    """interleaved I, Q integers -> complex64 samples"""
    return (raw[0::2].astype(np.float32) + 1j * raw[1::2].astype(np.float32)).astype(np.complex64)


def _call(name, *args):
    from gnss_sdr_b200 import capi
    rc = getattr(capi.lib, name)(*args)
    if rc:
        raise capi.B200Error(rc, name)


def search_i16(acq, raw, slots, dwell=1):
    """b200_acq_search_i16 on interleaved int16 I, Q samples -> one result record per slot"""
    from gnss_sdr_b200.abi import ACQ_RESULT_DTYPE
    raw, slots = np.ascontiguousarray(raw, np.int16), np.ascontiguousarray(slots, np.uint32)
    res = np.zeros(slots.size, ACQ_RESULT_DTYPE)
    _call("b200_acq_search_i16", acq.h, raw.ctypes.data, slots.ctypes.data, slots.size, dwell, res.ctypes.data)
    return res


def search_step_two_i16(acq, raw, slot, prev_input_power, dwell=1):
    """b200_acq_search_step_two_i16 on interleaved int16 I, Q samples -> the result record"""
    from gnss_sdr_b200.abi import ACQ_RESULT_DTYPE
    raw = np.ascontiguousarray(raw, np.int16)
    res = np.zeros(1, ACQ_RESULT_DTYPE)
    _call("b200_acq_search_step_two_i16", acq.h, raw.ctypes.data, slot, dwell, prev_input_power, res.ctypes.data)
    return res[0]
