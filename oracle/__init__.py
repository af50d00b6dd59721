"""TEST INFRASTRUCTURE ONLY.

ctypes bindings to the CPU oracles:

* ``oracle.ref``  -> oracle/_ref/liboracle_ref.so: the reference's OWN volk_gnsssdr kernels and
  ``Cpu_Multicorrelator_Real_Codes`` compiled in place from /root/reference by oracle/Makefile
  (built in the authoring container; the prebuilt .so travels to the GPU box).
* ``oracle.port`` -> oracle/liboracle_port.so: our plain-C restatement (always buildable),
  pinned bit-exact against ``oracle.ref`` by tests/test_oracle_port_vs_ref.py.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / ``--impl reference`` legs may
import this package.  The product (gnss_sdr_b200/) never does.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_REF_SO = os.path.join(_HERE, "_ref", "liboracle_ref.so")
_PORT_SO = os.path.join(_HERE, "liboracle_port.so")

c_float_p = C.POINTER(C.c_float)
c_int_p = C.POINTER(C.c_int)


def build(verbose: bool = False) -> None:
    """Compile the oracles (port always; ref only when /root/reference is present)."""
    out = None if verbose else subprocess.DEVNULL
    subprocess.check_call(["make", "-C", _HERE, "port"], stdout=out)
    subprocess.check_call(["make", "-C", _HERE, "ref"], stdout=out)
    # the reference's blocks compiled where they lie + the build check of integration/src (needs libb200gnss.so, which
    # gnss_sdr_b200.build produces first); both are skipped, keeping prebuilt libraries, where /root/reference is absent
    subprocess.check_call(["make", "-C", _HERE, "blocks"], stdout=out)
    subprocess.check_call(["make", "-C", _HERE, "patchcheck"], stdout=out)


def _fp(a: np.ndarray):
    return a.ctypes.data_as(c_float_p)


def _f32(a) -> np.ndarray:
    return np.ascontiguousarray(a, dtype=np.float32)


def _c64(a) -> np.ndarray:
    return np.ascontiguousarray(a, dtype=np.complex64)


class _Port:
    """Our C restatement (oracle/port_*.c)."""

    def __init__(self):
        if not os.path.exists(_PORT_SO):
            subprocess.check_call(["make", "-C", _HERE, "port"], stdout=subprocess.DEVNULL)
        self.lib = C.CDLL(_PORT_SO)

    # -- tracking ---------------------------------------------------------------------------
    def resampler(self, assoc, code, rem, step, shifts, n, return_idx=False):
        code = _f32(code)
        shifts = _f32(shifts)
        taps = len(shifts)
        out = np.empty((taps, n), np.float32)
        idx = np.empty((taps, n), np.int32)
        self.lib.port_resampler_32f(C.c_int(assoc), _fp(out), idx.ctypes.data_as(c_int_p), _fp(code), C.c_float(rem),
                                    C.c_float(step), _fp(shifts), C.c_uint(len(code)), C.c_int(taps), C.c_uint(n))
        return (out, idx) if return_idx else out

    def hd_resampler(self, code, rem, step, rate, shifts, n):
        code = _f32(code)
        shifts = _f32(shifts)
        taps = len(shifts)
        out = np.empty((taps, n), np.float32)
        self.lib.port_hd_resampler_32f(_fp(out), _fp(code), C.c_float(rem), C.c_float(step), C.c_float(rate),
                                       _fp(shifts), C.c_uint(len(code)), C.c_int(taps), C.c_uint(n))
        return out

    def hd_resampler_avx(self, code, rem, step, rate, shifts, n, return_idx=False):
        code = _f32(code)
        shifts = _f32(shifts)
        taps = len(shifts)
        out = np.empty((taps, n), np.float32)
        idx = np.empty(n, np.int32)
        self.lib.port_hd_resampler_avx_32f(_fp(out), idx.ctypes.data_as(c_int_p), _fp(code), C.c_float(rem), C.c_float(step),
                                           C.c_float(rate), _fp(shifts), C.c_uint(len(code)), C.c_int(taps), C.c_uint(n))
        return (out, idx) if return_idx else out

    def _rot(self, fn, iq, phase_inc, phase, codes):
        iq = _c64(iq)
        codes = _f32(codes)
        taps, n = codes.shape
        res = np.empty(taps, np.complex64)
        inc = np.array([phase_inc], np.complex64)
        ph = np.array([phase], np.complex64)

        class CF(C.Structure):
            _fields_ = [("re", C.c_float), ("im", C.c_float)]

        fn.argtypes = [C.c_void_p, C.c_void_p, CF, C.c_void_p, C.c_void_p, C.c_int, C.c_uint]
        fn(res.ctypes.data, iq.ctypes.data, CF(float(inc[0].real), float(inc[0].imag)), ph.ctypes.data,
           codes.ctypes.data, taps, n)
        return res, ph[0]

    def rotator_generic(self, iq, phase_inc, phase, codes):
        return self._rot(self.lib.port_rotator_generic, iq, phase_inc, phase, codes)

    def rotator_avx(self, iq, phase_inc, phase, codes):
        return self._rot(self.lib.port_rotator_avx, iq, phase_inc, phase, codes)

    def hd_rotator_generic(self, iq, phase_inc, phase_inc_rate, phase, codes):
        iq = _c64(iq)
        codes = _f32(codes)
        taps, n = codes.shape
        res = np.empty(taps, np.complex64)
        ph = np.array([phase], np.complex64)

        class CF(C.Structure):
            _fields_ = [("re", C.c_float), ("im", C.c_float)]

        fn = self.lib.port_hd_rotator_generic
        fn.argtypes = [C.c_void_p, C.c_void_p, CF, CF, C.c_void_p, C.c_void_p, C.c_int, C.c_uint]
        i1 = np.complex64(phase_inc)
        i2 = np.complex64(phase_inc_rate)
        fn(res.ctypes.data, iq.ctypes.data, CF(float(i1.real), float(i1.imag)), CF(float(i2.real), float(i2.imag)),
           ph.ctypes.data, codes.ctypes.data, taps, n)
        return res, ph[0]

    def multicorrelator(self, arch, iq, code, shifts, rem_carr, phase_step, rem_code, code_step, n=None):
        iq = _c64(iq)
        code = _f32(code)
        shifts = _f32(shifts)
        n = len(iq) if n is None else n
        taps = len(shifts)
        out = np.empty(taps, np.complex64)
        scratch = np.empty(taps * n, np.float32)
        fn = self.lib.port_multicorrelator
        fn.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint, C.c_void_p, C.c_int, C.c_float, C.c_float,
                       C.c_float, C.c_float, C.c_uint, C.c_void_p]
        fn(arch, out.ctypes.data, iq.ctypes.data, code.ctypes.data, len(code), shifts.ctypes.data, taps,
           rem_carr, phase_step, rem_code, code_step, n, scratch.ctypes.data)
        return out

    def multicorrelator_f64(self, assoc, iq, code, shifts, rem_carr, phase_step, rem_code, code_step, n=None):
        iq = _c64(iq)
        code = _f32(code)
        shifts = _f32(shifts)
        n = len(iq) if n is None else n
        taps = len(shifts)
        out = np.empty(2 * taps, np.float64)
        fn = self.lib.port_multicorrelator_f64
        fn.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint, C.c_void_p, C.c_int, C.c_float, C.c_float,
                       C.c_float, C.c_float, C.c_uint]
        fn(assoc, out.ctypes.data, iq.ctypes.data, code.ctypes.data, len(code), shifts.ctypes.data, taps,
           rem_carr, phase_step, rem_code, code_step, n)
        return out[0::2] + 1j * out[1::2]

    def multicorrelator_batch(self, arch, threads, iq, in_stride, code, shifts, params, n):
        """iq: flat complex64; item i reads iq[i*in_stride : i*in_stride+n]; params (items,4) f32."""
        iq = _c64(iq)
        code = _f32(code)
        shifts = _f32(shifts)
        params = _f32(params)
        items = params.shape[0]
        taps = len(shifts)
        out = np.empty((items, taps), np.complex64)
        fn = self.lib.port_multicorrelator_batch
        fn.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_uint, C.c_void_p, C.c_int,
                       C.c_void_p, C.c_uint, C.c_int]
        fn(arch, threads, out.ctypes.data, iq.ctypes.data, in_stride, code.ctypes.data, len(code), shifts.ctypes.data,
           taps, params.ctypes.data, n, items)
        return out

    # -- codes ------------------------------------------------------------------------------
    def gps_ca_code(self, prn, chip_shift=0) -> np.ndarray:
        out = np.empty(1023, np.float32)
        rc = self.lib.port_gps_l1_ca_code_gen_float(_fp(out), C.c_int32(prn), C.c_uint32(chip_shift))
        if rc:
            raise ValueError("bad PRN %d" % prn)
        return out

    def gps_ca_code_complex_sampled(self, prn, fs, chip_shift=0) -> np.ndarray:
        n = int(fs / (1023000.0 / 1023.0))
        out = np.empty(n, np.complex64)
        rc = self.lib.port_gps_l1_ca_code_gen_complex_sampled(out.ctypes.data_as(c_float_p), C.c_uint32(prn),
                                                              C.c_int32(int(fs)), C.c_uint32(chip_shift))
        assert rc == n
        return out

    def sinboc11(self, primary) -> np.ndarray:
        primary = np.ascontiguousarray(primary, np.int32)
        out = np.empty(2 * len(primary), np.float32)
        self.lib.port_sinboc11_from_primary(_fp(out), primary.ctypes.data_as(C.POINTER(C.c_int32)),
                                            C.c_uint32(len(primary)))
        return out


class _Ref:
    """The reference's own kernels (oracle/ref_kernels.c, oracle/ref_engine.cc wrappers)."""

    RESAMPLER = {"generic": 0, "a_avx": 1, "u_avx": 2, "a_sse3": 3, "a_sse4_1": 4}
    ROTATOR = {"generic": 0, "generic_reload": 1, "u_avx": 2, "a_avx": 3}
    SINCOS = {"generic": 0, "generic_fxpt": 1, "a_sse2": 2, "u_sse2": 3, "a_avx2": 4, "u_avx2": 5}
    INDEX_MAX = {"generic": 0, "a_avx": 1, "u_avx": 2, "a_sse4_1": 3, "a_sse": 4}

    def __init__(self):
        self.lib = C.CDLL(_REF_SO)
        self.lib.ref_mc_create.restype = C.c_void_p
        self.lib.ref_mc_bench.restype = C.c_double
        self.lib.ref_mc_bench_pinned.restype = C.c_double

    def select_arch(self, arch: str):
        assert self.lib.ref_select_arch(arch.encode()) == 0

    def resampler(self, variant, code, rem, step, shifts, n):
        code = _f32(code)
        shifts = _f32(shifts)
        taps = len(shifts)
        out = np.empty((taps, n), np.float32)
        rc = self.lib.ref_resampler_32f(C.c_int(self.RESAMPLER[variant]), _fp(out), _fp(code), C.c_float(rem),
                                        C.c_float(step), _fp(shifts), C.c_uint(len(code)), C.c_int(taps), C.c_uint(n))
        assert rc == 0
        return out

    def hd_resampler(self, variant, code, rem, step, rate, shifts, n):
        code = _f32(code)
        shifts = _f32(shifts)
        taps = len(shifts)
        out = np.empty((taps, n), np.float32)
        rc = self.lib.ref_hd_resampler_32f(C.c_int({"generic": 0, "a_avx": 1, "u_avx": 2}[variant]), _fp(out), _fp(code),
                                           C.c_float(rem), C.c_float(step), C.c_float(rate), _fp(shifts),
                                           C.c_uint(len(code)), C.c_int(taps), C.c_uint(n))
        assert rc == 0
        return out

    def rotator(self, variant, iq, phase_inc, phase, codes):
        iq = _c64(iq)
        codes = _f32(codes)
        taps, n = codes.shape
        res = np.empty(taps, np.complex64)
        inc = np.array([phase_inc], np.complex64)
        ph = np.array([phase], np.complex64)
        rc = self.lib.ref_rotator_dot_prod_32fc_32f(C.c_int(self.ROTATOR[variant]), C.c_void_p(res.ctypes.data),
                                                    C.c_void_p(iq.ctypes.data), C.c_void_p(inc.ctypes.data),
                                                    C.c_void_p(ph.ctypes.data), C.c_void_p(codes.ctypes.data),
                                                    C.c_int(taps), C.c_uint(n))
        assert rc == 0
        return res, ph[0]

    def hd_rotator(self, variant, iq, phase_inc, phase_inc_rate, phase, codes):
        iq = _c64(iq)
        codes = _f32(codes)
        taps, n = codes.shape
        res = np.empty(taps, np.complex64)
        inc = np.array([phase_inc], np.complex64)
        rate = np.array([phase_inc_rate], np.complex64)
        ph = np.array([phase], np.complex64)
        rc = self.lib.ref_hd_rotator_dot_prod_32fc_32f(C.c_int({"generic": 0, "generic_arg": 1}[variant]),
                                                       C.c_void_p(res.ctypes.data), C.c_void_p(iq.ctypes.data),
                                                       C.c_void_p(inc.ctypes.data), C.c_void_p(rate.ctypes.data),
                                                       C.c_void_p(ph.ctypes.data), C.c_void_p(codes.ctypes.data),
                                                       C.c_int(taps), C.c_uint(n))
        assert rc == 0
        return res, ph[0]

    def sincos(self, variant, phase_inc, phase, n):
        out = np.empty(n, np.complex64)
        ph = C.c_float(phase)
        rc = self.lib.ref_sincos_32fc(C.c_int(self.SINCOS[variant]), C.c_void_p(out.ctypes.data), C.c_float(phase_inc),
                                      C.byref(ph), C.c_uint(n))
        assert rc == 0
        return out, ph.value

    def index_max(self, variant, src):
        src = _f32(src)
        idx = C.c_uint(0)
        rc = self.lib.ref_index_max_32u(C.c_int(self.INDEX_MAX[variant]), C.byref(idx), _fp(src), C.c_uint(len(src)))
        assert rc == 0
        return idx.value

    # -- the reference's Cpu_Multicorrelator_Real_Codes class ---------------------------------
    def mc_create(self, max_len, taps, high_dyn=False):
        return C.c_void_p(self.lib.ref_mc_create(C.c_int(max_len), C.c_int(taps), C.c_int(int(high_dyn))))

    def mc_set_code(self, h, code, shifts):
        code = _f32(code)
        shifts = _f32(shifts)
        self.lib.ref_mc_set_code(h, _fp(code), C.c_int(len(code)), _fp(shifts))

    def mc_correlate(self, h, iq, taps, rem_carr, phase_step, phase_rate, rem_code, code_step, code_rate, n=None):
        iq = _c64(iq)
        n = len(iq) if n is None else n
        out = np.empty(taps, np.complex64)
        rc = self.lib.ref_mc_correlate(h, C.c_void_p(iq.ctypes.data), C.c_float(rem_carr), C.c_float(phase_step),
                                       C.c_float(phase_rate), C.c_float(rem_code), C.c_float(code_step),
                                       C.c_float(code_rate), C.c_int(n), C.c_void_p(out.ctypes.data))
        assert rc == 0
        return out

    def mc_destroy(self, h):
        self.lib.ref_mc_destroy(h)

    def mc_bench(self, threads, n, taps, code_len, iters, n_epochs_buf=8, high_dyn=False, pin=True) -> float:
        """seconds for `threads` concurrent reference correlators doing `iters` calls each (threads pinned round robin)"""
        return float(self.lib.ref_mc_bench_pinned(C.c_int(threads), C.c_int(n), C.c_int(taps), C.c_int(code_len),
                                                  C.c_int(iters), C.c_int(n_epochs_buf), C.c_int(1 if high_dyn else 0), C.c_int(1 if pin else 0)))

port = _Port()
ref = _Ref() if os.path.exists(_REF_SO) else None
