"""TEST INFRASTRUCTURE ONLY.  ctypes bindings to the DLL/PLL loop oracles:

* ``PortLoop`` -> oracle/port_loop.c (our C restatement, in liboracle_port.so)
* ``RefLoop``  -> oracle/ref_loop.cc over the reference's own tracking libs (oracle/_ref/liboracle_ref_loop.so)
* ``ref_dump_read`` -> the reference's own Tracking_Dump_Reader

The structures are include/b200gnss.h's (b200_trk_loop_conf, b200_trk_dump_record, b200_trk_loop_status), from
gnss_sdr_b200.abi, which declares them without loading the product library: the C port includes the same header.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from gnss_sdr_b200.abi import TRK_DUMP_RECORD_DTYPE, TrkLoopConf, TrkLoopStatus

# the names this module has always exported, for the code that still uses them: the same objects, not copies
LoopConf, LoopStatus, DUMP_RECORD_DTYPE = TrkLoopConf, TrkLoopStatus, TRK_DUMP_RECORD_DTYPE

_HERE = os.path.dirname(os.path.abspath(__file__))
_REF_LOOP_SO = os.path.join(_HERE, "_ref", "liboracle_ref_loop.so")
_PORT_SO = os.path.join(_HERE, "liboracle_port.so")


def default_conf(fs_in=4e6, prn=1, **kw) -> TrkLoopConf:
    """GPS L1 C/A defaults of Dll_Pll_Conf (dll_pll_conf.h:32-89, gnss_sdr_flags.cc:44-53) with
    early_late_space_chips = 0.5 as gps_l1_ca_dll_pll_tracking_test.cc:291 sets it."""
    c = TrkLoopConf()
    c.fs_in = fs_in
    c.code_chip_rate = 1.023e6
    c.signal_carrier_freq = 1575.42e6
    c.code_period = 0.001
    c.carrier_lock_th = 0.7
    c.code_length_chips = 1023
    c.vector_length = int(round(fs_in / (1.023e6 / 1023.0)))
    c.pull_in_time_s = 5
    c.bit_synchronization_time_limit_s = 0xFFFFFFFF
    c.prn = prn
    c.code_samples_per_chip = 1
    c.pll_filter_order = 3
    c.dll_filter_order = 2
    c.cn0_samples = 20
    c.cn0_min = 25
    c.max_code_lock_fail = 50
    c.max_carrier_lock_fail = 5000
    c.cn0_smoother_samples = 200
    c.carrier_lock_test_smoother_samples = 25
    c.veml = 0
    c.cloop = 1
    c.carrier_aiding = 1
    c.enable_fll_pull_in = 0
    c.enable_fll_steady_state = 0
    c.pll_bw_hz = 35.0
    c.dll_bw_hz = 2.0
    c.fll_bw_hz = 35.0
    c.early_late_space_chips = 0.5
    c.slope = 1.0
    c.y_intercept = 1.0
    c.cn0_smoother_alpha = 0.002
    c.carrier_lock_test_smoother_alpha = 0.002
    for k, v in kw.items():
        if not hasattr(c, k):
            raise AttributeError(k)
        setattr(c, k, v)
    return c


class _Loop:
    def __init__(self, lib, prefix, conf: TrkLoopConf):
        self.lib, self.p = lib, prefix
        f = lambda name: getattr(lib, prefix + name)
        f("create").restype = C.c_void_p
        f("create").argtypes = [C.POINTER(TrkLoopConf)]
        f("destroy").argtypes = [C.c_void_p]
        f("start").argtypes = [C.c_void_p, C.c_double, C.c_double, C.c_uint64, C.c_uint64]
        f("prepare").argtypes = [C.c_void_p, C.POINTER(C.c_uint64), C.POINTER(C.c_int32), C.POINTER(C.c_float)]
        f("update").argtypes = [C.c_void_p, C.POINTER(C.c_float), C.c_void_p]
        f("status").argtypes = [C.c_void_p, C.POINTER(TrkLoopStatus)]
        self.conf = conf
        self.h = f("create")(C.byref(conf))
        if not self.h:
            raise ValueError("loop_create failed")

    def start(self, acq_delay_samples, acq_doppler_hz, acq_samplestamp, nitems_read):
        getattr(self.lib, self.p + "start")(self.h, acq_delay_samples, acq_doppler_hz, acq_samplestamp, nitems_read)

    def prepare(self):
        """-> None in standby, else (sample_index, n, float32[6])"""
        si, n = C.c_uint64(), C.c_int32()
        p6 = np.zeros(6, np.float32)
        ok = getattr(self.lib, self.p + "prepare")(self.h, C.byref(si), C.byref(n), p6.ctypes.data_as(C.POINTER(C.c_float)))
        return (si.value, n.value, p6) if ok else None

    def update(self, taps):
        """taps complex64[3 or 5] -> (logged, record)"""
        t = np.ascontiguousarray(taps, np.complex64)
        rec = np.zeros(1, TRK_DUMP_RECORD_DTYPE)
        logged = getattr(self.lib, self.p + "update")(self.h, t.ctypes.data_as(C.POINTER(C.c_float)), rec.ctypes.data)
        return bool(logged), rec[0]

    def status(self) -> TrkLoopStatus:
        s = TrkLoopStatus()
        getattr(self.lib, self.p + "status")(self.h, C.byref(s))
        return s

    def close(self):
        if self.h:
            getattr(self.lib, self.p + "destroy")(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


_port_lib = None
_ref_lib = None


def port_lib():
    global _port_lib
    if _port_lib is None:
        _port_lib = C.CDLL(_PORT_SO)
        for name, res, args in [
            ("disc_pll_cloop", C.c_double, [C.c_float] * 2),
            ("disc_fll_diff_atan", C.c_double, [C.c_float] * 4 + [C.c_double] * 2),
            ("disc_dll_e_minus_l", C.c_double, [C.c_float] * 7),
            ("disc_dll_vemlp", C.c_double, [C.POINTER(C.c_float)]),
            ("cn0_m2m4", C.c_float, [C.POINTER(C.c_float), C.c_int, C.c_float]),
            ("carrier_lock_detector", C.c_float, [C.POINTER(C.c_float), C.c_int]),
        ]:
            getattr(_port_lib, "port_" + name).restype = res
            getattr(_port_lib, "port_" + name).argtypes = args
    return _port_lib


def ref_lib():
    global _ref_lib
    if _ref_lib is None:
        if not os.path.exists(_REF_LOOP_SO):
            return None
        _ref_lib = C.CDLL(_REF_LOOP_SO)
        for name, res, args in [
            ("disc_pll_cloop", C.c_double, [C.c_float] * 2),
            ("disc_fll_diff_atan", C.c_double, [C.c_float] * 4 + [C.c_double] * 2),
            ("disc_dll_e_minus_l", C.c_double, [C.c_float] * 7),
            ("disc_dll_vemlp", C.c_double, [C.POINTER(C.c_float)]),
            ("cn0_m2m4", C.c_float, [C.POINTER(C.c_float), C.c_int, C.c_float]),
            ("carrier_lock_detector", C.c_float, [C.POINTER(C.c_float), C.c_int]),
        ]:
            getattr(_ref_lib, "ref_" + name).restype = res
            getattr(_ref_lib, "ref_" + name).argtypes = args
        _ref_lib.ref_trk_dump_read.restype = C.c_int64
        _ref_lib.ref_trk_dump_read.argtypes = [C.c_char_p, C.POINTER(C.c_double), C.c_int64]
    return _ref_lib


def PortLoop(conf: TrkLoopConf) -> _Loop:
    return _Loop(port_lib(), "port_loop_", conf)


def RefLoop(conf: TrkLoopConf) -> _Loop:
    lib = ref_lib()
    if lib is None:
        raise RuntimeError("oracle/_ref/liboracle_ref_loop.so not built")
    return _Loop(lib, "ref_loop_", conf)


def ref_dump_read(filename: str, max_epochs: int = 1 << 20) -> np.ndarray:
    """Read a tracking dump file with the reference's own Tracking_Dump_Reader -> float64[n, 24]."""
    lib = ref_lib()
    out = np.zeros((max_epochs, 24), np.float64)
    n = lib.ref_trk_dump_read(filename.encode(), out.ctypes.data_as(C.POINTER(C.c_double)), max_epochs)
    if n < 0:
        raise IOError(filename)
    return out[:n].copy()
