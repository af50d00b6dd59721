"""ctypes wrapper of oracle/blocks_harness.cc (TEST INFRASTRUCTURE): one receiver channel - acquisition adapter,
tracking adapter, the reference's ChannelFsm - created by implementation string and driven over in-memory samples.

  ref_lib()   oracle/_ref/liboracle_ref_blocks.so   the reference's own blocks compiled where they lie
  b200_lib()  oracle/_ref/libb200_blocks_check.so   + the B200 blocks of integration/src (needs libb200gnss.so)
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
E1C_SECONDARY = "0011100000001010110110010"  # GALILEO_E1_C_SECONDARY_CODE, src/core/system_parameters/Galileo_E1.h


class Synchro(C.Structure):
    _fields_ = [("System", C.c_char), ("Signal", C.c_char * 3), ("PRN", C.c_uint32), ("Channel_ID", C.c_int32),
                ("Acq_delay_samples", C.c_double), ("Acq_doppler_hz", C.c_double), ("Acq_samplestamp_samples", C.c_uint64),
                ("Acq_doppler_step", C.c_uint32), ("Flag_valid_acquisition", C.c_int32), ("fs", C.c_int64),
                ("Prompt_I", C.c_double), ("Prompt_Q", C.c_double), ("CN0_dB_hz", C.c_double), ("Carrier_Doppler_hz", C.c_double),
                ("Carrier_phase_rads", C.c_double), ("Code_phase_samples", C.c_double), ("Tracking_sample_counter", C.c_uint64),
                ("Flag_valid_symbol_output", C.c_int32), ("correlation_length_ms", C.c_int32),
                ("Flag_PLL_180_deg_phase_locked", C.c_int32), ("pad", C.c_int32)]


SYNCHRO_DTYPE = np.dtype([("System", "S1"), ("Signal", "S3"), ("PRN", "<u4"), ("Channel_ID", "<i4"), ("Acq_delay_samples", "<f8"),
                          ("Acq_doppler_hz", "<f8"), ("Acq_samplestamp_samples", "<u8"), ("Acq_doppler_step", "<u4"),
                          ("Flag_valid_acquisition", "<i4"), ("fs", "<i8"), ("Prompt_I", "<f8"), ("Prompt_Q", "<f8"), ("CN0_dB_hz", "<f8"),
                          ("Carrier_Doppler_hz", "<f8"), ("Carrier_phase_rads", "<f8"), ("Code_phase_samples", "<f8"),
                          ("Tracking_sample_counter", "<u8"), ("Flag_valid_symbol_output", "<i4"), ("correlation_length_ms", "<i4"),
                          ("Flag_PLL_180_deg_phase_locked", "<i4"), ("pad", "<i4")], align=True)
assert SYNCHRO_DTYPE.itemsize == C.sizeof(Synchro)

_libs = {}


def _load(name):
    if name in _libs:
        return _libs[name]
    path = os.path.join(ROOT, "oracle", "_ref", name)
    if not os.path.exists(path):
        _libs[name] = None
        return None
    lib = C.CDLL(path, mode=C.RTLD_LOCAL)
    lib.itf_config_create.restype = C.c_void_p
    lib.itf_config_set.argtypes = [C.c_void_p, C.c_char_p, C.c_char_p]
    lib.itf_config_destroy.argtypes = [C.c_void_p]
    lib.itf_channel_create.restype = C.c_void_p
    lib.itf_channel_create.argtypes = [C.c_void_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_int]
    lib.itf_channel_destroy.argtypes = [C.c_void_p]
    lib.itf_implementation.restype = C.c_char_p
    lib.itf_implementation.argtypes = [C.c_void_p, C.c_int]
    lib.itf_set_satellite.argtypes = [C.c_void_p, C.c_char, C.c_char_p, C.c_uint32]
    lib.itf_acq_start.argtypes = [C.c_void_p]
    lib.itf_acq_set_doppler_center.argtypes = [C.c_void_p, C.c_int]
    lib.itf_acq_run.restype = C.c_long
    lib.itf_acq_run.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_long]
    lib.itf_events.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_int), C.c_int]
    lib.itf_fsm_tracking_started.argtypes = [C.c_void_p]
    lib.itf_get_synchro.argtypes = [C.c_void_p, C.POINTER(Synchro)]
    lib.itf_set_acq_result.argtypes = [C.c_void_p, C.c_double, C.c_double, C.c_uint64]
    lib.itf_trk_start.argtypes = [C.c_void_p]
    lib.itf_trk_stop.argtypes = [C.c_void_p]
    lib.itf_trk_post_telemetry_event.argtypes = [C.c_void_p, C.c_int]
    lib.itf_trk_run.restype = C.c_long
    lib.itf_trk_run.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_long, C.c_long]
    lib.itf_nitems_read.restype = C.c_uint64
    lib.itf_nitems_read.argtypes = [C.c_void_p, C.c_int]
    lib.itf_select_arch.argtypes = [C.c_char_p]
    lib.itf_trk_run_parallel.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_uint64, C.c_void_p, C.c_long, C.c_void_p]
    lib.itf_code_float.argtypes = [C.c_char, C.c_char_p, C.c_uint32, C.c_void_p, C.c_int]
    lib.itf_coalescer_stats.argtypes = [C.c_void_p, C.c_int]
    lib.itf_acq_bench.restype = C.c_double
    lib.itf_acq_bench.argtypes = [C.c_void_p, C.c_char_p, C.c_char_p, C.c_char, C.c_char_p, C.c_int, C.c_int, C.c_void_p, C.c_uint64, C.c_int,
                                  C.POINTER(C.c_int)]
    _libs[name] = lib
    return lib


def ref_lib():
    return _load("liboracle_ref_blocks.so")


def b200_lib():
    return _load("libb200_blocks_check.so")


class Channel:
    """One receiver channel.  conf: dict of configuration-file properties ("Acquisition_1C.doppler_max": 5000 ...)."""

    def __init__(self, lib, conf: dict, acq_impl="", trk_impl="", acq_role="Acquisition_1C", trk_role="Tracking_1C", channel=0):
        self.lib = lib
        self.cfg = lib.itf_config_create()
        for k, v in conf.items():
            if isinstance(v, bool):
                v = "true" if v else "false"
            lib.itf_config_set(self.cfg, str(k).encode(), str(v).encode())
        self.h = lib.itf_channel_create(self.cfg, acq_impl.encode(), acq_role.encode(), trk_impl.encode(), trk_role.encode(), channel)
        if not self.h:
            lib.itf_config_destroy(self.cfg)
            self.cfg = None
            raise ValueError(f"no such implementation (or unusable item type): {acq_impl!r} / {trk_impl!r}")

    def close(self):
        if self.h:
            self.lib.itf_channel_destroy(self.h)
            self.h = None
        if self.cfg:
            self.lib.itf_config_destroy(self.cfg)
            self.cfg = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def implementation(self, which):
        return self.lib.itf_implementation(self.h, 0 if which == "acq" else 1).decode()

    def set_satellite(self, system: str, signal: str, prn: int):
        self.lib.itf_set_satellite(self.h, system.encode(), signal.encode(), prn)

    def acq_start(self):
        return self.lib.itf_acq_start(self.h)

    def acq_set_doppler_center(self, center):
        return self.lib.itf_acq_set_doppler_center(self.h, int(center))

    def acq_run(self, samples: np.ndarray, max_calls=-1):
        samples = np.ascontiguousarray(samples)
        n = len(samples) if samples.dtype != np.int16 else len(samples) // 2
        return self.lib.itf_acq_run(self.h, samples.ctypes.data, n, max_calls)

    def events(self, which):
        buf = (C.c_int * 256)()
        n = self.lib.itf_events(self.h, 0 if which == "acq" else 1, buf, 256)
        return list(buf[:n])

    def tracking_started(self):
        return self.lib.itf_fsm_tracking_started(self.h)

    def synchro(self):
        s = Synchro()
        self.lib.itf_get_synchro(self.h, C.byref(s))
        return s

    def set_acq_result(self, delay_samples, doppler_hz, samplestamp):
        self.lib.itf_set_acq_result(self.h, float(delay_samples), float(doppler_hz), int(samplestamp))

    def trk_start(self):
        return self.lib.itf_trk_start(self.h)

    def trk_stop(self):
        return self.lib.itf_trk_stop(self.h)

    def trk_post_telemetry_event(self, event):
        return self.lib.itf_trk_post_telemetry_event(self.h, int(event))

    def trk_run(self, samples: np.ndarray, max_out=100000, max_calls=-1):
        samples = np.ascontiguousarray(samples, np.complex64)
        out = np.zeros(max_out, SYNCHRO_DTYPE)
        n = self.lib.itf_trk_run(self.h, samples.ctypes.data, len(samples), out.ctypes.data, max_out, max_calls)
        return out[:min(n, max_out)]

    def nitems_read(self, which):
        return int(self.lib.itf_nitems_read(self.h, 0 if which == "acq" else 1))


def code_table(lib, system: str, signal: str, prn: int) -> np.ndarray:
    """Tracking replica of the reference's generators: 'G','1C' | 'E','1B' / '1C' (sinBOC(1,1), 2 per chip) | 'G','5I' / '5Q'."""
    buf = np.zeros(16384, np.float32)
    n = lib.itf_code_float(system.encode(), signal.encode(), prn, buf.ctypes.data, len(buf))
    if n < 0:
        raise ValueError(f"no generator for {system} {signal}")
    return buf[:n].copy()


def trk_run_parallel(lib, channels, samples: np.ndarray, max_out=20000):
    """Run the tracking blocks of `channels` concurrently (one thread each) over the same samples."""
    samples = np.ascontiguousarray(samples, np.complex64)
    n = len(channels)
    hs = (C.c_void_p * n)(*[ch.h for ch in channels])
    out = np.zeros((n, max_out), SYNCHRO_DTYPE)
    n_out = np.zeros(n, np.int64)
    lib.itf_trk_run_parallel(hs, n, samples.ctypes.data, len(samples), out.ctypes.data, max_out, n_out.ctypes.data)
    return [out[c, :min(int(n_out[c]), max_out)] for c in range(n)]


def coalescer_stats(lib, reset=False):
    buf = np.zeros(8, np.float64)
    if lib.itf_coalescer_stats(buf.ctypes.data, 1 if reset else 0) != 0:
        return None
    keys = ["batches", "items", "window_expired", "mean_batch_us", "mean_latency_us", "max_latency_us", "samples_copied", "samples_offered"]
    return dict(zip(keys, buf.tolist()))


def acq_bench(lib, conf: dict, impl: str, samples: np.ndarray, threads: int, searches_per_thread: int, role="Acquisition_1C", system="G",
              signal="1C", pin=True):
    """(seconds, positives) for threads x searches_per_thread complete acquisitions through adapter + block on the CPU."""
    cfg = lib.itf_config_create()
    for k, v in conf.items():
        if isinstance(v, bool):
            v = "true" if v else "false"
        lib.itf_config_set(cfg, str(k).encode(), str(v).encode())
    samples = np.ascontiguousarray(samples, np.complex64)
    pos = C.c_int(0)
    dt = lib.itf_acq_bench(cfg, impl.encode(), role.encode(), system.encode(), signal.encode(), threads, searches_per_thread,
                           samples.ctypes.data, len(samples), 1 if pin else 0, C.byref(pos))
    lib.itf_config_destroy(cfg)
    return float(dt), int(pos.value)


def ref_mc_cplx_code(lib, sig, code, shifts, rem_carr, dphi, rem_code, step):
    """Cpu_Multicorrelator (complex local code) of the reference, compiled in place."""
    sig = np.ascontiguousarray(sig, np.complex64)
    code = np.ascontiguousarray(code, np.complex64)
    sh = np.ascontiguousarray(shifts, np.float32)
    out = np.zeros(len(sh), np.complex64)
    lib.ref_mc_cplx_code(C.c_void_p(sig.ctypes.data), len(sig), C.c_void_p(code.ctypes.data), len(code), C.c_void_p(sh.ctypes.data), len(sh),
                         C.c_float(rem_carr), C.c_float(dphi), C.c_float(rem_code), C.c_float(step), C.c_void_p(out.ctypes.data))
    return out


def ref_mc_16sc(lib, sig_iq, code_iq, shifts, rem_carr, dphi, rem_code, step):
    """Cpu_Multicorrelator_16sc of the reference, compiled in place (interleaved int16 I,Q in and out)."""
    sig_iq = np.ascontiguousarray(sig_iq, np.int16)
    code_iq = np.ascontiguousarray(code_iq, np.int16)
    sh = np.ascontiguousarray(shifts, np.float32)
    out = np.zeros(2 * len(sh), np.int16)
    lib.ref_mc_16sc(C.c_void_p(sig_iq.ctypes.data), len(sig_iq) // 2, C.c_void_p(code_iq.ctypes.data), len(code_iq) // 2, C.c_void_p(sh.ctypes.data),
                    len(sh), C.c_float(rem_carr), C.c_float(dphi), C.c_float(rem_code), C.c_float(step), C.c_void_p(out.ctypes.data))
    return out
