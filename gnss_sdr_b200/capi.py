"""ctypes binding of include/b200gnss.h.  Loads the in-tree libb200gnss.so; fails loudly if absent."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from .abi import (ACQ_RESULT_DTYPE, TRK_DUMP_RECORD_DTYPE, TRK_ITEM_DTYPE, AcqConf, AcqDump, AcqResult,  # noqa: F401
                  NotchStatus, PulseBlankingStatus, TrkDumpRecord, TrkItem, TrkLoopConf, TrkLoopStatus)

_HERE = os.path.dirname(os.path.abspath(__file__))
# B200_LIB selects an alternative build of the SAME library (A/B kernel experiments); default = in-tree build
LIB_PATH = os.environ.get("B200_LIB") or os.path.join(_HERE, "libb200gnss.so")

if not os.path.exists(LIB_PATH):
    raise ImportError(
        f"{LIB_PATH} is missing: build it with `python -m gnss_sdr_b200.build` "
        "(there is no CPU fallback for the B200 hot path)")

lib = C.CDLL(LIB_PATH)

B200_MAX_TAPS = 8
B200_ACQ_MAX_RESAMPLER_TAPS = 1024
B200_IQ_MAX_CONDITIONER_TAPS = 4096
B200_IQ_MAX_CONDITIONER_DECIMATION = 4096
B200_IQ_MAX_BLANKING_LENGTH = 4096
B200_NOTCH = 0
B200_NOTCH_LITE = 1
B200_IQ_MAX_NOTCH_LENGTH = 1024
ERRORS = {0: "OK", -1: "ERR_ARG", -2: "ERR_CUDA", -3: "ERR_NOMEM", -4: "ERR_STATE", -5: "ERR_RANGE", -6: "ERR_NODEV"}


class B200Error(RuntimeError):
    def __init__(self, code: int, where: str):
        self.code = code
        msg = lib.b200_last_error()
        super().__init__(f"{where}: {ERRORS.get(code, code)}: {msg.decode() if msg else ''}")


lib.b200_last_error.restype = C.c_char_p
_vp = C.c_void_p

_SIGS = {
    "b200_version": ([], C.c_int),
    "b200_device_count": ([C.POINTER(C.c_int)], C.c_int),
    "b200_engine_create": ([C.POINTER(_vp), C.c_int, _vp], C.c_int),
    "b200_engine_destroy": ([_vp], C.c_int),
    "b200_engine_sync": ([_vp], C.c_int),
    "b200_engine_timer_start": ([_vp], C.c_int),
    "b200_engine_timer_stop_ms": ([_vp, C.POINTER(C.c_float)], C.c_int),
    "b200_engine_launch_count": ([_vp, C.POINTER(C.c_uint64)], C.c_int),
    "b200_iq_create": ([_vp, C.c_int, C.c_uint64], C.c_int),
    "b200_iq_create_typed": ([_vp, C.c_int, C.c_uint64, C.c_char_p], C.c_int),
    "b200_iq_push": ([_vp, C.c_int, _vp, C.c_uint64, C.POINTER(C.c_uint64)], C.c_int),
    "b200_iq_push_at": ([_vp, C.c_int, C.c_uint64, _vp, C.c_uint64, C.POINTER(C.c_uint64)], C.c_int),
    "b200_iq_window": ([_vp, C.c_int, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)], C.c_int),
    "b200_iq_forget": ([_vp, C.c_int], C.c_int),
    "b200_trk_kernel_choice": ([_vp, C.c_int], C.c_int),
    "b200_iq_refill": ([_vp, C.c_int, _vp, C.c_uint64, C.c_uint64], C.c_int),
    "b200_iq_read": ([_vp, C.c_int, C.c_uint64, C.c_uint64, _vp], C.c_int),
    "b200_iq_set_conditioner": ([_vp, C.c_int, C.c_int, C.c_uint32, _vp, C.c_uint32, C.c_double, C.c_double], C.c_int),
    "b200_iq_conditioner_lowpass": ([C.c_double, C.c_uint32, C.c_double, C.c_double, C.c_uint32, _vp, C.POINTER(C.c_uint32)], C.c_int),
    "b200_iq_set_pulse_blanking": ([_vp, C.c_int, C.c_int, C.c_float, C.c_int32, C.c_int32, C.c_int32], C.c_int),
    "b200_iq_pulse_blanking_threshold": ([C.c_float, C.c_int32, C.POINTER(C.c_float)], C.c_int),
    "b200_iq_pulse_blanking_status": ([_vp, C.c_int, C.POINTER(PulseBlankingStatus)], C.c_int),
    "b200_iq_set_notch": ([_vp, C.c_int, C.c_int, C.c_int, C.c_float, C.c_float, C.c_int32, C.c_int32, C.c_int32, C.c_int32], C.c_int),
    "b200_iq_notch_status": ([_vp, C.c_int, C.POINTER(NotchStatus)], C.c_int),
    "b200_trk_set_taps": ([_vp, _vp], C.c_int),
    "b200_trk_set_local_code_and_taps_cplx": ([_vp, C.c_int, _vp, _vp], C.c_int),
    "b200_trk_correlate_cplx": ([_vp, _vp, C.c_float, C.c_float, C.c_float, C.c_float, C.c_int, _vp], C.c_int),
    "b200_trk_set_local_code_and_taps_16sc": ([_vp, C.c_int, _vp, _vp], C.c_int),
    "b200_trk_correlate_16sc": ([_vp, _vp, C.c_float, C.c_float, C.c_float, C.c_float, C.c_int, _vp], C.c_int),
    "b200_trk_channel_set_taps": ([_vp, C.c_int, _vp], C.c_int),
    "b200_acq_sweep_best_dev": ([_vp, _vp, _vp, C.c_uint32, _vp], C.c_int),
    "b200_acq_search_i16": ([_vp, _vp, _vp, C.c_uint32, C.c_uint32, _vp], C.c_int),
    "b200_acq_search_step_two_i16": ([_vp, _vp, C.c_uint32, C.c_uint32, C.c_float, _vp], C.c_int),
    "b200_iq_push_i16": ([_vp, C.c_int, _vp, C.c_uint64, C.POINTER(C.c_uint64)], C.c_int),
    "b200_iq_push_i8": ([_vp, C.c_int, _vp, C.c_uint64, C.POINTER(C.c_uint64)], C.c_int),
    "b200_iq_attach_dev": ([_vp, C.c_int, _vp, C.c_uint64, C.c_uint64], C.c_int),
    "b200_iq_push_file": ([_vp, C.c_int, C.c_char_p, C.c_char_p, C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint64,
                           C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)], C.c_int),
    "b200_trk_create": ([_vp, C.POINTER(_vp), C.c_int, C.c_int], C.c_int),
    "b200_trk_set_high_dynamics_resampler": ([_vp, C.c_int], C.c_int),
    "b200_trk_set_local_code_and_taps": ([_vp, C.c_int, _vp, _vp], C.c_int),
    "b200_trk_correlate": ([_vp, _vp, C.c_float, C.c_float, C.c_float, C.c_float, C.c_float, C.c_float, C.c_int, _vp], C.c_int),
    "b200_trk_destroy": ([_vp], C.c_int),
    "b200_trk_channel_create": ([_vp, C.c_int, C.c_int, C.POINTER(C.c_int)], C.c_int),
    "b200_trk_channel_set_code": ([_vp, C.c_int, C.c_int, _vp, _vp, C.c_int], C.c_int),
    "b200_trk_batch": ([_vp, _vp, C.c_int, _vp, C.c_int], C.c_int),
    "b200_trk_batch_dev": ([_vp, _vp, C.c_int, _vp, C.c_int, C.c_int], C.c_int),
    "b200_trk_submit": ([_vp, _vp, C.c_int, C.c_int, C.POINTER(C.c_uint64)], C.c_int),
    "b200_trk_wait": ([_vp, C.c_uint64, _vp], C.c_int),
    "b200_acq_create": ([_vp, C.POINTER(AcqConf), C.POINTER(_vp)], C.c_int),
    "b200_acq_set_local_code": ([_vp, C.c_uint32, _vp], C.c_int),
    "b200_acq_set_doppler_center": ([_vp, C.c_int32, C.c_int32], C.c_int),
    "b200_acq_search": ([_vp, _vp, _vp, C.c_uint32, C.c_uint32, _vp], C.c_int),
    "b200_acq_search_submit": ([_vp, _vp, _vp, C.c_uint32, C.c_uint32], C.c_int),
    "b200_acq_search_wait": ([_vp, _vp], C.c_int),
    "b200_acq_set_step_two": ([_vp, C.c_float, C.c_float, C.c_uint32], C.c_int),
    "b200_acq_search_step_two": ([_vp, _vp, C.c_uint32, C.c_uint32, C.c_float, _vp], C.c_int),
    "b200_acq_search_dev": ([_vp, _vp, _vp, C.c_uint32, C.c_uint32, _vp], C.c_int),
    "b200_acq_search_band": ([_vp, C.c_int, C.c_uint64, _vp, C.c_uint32, C.c_uint32, _vp], C.c_int),
    "b200_acq_search_band_submit": ([_vp, C.c_int, C.c_uint64, _vp, C.c_uint32, C.c_uint32], C.c_int),
    "b200_acq_search_step_two_band": ([_vp, C.c_int, C.c_uint64, C.c_uint32, C.c_uint32, C.c_float, _vp], C.c_int),
    "b200_acq_resampler_design": ([C.c_int64, C.c_int64, C.c_uint32, C.POINTER(C.c_uint32), _vp, C.POINTER(C.c_uint32)], C.c_int),
    "b200_acq_set_band_resampler": ([_vp, C.c_uint32, _vp, C.c_uint32], C.c_int),
    "b200_acq_read_grid": ([_vp, C.c_uint32, _vp], C.c_int),
    "b200_acq_selftest_dft": ([_vp, _vp, _vp], C.c_int),
    "b200_acq_read_wipeoffs": ([_vp, _vp], C.c_int),
    "b200_acq_destroy": ([_vp], C.c_int),
    "b200_trk_loop_create": ([_vp, C.c_int, C.POINTER(TrkLoopConf), C.POINTER(C.c_int)], C.c_int),
    "b200_trk_loop_start": ([_vp, C.c_int, C.c_double, C.c_double, C.c_uint64, C.c_uint64], C.c_int),
    "b200_trk_loop_run": ([_vp, C.c_int, _vp, _vp], C.c_int),
    "b200_trk_loop_run_prompts": ([_vp, C.c_int, _vp, _vp, _vp], C.c_int),
    "b200_trk_loop_set_data_channel": ([_vp, C.c_int, C.c_int], C.c_int),
    "b200_trk_loop_peek_items": ([_vp, _vp], C.c_int),
    "b200_trk_loop_set_mode": ([_vp, C.c_int], C.c_int),
    "b200_trk_loop_step_taps": ([_vp, _vp, _vp, _vp], C.c_int),
    "b200_trk_loop_status_get": ([_vp, C.c_int, C.POINTER(TrkLoopStatus)], C.c_int),
    "b200_trk_dump_write": ([C.c_char_p, _vp, C.c_int, C.c_int], C.c_int),
    "b200_acq_fine_create": ([_vp, C.c_uint32, C.POINTER(_vp)], C.c_int),
    "b200_acq_fine_estimate": ([_vp, _vp, _vp, C.POINTER(C.c_uint32), C.POINTER(C.c_float)], C.c_int),
    "b200_acq_fine_read_spectrum": ([_vp, _vp], C.c_int),
    "b200_acq_fine_destroy": ([_vp], C.c_int),
    "b200_acq_dump_write": ([C.c_char_p, C.POINTER(AcqDump)], C.c_int),
    "b200_acq_dump_filename": ([C.c_char_p, C.c_char, C.c_char_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_char_p, C.c_size_t], C.c_int),
}

for _name, (_args, _res) in _SIGS.items():
    _fn = getattr(lib, _name)
    _fn.argtypes = _args
    _fn.restype = _res


def exported_symbols():
    """Names declared in include/b200gnss.h that this binding knows about."""
    return list(_SIGS) + ["b200_last_error"]


def _chk(rc: int, where: str):
    if rc != 0:
        raise B200Error(rc, where)


def device_count() -> int:
    n = C.c_int(0)
    lib.b200_device_count(C.byref(n))
    return n.value


class Engine:
    """b200_engine handle."""

    def __init__(self, device: int = 0, stream: int | None = None):
        h = _vp()
        _chk(lib.b200_engine_create(C.byref(h), device, _vp(stream) if stream else None), "b200_engine_create")
        self.h = h
        self.device = device
        self._band_types = {}   # item type of each band made by iq_create (iq_read's output format)

    def close(self):
        if self.h:
            lib.b200_engine_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def sync(self):
        _chk(lib.b200_engine_sync(self.h), "b200_engine_sync")

    def timer_start(self):
        _chk(lib.b200_engine_timer_start(self.h), "timer_start")

    def timer_stop_ms(self) -> float:
        ms = C.c_float(0)
        _chk(lib.b200_engine_timer_stop_ms(self.h, C.byref(ms)), "timer_stop")
        return ms.value

    def launch_count(self) -> int:
        n = C.c_uint64(0)
        _chk(lib.b200_engine_launch_count(self.h, C.byref(n)), "launch_count")
        return n.value

    # bands
    def iq_create(self, band: int, capacity: int, item_type: str = "gr_complex"):
        """item_type: "gr_complex" (float samples), "ishort" or "ibyte" (interleaved int16 / int8 I,Q kept at their own
        width; such a band takes only iq_push_int / iq_push_file pushes of its own type)"""
        _chk(lib.b200_iq_create_typed(self.h, band, capacity, item_type.encode()), "b200_iq_create_typed")
        self._band_types[band] = item_type

    def iq_push(self, band: int, iq: np.ndarray) -> int:
        iq = np.ascontiguousarray(iq, np.complex64)
        first = C.c_uint64(0)
        _chk(lib.b200_iq_push(self.h, band, iq.ctypes.data, iq.size, C.byref(first)), "b200_iq_push")
        return first.value

    def iq_push_at(self, band: int, abs_index: int, iq: np.ndarray) -> int:
        """idempotent push by absolute index; returns how many samples were actually copied"""
        iq = np.ascontiguousarray(iq, np.complex64)
        n_new = C.c_uint64(0)
        _chk(lib.b200_iq_push_at(self.h, band, int(abs_index), iq.ctypes.data, iq.size, C.byref(n_new)), "b200_iq_push_at")
        return n_new.value

    def iq_refill_ptr(self, band: int, host_ptr: int, n: int, first_index: int = 0):
        _chk(lib.b200_iq_refill(self.h, band, host_ptr, n, first_index), "b200_iq_refill")

    def trk_kernel_choice(self, mode: int):
        _chk(lib.b200_trk_kernel_choice(self.h, mode), "b200_trk_kernel_choice")

    def iq_forget(self, band: int):
        _chk(lib.b200_iq_forget(self.h, band), "b200_iq_forget")

    def iq_window(self, band: int):
        lo, hi = C.c_uint64(0), C.c_uint64(0)
        _chk(lib.b200_iq_window(self.h, band, C.byref(lo), C.byref(hi)), "b200_iq_window")
        return lo.value, hi.value

    def iq_push_ptr(self, band: int, host_ptr: int, n: int) -> int:
        first = C.c_uint64(0)
        _chk(lib.b200_iq_push(self.h, band, host_ptr, n, C.byref(first)), "b200_iq_push")
        return first.value

    def iq_push_int(self, band: int, host_ptr_or_array, n: int = None) -> int:
        """interleaved int16 or int8 (I,Q) samples; n = number of complex samples"""
        first = C.c_uint64(0)
        if isinstance(host_ptr_or_array, np.ndarray):
            a = np.ascontiguousarray(host_ptr_or_array)
            assert a.dtype in (np.int16, np.int8)
            fn = lib.b200_iq_push_i16 if a.dtype == np.int16 else lib.b200_iq_push_i8
            _chk(fn(self.h, band, a.ctypes.data, a.size // 2, C.byref(first)), "b200_iq_push_int")
        else:
            ptr, bits = host_ptr_or_array
            fn = lib.b200_iq_push_i16 if bits == 16 else lib.b200_iq_push_i8
            _chk(fn(self.h, band, ptr, n, C.byref(first)), "b200_iq_push_int")
        return first.value

    def iq_push_file(self, band: int, path: str, item_type: str = "gr_complex", header_bytes: int = 0, skip_samples: int = 0,
                     max_samples: int = 0, chunk_samples: int = 0):
        """-> (first_index, samples_pushed)"""
        first, n = C.c_uint64(0), C.c_uint64(0)
        _chk(lib.b200_iq_push_file(self.h, band, path.encode(), item_type.encode(), header_bytes, skip_samples, max_samples,
                                   chunk_samples, C.byref(first), C.byref(n)), "b200_iq_push_file")
        return first.value, n.value

    def iq_attach_dev(self, band: int, dev_ptr: int, n_samples: int, first_index: int = 0):
        self._band_types[band] = "gr_complex"
        _chk(lib.b200_iq_attach_dev(self.h, band, dev_ptr, n_samples, first_index), "b200_iq_attach_dev")

    def iq_read(self, band: int, abs_index: int, n: int) -> np.ndarray:
        """samples [abs_index, abs_index + n) of the band's window in its own format: complex64 for a gr_complex band,
        interleaved (I, Q) int16 / int8 (2 n values) for an ishort / ibyte band"""
        fmt = self._band_types.get(band, "gr_complex")
        out = np.zeros(n, np.complex64) if fmt == "gr_complex" else np.zeros(2 * n, np.int16 if fmt == "ishort" else np.int8)
        _chk(lib.b200_iq_read(self.h, band, int(abs_index), int(n), out.ctypes.data if n else None), "b200_iq_read")
        return out

    def iq_set_conditioner(self, dst_band: int, src_band: int, decimation: int, taps, intermediate_freq_hz: float,
                           sampling_freq_hz: float):
        """fill dst_band with the frequency-translating decimating FIR of every push into src_band
        (freq_xlating_fir_filter_ccf(decimation, taps, IF, fs)); empty taps remove dst_band's conditioner"""
        taps = np.ascontiguousarray(taps, np.float32)
        _chk(lib.b200_iq_set_conditioner(self.h, dst_band, src_band, int(decimation), taps.ctypes.data if taps.size else None,
                                         taps.size, float(intermediate_freq_hz), float(sampling_freq_hz)), "b200_iq_set_conditioner")

    def iq_remove_conditioner(self, dst_band: int):
        _chk(lib.b200_iq_set_conditioner(self.h, dst_band, 0, 1, None, 0, 0.0, 1.0), "b200_iq_set_conditioner")

    def iq_set_pulse_blanking(self, dst_band: int, src_band: int, pfa: float = 0.04, length: int = 32, segments_est: int = 12500,
                              segments_reset: int = 5000000):
        """fill dst_band with the pulse-blanking input filter of every push into src_band (pulse_blanking_cc(pfa, length,
        segments_est, segments_reset); the defaults are the adapter's)"""
        _chk(lib.b200_iq_set_pulse_blanking(self.h, dst_band, src_band, float(pfa), int(length), int(segments_est), int(segments_reset)),
             "b200_iq_set_pulse_blanking")

    def iq_remove_pulse_blanking(self, dst_band: int):
        _chk(lib.b200_iq_set_pulse_blanking(self.h, dst_band, 0, 0.04, 0, 0, 0), "b200_iq_set_pulse_blanking")

    def iq_pulse_blanking_status(self, dst_band: int) -> dict:
        """origin, segments (processed), blanked, n, noise_power (est), threshold, last_filtered and length of dst_band's
        blanker, after every push queued so far"""
        st = PulseBlankingStatus()
        _chk(lib.b200_iq_pulse_blanking_status(self.h, dst_band, C.byref(st)), "b200_iq_pulse_blanking_status")
        return {name: getattr(st, name) for name, _ in PulseBlankingStatus._fields_}

    def iq_set_notch(self, dst_band: int, src_band: int, variant: int = B200_NOTCH_LITE, pfa: float = 0.001, p_c_factor: float = 0.9,
                     length: int = 32, segments_est: int = 12500, segments_reset: int = 5000000, segments_coeff: int = 1):
        """fill dst_band with the notch input filter of every push into src_band: variant B200_NOTCH (Notch(pfa, p_c_factor,
        length, segments_est, segments_reset)) or B200_NOTCH_LITE (NotchLite(p_c_factor, pfa, length, segments_est,
        segments_reset, segments_coeff)); the defaults are the adapters'"""
        _chk(lib.b200_iq_set_notch(self.h, dst_band, src_band, int(variant), float(pfa), float(p_c_factor), int(length), int(segments_est),
                                   int(segments_reset), int(segments_coeff)), "b200_iq_set_notch")

    def iq_remove_notch(self, dst_band: int):
        _chk(lib.b200_iq_set_notch(self.h, dst_band, 0, B200_NOTCH_LITE, 0.001, 0.9, 0, 0, 0, 1), "b200_iq_set_notch")

    def iq_notch_status(self, dst_band: int) -> dict:
        """origin, segments, filtered, n, noise_power (est), threshold, z0, last_out (complex), filter_state, n_coeff,
        length and variant of dst_band's notch, after every push queued so far"""
        st = NotchStatus()
        _chk(lib.b200_iq_notch_status(self.h, dst_band, C.byref(st)), "b200_iq_notch_status")
        d = {name: getattr(st, name) for name, _ in NotchStatus._fields_}
        d["z0"] = complex(d.pop("z0_re"), d.pop("z0_im"))
        d["last_out"] = complex(d.pop("last_out_re"), d.pop("last_out_im"))
        return d

    # channels
    def channel_create(self, band: int, taps: int) -> int:
        cid = C.c_int(-1)
        _chk(lib.b200_trk_channel_create(self.h, band, taps, C.byref(cid)), "b200_trk_channel_create")
        return cid.value

    def channel_set_code(self, cid: int, code, shifts, high_dyn: bool = False):
        code = np.ascontiguousarray(code, np.float32)
        shifts = np.ascontiguousarray(shifts, np.float32)
        _chk(lib.b200_trk_channel_set_code(self.h, cid, code.size, code.ctypes.data, shifts.ctypes.data, int(high_dyn)),
             "b200_trk_channel_set_code")

    def channel_set_taps(self, cid: int, shifts):
        shifts = np.ascontiguousarray(shifts, np.float32)
        _chk(lib.b200_trk_channel_set_taps(self.h, cid, shifts.ctypes.data), "b200_trk_channel_set_taps")

    def trk_batch(self, items: np.ndarray, out_stride: int) -> np.ndarray:
        items = np.ascontiguousarray(items, TRK_ITEM_DTYPE)
        out = np.zeros((items.size, out_stride), np.complex64)
        _chk(lib.b200_trk_batch(self.h, items.ctypes.data, items.size, out.ctypes.data, out_stride), "b200_trk_batch")
        return out

    def trk_submit(self, items: np.ndarray, out_stride: int) -> tuple:
        items = np.ascontiguousarray(items, TRK_ITEM_DTYPE)
        t = C.c_uint64(0)
        _chk(lib.b200_trk_submit(self.h, items.ctypes.data, items.size, out_stride, C.byref(t)), "b200_trk_submit")
        return (t.value, items.size, out_stride)

    def trk_wait(self, ticket: tuple) -> np.ndarray:
        t, n, stride = ticket
        out = np.zeros((n, stride), np.complex64)
        _chk(lib.b200_trk_wait(self.h, t, out.ctypes.data), "b200_trk_wait")
        return out

    def trk_batch_dev(self, items_dev_ptr: int, n_items: int, out_dev_ptr: int, out_stride: int, slices: int = 1):
        _chk(lib.b200_trk_batch_dev(self.h, items_dev_ptr, n_items, out_dev_ptr, out_stride, slices), "b200_trk_batch_dev")

    # free-running DLL/PLL loops on the device
    def loop_create(self, channel: int, conf: TrkLoopConf) -> int:
        lid = C.c_int(-1)
        _chk(lib.b200_trk_loop_create(self.h, channel, C.byref(conf), C.byref(lid)), "b200_trk_loop_create")
        self._n_loops = getattr(self, "_n_loops", 0) + 1
        return lid.value

    def loop_start(self, loop_id: int, acq_delay_samples: float, acq_doppler_hz: float, acq_samplestamp: int, nitems_read: int):
        _chk(lib.b200_trk_loop_start(self.h, loop_id, acq_delay_samples, acq_doppler_hz, acq_samplestamp, nitems_read),
             "b200_trk_loop_start")

    def loop_run(self, max_epochs: int):
        """-> (records[n_loops, max_epochs] of TRK_DUMP_RECORD_DTYPE, n_records[n_loops])"""
        n = getattr(self, "_n_loops", 0)
        rec = np.zeros((n, max_epochs), TRK_DUMP_RECORD_DTYPE)
        cnt = np.zeros(n, np.int32)
        _chk(lib.b200_trk_loop_run(self.h, max_epochs, rec.ctypes.data, cnt.ctypes.data), "b200_trk_loop_run")
        return rec, cnt

    def loop_set_data_channel(self, loop_id: int, channel: int):
        """correlate the 1-tap `channel` beside the loop's pilot; the records then carry its prompt"""
        _chk(lib.b200_trk_loop_set_data_channel(self.h, loop_id, channel), "b200_trk_loop_set_data_channel")

    def loop_run_prompts(self, max_epochs: int):
        """-> (records[n_loops, max_epochs], n_records[n_loops], pilot prompts complex64[n_loops, max_epochs])"""
        n = getattr(self, "_n_loops", 0)
        rec = np.zeros((n, max_epochs), TRK_DUMP_RECORD_DTYPE)
        cnt = np.zeros(n, np.int32)
        prm = np.zeros((n, max_epochs), np.complex64)
        _chk(lib.b200_trk_loop_run_prompts(self.h, max_epochs, rec.ctypes.data, cnt.ctypes.data, prm.ctypes.data), "b200_trk_loop_run_prompts")
        return rec, cnt, prm

    def loop_set_mode(self, mode: int):
        _chk(lib.b200_trk_loop_set_mode(self.h, mode), "b200_trk_loop_set_mode")

    def loop_peek_items(self) -> np.ndarray:
        n = getattr(self, "_n_loops", 0)
        items = np.zeros(n, TRK_ITEM_DTYPE)
        _chk(lib.b200_trk_loop_peek_items(self.h, items.ctypes.data), "b200_trk_loop_peek_items")
        return items

    def loop_step_taps(self, taps: np.ndarray):
        """taps complex64[n_loops, 8] -> (records[n_loops], logged[n_loops])"""
        n = getattr(self, "_n_loops", 0)
        t = np.zeros((n, B200_MAX_TAPS), np.complex64)
        taps = np.asarray(taps, np.complex64).reshape(n, -1)
        t[:, :taps.shape[1]] = taps
        rec = np.zeros(n, TRK_DUMP_RECORD_DTYPE)
        logged = np.zeros(n, np.int32)
        _chk(lib.b200_trk_loop_step_taps(self.h, t.ctypes.data, rec.ctypes.data, logged.ctypes.data), "b200_trk_loop_step_taps")
        return rec, logged

    def loop_status(self, loop_id: int) -> TrkLoopStatus:
        s = TrkLoopStatus()
        _chk(lib.b200_trk_loop_status_get(self.h, loop_id, C.byref(s)), "b200_trk_loop_status_get")
        return s


def trk_dump_write(filename: str, records: np.ndarray, append: bool = False):
    """Write records in the reference's tracking dump format (dll_pll_veml_tracking.cc:1599-1694)."""
    records = np.ascontiguousarray(records, TRK_DUMP_RECORD_DTYPE)
    _chk(lib.b200_trk_dump_write(filename.encode(), records.ctypes.data, records.size, int(append)), "b200_trk_dump_write")


class Multicorrelator:
    """b200_trk handle; same call sequence as the reference's Cpu_Multicorrelator_Real_Codes."""

    def __init__(self, engine: Engine, max_signal_length_samples: int, n_correlators: int):
        h = _vp()
        _chk(lib.b200_trk_create(engine.h, C.byref(h), max_signal_length_samples, n_correlators), "b200_trk_create")
        self.h = h
        self.engine = engine
        self.taps = n_correlators

    def set_high_dynamics_resampler(self, flag: bool):
        _chk(lib.b200_trk_set_high_dynamics_resampler(self.h, int(flag)), "set_high_dynamics_resampler")

    def set_local_code_and_taps(self, code, shifts):
        code = np.ascontiguousarray(code, np.float32)
        shifts = np.ascontiguousarray(shifts, np.float32)
        assert shifts.size == self.taps
        _chk(lib.b200_trk_set_local_code_and_taps(self.h, code.size, code.ctypes.data, shifts.ctypes.data),
             "set_local_code_and_taps")

    def Carrier_wipeoff_multicorrelator_resampler(self, sig_in, rem_carrier_phase_in_rad, phase_step_rad,
                                                  phase_rate_step_rad, rem_code_phase_chips, code_phase_step_chips,
                                                  code_phase_rate_step_chips, signal_length_samples=None) -> np.ndarray:
        sig_in = np.ascontiguousarray(sig_in, np.complex64)
        n = sig_in.size if signal_length_samples is None else signal_length_samples
        out = np.zeros(self.taps, np.complex64)
        _chk(lib.b200_trk_correlate(self.h, sig_in.ctypes.data, rem_carrier_phase_in_rad, phase_step_rad,
                                    phase_rate_step_rad, rem_code_phase_chips, code_phase_step_chips,
                                    code_phase_rate_step_chips, n, out.ctypes.data), "b200_trk_correlate")
        return out

    # Cpu_Multicorrelator (complex local code)
    def set_local_code_and_taps_cplx(self, code, shifts):
        code = np.ascontiguousarray(code, np.complex64)
        shifts = np.ascontiguousarray(shifts, np.float32)
        _chk(lib.b200_trk_set_local_code_and_taps_cplx(self.h, code.size, code.ctypes.data, shifts.ctypes.data), "set_local_code_and_taps_cplx")

    def correlate_cplx(self, sig_in, rem_carrier_phase_in_rad, phase_step_rad, rem_code_phase_chips, code_phase_step_chips) -> np.ndarray:
        sig_in = np.ascontiguousarray(sig_in, np.complex64)
        out = np.zeros(self.taps, np.complex64)
        _chk(lib.b200_trk_correlate_cplx(self.h, sig_in.ctypes.data, rem_carrier_phase_in_rad, phase_step_rad, rem_code_phase_chips,
                                         code_phase_step_chips, sig_in.size, out.ctypes.data), "b200_trk_correlate_cplx")
        return out

    # Cpu_Multicorrelator_16sc (interleaved int16 I,Q)
    def set_local_code_and_taps_16sc(self, code_iq, shifts):
        code_iq = np.ascontiguousarray(code_iq, np.int16)
        shifts = np.ascontiguousarray(shifts, np.float32)
        _chk(lib.b200_trk_set_local_code_and_taps_16sc(self.h, code_iq.size // 2, code_iq.ctypes.data, shifts.ctypes.data), "set_local_code_and_taps_16sc")

    def correlate_16sc(self, sig_iq, rem_carrier_phase_in_rad, phase_step_rad, rem_code_phase_chips, code_phase_step_chips) -> np.ndarray:
        sig_iq = np.ascontiguousarray(sig_iq, np.int16)
        out = np.zeros(2 * self.taps, np.int16)
        _chk(lib.b200_trk_correlate_16sc(self.h, sig_iq.ctypes.data, rem_carrier_phase_in_rad, phase_step_rad, rem_code_phase_chips,
                                         code_phase_step_chips, sig_iq.size // 2, out.ctypes.data), "b200_trk_correlate_16sc")
        return out

    def free(self):
        if self.h:
            lib.b200_trk_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class PcpsAcquisition:
    """b200_acq handle: the arithmetic of one pcps_acquisition block (or of a multi-PRN sweep).

    Construction mirrors pcps_acquisition's constructor (pcps_acquisition.cc:100-193): sizes are
    derived from the Acq_Conf fields exactly as there."""

    def __init__(self, engine: Engine, *, fs_in: int, samples_per_ms: float, samples_per_chip: int, doppler_max: int,
                 doppler_step: int, sampled_ms: int = 1, ms_per_code: int = 1, bit_transition_flag: bool = False,
                 use_CFAR_algorithm_flag: bool = True, max_dwells: int = 1, n_code_slots: int = 1,
                 keep_grid: bool = False, num_doppler_bins: int = None):
        import math
        consumed = int(sampled_ms * samples_per_ms * (2.0 if bit_transition_flag else 1.0))
        fft_size = consumed if sampled_ms == ms_per_code else consumed * 2
        eff = fft_size // 2 if bit_transition_flag else fft_size
        bins = int(math.ceil(float(2 * doppler_max) / float(doppler_step))) if num_doppler_bins is None else int(num_doppler_bins)
        layout = 1 if bit_transition_flag else (0 if sampled_ms == ms_per_code else 2)
        self.conf = AcqConf(fft_size, eff, consumed, bins, doppler_max, doppler_step, int(fs_in), samples_per_chip,
                            layout, int(bit_transition_flag), int(use_CFAR_algorithm_flag), max_dwells, n_code_slots,
                            int(keep_grid))
        h = _vp()
        _chk(lib.b200_acq_create(engine.h, C.byref(self.conf), C.byref(h)), "b200_acq_create")
        self.h = h
        self.engine = engine

    def set_local_code(self, slot: int, code):
        code = np.ascontiguousarray(code, np.complex64)
        need = self.conf.fft_size // 2 if self.conf.code_layout == 1 else self.conf.consumed_samples
        assert code.size >= need, (code.size, need)
        _chk(lib.b200_acq_set_local_code(self.h, slot, code.ctypes.data), "b200_acq_set_local_code")

    def set_doppler_center(self, center: int, bias: int = 0):
        _chk(lib.b200_acq_set_doppler_center(self.h, center, bias), "b200_acq_set_doppler_center")

    def search(self, iq, slots, dwell_counter: int = 1) -> np.ndarray:
        iq = np.ascontiguousarray(iq, np.complex64)
        assert iq.size >= self.conf.consumed_samples
        slots = np.ascontiguousarray(slots, np.uint32)
        res = np.zeros(slots.size, ACQ_RESULT_DTYPE)
        _chk(lib.b200_acq_search(self.h, iq.ctypes.data, slots.ctypes.data, slots.size, dwell_counter, res.ctypes.data),
             "b200_acq_search")
        return res

    def search_submit(self, iq, slots, dwell_counter: int = 1):
        iq = np.ascontiguousarray(iq, np.complex64)
        assert iq.size >= self.conf.consumed_samples
        slots = np.ascontiguousarray(slots, np.uint32)
        _chk(lib.b200_acq_search_submit(self.h, iq.ctypes.data, slots.ctypes.data, slots.size, dwell_counter), "b200_acq_search_submit")
        self._pending_n = slots.size      # only once the sweep is really in flight: wait() sizes its buffer from it

    def search_wait(self) -> np.ndarray:
        res = np.zeros(max(getattr(self, "_pending_n", 0), self.conf.n_code_slots), ACQ_RESULT_DTYPE)[:getattr(self, "_pending_n", 0)]
        _chk(lib.b200_acq_search_wait(self.h, res.ctypes.data), "b200_acq_search_wait")
        return res

    def set_step_two(self, center: float, step2: float, bins2: int):
        _chk(lib.b200_acq_set_step_two(self.h, center, step2, bins2), "b200_acq_set_step_two")

    def search_step_two(self, iq, slot: int, prev_input_power: float, dwell_counter: int = 1) -> np.ndarray:
        iq = np.ascontiguousarray(iq, np.complex64)
        res = np.zeros(1, ACQ_RESULT_DTYPE)
        _chk(lib.b200_acq_search_step_two(self.h, iq.ctypes.data, slot, dwell_counter, prev_input_power, res.ctypes.data),
             "b200_acq_search_step_two")
        return res[0]

    def search_dev(self, in_dev_ptr: int, slots, results_dev_ptr: int, dwell_counter: int = 1):
        slots = np.ascontiguousarray(slots, np.uint32)
        _chk(lib.b200_acq_search_dev(self.h, in_dev_ptr, slots.ctypes.data, slots.size, dwell_counter, results_dev_ptr),
             "b200_acq_search_dev")

    def set_band_resampler(self, decimation: int, taps):
        """decimate the band searches' input by `decimation` through the FIR `taps` (acq_resampler_design); decimation 1
        turns the resampler off.  The object works at the decimated rate, its bands hold the full rate."""
        taps = np.ascontiguousarray(taps, np.float32)
        _chk(lib.b200_acq_set_band_resampler(self.h, int(decimation), taps.ctypes.data if taps.size else None, taps.size),
             "b200_acq_set_band_resampler")

    def search_band(self, band: int, abs_index: int, slots, dwell_counter: int = 1) -> np.ndarray:
        """search samples [abs_index, abs_index + consumed_samples) of one of the engine's bands; the result's sample stamp
        for loop_start is abs_index + consumed_samples.  Dwell k takes the window k * consumed_samples further on.

        With a band resampler of decimation D and T taps, the search reads [abs_index - (T - 1), abs_index + (consumed - 1) D
        + 1) and searches y[j] = sum_k taps[k] x[abs_index + j D - k]; dwell k takes abs_index + k consumed D.  Mapped to the
        full rate as the reference does (pcps_acquisition.cc:583-597): the sample stamp is abs_index + consumed D and the
        delay fmod(index_time, samples_per_code) D - (T - 1) / 2."""
        slots = np.ascontiguousarray(slots, np.uint32)
        res = np.zeros(slots.size, ACQ_RESULT_DTYPE)
        _chk(lib.b200_acq_search_band(self.h, band, int(abs_index), slots.ctypes.data, slots.size, dwell_counter, res.ctypes.data),
             "b200_acq_search_band")
        return res

    def search_band_submit(self, band: int, abs_index: int, slots, dwell_counter: int = 1):
        """queue search_band's sweep (the same window, resampler and stamp rules); search_wait() collects its results"""
        slots = np.ascontiguousarray(slots, np.uint32)
        _chk(lib.b200_acq_search_band_submit(self.h, band, int(abs_index), slots.ctypes.data, slots.size, dwell_counter),
             "b200_acq_search_band_submit")
        self._pending_n = slots.size

    def search_step_two_band(self, band: int, abs_index: int, slot: int, prev_input_power: float, dwell_counter: int = 1) -> np.ndarray:
        res = np.zeros(1, ACQ_RESULT_DTYPE)
        _chk(lib.b200_acq_search_step_two_band(self.h, band, int(abs_index), slot, dwell_counter, prev_input_power, res.ctypes.data),
             "b200_acq_search_step_two_band")
        return res[0]

    def sweep_best_dev(self, results_dev_ptr: int, prn_of_result_dev_ptr: int, n_results: int, peak_dev_ptr: int):
        """one 16-byte b200_acq_peak record of the sweep, written on the device (no host synchronisation)"""
        _chk(lib.b200_acq_sweep_best_dev(self.h, results_dev_ptr, prn_of_result_dev_ptr, n_results, peak_dev_ptr), "b200_acq_sweep_best_dev")

    def selftest_dft(self, x) -> np.ndarray:
        x = np.ascontiguousarray(x, np.complex64)
        assert x.size == self.conf.fft_size
        out = np.empty(x.size, np.complex64)
        _chk(lib.b200_acq_selftest_dft(self.h, x.ctypes.data, out.ctypes.data), "b200_acq_selftest_dft")
        return out

    def read_grid(self, slot: int) -> np.ndarray:
        g = np.empty((self.conf.num_doppler_bins, self.conf.effective_fft_size), np.float32)
        _chk(lib.b200_acq_read_grid(self.h, slot, g.ctypes.data), "b200_acq_read_grid")
        return g

    def read_wipeoffs(self) -> np.ndarray:
        w = np.empty((self.conf.num_doppler_bins, self.conf.fft_size), np.complex64)
        _chk(lib.b200_acq_read_wipeoffs(self.h, w.ctypes.data), "b200_acq_read_wipeoffs")
        return w

    def close(self):
        if self.h:
            lib.b200_acq_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def acq_dump_write(filename: str, grid: np.ndarray, *, doppler_max: int, doppler_step: int, positive_acq: bool, acq_doppler_hz: float,
                   acq_delay_samples: float, test_statistic: float, threshold: float, input_power: float, sample_counter: int,
                   prn: int, num_dwells: int, grid_narrow: np.ndarray = None, doppler_step_narrow: float = 0.0,
                   doppler_grid_narrow_min: float = 0.0):
    """Write the acquisition dump of pcps_acquisition::dump_results (:354-406) as a Level-5 MAT-file.
    grid: float32[num_doppler_bins, effective_fft_size] as PcpsAcquisition.read_grid returns it."""
    grid = np.ascontiguousarray(grid, np.float32)
    d = AcqDump()
    d.acq_grid = grid.ctypes.data
    d.num_doppler_bins, d.effective_fft_size = grid.shape
    if grid_narrow is not None:
        grid_narrow = np.ascontiguousarray(grid_narrow, np.float32)
        d.acq_grid_narrow = grid_narrow.ctypes.data
        d.num_doppler_bins_step2 = grid_narrow.shape[0]
    d.doppler_max, d.doppler_step, d.positive_acq, d.num_dwells, d.prn = doppler_max, doppler_step, int(positive_acq), num_dwells, prn
    d.acq_doppler_hz, d.acq_delay_samples, d.test_statistic, d.threshold = acq_doppler_hz, acq_delay_samples, test_statistic, threshold
    d.input_power, d.doppler_step_narrow, d.doppler_grid_narrow_min, d.sample_counter = input_power, doppler_step_narrow, doppler_grid_narrow_min, sample_counter
    _chk(lib.b200_acq_dump_write(filename.encode(), C.byref(d)), "b200_acq_dump_write")


def acq_resampler_design(fs_in: int, opt_acq_fs: int) -> tuple:
    """-> (decimation, float32 taps): the acquisition resampler the reference inserts for a stream at fs_in and a signal
    acquired at opt_acq_fs (gnss_flowgraph.cc:1117-1212); (1, no taps) where it inserts none"""
    d, n = C.c_uint32(0), C.c_uint32(0)
    rc = lib.b200_acq_resampler_design(int(fs_in), int(opt_acq_fs), 0, C.byref(d), None, C.byref(n))
    if rc == 0:
        return d.value, np.zeros(0, np.float32)
    if rc != -5:
        _chk(rc, "b200_acq_resampler_design")
    taps = np.zeros(n.value, np.float32)
    _chk(lib.b200_acq_resampler_design(int(fs_in), int(opt_acq_fs), taps.size, C.byref(d), taps.ctypes.data, C.byref(n)),
         "b200_acq_resampler_design")
    return d.value, taps


def iq_conditioner_lowpass(sampling_freq_hz: float, decimation: int, bw_hz: float = 0.0, tw_hz: float = 0.0) -> np.ndarray:
    """float32 taps of the input filter's filter_type = lowpass design (freq_xlating_fir_filter.cc:103-110): firdes::low_pass(1,
    fs, bw, tw), bw = (fs / decimation) / 2 and tw = bw / 10 where not given (<= 0)"""
    n = C.c_uint32(0)
    rc = lib.b200_iq_conditioner_lowpass(float(sampling_freq_hz), int(decimation), float(bw_hz), float(tw_hz), 0, None, C.byref(n))
    if rc != -5:
        _chk(rc, "b200_iq_conditioner_lowpass")
    taps = np.zeros(n.value, np.float32)
    _chk(lib.b200_iq_conditioner_lowpass(float(sampling_freq_hz), int(decimation), float(bw_hz), float(tw_hz), taps.size,
                                         taps.ctypes.data, C.byref(n)), "b200_iq_conditioner_lowpass")
    return taps


def pulse_blanking_threshold(pfa: float, length: int) -> float:
    """the blanker's float threshold (pulse_blanking_cc.cc:57-58): the chi-squared upper quantile with 2 length degrees of
    freedom at the float pfa"""
    t = C.c_float(0.0)
    _chk(lib.b200_iq_pulse_blanking_threshold(float(pfa), int(length), C.byref(t)), "b200_iq_pulse_blanking_threshold")
    return t.value


def acq_dump_filename(base: str, system: str, signal: str, channel: int, dump_number: int, prn: int) -> str:
    buf = C.create_string_buffer(1024)
    _chk(lib.b200_acq_dump_filename(base.encode(), system.encode()[:1], signal.encode(), channel, dump_number, prn, buf, 1024),
         "b200_acq_dump_filename")
    return buf.value.decode()


class AcqFineDoppler:
    """b200_acq_fine: estimate_Doppler() of pcps_acquisition_fine_doppler_cc on the device."""

    def __init__(self, engine: Engine, fft_size: int):
        self.h = _vp()
        self.fft_size = fft_size
        _chk(lib.b200_acq_fine_create(engine.h, fft_size, C.byref(self.h)), "b200_acq_fine_create")

    def estimate(self, buffer_10ms, code_replica):
        """-> (tmp_index_freq, peak)"""
        buf = np.ascontiguousarray(buffer_10ms, np.complex64)
        code = np.ascontiguousarray(code_replica, np.complex64)
        assert buf.size == 10 * self.fft_size and code.size == self.fft_size
        idx, peak = C.c_uint32(0), C.c_float(0)
        _chk(lib.b200_acq_fine_estimate(self.h, buf.ctypes.data, code.ctypes.data, C.byref(idx), C.byref(peak)), "b200_acq_fine_estimate")
        return idx.value, peak.value

    def read_spectrum(self) -> np.ndarray:
        out = np.zeros(80 * self.fft_size, np.float32)
        _chk(lib.b200_acq_fine_read_spectrum(self.h, out.ctypes.data), "b200_acq_fine_read_spectrum")
        return out

    def close(self):
        if self.h:
            lib.b200_acq_fine_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
