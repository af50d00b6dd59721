"""The structures of include/b200gnss.h, stated once for Python: a ctypes class per struct, and for the structs that
travel in arrays the numpy dtype derived from it.  Declarations only: this module never loads libb200gnss.so, so the CPU
oracles (oracle/loop.py) share these layouts on a box without the library, as oracle/port_loop.c shares the header."""
from __future__ import annotations

import ctypes as C

import numpy as np


class TrkItem(C.Structure):
    """b200_trk_item"""
    _fields_ = [("channel", C.c_int32), ("n", C.c_int32), ("sample_index", C.c_uint64),
                ("rem_carrier_phase_rad", C.c_float), ("phase_step_rad", C.c_float), ("phase_rate_step_rad", C.c_float),
                ("rem_code_phase_chips", C.c_float), ("code_phase_step_chips", C.c_float),
                ("code_phase_rate_step_chips", C.c_float)]


class AcqConf(C.Structure):
    """b200_acq_conf"""
    _fields_ = [("fft_size", C.c_uint32), ("effective_fft_size", C.c_uint32), ("consumed_samples", C.c_uint32),
                ("num_doppler_bins", C.c_uint32), ("doppler_max", C.c_int32), ("doppler_step", C.c_int32),
                ("fs_in", C.c_int64), ("samples_per_chip", C.c_uint32), ("code_layout", C.c_uint32),
                ("bit_transition_flag", C.c_int32), ("use_cfar", C.c_int32), ("max_dwells", C.c_uint32),
                ("n_code_slots", C.c_uint32), ("keep_grid", C.c_int32)]


class AcqResult(C.Structure):
    """b200_acq_result"""
    _fields_ = [("index_time", C.c_uint32), ("index_doppler", C.c_uint32), ("doppler", C.c_int32),
                ("test_statistics", C.c_float), ("grid_maximum", C.c_float), ("input_power", C.c_float),
                ("second_peak", C.c_float)]


class TrkLoopConf(C.Structure):
    """b200_trk_loop_conf: Dll_Pll_Conf / dll_pll_veml_tracking members the device loop needs."""
    _fields_ = [
        ("fs_in", C.c_double), ("code_chip_rate", C.c_double), ("signal_carrier_freq", C.c_double),
        ("code_period", C.c_double), ("carrier_lock_th", C.c_double),
        ("code_length_chips", C.c_uint32), ("vector_length", C.c_uint32), ("pull_in_time_s", C.c_uint32),
        ("bit_synchronization_time_limit_s", C.c_uint32), ("prn", C.c_uint32),
        ("code_samples_per_chip", C.c_int32), ("pll_filter_order", C.c_int32), ("dll_filter_order", C.c_int32),
        ("cn0_samples", C.c_int32), ("cn0_min", C.c_int32), ("max_code_lock_fail", C.c_int32),
        ("max_carrier_lock_fail", C.c_int32), ("cn0_smoother_samples", C.c_int32),
        ("carrier_lock_test_smoother_samples", C.c_int32), ("veml", C.c_int32), ("cloop", C.c_int32),
        ("carrier_aiding", C.c_int32), ("enable_fll_pull_in", C.c_int32), ("enable_fll_steady_state", C.c_int32),
        ("pll_bw_hz", C.c_float), ("dll_bw_hz", C.c_float), ("fll_bw_hz", C.c_float),
        ("early_late_space_chips", C.c_float), ("slope", C.c_float), ("y_intercept", C.c_float),
        ("cn0_smoother_alpha", C.c_float), ("carrier_lock_test_smoother_alpha", C.c_float),
    ]


class TrkLoopStatus(C.Structure):
    """b200_trk_loop_status"""
    _fields_ = [
        ("state", C.c_int32), ("loss_of_lock", C.c_int32), ("sample_counter", C.c_uint64), ("epochs", C.c_uint64),
        ("carrier_doppler_hz", C.c_double), ("code_freq_chips", C.c_double), ("rem_code_phase_samples", C.c_double),
        ("acc_carrier_phase_rad", C.c_double), ("CN0_SNV_dB_Hz", C.c_double), ("carrier_lock_test", C.c_double),
    ]


class TrkDumpRecord(C.Structure):
    """b200_trk_dump_record: one epoch of the reference's tracking dump file, unpadded as the header packs it (the u64 at
    offset 28 and the double sit on 4-byte boundaries)."""
    _pack_ = 1
    _fields_ = [
        ("abs_VE", C.c_float), ("abs_E", C.c_float), ("abs_P", C.c_float), ("abs_L", C.c_float), ("abs_VL", C.c_float),
        ("prompt_I", C.c_float), ("prompt_Q", C.c_float), ("PRN_start_sample_count", C.c_uint64),
        ("acc_carrier_phase_rad", C.c_float), ("carrier_doppler_hz", C.c_float), ("carrier_doppler_rate_hz_s", C.c_float),
        ("code_freq_chips", C.c_float), ("code_freq_rate_chips", C.c_float), ("carr_error_hz", C.c_float),
        ("carr_error_filt_hz", C.c_float), ("code_error_chips", C.c_float), ("code_error_filt_chips", C.c_float),
        ("CN0_SNV_dB_Hz", C.c_float), ("carrier_lock_test", C.c_float), ("aux1", C.c_float), ("aux2", C.c_double),
        ("PRN", C.c_uint32), ("TOW_ms", C.c_uint64), ("WN", C.c_uint32),
    ]


class AcqDump(C.Structure):
    """b200_acq_dump"""
    _fields_ = [("acq_grid", C.c_void_p), ("acq_grid_narrow", C.c_void_p), ("effective_fft_size", C.c_uint32),
                ("num_doppler_bins", C.c_uint32), ("num_doppler_bins_step2", C.c_uint32), ("doppler_max", C.c_int32),
                ("doppler_step", C.c_int32), ("positive_acq", C.c_int32), ("num_dwells", C.c_int32), ("prn", C.c_uint32),
                ("acq_doppler_hz", C.c_float), ("acq_delay_samples", C.c_float), ("test_statistic", C.c_float),
                ("threshold", C.c_float), ("input_power", C.c_float), ("doppler_step_narrow", C.c_float),
                ("doppler_grid_narrow_min", C.c_float), ("sample_counter", C.c_uint64)]


TRK_ITEM_DTYPE = np.dtype(TrkItem)
ACQ_RESULT_DTYPE = np.dtype(AcqResult)
TRK_DUMP_RECORD_DTYPE = np.dtype(TrkDumpRecord)

assert C.sizeof(TrkItem) == TRK_ITEM_DTYPE.itemsize == 40
assert C.sizeof(AcqConf) == 64
assert C.sizeof(AcqResult) == ACQ_RESULT_DTYPE.itemsize == 28
assert C.sizeof(TrkLoopConf) == 152
assert C.sizeof(TrkLoopStatus) == 72
assert C.sizeof(TrkDumpRecord) == TRK_DUMP_RECORD_DTYPE.itemsize == 108
