"""gnss_sdr_b200 -- H100 (sm_90a) implementation of gnss-sdr's tracking-correlator and PCPS
acquisition hot paths behind a C ABI (include/b200gnss.h, libb200gnss.so).

This package is only the thin Python face of that library (ctypes) used by tests and bench.py;
the product is the CUDA library and the C++ host mirror in gnss_sdr_b200/host/.
There is NO CPU fallback: importing `gnss_sdr_b200.capi` raises if libb200gnss.so is missing.
"""
__version__ = "0.1.0"
