"""Build recipe of the C++ host program tests/host/test_host_mirror.cc, linked against libb200gnss.so and the C++ host
mirror (gnss_sdr_b200/host/), and against the reference's correlator where oracle/_ref has it."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "tests", "host", "test_host_mirror")


def build(exe=EXE):
    """the host program, by default into tests/host/ where bench.py runs it; the tests build their own copy under tmp_path,
    so that they also run from a read-only tree"""
    libdir = os.path.join(ROOT, "gnss_sdr_b200")
    ref = os.path.join(ROOT, "oracle", "_ref", "liboracle_ref.so")
    cmd = ["g++", "-std=c++20", "-O2", os.path.join(ROOT, "tests", "host", "test_host_mirror.cc"),
           os.path.join(libdir, "host", "b200_multicorrelator_real_codes.cc"),
           os.path.join(libdir, "host", "b200_trk_coalescer.cc"),
           os.path.join(libdir, "host", "b200_multicorrelator_variants.cc"),
           os.path.join(libdir, "host", "b200_pcps_acquisition_core.cc"),
           os.path.join(libdir, "host", "b200_pcps_acquisition_fine_doppler_core.cc"),
           os.path.join(libdir, "host", "b200_dll_pll_veml_loop.cc"),
           "-I" + os.path.join(ROOT, "include"), "-I" + os.path.join(libdir, "host"),
           "-L" + libdir, "-lb200gnss", "-Wl,-rpath," + libdir, "-lpthread", "-o", str(exe)]
    if os.path.exists(ref):
        cmd += ["-DHAVE_REF", ref, "-Wl,-rpath," + os.path.dirname(ref)]
    subprocess.check_call(cmd)
    return str(exe)
