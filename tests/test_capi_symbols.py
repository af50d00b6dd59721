"""The C-ABI library loads on a CPU-only box and exports every symbol include/b200gnss.h declares
(no compute calls without a GPU).  Also: the product path has no CPU fallback."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    src = open(os.path.join(ROOT, "include", "b200gnss.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(b200_[a-z0-9_]+)\s*\(", src)))


def test_header_symbols_are_exported():
    import gnss_sdr_b200.capi as capi
    names = declared_symbols()
    assert len(names) >= 28
    lib = ctypes.CDLL(capi.LIB_PATH)
    missing = [n for n in names if not hasattr(lib, n)]
    assert not missing, missing
    # and the ctypes binding knows each of them
    known = set(capi.exported_symbols())
    assert set(names) <= known, sorted(set(names) - known)


def test_struct_layouts_match_header():
    import gnss_sdr_b200.capi as capi
    assert ctypes.sizeof(capi.TrkItem) == 40
    assert ctypes.sizeof(capi.AcqResult) == 28
    assert ctypes.sizeof(capi.AcqConf) == 64
    assert ctypes.sizeof(capi.TrkLoopConf) == 152
    assert ctypes.sizeof(capi.TrkLoopStatus) == 72
    assert ctypes.sizeof(capi.TrkDumpRecord) == capi.TRK_DUMP_RECORD_DTYPE.itemsize == 108


def test_no_gpu_means_loud_failure_not_fallback():
    import torch
    import gnss_sdr_b200.capi as capi
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    assert capi.device_count() == 0
    with pytest.raises(capi.B200Error) as ei:
        capi.Engine(0)
    assert ei.value.code == -6   # B200_ERR_NODEV


def test_product_never_imports_oracle():
    pkg = os.path.join(ROOT, "gnss_sdr_b200")
    offenders = []
    for dp, _, files in os.walk(pkg):
        if "build" in dp.split(os.sep):
            continue
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".cc", ".h")):
                txt = open(os.path.join(dp, f)).read()
                if re.search(r"^\s*(import|from)\s+oracle\b", txt, flags=re.M) and f != "acq_smoke.py":
                    offenders.append(os.path.join(dp, f))
                if "liboracle" in txt:
                    offenders.append(os.path.join(dp, f))
    assert not offenders, offenders
