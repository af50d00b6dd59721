"""The engine's launch counter (b200_engine_launch_count) grows by exactly the kernels one acquisition search issues, for
single-level and two-level mixed-radix plans.

A single-level plan (fft_size <= 27 648) runs 1 forward + 1 correlation + 1 statistics kernel; without CFAR, + 1
second-peak pass + 1 finish.  A two-level plan runs 2 forward kernels (global radix-n1 stage, in-shared-memory blocks) and
3 correlation kernels (blocks, final radix-n1 stage, row reduction) + 1 statistics; without CFAR the second-peak pass is
one kernel over the stored grid row when there is a grid, else the same 3 kernels again, + 1 finish.  Chirp-z counts are
checked in test_acq_chirpz_modes_gpu.py.
"""
import numpy as np
import pytest

import acq_rig as ar
from gpu_fixtures import capi, engine  # noqa: F401

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("fs,sampled_ms,cfar,keep_grid,launches", [
    (4e6, 1, True, False, 3),      # N = 4000, single level
    (4e6, 1, False, True, 5),      # N = 4000, single level, first/second peak
    (50e6, 1, True, False, 6),     # N = 50000 = 2 x 25000
    (8e6, 7, True, False, 6),      # N = 56000 = 4 x 14000 (56000 / 2 = 28000 exceeds 27648)
    (50e6, 4, False, True, 8),     # N = 200000 = 8 x 25000, second peak from the stored grid row
    (50e6, 1, False, False, 10),   # N = 50000, no grid: the second-peak row is recomputed
])
def test_search_counts_the_kernels_it_issues(capi, engine, fs, sampled_ms, cfar, keep_grid, launches):
    acq = ar.make(capi, engine, fs, doppler_max=1000, doppler_step=500, use_CFAR_algorithm_flag=cfar, sampled_ms=sampled_ms,
                  ms_per_code=sampled_ms, keep_grid=keep_grid)
    n = acq.conf.fft_size
    assert n == int(fs / 1000.0) * sampled_ms
    rng = np.random.default_rng(n)
    acq.set_local_code(0, rng.choice([-1.0, 1.0], n).astype(np.complex64))
    iq = (rng.normal(size=n) + 1j * rng.normal(size=n)).astype(np.complex64)
    k0 = engine.launch_count()
    acq.search(iq, [0])
    assert engine.launch_count() - k0 == launches
    acq.close()
