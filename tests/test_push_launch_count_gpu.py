"""The engine's launch counter (b200_engine_launch_count) across the sample writes into a band.

Float samples are copied into the band without a kernel (b200_iq_push, b200_iq_push_at, b200_iq_refill); integer samples
are converted on the device, one launch per non-empty int16 or int8 block, so b200_iq_push_file with "ishort" is one
launch per chunk.  The tracking calls' counts are in test_trk_launch_count_gpu.py."""
import numpy as np
import pytest

from gpu_fixtures import capi  # noqa: F401

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("kind,launches", [
    ("cf32", 0),
    ("push_at", 0),
    ("refill", 0),
    ("i16", 1),
    ("i8", 1),
    ("i16_empty", 0),
    ("file_ishort", 3),   # 3000 samples in chunks of 1000
])
def test_sample_pushes_count_their_conversions(capi, tmp_path, kind, launches):
    rng = np.random.default_rng(11)
    n = 3000
    iq = rng.integers(-100, 100, 2 * n)
    x = (iq[0::2] + 1j * iq[1::2]).astype(np.complex64)
    e = capi.Engine(0)
    if kind == "refill":
        import torch
        buf = torch.zeros(2 * n, dtype=torch.float32, device="cuda")
        torch.cuda.synchronize()
        e.iq_attach_dev(0, buf.data_ptr(), n)
    else:
        e.iq_create(0, 1 << 14)
    k0 = e.launch_count()
    if kind == "cf32":
        e.iq_push(0, x)
    elif kind == "push_at":
        assert e.iq_push_at(0, 0, x) == n
    elif kind == "refill":
        e.iq_refill_ptr(0, x.ctypes.data, n)
    elif kind == "i16_empty":
        e.iq_push_int(0, iq[:0].astype(np.int16))
    elif kind in ("i16", "i8"):
        e.iq_push_int(0, iq.astype(np.int16 if kind == "i16" else np.int8))
    else:
        path = tmp_path / "iq.bin"
        iq.astype(np.int16).tofile(path)
        assert e.iq_push_file(0, str(path), "ishort", chunk_samples=1000) == (0, n)
    e.sync()
    assert e.launch_count() - k0 == launches
    assert e.iq_window(0) == (0, 0 if kind == "i16_empty" else n)
    e.close()
