"""The device loops' sample window on an attached band is [valid_from, write_index), the window b200_iq_window reports.

b200_iq_refill with fewer samples than the attached buffer holds moves write_index to first_index + n; the buffer's slots
past it still hold the previous fill.  A loop must track the refilled samples exactly and stall where they end, never
correlating what the buffer held before.  Helpers and configurations are those of test_loop_correlator_gpu.py, from
tests/loop_rig.py."""
import numpy as np
import pytest

from gpu_fixtures import capi  # noqa: F401
import loop_rig as tl
from oracle import loop as ol

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("mode", list(tl.MODES))
def test_loops_stall_past_a_partial_refill(capi, mode):
    """A device buffer of 60_000 samples attached at 2_000_000 and filled with stream A, then b200_iq_refill of B[:30_000] at
    the same index.  A loop started at 2_000_000 tracks B exactly for the epochs inside the refill, then stalls (no record,
    sample counter frozen); a loop on another band is unaffected."""
    import torch
    rng = np.random.default_rng(8)
    x0 = 2_000_000
    _, a = tl.gps_stream(rng, 14, x0, 60_000)
    code, b = tl.gps_stream(rng, 3, x0, 30_000)
    loop = tl.LoopSpec(0, code, ol.default_conf(fs_in=tl.FS, prn=3), (tl.DELAY + 0.3, 0.0, x0, x0), b)
    oth = tl.other_band(rng, 16)
    e, ids = tl.window_engine(capi, mode, [loop, oth], {1: len(oth.stream.x) + 16})
    buf = torch.zeros(2 * len(a.x), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    e.iq_attach_dev(0, buf.data_ptr(), len(a.x), x0)
    ax, bx = a.x.astype(np.complex64), b.x.astype(np.complex64)
    e.iq_refill_ptr(0, ax.ctypes.data, ax.size, x0)
    e.iq_refill_ptr(0, bx.ctypes.data, bx.size, x0)
    tl.push_all(e, [oth])
    assert e.iq_window(0) == (x0, x0 + bx.size)
    tl.start_all(e, ids, [loop, oth])
    first = tl.run_per_epoch(e, ids, 12)
    tl.check_loop(loop, first[0], 6, "inside the refill")
    frozen = e.loop_status(ids[0]).sample_counter
    assert frozen + loop.conf.vector_length > x0 + bx.size, frozen
    more = tl.run_per_epoch(e, ids, 4)
    s = e.loop_status(ids[0])
    assert len(more[0][1]) == 0 and s.sample_counter == frozen and s.state == 2, (len(more[0][1]), s.sample_counter)
    tl.check_loop(oth, (np.concatenate([first[1][0], more[1][0]]), np.concatenate([first[1][1], more[1][1]])), 16, "other band")
    e.close()
    del buf
