"""The engine's launch counter (b200_engine_launch_count) grows by exactly the kernels one tracking call issues.

A batch on the per-item kernel is one launch per tap count among the channels with a code table; on the shared-window
kernel it is one launch.  The single correlators are one launch each.  A device-loop run is one launch in mode 0 (the
persistent kernel); in modes 1 and 2 it is one prepare launch, then per epoch the correlator's launches (one per tap
count: a loop with a data channel has 3- or 5-tap pilot items and 1-tap data items) and one loop-cycle launch.
"""
import numpy as np
import pytest

from gpu_fixtures import capi, torch  # noqa: F401
import loop_rig as tl
import trk_rig as tr

pytestmark = pytest.mark.gpu

N = 4000


def batch_engine(capi, taps_list):
    """one band of random samples, one channel per entry of taps_list, one 4000-sample item per channel"""
    rng = np.random.default_rng(len(taps_list))
    e = capi.Engine(0)
    tr.ring(e, 0, (rng.normal(size=1 << 15) + 1j * rng.normal(size=1 << 15)).astype(np.complex64), 1 << 16)
    chans = [tr.channel(e, 0, rng.choice([-1.0, 1.0], 1023), list(np.linspace(-0.5, 0.5, taps))) for taps in taps_list]
    return e, tr.items((ch, N, 100 * i, 0.3, 0.01, 0.0, 0.2, 1.023e6 / 4e6) for i, ch in enumerate(chans))


@pytest.mark.parametrize("taps_list,launches", [
    ([3, 3, 3], 1),        # uniform
    ([5, 1, 5, 1], 2),     # a pilot's 5 taps and its data channel's 1
    ([5, 1, 2], 3),        # a tap count outside 1, 3 and 5
    ([4, 6, 7, 8], 4),
])
def test_per_item_batch_counts_one_launch_per_tap_count(capi, taps_list, launches):
    e, items = batch_engine(capi, taps_list)
    e.trk_kernel_choice(0)
    k0 = e.launch_count()
    e.trk_batch(items, 8)
    assert e.launch_count() - k0 == launches
    e.close()


def test_shared_window_batch_counts_one_launch(capi, torch):
    e, items = batch_engine(capi, [3] * 16)
    e.trk_kernel_choice(1)
    k0 = e.launch_count()
    tr.run_dev(torch, e, items, 8)
    assert e.launch_count() - k0 == 1
    e.close()


def test_single_correlators_count_one_launch_each(capi):
    rng = np.random.default_rng(7)
    e = capi.Engine(0)
    mc = capi.Multicorrelator(e, N, 3)
    sig = (rng.normal(size=N) + 1j * rng.normal(size=N)).astype(np.complex64)
    shifts = [-0.5, 0.0, 0.5]
    mc.set_local_code_and_taps(rng.choice([-1.0, 1.0], 1023).astype(np.float32), shifts)
    mc.set_local_code_and_taps_cplx(rng.choice([-1.0, 1.0], 1023).astype(np.complex64), shifts)
    mc.set_local_code_and_taps_16sc(rng.integers(-1, 2, 2 * 1023).astype(np.int16), shifts)
    k0 = e.launch_count()
    mc.Carrier_wipeoff_multicorrelator_resampler(sig, 0.3, 0.01, 0.0, 0.2, 1.023e6 / 4e6, 0.0)
    assert e.launch_count() - k0 == 1
    mc.correlate_cplx(sig, 0.3, 0.01, 0.2, 1.023e6 / 4e6)
    assert e.launch_count() - k0 == 2
    mc.correlate_16sc(rng.integers(-100, 100, 2 * N).astype(np.int16), 0.3, 0.01, 0.2, 1.023e6 / 4e6)
    assert e.launch_count() - k0 == 3
    mc.free()
    e.close()


@pytest.mark.parametrize("mode,with_data,launches", [
    ("persistent256", True, lambda ep: 1),
    ("per_epoch", False, lambda ep: 1 + ep * 2),
    ("per_epoch", True, lambda ep: 1 + ep * 3),   # pilot items and data items: two correlator launches per epoch
    ("sliced", True, lambda ep: 1 + ep * 3),
])
def test_loop_run_counts_its_launches(capi, mode, with_data, launches):
    n_ep = 5
    sp, dt = tl.pilot_data_spec(5, 25, 1234.0, 1777, n_ep)
    e, ids, _ = tl.make_engine_with_data(capi, [sp], [dt if with_data else None], {0: len(sp.stream.x) + 16})
    tl.set_mode(e, mode, sp)
    tl.push_all(e, [sp])
    tl.start_all(e, ids, [sp])
    k0 = e.launch_count()
    e.loop_run(n_ep)
    assert e.launch_count() - k0 == launches(n_ep)
    e.close()


def test_loop_mode_only_through_the_api(capi, monkeypatch):
    """B200_LOOP_MODE in the environment selects nothing: an engine whose mode was never set runs the persistent kernel,
    one launch per run (mode 1 would issue 1 + 2 per epoch)."""
    n_ep = 5
    monkeypatch.setenv("B200_LOOP_MODE", "1")
    sp, _ = tl.pilot_data_spec(5, 25, 1234.0, 1777, n_ep)
    e, ids, _ = tl.make_engine_with_data(capi, [sp], [None], {0: len(sp.stream.x) + 16})
    tl.push_all(e, [sp])
    tl.start_all(e, ids, [sp])
    k0 = e.launch_count()
    e.loop_run(n_ep)
    assert e.launch_count() - k0 == 1
    e.close()
