"""Stress test of the TMA sample ring of trk_shared_kernel (DESIGN.md 4.2): compute-sanitizer's racecheck flags the slot
reuse (consumer LDS vs the producer's bulk copy into the same slot) as potential WAR hazards because it does not model
ordering through mbarrier arrive / try_wait for async-proxy writes.  This test puts data behind the dismissal: builds of
the library with 2, 4 and 8 ring stages and pseudo-random delays injected into the producer and into every consumer warp
(-DSH_STRESS=1: warps drift apart by whole tiles, every full/empty hand-over happens under contention) must produce, over
thousands of launches, results bitwise equal to the production build's and to the integer-exact oracle."""
import pytest

from gnss_sdr_b200.build import LIB, build_variant
from ring_worker import run_worker

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("stages", [2, 4, 8])
def test_ring_under_injected_delays_is_bitwise_stable(stages):
    """Integer-valued samples and +-1 codes with a zero carrier make every tap an exact integer sum: any sample read from
    a slot the producer had already overwritten (or not yet filled) changes the result.  2000 launches per variant x 120
    groups x ~90 tiles with delays; compared with the production build (4 stages, no delays) on the same input."""
    prod = run_worker(LIB, 3)
    lib = build_variant(stages, stress=True)
    got = run_worker(lib, 2000)
    assert got["bad"] == 0, got
    assert got["sha"] == prod["sha"], (got, prod)
