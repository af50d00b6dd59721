"""Stress test of the TMA sample ring of trk_shared_kernel (DESIGN.md 4.2): compute-sanitizer's racecheck flags the slot
reuse (consumer LDS vs the producer's bulk copy into the same slot) as potential WAR hazards because it does not model
ordering through mbarrier arrive / try_wait for async-proxy writes.  This test puts data behind the dismissal: builds of
the library with 2, 4 and 8 ring stages and pseudo-random delays injected into the producer and into every consumer warp
(-DSH_STRESS=1: warps drift apart by whole tiles, every full/empty hand-over happens under contention) must produce, over
thousands of launches, results bitwise equal to the production build's and to the integer-exact oracle."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

WORKER = r'''
import json, os, sys
import numpy as np
sys.path.insert(0, os.environ["B200_ROOT"]); sys.path.insert(0, os.path.join(os.environ["B200_ROOT"], "tests"))
import gnss_sdr_b200.capi as capi
launches = int(sys.argv[1])
rng = np.random.default_rng(99)
n_ch, n, n_ep = 24, 6000, 40
eng = capi.Engine(0)
iq = (rng.integers(-40, 40, n * n_ep + 7000) + 1j * rng.integers(-40, 40, n * n_ep + 7000)).astype(np.complex64)
eng.iq_create(0, 1 << 19)
eng.iq_push(0, iq)
items = []
for c in range(n_ch):
    code = np.where(rng.integers(0, 2, 1023) > 0, 1.0, -1.0).astype(np.float32)
    cid = eng.channel_create(0, 3)
    eng.channel_set_code(cid, code, [-0.5, 0.0, 0.5])
    off = int(rng.integers(0, 5000))            # staggered epochs: the hull of a group spans several extra tiles
    step = 1023.0 / n * (1.0 + rng.uniform(-1e-5, 1e-5))
    for k in range(n_ep):
        items.append((cid, n, off + k * n, 0.0, 0.0, 0.0, float(rng.uniform(0, 1)), step, 0.0))
items = np.array(items, dtype=capi.TRK_ITEM_DTYPE)
items = items[np.argsort(items["sample_index"], kind="stable")]
eng.trk_kernel_choice(1)                        # 960 items: below the automatic choice's 1024
first = None
bad = 0
for it in range(launches):
    out = eng.trk_batch(items, 3)
    if first is None:
        first = out.copy()
    elif out.tobytes() != first.tobytes():
        bad += 1
eng.close()
import hashlib
print("RESULT " + json.dumps({"bad": bad, "launches": launches, "sha": hashlib.sha256(first.tobytes()).hexdigest(),
                              "sum": [float(np.sum(first.real)), float(np.sum(first.imag))]}))
'''


def _source_hash():
    import glob
    import hashlib
    h = hashlib.sha1()
    for pat in ("gnss_sdr_b200/csrc/*", "include/*.h"):
        for f in sorted(glob.glob(os.path.join(ROOT, pat))):
            h.update(os.path.basename(f).encode())
            with open(f, "rb") as fh:
                h.update(fh.read())
    return h.hexdigest()


def build_variant(stages, stress):
    """Same sources as the production library with -DSH_STAGES / -DSH_STRESS.  Staleness is decided on a hash of the sources
    (kept beside the .so), not on file times: a snapshot copied to another machine keeps contents, not necessarily mtimes."""
    from gnss_sdr_b200 import build as b
    os.makedirs(os.path.join(ROOT, "gnss_sdr_b200", "variants"), exist_ok=True)
    out = os.path.join(ROOT, "gnss_sdr_b200", "variants", f"libb200gnss_ring{stages}_{'stress' if stress else 'plain'}.so")
    want = _source_hash()
    stamp = out + ".srchash"
    have = open(stamp).read().strip() if os.path.exists(stamp) else ""
    if not os.path.exists(out) or have != want:
        b.build(extra=[f"-DSH_STAGES={stages}", f"-DSH_STRESS={1 if stress else 0}"], out=out)
        with open(stamp, "w") as fh:
            fh.write(want)
    return out


def run_worker(lib, launches, tmp_path):
    script = tmp_path / "ring_worker.py"
    script.write_text(WORKER)
    env = dict(os.environ, B200_ROOT=ROOT, B200_LIB=lib)
    r = subprocess.run([sys.executable, str(script), str(launches)], env=env, capture_output=True, text=True, timeout=1500)
    assert r.returncode == 0, r.stdout + r.stderr
    line = [ln for ln in r.stdout.splitlines() if ln.startswith("RESULT ")][0]
    return json.loads(line[len("RESULT "):])


@pytest.mark.parametrize("stages", [2, 4, 8])
def test_ring_under_injected_delays_is_bitwise_stable(stages, tmp_path):
    """Integer-valued samples and +-1 codes with a zero carrier make every tap an exact integer sum: any sample read from
    a slot the producer had already overwritten (or not yet filled) changes the result.  2000 launches per variant x 120
    groups x ~90 tiles with delays; compared with the production build (4 stages, no delays) on the same input."""
    prod = run_worker(os.path.join(ROOT, "gnss_sdr_b200", "libb200gnss.so"), 3, tmp_path)
    lib = build_variant(stages, stress=True)
    got = run_worker(lib, 2000, tmp_path)
    assert got["bad"] == 0, got
    assert got["sha"] == prod["sha"], (got, prod)
