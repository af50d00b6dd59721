"""The worker of the TMA sample-ring stress tests (test_ring_stress_gpu.py, test_trk_shared_chunks_gpu.py).

run_worker(lib, launches, step) runs this file in a fresh process with B200_LIB = lib, so each build of the library loads
into its own process: 24 channels x 40 epochs of 6000 integer-valued samples with +-1 codes and a zero carrier (every tap
an exact integer sum), as one 960-item batch on the shared-window kernel, `launches` times.  It reports how many launches
differed from the first and the SHA-256 of the first.  `step` is the code step in chips per sample (each channel's
differs from it by up to 1e-5 relative): about 0.17 runs warp_tile only, a C2-like 0.041 the chunk path."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N = 6000
STEP = 1023.0 / N


def work(launches, step):
    import hashlib

    import numpy as np

    import gnss_sdr_b200.capi as capi
    rng = np.random.default_rng(99)
    n_ch, n, n_ep = 24, N, 40
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
        st = step * (1.0 + rng.uniform(-1e-5, 1e-5))
        for k in range(n_ep):
            items.append((cid, n, off + k * n, 0.0, 0.0, 0.0, float(rng.uniform(0, 1)), st, 0.0))
    items = np.array(items, dtype=capi.TRK_ITEM_DTYPE)
    items = items[np.argsort(items["sample_index"], kind="stable")]
    eng.trk_kernel_choice(1)                        # 960 items: below the automatic choice's 1024
    first = None
    bad = 0
    for _ in range(launches):
        out = eng.trk_batch(items, 3)
        if first is None:
            first = out.copy()
        elif out.tobytes() != first.tobytes():
            bad += 1
    eng.close()
    print("RESULT " + json.dumps({"bad": bad, "launches": launches, "sha": hashlib.sha256(first.tobytes()).hexdigest(),
                                  "sum": [float(np.sum(first.real)), float(np.sum(first.imag))]}))


def run_worker(lib, launches, step=STEP):
    env = dict(os.environ, B200_LIB=lib)
    r = subprocess.run([sys.executable, os.path.abspath(__file__), str(launches), repr(float(step))], env=env,
                       capture_output=True, text=True, timeout=1500)
    assert r.returncode == 0, r.stdout + r.stderr
    line = [ln for ln in r.stdout.splitlines() if ln.startswith("RESULT ")][0]
    return json.loads(line[len("RESULT "):])


if __name__ == "__main__":
    sys.path.insert(0, ROOT)
    work(int(sys.argv[1]), float(sys.argv[2]))
