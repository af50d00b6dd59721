#!/usr/bin/env python
"""CUDA-event timing of the C4 acquisition sweep (GPS L1 C/A, 32 PRNs x 81 Doppler bins x N = 25 000 at 25 Msps, CFAR)
from three places the samples can be, alternating in one run, one JSON line per mode:

  host  b200_acq_search_submit / _wait: the 200 kB window crosses PCIe first (pinned staging, H2D on the search's stream);
  band  b200_acq_search_band_submit / _wait: the window is read where it lies in a device IQ band (here it wraps around
        the ring's end, so the forward stage reads two runs);
  dev   b200_acq_search_dev from a linear device buffer, then the same 896-byte copy of the results into pinned host
        memory that the other two modes make.

Each sample is one sweep: a CUDA event before its first launch and one after its last operation on the search's stream
(the result copy down), so the times are device time, without the host wake-up after the wait.  All three modes run the
same kernels; band and dev differ only in where the forward stage loads its input.  The first line
reports the card, its power limit and SM clock, read in the same run; the three result tables are checked equal.

usage: python tools/acq_band_time.py [--rounds 40]
"""
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

FS, N, PRNS, DMAX, DSTEP = 25_000_000, 25000, 32, 10125, 250


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                             timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        out = f"nvidia-smi unavailable: {e}"
    return dict(zip(q.split(","), [s.strip() for s in out.split(",")])) if out.count(",") == 3 else {"nvidia-smi": out}


def main(rounds):
    import torch
    import gnss_sdr_b200.capi as capi
    from gnss_synth import gps_ca_code, gps_ca_code_complex_sampled, make_iq
    dev = torch.device("cuda", 0)
    st = torch.cuda.Stream(device=dev)
    torch.cuda.set_stream(st)
    eng = capi.Engine(0, st.cuda_stream)  # the search runs on torch's stream, so torch's events bracket it
    print(json.dumps({"gpu": torch.cuda.get_device_name(dev), **card()}), flush=True)

    rng = np.random.default_rng(4)
    present = [2, 5, 9, 13, 17, 21, 26, 30]
    svs = [dict(prn=p, doppler=float(rng.uniform(-9000, 9000)), code_phase_chips=float(rng.uniform(0, 1023)), cn0=45.0) for p in present]
    iq = make_iq({p: gps_ca_code(p) for p in present}, float(FS), 2 * N, svs, seed=4)
    acq = capi.PcpsAcquisition(eng, fs_in=FS, samples_per_ms=float(N), samples_per_chip=24, doppler_max=DMAX, doppler_step=DSTEP,
                               n_code_slots=PRNS)
    for p in range(1, PRNS + 1):
        acq.set_local_code(p - 1, gps_ca_code_complex_sampled(p, FS))
    slots = np.arange(PRNS, dtype=np.uint32)
    cap = 32768
    eng.iq_create(0, cap)
    eng.iq_push(0, iq[:N])
    eng.iq_push(0, iq[N:])
    idx = 20000                                  # [20 000, 45 000) wraps around the ring's end at 32 768
    window = iq[idx:idx + N].copy()
    x_dev = torch.from_numpy(window.view(np.float32)).to(dev)
    res_dev = torch.zeros(PRNS * capi.ACQ_RESULT_DTYPE.itemsize, dtype=torch.uint8, device=dev)
    res_pin = torch.zeros(res_dev.numel(), dtype=torch.uint8).pin_memory()
    torch.cuda.synchronize()

    out = {}

    def host():
        acq.search_submit(window, slots)
        e1.record()
        out["host"] = acq.search_wait()

    def band():
        acq.search_band_submit(0, idx, slots)
        e1.record()
        out["band"] = acq.search_wait()

    def dev_():
        acq.search_dev(x_dev.data_ptr(), slots, res_dev.data_ptr())
        res_pin.copy_(res_dev, non_blocking=True)
        e1.record()

    modes = {"host": host, "band": band, "dev": dev_}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    times = {m: [] for m in modes}
    for r in range(rounds + 3):                 # 3 warm-up rounds
        names = list(modes)
        names = names[r % 3:] + names[:r % 3]   # rotate the order: no mode always runs first
        for m in names:
            e0.record()
            modes[m]()
            e1.synchronize()
            if r >= 3:
                times[m].append(e0.elapsed_time(e1))
    torch.cuda.synchronize()
    out["dev"] = np.frombuffer(res_pin.numpy().tobytes(), capi.ACQ_RESULT_DTYPE)
    same = out["host"].tobytes() == out["band"].tobytes() == out["dev"].tobytes()
    for m, t in times.items():
        t = np.array(t)
        print(json.dumps({m: {"ms_median": float(np.median(t)), "ms_min": float(t.min()), "ms_p10": float(np.percentile(t, 10)),
                              "ms_p90": float(np.percentile(t, 90)), "ms_max": float(t.max()), "sweeps": int(t.size)}}), flush=True)
    print(json.dumps({"workload": f"C4: {PRNS} PRNs x {acq.conf.num_doppler_bins} bins x N={N} (25 Msps, 1 ms), CFAR",
                      "results_identical": bool(same), "after": card()}), flush=True)
    acq.close()
    eng.close()
    return 0 if same else 1


if __name__ == "__main__":
    sys.exit(main(int(sys.argv[sys.argv.index("--rounds") + 1]) if "--rounds" in sys.argv else 40))
