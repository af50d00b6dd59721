#!/usr/bin/env python
"""CUDA-event timing of the acquisition options at a chirp-z size (16.368 Msps, N with prime factors 11 and 31), one JSON
line each:

  bit_transition_sweep  32 PRNs x 40 Doppler bins, bit_transition_flag (N = 32 736, M = 65 536), input on the device
                        (b200_acq_search_dev);
  plain_sweep           the same sweep without bit transition (N = 16 368, M = 32 768), for scale;
  step_two              one PRN, 4 bins of 125 Hz (N = 16 368), through b200_acq_search_step_two: host input, so the
                        time includes the 131 kB copy up, the result copy down and the host synchronisation.

usage: python tools/acq_chirpz_modes_time.py [--reps 20]
"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

FS, N1, PRNS, DMAX, DSTEP = 16_368_000, 16368, 32, 5000, 250


def time_ms(torch, fn, reps, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    c0, c1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    c0.record()
    for _ in range(reps):
        fn()
    c1.record()
    torch.cuda.synchronize()
    return c0.elapsed_time(c1) / reps


def sweep(torch, capi, eng, dev, reps, bit_transition):
    from gnss_synth import gps_ca_code_complex_sampled
    acq = capi.PcpsAcquisition(eng, fs_in=FS, samples_per_ms=float(N1), samples_per_chip=16, doppler_max=DMAX, doppler_step=DSTEP,
                               n_code_slots=PRNS, bit_transition_flag=bit_transition)
    for p in range(1, PRNS + 1):
        code = gps_ca_code_complex_sampled(p, FS)
        acq.set_local_code(p - 1, np.tile(code, 2) if bit_transition else code)
    slots = np.arange(PRNS, dtype=np.uint32)
    x = torch.randn((acq.conf.consumed_samples, 2), device=dev, dtype=torch.float32)
    res = torch.zeros(PRNS * capi.ACQ_RESULT_DTYPE.itemsize, dtype=torch.uint8, device=dev)
    ms = time_ms(torch, lambda: acq.search_dev(x.data_ptr(), slots, res.data_ptr()), reps)
    out = {"workload": f"{PRNS} PRNs x {acq.conf.num_doppler_bins} bins, N={acq.conf.fft_size}, effective {acq.conf.effective_fft_size}",
           "ms_per_sweep": ms, "acquisitions_per_s": PRNS / (ms * 1e-3)}
    acq.close()
    return out


def step_two(torch, capi, eng, reps):
    from gnss_synth import gps_ca_code_complex_sampled
    acq = capi.PcpsAcquisition(eng, fs_in=FS, samples_per_ms=float(N1), samples_per_chip=16, doppler_max=DMAX, doppler_step=500)
    acq.set_local_code(0, gps_ca_code_complex_sampled(1, FS))
    acq.set_step_two(1500.0, 125.0, 4)
    rng = np.random.default_rng(1)
    iq = (rng.standard_normal(N1) + 1j * rng.standard_normal(N1)).astype(np.complex64)
    ms = time_ms(torch, lambda: acq.search_step_two(iq, 0, 1.0), reps)
    out = {"workload": f"1 PRN x 4 bins (125 Hz), N={acq.conf.fft_size}, host input", "ms_per_search": ms}
    acq.close()
    return out


if __name__ == "__main__":
    import torch
    import gnss_sdr_b200.capi as capi
    reps = int(sys.argv[sys.argv.index("--reps") + 1]) if "--reps" in sys.argv else 20
    dev = torch.device("cuda", 0)
    st = torch.cuda.Stream(device=dev)
    torch.cuda.set_stream(st)
    eng = capi.Engine(0, st.cuda_stream)
    print(json.dumps({"gpu": torch.cuda.get_device_name(dev)}), flush=True)
    print(json.dumps({"bit_transition_sweep": sweep(torch, capi, eng, dev, reps, True)}), flush=True)
    print(json.dumps({"plain_sweep": sweep(torch, capi, eng, dev, reps, False)}), flush=True)
    print(json.dumps({"step_two": step_two(torch, capi, eng, reps)}), flush=True)
    eng.close()
