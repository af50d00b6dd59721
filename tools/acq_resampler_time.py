#!/usr/bin/env python
"""CUDA-event timing of acquisition band searches at the full rate against the same searches through the acquisition
resampler (b200_acq_set_band_resampler), legs alternating in one run, one JSON line per leg:

  c4_full   32 PRNs x 81 Doppler bins, 1 ms of GPS L1 C/A from a 25 Msps band: N = 25 000 points per row;
  c4_dec    the same sweep decimated by 10 (49 taps) to 2.5 Msps: N = 2 500, plus one filter launch;
  e4_full   one PRN x 81 bins, 4 ms of GPS L1 C/A from a 50 Msps band: N = 200 000 points on the two-level plan;
  e4_dec    the same search decimated by 25 (121 taps) to 2 Msps: N = 8 000;
  filter    the decimation kernel alone, per search, from torch.profiler in a separate pass (c4_dec and e4_dec).

Each sample is one search: a CUDA event before its first launch and one after the result copy down, on the search's
stream.  The first line reports the card, its power limit and SM clock, read in the same run.  The decimated sweeps are
also checked to find the satellites the full-rate sweeps find (PRN, and Doppler within a bin).

usage: python tools/acq_resampler_time.py [--rounds 30]
"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from acq_band_time import card  # noqa: E402  (same directory)

DMAX, DSTEP = 10125, 250


def main(rounds):
    import torch
    import gnss_sdr_b200.capi as capi
    from gnss_synth import gps_ca_code, gps_ca_code_complex_sampled, make_iq
    dev = torch.device("cuda", 0)
    st = torch.cuda.Stream(device=dev)
    torch.cuda.set_stream(st)
    eng = capi.Engine(0, st.cuda_stream)  # the searches run on torch's stream, so torch's events bracket them
    print(json.dumps({"gpu": torch.cuda.get_device_name(dev), **card()}), flush=True)

    rng = np.random.default_rng(4)
    present = [2, 5, 9, 13, 17, 21, 26, 30]
    svs = [dict(prn=p, doppler=float(rng.uniform(-9000, 9000)), code_phase_chips=float(rng.uniform(0, 1023)), cn0=45.0) for p in present]
    legs, checks = {}, {}

    def leg(name, band, fs, ms, prns, decimate):
        d, taps = capi.acq_resampler_design(fs, 2_000_000) if decimate else (1, np.zeros(0, np.float32))
        fa = fs // d
        acq = capi.PcpsAcquisition(eng, fs_in=fa, samples_per_ms=fa / 1000.0, samples_per_chip=max(1, fa // 1_023_000),
                                   doppler_max=DMAX, doppler_step=DSTEP, sampled_ms=ms, ms_per_code=ms, n_code_slots=len(prns))
        for s, p in enumerate(prns):
            acq.set_local_code(s, np.tile(gps_ca_code_complex_sampled(p, fa), ms))
        if decimate:
            acq.set_band_resampler(d, taps)
        slots = np.arange(len(prns), dtype=np.uint32)
        legs[name] = (acq, lambda: acq.search_band_submit(band, 1000, slots))
        checks[name] = (acq, prns)

    for band, fs, ms, prns in ((0, 25_000_000, 1, list(range(1, 33))), (1, 50_000_000, 4, [present[0]])):
        n = 1000 + ms * (fs // 1000) + 1000
        eng.iq_create(band, 1 << (n - 1).bit_length())
        eng.iq_push(band, make_iq({p: gps_ca_code(p) for p in present}, float(fs), n, svs, seed=band))
        tag = "c4" if band == 0 else "e4"
        leg(f"{tag}_full", band, fs, ms, prns, False)
        leg(f"{tag}_dec", band, fs, ms, prns, True)
    torch.cuda.synchronize()

    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    times = {m: [] for m in legs}
    results = {}
    names = list(legs)
    for r in range(rounds + 3):                 # 3 warm-up rounds
        order = names[r % len(names):] + names[:r % len(names)]
        for m in order:
            acq, submit = legs[m]
            e0.record()
            submit()
            e1.record()
            results[m] = acq.search_wait()
            e1.synchronize()
            if r >= 3:
                times[m].append(e0.elapsed_time(e1))
    for m, t in times.items():
        t = np.array(t)
        c = legs[m][0].conf
        print(json.dumps({m: {"fft_size": int(c.fft_size), "bins": int(c.num_doppler_bins), "slots": int(c.n_code_slots),
                              "ms_median": float(np.median(t)), "ms_min": float(t.min()), "ms_p10": float(np.percentile(t, 10)),
                              "ms_p90": float(np.percentile(t, 90)), "sweeps": int(t.size)}}), flush=True)

    # the filter kernel alone: its device time per search, from the profiler's kernel records
    from torch.profiler import ProfilerActivity, profile
    filt = {}
    for m in ("c4_dec", "e4_dec"):
        acq, submit = legs[m]
        k = 20
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(k):
                submit()
                acq.search_wait()
            torch.cuda.synchronize()
        us = [ev.device_time_total for ev in prof.key_averages() if "acq_decimate_kernel" in ev.key]
        filt[m] = {"filter_us_per_search": float(sum(us)) / k if us else None}
    print(json.dumps({"filter": filt}), flush=True)

    found = {}
    for m, (acq, prns) in checks.items():
        res = results[m]
        best = int(np.argmax(res["test_statistics"]))
        found[m] = (prns[best], int(res[best]["doppler"]))
    same = all(found[f"{t}_full"][0] == found[f"{t}_dec"][0] and abs(found[f"{t}_full"][1] - found[f"{t}_dec"][1]) <= DSTEP
               for t in ("c4", "e4"))
    print(json.dumps({"strongest": found, "decimated_finds_the_same": bool(same), "after": card()}), flush=True)
    for acq, _ in legs.values():
        acq.close()
    eng.close()
    return 0 if same else 1


if __name__ == "__main__":
    sys.exit(main(int(sys.argv[sys.argv.index("--rounds") + 1]) if "--rounds" in sys.argv else 30))
