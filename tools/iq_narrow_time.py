#!/usr/bin/env python
"""CUDA-event timing of gr_complex, ishort and ibyte IQ bands (b200_iq_create_typed), the band types alternating in one run.
One JSON line per measurement; the first line reports the card, its power limit and SM clock, read in the same run.

  distinct   bench.py's C2_distinct_iq shape: 32 channels x 25 Msps x 0.5 s, every (channel, epoch) reading its own 25 000
             samples of an owned ring of 2^29 samples (4.3 / 2.1 / 1.1 GB), per-item kernel.  Msamples/s, and the
             algorithmic bytes/s at 8 / 4 / 2 B per channel-sample as a fraction of the H100 SXM data sheet's 3.35 TB/s.
  c2_item    the C2 shared layout (32 channels on one 25 Msps x 1 s stream, epoch-major, the stream L2-resident per
             epoch group) on the per-item kernel (b200_trk_kernel_choice(0)): the per-item kernel's rate when HBM is not
             the limit.
  c2_auto    the same under the default kernel choice: the shared-window kernel on the gr_complex band, the per-item
             kernel on the narrow bands (the shared-window kernel reads float bands only).
  c4         the C4 sweep (GPS L1 C/A, 32 PRNs x 81 Doppler bins x N = 25 000 at 25 Msps, CFAR) from a window of a
             gr_complex and of an ishort band that wraps around the ring's end (b200_acq_search_band_submit / _wait).
  push       b200_iq_push_i16 of 2^24 samples from pinned memory into a gr_complex band (raw copy + conversion launch) and
             into an ishort band (raw copy only), host clock around pushes ending in a synchronise.

usage: python tools/iq_narrow_time.py [--legs distinct,c2_item,c2_auto,c4,push] [--rounds 3] [--steps 10]
The integers pushed are the same for every band type, and each leg checks that the band types' outputs are identical.
"""
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

TYPES = ["gr_complex", "ishort", "ibyte"]
BYTES = {"gr_complex": 8, "ishort": 4, "ibyte": 2}
HBM_TBPS = 3.35
FS, N_CH, EPOCH, SHIFTS = 25_000_000, 32, 25000, [-0.5, 0.0, 0.5]


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                             timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        out = f"nvidia-smi unavailable: {e}"
    return dict(zip(q.split(","), [s.strip() for s in out.split(",")])) if out.count(",") == 3 else {"nvidia-smi": out}


def fill(eng, band, item_type, n, block):
    """n samples of the int8-range block (int16 for gr_complex and ishort bands, int8 for ibyte), pushed block by block"""
    src = block if item_type == "ibyte" else block.astype(np.int16)
    m = src.size // 2
    pushed = 0
    while pushed < n:
        k = min(m, n - pushed)
        eng.iq_push_int(band, src[:2 * k])
        pushed += k
    eng.sync()


def trk_engine(capi, st, item_type, cap, n_samples, block, kernel):
    eng = capi.Engine(0, st.cuda_stream)
    eng.iq_create(0, cap, item_type)
    fill(eng, 0, item_type, n_samples, block)
    eng.trk_kernel_choice(kernel)
    return eng


def trk_items(capi, eng, seconds, distinct):
    """C2's 32 channels x 1000 epochs/s; distinct: channel c reads its own stream at c * fs * seconds"""
    rng = np.random.default_rng(3)
    n_iq = int(FS * seconds)
    n_ep = n_iq // EPOCH
    items = []
    for c in range(N_CH):
        cid = eng.channel_create(0, 3)
        eng.channel_set_code(cid, rng.choice([-1.0, 1.0], 1023).astype(np.float32), SHIFTS)
        doppler = rng.uniform(-5000, 5000)
        step = 1.023e6 * (1 + doppler / 1575.42e6) / FS
        k = np.arange(n_ep)
        arr = np.zeros(n_ep, capi.TRK_ITEM_DTYPE)
        arr["channel"] = cid
        arr["n"] = EPOCH
        arr["sample_index"] = k * EPOCH + (c * n_iq if distinct else 0)
        arr["rem_carrier_phase_rad"] = np.mod(2 * np.pi * doppler / FS * k * EPOCH, 2 * np.pi)
        arr["phase_step_rad"] = 2 * np.pi * doppler / FS
        arr["rem_code_phase_chips"] = -np.mod(rng.uniform(0, 1023) + step * k * EPOCH, 1023)
        arr["code_phase_step_chips"] = step
        items.append(arr)
    items = np.concatenate(items)
    if not distinct:
        items = items[np.argsort(items["sample_index"], kind="stable")]
    return items


def time_batches(torch, st, eng, it_dev, n, out, steps):
    for _ in range(2):
        eng.trk_batch_dev(it_dev.data_ptr(), n, out.data_ptr(), 3, 1)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    k0 = eng.launch_count()
    e0.record(st)
    for _ in range(steps):
        eng.trk_batch_dev(it_dev.data_ptr(), n, out.data_ptr(), 3, 1)
    e1.record(st)
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps, (eng.launch_count() - k0) // steps


def trk_leg(torch, capi, st, leg, block, rounds, steps):
    distinct = leg == "distinct"
    seconds = 0.5 if distinct else 1.0
    cap = 1 << 29 if distinct else 1 << 25
    n_samples = int(FS * seconds) * (N_CH if distinct else 1)
    kernel = 2 if leg == "c2_auto" else 0
    engines, outs = {}, {}
    for t in TYPES:
        engines[t] = trk_engine(capi, st, t, cap, n_samples, block, kernel)
    items = trk_items(capi, engines[TYPES[0]], seconds, distinct)
    for t in TYPES[1:]:
        assert np.array_equal(trk_items(capi, engines[t], seconds, distinct), items)
    it_dev = torch.from_numpy(items.view(np.uint8)).cuda()
    ch_samples = int(items["n"].astype(np.int64).sum())
    times = {t: [] for t in TYPES}
    launches = {}
    for _ in range(rounds):
        for t in TYPES:
            out = torch.zeros((items.size, 3, 2), dtype=torch.float32, device="cuda")
            ms, launches[t] = time_batches(torch, st, engines[t], it_dev, items.size, out, steps)
            times[t].append(ms)
            outs[t] = out.cpu().numpy()
    same = all(outs[t].tobytes() == outs[TYPES[0]].tobytes() for t in TYPES) if kernel == 0 else None
    for t in TYPES:
        ms = min(times[t])
        line = {"leg": leg, "band": t, "items": int(items.size), "channel_samples_per_step": ch_samples,
                "ms_per_step": [round(x, 4) for x in times[t]], "launches_per_step": launches[t],
                "Msamples_per_s": round(ch_samples / (ms * 1e-3) / 1e6), "outputs_equal_across_types": same}
        if distinct:
            bps = ch_samples * BYTES[t] / (ms * 1e-3)
            line.update(algorithmic_TBps=round(bps / 1e12, 3), frac_of_hbm=round(bps / 1e12 / HBM_TBPS, 3))
        print(json.dumps(line), flush=True)
    for e in engines.values():
        e.close()


def c4_leg(torch, capi, st, rounds):
    from gnss_synth import gps_ca_code, gps_ca_code_complex_sampled, make_iq
    n, prns = 25000, 32
    present = [2, 5, 9, 13, 17, 21, 26, 30]
    rng = np.random.default_rng(4)
    svs = [dict(prn=p, doppler=float(rng.uniform(-9000, 9000)), code_phase_chips=float(rng.uniform(0, 1023)), cn0=45.0) for p in present]
    x = make_iq({p: gps_ca_code(p) for p in present}, float(FS), 2 * n, svs, seed=4)
    iq = np.empty(2 * x.size, np.int16)
    iq[0::2] = np.clip(np.round(300 * x.real), -32768, 32767)
    iq[1::2] = np.clip(np.round(300 * x.imag), -32768, 32767)
    eng = capi.Engine(0, st.cuda_stream)
    cap = 1 << 16
    for b, t in ((0, "gr_complex"), (1, "ishort")):
        eng.iq_create(b, cap, t)
        eng.iq_push_int(b, np.zeros(2 * (cap - n // 2), np.int16))   # the searched window wraps around the ring's end
        eng.iq_push_int(b, iq)
    s0 = cap - n // 2
    acq = capi.PcpsAcquisition(eng, fs_in=FS, samples_per_ms=float(n), samples_per_chip=24, doppler_max=10125, doppler_step=250,
                               n_code_slots=prns)
    for p in range(1, prns + 1):
        acq.set_local_code(p - 1, gps_ca_code_complex_sampled(p, FS))
    slots = np.arange(prns, dtype=np.uint32)
    res, times = {}, {0: [], 1: []}
    for _ in range(3):
        for b in (0, 1):
            acq.search_band_submit(b, s0, slots)
            res[b] = acq.search_wait()
    for _ in range(rounds * 20):
        for b in (0, 1):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(st)
            acq.search_band_submit(b, s0, slots)
            e1.record(st)
            res[b] = acq.search_wait()
            e1.synchronize()
            times[b].append(e0.elapsed_time(e1))
    for b, t in ((0, "gr_complex"), (1, "ishort")):
        print(json.dumps({"leg": "c4", "band": t, "ms_median": round(float(np.median(times[b])), 4),
                          "ms_min": round(float(np.min(times[b])), 4), "sweeps": len(times[b]),
                          "records_equal": res[b].tobytes() == res[0].tobytes()}), flush=True)
    acq.close()
    eng.close()


def push_leg(torch, capi, st, block, rounds):
    n = 1 << 24
    src = torch.from_numpy(np.resize(block.astype(np.int16), 2 * n)).pin_memory()
    eng = capi.Engine(0, st.cuda_stream)
    for b, t in ((0, "gr_complex"), (1, "ishort")):
        eng.iq_create(b, 1 << 26, t)
    times = {0: [], 1: []}
    for r in range(rounds + 1):
        for b in (0, 1):
            eng.sync()
            t0 = time.perf_counter()
            for _ in range(8):
                eng.iq_push_int(b, (src.data_ptr(), 16), n)
            eng.sync()
            if r:
                times[b].append(time.perf_counter() - t0)
    for b, t in ((0, "gr_complex"), (1, "ishort")):
        s = min(times[b])
        print(json.dumps({"leg": "push_i16", "band": t, "samples": 8 * n, "s": [round(x, 4) for x in times[b]],
                          "Msamples_per_s": round(8 * n / s / 1e6), "host_GBps": round(8 * n * 4 / s / 1e9, 2)}), flush=True)
    eng.close()


def main():
    import torch
    import gnss_sdr_b200.capi as capi
    legs = sys.argv[sys.argv.index("--legs") + 1].split(",") if "--legs" in sys.argv else ["distinct", "c2_item", "c2_auto", "c4", "push"]
    rounds = int(sys.argv[sys.argv.index("--rounds") + 1]) if "--rounds" in sys.argv else 3
    steps = int(sys.argv[sys.argv.index("--steps") + 1]) if "--steps" in sys.argv else 10
    dev = torch.device("cuda", 0)
    st = torch.cuda.Stream(device=dev)
    torch.cuda.set_stream(st)
    print(json.dumps({"gpu": torch.cuda.get_device_name(dev), "lib": capi.LIB_PATH, **card()}), flush=True)
    block = np.random.default_rng(1).integers(-128, 128, 2 * (1 << 24)).astype(np.int8)
    for leg in legs:
        if leg in ("distinct", "c2_item", "c2_auto"):
            trk_leg(torch, capi, st, leg, block, rounds, steps)
        elif leg == "c4":
            c4_leg(torch, capi, st, rounds)
        elif leg == "push":
            push_leg(torch, capi, st, block, rounds)
    print(json.dumps({"end": card()}), flush=True)


if __name__ == "__main__":
    main()
