"""Time the pulse blanker (b200_iq_set_pulse_blanking) on the device.

Push throughput: half a second of signal at 25 and 100 Msps is pushed from pinned host memory in blocks of 2^20 samples into
a source band with no blanker, one, two, and a conditioner (D = 1, 97 taps, at an IF) followed by a blanker, from gr_complex
and ibyte bands; CUDA events on the engine's compute stream (which every push's copy and every stage launch are ordered
into) time the whole stream.  Reported as Msamples/s of input, the median of `--repeats` runs, the configurations
alternating within each repeat.  The blankers run at the adapter's defaults (pfa 0.04, L = 32, E = 12 500, R = 5 000 000),
so the first 400 000 samples are the estimation phase.

Scan kernel: torch.profiler's CUDA activity gives blank_scan_kernel's time per push of 2^20 samples (32 768 segments of 32),
once with every segment in estimation (E above the stream length: the serial recurrence, thread 0 alone) and once with every
segment in detection (E = 1), and the energy and apply kernels' times beside them.

    python tools/iq_blanking_time.py [--seconds 0.5] [--repeats 5] [--out result.json]

The card's name and power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

BLOCK = 1 << 20
DEFAULTS = (0.04, 32, 12500, 5000000)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def make_stream(torch, item_type, n, rng):
    """pinned host samples of item_type: (tensor, bits) with bits 0 for gr_complex"""
    if item_type == "gr_complex":
        return torch.from_numpy(rng.normal(0, 30, 2 * n).astype(np.float32)).pin_memory(), 0
    return torch.from_numpy(rng.integers(-100, 100, 2 * n).astype(np.int8)).pin_memory(), 8


def setup(capi, item_type, fs, stages, blank=DEFAULTS):
    """an engine with the source in band 0 and stages: "blank" (a blanker on band 0) or "cond_blank" (a conditioner at an IF
    into a band, then a blanker on it)"""
    e = capi.Engine(0)
    e.iq_create(0, 1 << 22, item_type)
    b = 1
    for s in stages:
        if s == "blank":
            e.iq_create(b, 1 << 22)
            e.iq_set_pulse_blanking(b, 0, *blank)
            b += 1
        else:
            taps = capi.iq_conditioner_lowpass(fs, 1, fs / 4, fs / 40)
            e.iq_create(b, 1 << 22)
            e.iq_create(b + 1, 1 << 22)
            e.iq_set_conditioner(b, 0, 1, taps, fs / 8, fs)
            e.iq_set_pulse_blanking(b + 1, b, *blank)
            b += 2
    return e


def pusher(e, host, bits):
    item = host.element_size() * 2
    ptr = host.data_ptr()

    def push(a, b):
        if bits == 0:
            e.iq_push_ptr(0, ptr + a * item, b - a)
        else:
            e.iq_push_int(0, (ptr + a * item, bits), b - a)
    return push


def run_once(capi, item_type, fs, stages, host, bits, n):
    """ms to push n samples through a source with the given stages"""
    e = setup(capi, item_type, fs, stages)
    push = pusher(e, host, bits)
    push(0, BLOCK)                                                         # warm-up: modules, staging buffers
    e.sync()
    e.timer_start()
    for a in range(BLOCK, n, BLOCK):
        push(a, min(n, a + BLOCK))
    ms = e.timer_stop_ms()
    e.sync()
    e.close()
    return ms


def kernel_times(capi, torch, host, bits, est, pushes=12):
    """mean us per push of each blanker kernel, profiled over `pushes` pushes of BLOCK gr_complex samples"""
    from torch.profiler import ProfilerActivity, profile
    e = setup(capi, "gr_complex", 25e6, ["blank"], blank=(0.04, 32, est, 5000000))
    push = pusher(e, host, bits)
    push(0, BLOCK)
    e.sync()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for k in range(1, pushes + 1):
            push(k * BLOCK, (k + 1) * BLOCK)
        e.sync()
    out = {}
    for ev in prof.key_averages():
        for name in ("blank_energy_kernel", "blank_scan_kernel", "blank_apply_kernel"):
            if name in ev.key:
                out[name] = out.get(name, 0.0) + ev.device_time_total / pushes
    e.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=0.5)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from gnss_sdr_b200 import capi
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: the blanker is timed on the GPU only")
    rng = np.random.default_rng(1)
    configs = []
    for fs in (25e6, 100e6):
        for item_type in ("gr_complex", "ibyte"):
            for name, stages in (("none", []), ("one_blanker", ["blank"]), ("two_blankers", ["blank", "blank"]),
                                 ("conditioner_then_blanker", ["cond_blank"])):
                configs.append((f"{int(fs / 1e6)}Msps_{item_type}_{name}", item_type, fs, stages))
    streams = {}
    times = {c[0]: [] for c in configs}
    for _ in range(args.repeats):
        for name, item_type, fs, stages in configs:
            n = int(fs * args.seconds)
            key = (item_type, n)
            if key not in streams:
                streams[key] = make_stream(torch, item_type, n, rng)
            host, bits = streams[key]
            times[name].append(run_once(capi, item_type, fs, stages, host, bits, n))
    gpu = card()
    rows = []
    for name, item_type, fs, stages in configs:
        n = int(fs * args.seconds) - BLOCK
        ms = float(np.median(times[name]))
        rows.append(dict(config=name, input_msps=n / ms / 1e3, realtime_factor=n / ms / 1e3 / (fs / 1e6), ms=ms,
                         spread_ms=[float(min(times[name])), float(max(times[name]))]))
        print(f"{name:44s} {n / ms / 1e3:9.1f} Msamples/s  x{n / ms / 1e3 / (fs / 1e6):6.1f} real time  "
              f"({ms:.2f} ms, {args.repeats} runs {min(times[name]):.2f}-{max(times[name]):.2f})")
    host, bits = make_stream(torch, "gr_complex", 14 * BLOCK, rng)
    kt = {"estimation": kernel_times(capi, torch, host, bits, est=1 << 30), "detection": kernel_times(capi, torch, host, bits, est=1)}
    for phase, d in kt.items():
        print(f"per push of {BLOCK} samples (32768 segments), all {phase}: " + ", ".join(f"{k} {v:.1f} us" for k, v in d.items()))
    print(f"card: {gpu}")
    res = dict(card=gpu, seconds=args.seconds, block=BLOCK, rows=rows, kernel_us_per_push=kt)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
