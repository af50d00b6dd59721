"""Time the notch filters (b200_iq_set_notch) on the device.

Push throughput: half a second of signal at 25 and 100 Msps is pushed from pinned host memory in blocks of 2^20 samples into
a source band with no stage, a Lite notch at the adapter's defaults (p 0.9, pfa 0.001, L = 32, E = 12 500, R = 5 000 000) on
clean noise (where the reference's estimator keeps the filter on for most segments), the same with a strong CW on every
sample, a Notch at the same defaults, and a conditioner (D = 1, at an IF) followed by a Lite notch, from gr_complex and
ibyte bands.  CUDA events on the engine's compute stream time the whole stream.  Reported as Msamples/s of input, the median
of `--repeats` runs, the configurations alternating within each repeat.

Kernels: torch.profiler's CUDA activity gives each notch kernel's time per push of 2^20 samples (32 768 segments of 32),
once with every segment in estimation (E above the stream length) and once in detection (E = 1).

    python tools/iq_notch_time.py [--seconds 0.5] [--repeats 5] [--out result.json]

The card's name, power limit and SM clock are read in the same run."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

BLOCK = 1 << 20
KERNELS = ("notch_energy_kernel", "notch_floor_kernel", "notch_scan_kernel", "notch_compose_kernel", "notch_carry_kernel",
           "notch_apply_kernel")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def make_stream(torch, item_type, n, rng, cw):
    """pinned host samples of item_type, noise plus (cw) a CW ten times the noise's amplitude: (tensor, bits)"""
    sigma = 10.0 if item_type == "ibyte" else 30.0
    x = rng.normal(0, sigma, 2 * n).astype(np.float32)
    if cw:
        ph = 0.37 * np.arange(n)
        x[0::2] += 4 * sigma * np.cos(ph)
        x[1::2] += 4 * sigma * np.sin(ph)
    if item_type == "gr_complex":
        return torch.from_numpy(x).pin_memory(), 0
    return torch.from_numpy(np.clip(np.round(x), -127, 127).astype(np.int8)).pin_memory(), 8


def setup(capi, item_type, fs, stage, est=12500):
    e = capi.Engine(0)
    e.iq_create(0, 1 << 22, item_type)
    if stage in ("lite", "notch"):
        e.iq_create(1, 1 << 22)
        e.iq_set_notch(1, 0, capi.B200_NOTCH_LITE if stage == "lite" else capi.B200_NOTCH, 0.001, 0.9, 32, est, 5000000, 1)
    elif stage == "cond_lite":
        taps = capi.iq_conditioner_lowpass(fs, 1, fs / 4, fs / 40)
        e.iq_create(1, 1 << 22)
        e.iq_create(2, 1 << 22)
        e.iq_set_conditioner(1, 0, 1, taps, fs / 8, fs)
        e.iq_set_notch(2, 1, capi.B200_NOTCH_LITE, 0.001, 0.9, 32, est, 5000000, 1)
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


def run_once(capi, item_type, fs, stage, host, bits, n):
    """ms to push n samples through a source with the given stage"""
    e = setup(capi, item_type, fs, stage)
    push = pusher(e, host, bits)
    push(0, BLOCK)
    e.sync()
    e.timer_start()
    for a in range(BLOCK, n, BLOCK):
        push(a, min(n, a + BLOCK))
    ms = e.timer_stop_ms()
    e.sync()
    e.close()
    return ms


def kernel_times(capi, torch, host, bits, est, pushes=12):
    """mean us per push of each notch kernel (Lite), profiled over `pushes` pushes of BLOCK gr_complex samples"""
    from torch.profiler import ProfilerActivity, profile
    e = setup(capi, "gr_complex", 25e6, "lite", est=est)
    push = pusher(e, host, bits)
    push(0, BLOCK)
    e.sync()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for k in range(1, pushes + 1):
            push(k * BLOCK, (k + 1) * BLOCK)
        e.sync()
    out = {}
    for ev in prof.key_averages():
        for name in KERNELS:
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
        raise SystemExit("no CUDA device: the notch is timed on the GPU only")
    rng = np.random.default_rng(1)
    configs = []
    for fs in (25e6, 100e6):
        for item_type in ("gr_complex", "ibyte"):
            for name, stage, cw in (("none", None, False), ("lite_clean", "lite", False), ("lite_cw", "lite", True),
                                    ("notch_cw", "notch", True), ("conditioner_then_lite", "cond_lite", False)):
                configs.append((f"{int(fs / 1e6)}Msps_{item_type}_{name}", item_type, fs, stage, cw))
    streams = {}
    times = {c[0]: [] for c in configs}
    for _ in range(args.repeats):
        for name, item_type, fs, stage, cw in configs:
            n = int(fs * args.seconds)
            key = (item_type, n, cw)
            if key not in streams:
                streams[key] = make_stream(torch, item_type, n, rng, cw)
            host, bits = streams[key]
            times[name].append(run_once(capi, item_type, fs, stage, host, bits, n))
    gpu = card()
    rows = []
    for name, item_type, fs, stage, cw in configs:
        n = int(fs * args.seconds) - BLOCK
        ms = float(np.median(times[name]))
        rows.append(dict(config=name, input_msps=n / ms / 1e3, ms=ms, spread_ms=[float(min(times[name])), float(max(times[name]))]))
        print(f"{name:40s} {n / ms / 1e3:9.1f} Msamples/s  ({ms:.2f} ms, {args.repeats} runs {min(times[name]):.2f}-{max(times[name]):.2f})")
    host, bits = make_stream(torch, "gr_complex", 14 * BLOCK, rng, False)
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
