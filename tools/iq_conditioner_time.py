"""Time the signal conditioner (b200_iq_set_conditioner) on the device: a stream of `--seconds` of signal is pushed from pinned
host memory in blocks of 2^20 samples into a source band, with no, one or two conditioners attached, and CUDA events on the
engine's compute stream (which every push's copy and every conditioner launch are ordered into) time the whole stream.
Reported as Msamples/s of input, the median of `--repeats` runs, the configurations alternating within each repeat.

    python tools/iq_conditioner_time.py [--seconds 2] [--repeats 5] [--out result.json]

Configurations: 25 Msps at IF 0 with D = 10 (481 taps) and D = 5 (241 taps, the adapter's default low-pass) from each band
type; 50 Msps at an IF of 4.092 MHz with D = 25 and 121 taps; and one gr_complex push stream at 25 Msps with no conditioner,
one, and two (GPS L1 and Galileo E1 at different IFs).  The card's name and power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

BLOCK = 1 << 20


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def make_stream(torch, item_type, n, rng):
    """pinned host samples of item_type: (tensor, bits) with bits 0 for gr_complex"""
    if item_type == "gr_complex":
        x = torch.from_numpy(rng.normal(0, 30, 2 * n).astype(np.float32)).pin_memory()
        return x, 0
    dt, bits = (np.int16, 16) if item_type == "ishort" else (np.int8, 8)
    x = torch.from_numpy(rng.integers(-100, 100, 2 * n).astype(dt)).pin_memory()
    return x, bits


def run_once(capi, torch, item_type, fs, conds, host, bits, n):
    """ms to push n samples through a source with conditioners conds = [(D, taps, IF)]"""
    e = capi.Engine(0)
    e.iq_create(0, 1 << 22, item_type)
    for k, (d, taps, if_hz) in enumerate(conds):
        e.iq_create(1 + k, (1 << 22) // d + 1)
        e.iq_set_conditioner(1 + k, 0, d, taps, if_hz, fs)
    item = host.element_size() * 2
    ptr = host.data_ptr()

    def push(a, b):
        if bits == 0:
            e.iq_push_ptr(0, ptr + a * item, b - a)
        else:
            e.iq_push_int(0, (ptr + a * item, bits), b - a)

    push(0, BLOCK)                                                         # warm-up: modules, staging buffers
    e.sync()
    e.timer_start()
    for a in range(BLOCK, n, BLOCK):
        push(a, min(n, a + BLOCK))
    ms = e.timer_stop_ms()
    e.sync()
    e.close()
    return ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=2.0)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from gnss_sdr_b200 import capi
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: the conditioner is timed on the GPU only")
    rng = np.random.default_rng(1)
    lp = capi.iq_conditioner_lowpass
    configs = []
    for item_type in ("gr_complex", "ishort", "ibyte"):
        for d in (10, 5):
            configs.append((f"25Msps_IF0_D{d}_{item_type}", item_type, 25e6, [(d, lp(25e6, d), 0.0)]))
    configs.append(("50Msps_IF4.092MHz_D25_121taps_gr_complex", "gr_complex", 50e6, [(25, lp(50e6, 25, 1.0e6, 1.0e6), 4.092e6)]))
    t5 = lp(25e6, 5)
    configs += [("25Msps_gr_complex_no_conditioner", "gr_complex", 25e6, []),
                ("25Msps_gr_complex_one_conditioner", "gr_complex", 25e6, [(5, t5, 0.0)]),
                ("25Msps_gr_complex_two_conditioners", "gr_complex", 25e6, [(5, t5, 1.0e6), (5, t5, -1.0e6)])]
    for item_type in ("ishort", "ibyte"):
        configs.append((f"25Msps_{item_type}_no_conditioner", item_type, 25e6, []))
    streams = {}
    times = {c[0]: [] for c in configs}
    for _ in range(args.repeats):
        for name, item_type, fs, conds in configs:
            n = int(fs * args.seconds)
            key = (item_type, n)
            if key not in streams:
                streams[key] = make_stream(torch, item_type, n, rng)
            host, bits = streams[key]
            times[name].append(run_once(capi, torch, item_type, fs, conds, host, bits, n))
    gpu = card()
    rows = []
    for name, item_type, fs, conds in configs:
        n = int(fs * args.seconds) - BLOCK
        ms = float(np.median(times[name]))
        rows.append(dict(config=name, taps=[int(c[1].size) for c in conds], decimation=[c[0] for c in conds], input_msps=n / ms / 1e3,
                         ms=ms, spread_ms=[float(min(times[name])), float(max(times[name]))]))
        print(f"{name:48s} {n / ms / 1e3:9.1f} Msamples/s  ({ms:.2f} ms, {args.repeats} runs {min(times[name]):.2f}-{max(times[name]):.2f})")
    print(f"card: {gpu}")
    res = dict(card=gpu, seconds=args.seconds, block=BLOCK, rows=rows)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
