"""Time b200_trk_loop_run per epoch (CUDA events on the engine stream) on Galileo-E1-like loops, with and without a
data channel.

    python tools/loop_pilot_data_time.py [--baseline DIR] [--rounds 3] [--out FILE]

Each loop: 8184-entry sinBOC(1,1) pilot table, VEML taps, 4 ms epochs of 16 000 samples (4 Msps) or 200 000 samples
(50 Msps); each loop with a data channel also has its own 8184-entry data table.  32, 64 and 256 loops in mode 0, the
persistent kernel, which takes 512-thread CTAs while the loops are no more than the SMs and 256-thread CTAs beyond that: on
a 132-SM H100 the first two counts time the wide CTA, the third the narrow one.  The samples are noise: the lock detectors
are switched off so that every loop runs every epoch.

--baseline DIR: a checkout of another version with its library and oracle built.  Each round then runs both libraries, one after
the other, each in a fresh process; the baseline's legs without a data channel are timed if it has no
b200_trk_loop_set_data_channel.  One JSON line per measurement, and the card's name, power limit and SM clocks first."""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EPOCHS = {16000: (4e6, 100), 200000: (50e6, 30)}   # samples per epoch -> (fs, timed epochs per run)
LOOPS = (32, 64, 256)
WARM = 2
REPEATS = 5


def child(root: str, label: str):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, root)   # the library under test, its binding and its oracle: this tree's or the baseline's
    import numpy as np
    import gnss_sdr_b200.capi as capi
    from oracle import loop as ol
    import oracle

    has_data = hasattr(capi.lib, "b200_trk_loop_set_data_channel")
    rng = np.random.default_rng(1)
    tables = [oracle.port.sinboc11((2 * rng.integers(0, 2, 4092) - 1).astype(np.int32)) for _ in range(2 * LOOPS[-1])]
    shifts = [-1.0, -0.3, 0.0, 0.3, 1.0]
    for n_ep_samples, (fs, k) in EPOCHS.items():
        n_iq = n_ep_samples * (WARM + k + 2)
        iq = (rng.standard_normal(n_iq) + 1j * rng.standard_normal(n_iq)).astype(np.complex64)
        for n_loops in LOOPS:
            for data in ((False, True) if has_data else (False,)):
                e = capi.Engine(0)
                e.iq_create(0, n_iq + 16)
                e.iq_push(0, iq)
                ids = []
                for j in range(n_loops):
                    ch = e.channel_create(0, 5)
                    e.channel_set_code(ch, tables[2 * j], shifts)
                    conf = ol.default_conf(fs_in=fs, prn=j + 1, code_length_chips=4092, code_period=0.004, vector_length=n_ep_samples,
                                           code_samples_per_chip=2, veml=1, early_late_space_chips=0.15, cn0_min=-1000,
                                           max_code_lock_fail=1 << 30, max_carrier_lock_fail=1 << 30, cloop=0)
                    lid = e.loop_create(ch, capi.TrkLoopConf.from_buffer_copy(conf))   # an older tree's oracle has its own class
                    if data:
                        dch = e.channel_create(0, 1)
                        e.channel_set_code(dch, tables[2 * j + 1], [0.0])
                        e.loop_set_data_channel(lid, dch)
                    ids.append(lid)
                e.loop_set_mode(0)
                times = []
                for _ in range(REPEATS + 1):
                    for j, lid in enumerate(ids):
                        e.loop_start(lid, 100.0 + 37 * j, 0.0, 0, 0)
                    rc = capi.lib.b200_trk_loop_run(e.h, WARM, None, None)
                    assert rc == 0
                    e.timer_start()
                    rc = capi.lib.b200_trk_loop_run(e.h, k, None, None)
                    ms = e.timer_stop_ms()
                    assert rc == 0
                    times.append(ms)
                st = [e.loop_status(lid) for lid in ids]
                assert all(s.state == 2 for s in st), "a loop stopped"
                times = sorted(times[1:])
                print(json.dumps(dict(lib=label, samples_per_epoch=n_ep_samples, loops=n_loops, data_channel=data,
                                      us_per_epoch_median=round(1000.0 * times[len(times) // 2] / k, 3),
                                      us_per_epoch_min=round(1000.0 * times[0] / k, 3))), flush=True)
                e.close()


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
    except (OSError, subprocess.SubprocessError) as exc:
        out = f"nvidia-smi unavailable: {exc}"
    return out.strip().splitlines()[:1]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--baseline", default=None)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    ap.add_argument("--child", nargs=2, metavar=("ROOT", "LABEL"), help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.child:
        child(*a.child)
        return
    libs = [(ROOT, "this")] + ([(os.path.abspath(a.baseline), "baseline")] if a.baseline else [])
    lines = [json.dumps(dict(gpu=gpu_info()))]
    print(lines[0], flush=True)
    for _ in range(a.rounds):
        for root, label in libs:
            env = dict(os.environ)
            env.pop("B200_LIB", None)
            p = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", root, label], env=env, capture_output=True, text=True)
            if p.returncode != 0:
                sys.stderr.write(p.stderr)
                raise SystemExit(f"{label}: exit {p.returncode}")
            for ln in p.stdout.splitlines():
                print(ln, flush=True)
                lines.append(ln)
        lines.append(json.dumps(dict(gpu=gpu_info())))
        print(lines[-1], flush=True)
    if a.out:
        with open(a.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
