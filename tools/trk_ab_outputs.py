#!/usr/bin/env python
"""Every output of the tracking correlators and device loops on seeded random inputs, for byte-for-byte A/B runs of two builds.

  B200_LIB=<lib.so> python tools/trk_ab_outputs.py out.npz     # one .npz: taps of every batch, correlator and loop record
  python tools/trk_ab_outputs.py --compare a.npz b.npz         # names the first array that differs

Each case is sized for the path it names (STEP = 1.023 Mchip/s at 4 Msps, 0.2558 chips per sample):
  per-item kernel (extended table of 1023 + 64 entries on the main engine, 4092 + 64 on the pilot engine)
    item{1..8}       4000-sample epochs, about 1030 chips: the extended-table fast tiles, one and four slices, epochs that
                     cross the ring's end (both sample parities), every batch mixed (only_mask set)
    mixed_5_2_1      the same path with 5-, 2- and 1-tap channels in one batch, one and three slices
    large_index      rem = -5e6 chips, span still under the table: the extended table with the scalar main tiles
    modulo           40 000-sample epochs (10 230 chips): the integer-modulo path
    short_epochs     7 samples: no main tile, the remainder only
    submit_unsorted  b200_trk_submit / b200_trk_wait with the items in random order
    mixed_5_1        a pilot's 5 taps and its data channel's 1 tap, 8000 samples at 2 STEP on 4092-entry tables (4099 chips)
    high_dynamics    a high-dynamics channel
  shared-window kernel (forced; 16 items, 3 taps)
    whole_table_chunks   25 Msps (0.041 chips per sample), 25 000 samples: whole-epoch table, chunk path
    whole_table          STEP, 4000 samples (15 STEP > 1): whole-epoch table, warp_tile
    sliding_window       STEP, 16 000 samples on an 8184-entry code (4092 chips > 1152): the cp.async window
    no_share             items spread over 200 000 samples: every warp streams its own tiles
    off_table            rem = 2e6 chips: warp_correlate_general
    linear_band          an attached band whose last tiles are clipped at its end
  and the same items through the per-item kernel with a single tap count (only_mask = 0), two slices;
  the three single correlators; the device loops in modes 0 (at both CTA widths), 1 and 2 with and without a data channel
  (records, pilot prompts, final status).
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from acq_ab_outputs import compare  # noqa: E402  (same byte-for-byte comparison)

FS = 4e6
STEP = 1.023e6 / FS


def main(out_path):
    import torch
    import gnss_sdr_b200.capi as capi
    rng = np.random.default_rng(20261017)
    out = {}

    def noise(n):
        return (rng.normal(size=n) + 1j * rng.normal(size=n)).astype(np.complex64)

    def code(n):
        return rng.choice([-1.0, 1.0], n).astype(np.float32)

    def items_for(chans, n, starts, rem_code=0.2, step=STEP, rate=0.0):
        it = np.zeros(len(chans), capi.TRK_ITEM_DTYPE)
        for i, (ch, s0) in enumerate(zip(chans, starts)):
            it[i] = (ch, n, s0, rng.uniform(-3, 3), rng.uniform(-0.05, 0.05), 1e-7, rem_code + rng.uniform(0, 1), step, rate)
        return it

    def batch_dev(e, items, stride, slices):
        d = torch.from_numpy(items.view(np.uint8).copy()).cuda()
        o = torch.zeros(len(items) * stride, dtype=torch.complex64, device="cuda")
        torch.cuda.synchronize()
        e.trk_batch_dev(d.data_ptr(), len(items), o.data_ptr(), stride, slices)
        e.sync()
        return o.cpu().numpy()

    # ---- per-item kernel
    e = capi.Engine(0)
    e.iq_create(0, 1 << 20)
    e.iq_push(0, noise(1 << 20))
    e.iq_push(0, noise(3 << 18))  # the ring has wrapped: epochs across its end
    e.trk_kernel_choice(0)
    lo = e.iq_window(0)[0]
    taps_ch = {}
    for taps in range(1, 9):
        ch = e.channel_create(0, taps)
        e.channel_set_code(ch, code(1023), sorted(rng.uniform(-1, 1, taps)))
        taps_ch[taps] = ch
    ring_end = 1 << 20  # absolute index of the first sample stored at the ring's start again
    for taps in range(1, 9):
        starts = np.concatenate([lo + rng.integers(0, 1 << 19, 6), [ring_end - 2000, ring_end - 2001]])
        its = items_for([taps_ch[taps]] * 8, 4000, starts)
        out[f"item{taps}.batch"] = e.trk_batch(its, 8)
        for slices in (1, 4):
            out[f"item{taps}.dev_s{slices}"] = batch_dev(e, its, 8, slices)
    mixed = items_for([taps_ch[5], taps_ch[1], taps_ch[2], taps_ch[5], taps_ch[1]], 4000, lo + rng.integers(0, 1 << 19, 5))
    out["mixed_5_2_1.batch"] = e.trk_batch(mixed, 8)
    out["mixed_5_2_1.dev_s3"] = batch_dev(e, mixed, 8, 3)
    out["large_index"] = e.trk_batch(items_for([taps_ch[3]] * 4, 4000, lo + rng.integers(0, 1 << 19, 4), rem_code=-5.0e6), 8)
    out["modulo"] = e.trk_batch(items_for([taps_ch[5]] * 4, 40000, lo + rng.integers(0, 1 << 19, 4)), 8)
    out["short_epochs"] = e.trk_batch(items_for([taps_ch[3]] * 8, 7, lo + rng.integers(0, 1 << 19, 8)), 8)
    t = e.trk_submit(items_for([taps_ch[3]] * 40, 4000, lo + rng.permutation(1 << 19)[:40]), 8)
    out["submit_unsorted"] = e.trk_wait(t)
    e.close()

    e = capi.Engine(0)  # only 5 + 1 taps: the mixed batch of a tracked pilot
    e.iq_create(0, 1 << 18)
    e.iq_push(0, noise(1 << 18))
    p, d = e.channel_create(0, 5), e.channel_create(0, 1)
    e.channel_set_code(p, code(4092), [-1.0, -0.15, 0.0, 0.15, 1.0])
    e.channel_set_code(d, code(4092), [0.0])
    out["mixed_5_1"] = e.trk_batch(items_for([p, d, p, d], 8000, rng.integers(0, 1 << 17, 4), step=2 * STEP), 8)
    hd = e.channel_create(0, 3)
    e.channel_set_code(hd, code(1023), [-0.5, 0.0, 0.5], high_dyn=True)
    out["high_dynamics"] = e.trk_batch(items_for([hd] * 3, 4001, rng.integers(0, 1 << 17, 3), rate=3e-9), 8)
    e.close()

    # ---- shared-window kernel (forced): 3 taps, slices 1
    def shared_case(name, code_len, n, starts, step=STEP, rem_code=0.2, attach=False):
        e = capi.Engine(0)
        x = noise(1 << 18)
        if attach:
            xd = torch.from_numpy(x.view(np.float32).copy()).cuda()
            e.iq_attach_dev(0, xd.data_ptr(), len(x))
        else:
            e.iq_create(0, 1 << 18)
            e.iq_push(0, x)
        ch = e.channel_create(0, 3)
        e.channel_set_code(ch, code(code_len), [-0.5, 0.0, 0.5])
        its = items_for([ch] * len(starts), n, starts, rem_code=rem_code, step=step)
        e.trk_kernel_choice(1)
        out[f"shared.{name}"] = batch_dev(e, its, 4, 1)
        e.trk_kernel_choice(0)
        out[f"item_uniform.{name}"] = batch_dev(e, its, 4, 2)
        e.close()

    near = np.sort(rng.integers(1000, 3000, 16))
    shared_case("whole_table_chunks", 1023, 25000, near, step=1.023e6 / 25e6)
    shared_case("whole_table", 1023, 4000, near)
    shared_case("sliding_window", 8184, 16000, near)
    shared_case("no_share", 1023, 4000, np.sort(rng.integers(0, 200000, 16)))
    shared_case("off_table", 1023, 4000, near, rem_code=2.0e6)
    shared_case("linear_band", 1023, 4000, np.sort(rng.integers(254000, 258100, 16)), attach=True)

    # ---- single correlators
    e = capi.Engine(0)
    mc = capi.Multicorrelator(e, 20000, 5)
    sh = [-1.0, -0.5, 0.0, 0.5, 1.0]
    mc.set_high_dynamics_resampler(False)
    mc.set_local_code_and_taps(code(1023), sh)
    for n in (3, 4001, 20000):
        out[f"single.n{n}"] = mc.Carrier_wipeoff_multicorrelator_resampler(noise(n), 0.3, 0.012, 0.0, 0.2, STEP, 0.0)
    mc.set_local_code_and_taps_cplx(code(1023) + 1j * code(1023), sh)
    out["single.cplx"] = mc.correlate_cplx(noise(20000), 0.3, 0.012, 0.2, STEP)
    mc.set_local_code_and_taps_16sc(rng.integers(-2, 3, 2 * 1023).astype(np.int16), sh)
    out["single.16sc"] = mc.correlate_16sc(rng.integers(-60, 60, 2 * 20000).astype(np.int16), 0.3, 0.012, 0.2, STEP)
    mc.free()
    e.close()

    # ---- device loops
    import loop_rig as tl

    for mode in tl.MODES:
        for with_data in (False, True):
            sp, dt = tl.pilot_data_spec(5, 25, 1234.0, 1777, 60)
            e, ids, _ = tl.make_engine_with_data(capi, [sp], [dt if with_data else None], {0: len(sp.stream.x) + 16})
            tl.set_mode(e, mode, sp)
            tl.push_all(e, [sp])
            tl.start_all(e, ids, [sp])
            rec, cnt, prm = (a[:len(ids)] for a in e.loop_run_prompts(60))   # the started loop, not the standby ones
            name = f"loop.{mode}.{'data' if with_data else 'pilot'}"
            out[name + ".records"] = rec
            out[name + ".n_records"] = np.asarray(cnt)
            out[name + ".prompts"] = prm
            st = e.loop_status(ids[0])
            out[name + ".status"] = np.frombuffer(bytes(st), np.uint8)
            e.close()
    np.savez(out_path, **out)
    print(f"{out_path}: {len(out)} arrays")


if __name__ == "__main__":
    if sys.argv[1] == "--compare":
        sys.exit(compare(sys.argv[2], sys.argv[3]))
    main(sys.argv[1])
