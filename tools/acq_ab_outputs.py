#!/usr/bin/env python
"""Every output of the acquisition search on seeded random inputs, for byte-for-byte A/B runs of two builds.

  B200_LIB=<lib.so> python tools/acq_ab_outputs.py out.npz     # one .npz: result records, grids, wipe-offs, spectra
  python tools/acq_ab_outputs.py --compare a.npz b.npz         # names the first array that differs

Inputs are random +-1 codes and noisy code-modulated carriers from numpy's seeded generator.  The cases reach every plan
family: single-level N = 4000, 16 000 and 25 000, two-level N with each global radix 2, 3, 4, 5, 7, 8, 10, chirp-z sizes,
and the fine Doppler estimate at a single- and a two-level size.  On one single-level and one two-level size every search
option runs as well.
"""
import ctypes as C
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SINGLE = [4000, 16000, 25000]
TWO_LEVEL = [50000, 30375, 100000, 125000, 175000, 200000, 270000]  # global radix 2, 3, 4, 5, 7, 8, 10
CHIRP_Z = [16368, 5456, 13000]


def compare(a_path, b_path):
    a, b = np.load(a_path), np.load(b_path)
    if list(a.files) != list(b.files):
        print("different array names:", sorted(set(a.files) ^ set(b.files)))
        return 1
    for k in a.files:
        if a[k].dtype != b[k].dtype or a[k].shape != b[k].shape or a[k].tobytes() != b[k].tobytes():
            print("first difference:", k)
            return 1
    print(f"identical: {len(a.files)} arrays")
    return 0


def main(out_path):
    import torch
    import gnss_sdr_b200.capi as capi
    rng = np.random.default_rng(20261016)
    st = torch.cuda.Stream()
    torch.cuda.set_stream(st)  # the engine borrows torch's stream, so torch.cuda.synchronize() covers the device-side entry points
    eng = capi.Engine(0, st.cuda_stream)
    out = {}

    def signal(code, n, fs):
        t = np.arange(n)
        carrier = np.exp(2j * np.pi * rng.uniform(-1500, 1500) / fs * t)
        x = np.roll(np.resize(code, n), int(rng.integers(0, code.size))) * carrier
        return (x + rng.normal(0, 2.0, n) + 1j * rng.normal(0, 2.0, n)).astype(np.complex64)

    def i16(n):
        return rng.integers(-200, 200, 2 * n).astype(np.int16)

    def case(name, spms, *, cfar=True, keep_grid=True, dwells=1, bits=False, ms_per_code=1, sampled_ms=1, center=0, step_two=False,
             i16_search=False, dev=False, selftest=False):
        fs = int(spms * 1000)
        acq = capi.PcpsAcquisition(eng, fs_in=fs, samples_per_ms=float(spms), samples_per_chip=max(1, int(fs / 1.023e6)), doppler_max=1000,
                                   doppler_step=500, use_CFAR_algorithm_flag=cfar, keep_grid=keep_grid, max_dwells=dwells, n_code_slots=2,
                                   bit_transition_flag=bits, sampled_ms=sampled_ms, ms_per_code=ms_per_code)
        c = acq.conf
        need = c.fft_size // 2 if c.code_layout == 1 else c.consumed_samples
        codes = [rng.choice([-1.0, 1.0], need).astype(np.complex64) for _ in range(2)]
        for s, code in enumerate(codes):
            acq.set_local_code(s, code)
        if center:
            acq.set_doppler_center(center, 0)
        out[f"{name}.wipeoffs"] = acq.read_wipeoffs()
        n = c.consumed_samples
        for d in range(1, dwells + 1):
            out[f"{name}.search{d}"] = acq.search(signal(codes[1], n, fs), [1, 0], dwell_counter=d)
        if keep_grid or dwells > 1:
            for s in range(2):
                out[f"{name}.grid{s}"] = acq.read_grid(s)
        if step_two:
            first = out[f"{name}.search1"][0]
            acq.set_step_two(float(first["doppler"]), 125.0, 4)
            out[f"{name}.step_two"] = acq.search_step_two(signal(codes[1], n, fs), 1, float(first["input_power"]))
            got, raw = np.zeros(1, capi.ACQ_RESULT_DTYPE), i16(n)
            assert capi.lib.b200_acq_search_step_two_i16(acq.h, raw.ctypes.data, 1, 1, C.c_float(float(first["input_power"])),
                                                         got.ctypes.data) == 0
            out[f"{name}.step_two_i16"] = got
        if i16_search:
            got, raw, slots = np.zeros(2, capi.ACQ_RESULT_DTYPE), i16(n), np.array([0, 1], np.uint32)
            assert capi.lib.b200_acq_search_i16(acq.h, raw.ctypes.data, slots.ctypes.data, 2, 1, got.ctypes.data) == 0
            out[f"{name}.search_i16"] = got
        if dev:
            x = torch.from_numpy(signal(codes[0], n, fs).view(np.float32)).cuda()
            res = torch.zeros(2 * capi.ACQ_RESULT_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
            prn = torch.tensor([7, 21], dtype=torch.int32, device="cuda")
            peak = torch.zeros(16, dtype=torch.uint8, device="cuda")
            acq.search_dev(x.data_ptr(), [0, 1], res.data_ptr())
            acq.sweep_best_dev(res.data_ptr(), prn.data_ptr(), 2, peak.data_ptr())
            torch.cuda.synchronize()
            out[f"{name}.search_dev"] = res.cpu().numpy()
            out[f"{name}.sweep_best"] = peak.cpu().numpy()
        if selftest:
            x = (rng.normal(size=c.fft_size) + 1j * rng.normal(size=c.fft_size)).astype(np.complex64)
            out[f"{name}.selftest_dft"] = acq.selftest_dft(x)
        acq.close()

    for n in SINGLE + TWO_LEVEL:
        case(f"n{n}", n)
    for name, spms in (("single", 4000), ("two_level", 50000)):
        half = spms // 2  # bit transition and layout 2 keep fft_size = spms
        case(f"{name}_nocfar_grid", spms, cfar=False)
        case(f"{name}_nocfar_nogrid", spms, cfar=False, keep_grid=False)
        case(f"{name}_dwells", spms, dwells=2)
        case(f"{name}_bits", half, bits=True)
        case(f"{name}_layout2", half, ms_per_code=2)
        case(f"{name}_center", spms, center=750)
        case(f"{name}_modes", spms, step_two=True, i16_search=True, dev=True)
    for n in CHIRP_Z:
        case(f"chirpz{n}", n, dwells=2, selftest=True)
    case("chirpz32736", 16368, sampled_ms=2, ms_per_code=2, dwells=2, selftest=True)
    case("chirpz16368_bits", 16368, bits=True, selftest=True)
    case("chirpz16368_modes", 16368, step_two=True, i16_search=True, dev=True)
    for n1ms in (2000, 4000):  # M = 10 x fft_size: single-level 20 000, two-level 40 000
        fine = capi.AcqFineDoppler(eng, n1ms)
        code = rng.choice([-1.0, 1.0], n1ms).astype(np.complex64)
        idx, peak = fine.estimate(signal(code, 10 * n1ms, n1ms * 1000.0), code)
        out[f"fine{n1ms}.estimate"] = np.array([idx, np.float32(peak).view(np.uint32)], np.uint32)
        out[f"fine{n1ms}.spectrum"] = fine.read_spectrum()
        fine.close()
    eng.close()
    np.savez(out_path, **out)
    print(f"{out_path}: {len(out)} arrays")


if __name__ == "__main__":
    if sys.argv[1] == "--compare":
        sys.exit(compare(sys.argv[2], sys.argv[3]))
    main(sys.argv[1])
