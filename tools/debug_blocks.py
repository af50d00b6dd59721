"""Per-epoch comparison of the reference tracking block and the B200 block through their dump files (GPU box).
usage: python tools/debug_blocks.py [e1|l5] """
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import blocks_itf as bi  # noqa: E402
from gnss_synth import make_iq  # noqa: E402
from gnss_sdr_b200.abi import TRK_DUMP_RECORD_DTYPE  # noqa: E402


def run(which, coalesce):
    reflib, b200lib = bi.ref_lib(), bi.b200_lib()
    rng = np.random.default_rng(11)
    if which == "e1":
        prn, fs, role, sysc, sig = 11, 4_000_000, "Tracking_1B", "E", "1B"
        e1b = bi.code_table(reflib, "E", "1B", prn)
        e1c = bi.code_table(reflib, "E", "1C", prn)
        data = rng.choice([-1.0, 1.0], 300)
        sec = np.array([1.0 if c == "0" else -1.0 for c in bi.E1C_SECONDARY])
        n, delay = int(fs * 1.9), 1234
        cp = (-delay * 2 * 1.023e6 / fs) % 8184
        svs = [dict(prn="b", doppler=-850.0, code_phase_chips=cp, cn0=43.0, symbols=data, periods_per_symbol=1),
               dict(prn="c", doppler=-850.0, code_phase_chips=cp, cn0=43.0, symbols=-sec, periods_per_symbol=1)]
        iq = make_iq({"b": e1b, "c": e1c}, fs, n, svs, seed=5, chips_per_table_chip=2.0)
        conf = {"GNSS-SDR.internal_fs_sps": fs, f"{role}.item_type": "gr_complex", f"{role}.pll_bw_hz": 15.0, f"{role}.dll_bw_hz": 2.0,
                f"{role}.early_late_space_chips": 0.15, f"{role}.very_early_late_space_chips": 0.6, f"{role}.pull_in_time_s": 1,
                f"{role}.track_pilot": True}
        impls = ("Galileo_E1_DLL_PLL_VEML_Tracking", "Galileo_E1_DLL_PLL_VEML_Tracking_B200")
        acq = (float(delay), -840.0, 16000)
    else:
        rng = np.random.default_rng(31)
        prn, fs, role, sysc, sig = 6, 12_000_000, "Tracking_L5", "G", "L5"
        l5i = bi.code_table(reflib, "G", "5I", prn)
        l5q = bi.code_table(reflib, "G", "5Q", prn)
        nh10 = np.array([1.0 if c == "0" else -1.0 for c in "0000110101"])
        nh20 = np.array([1.0 if c == "0" else -1.0 for c in "00000100110101001110"])
        data = rng.choice([-1.0, 1.0], 200)
        sym_i = np.repeat(data, 10) * np.tile(nh10, len(data))
        n, delay = int(fs * 0.45), 4321
        cp = (-delay * 10.23e6 / fs) % 10230
        svs = [dict(prn="i", doppler=2100.0, code_phase_chips=cp, cn0=48.0, symbols=sym_i, periods_per_symbol=1),
               dict(prn="q", doppler=2100.0, code_phase_chips=cp, cn0=48.0, symbols=nh20, periods_per_symbol=1, phase0=np.pi / 2)]
        iq = make_iq({"i": l5i, "q": l5q}, float(fs), n, svs, seed=8, chips_per_table_chip=10.0)
        conf = {"GNSS-SDR.internal_fs_sps": fs, f"{role}.item_type": "gr_complex", f"{role}.pll_bw_hz": 20.0, f"{role}.dll_bw_hz": 1.5,
                f"{role}.early_late_space_chips": 0.5, f"{role}.pull_in_time_s": 1, f"{role}.track_pilot": True}
        impls = ("GPS_L5_DLL_PLL_Tracking", "GPS_L5_DLL_PLL_Tracking_B200")
        acq = (float(delay), 2080.0, 12000)
    tmp = tempfile.mkdtemp()
    dumps = {}
    for name, lib, impl in [("ref", reflib, impls[0]), ("b200", b200lib, impls[1])]:
        c = dict(conf)
        c[f"{role}.dump"] = True
        c[f"{role}.dump_mat"] = False
        c[f"{role}.dump_filename"] = os.path.join(tmp, name + "_")
        c[f"{role}.b200_coalesce"] = coalesce
        ch = bi.Channel(lib, c, "", impl, trk_role=role)
        ch.set_satellite(sysc, sig, prn)
        ch.set_acq_result(*acq)
        ch.trk_start()
        out = ch.trk_run(iq)
        print(name, "outputs", len(out), "events", ch.events("trk"))
        ch.close()
        fn = os.path.join(tmp, name + "_0.dat")
        dumps[name] = np.fromfile(fn, TRK_DUMP_RECORD_DTYPE)
    r, g = dumps["ref"], dumps["b200"]
    print(which, "coalesce", coalesce, "records", len(r), len(g))
    m = min(len(r), len(g))
    shown = 0
    for k in range(m):
        bad = (r["PRN_start_sample_count"][k] != g["PRN_start_sample_count"][k] or
               abs(r["abs_P"][k] - g["abs_P"][k]) > 0.02 * abs(r["abs_P"][k]) + 5 or
               abs(r["prompt_I"][k] - g["prompt_I"][k]) > 0.05 * abs(r["abs_P"][k]) + 5)
        if bad or k < 3:
            print(k, "ref", [r[f][k] for f in ("PRN_start_sample_count", "abs_E", "abs_P", "abs_L", "prompt_I", "prompt_Q", "carrier_doppler_hz", "code_freq_chips", "CN0_SNV_dB_Hz", "aux1")])
            print(k, "b200", [g[f][k] for f in ("PRN_start_sample_count", "abs_E", "abs_P", "abs_L", "prompt_I", "prompt_Q", "carrier_doppler_hz", "code_freq_chips", "CN0_SNV_dB_Hz", "aux1")])
            shown += bad
            if shown > 6:
                break


if __name__ == "__main__":
    which = sys.argv[1] if len(sys.argv) > 1 else "e1"
    for co in (False, True):
        run(which, co)
