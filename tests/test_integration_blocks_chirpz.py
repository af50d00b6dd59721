"""Drop-in acquisition blocks at chirp-z transform sizes (fft_size with a prime factor above 7) against the reference's own
blocks, both created by implementation string through the same harness (oracle/blocks_harness.cc) and run over the same
samples, as in test_integration_blocks.py:

  * Galileo E1 at 5.456 Msps with 4 ms coherent integration and bit_transition_flag=true, the acquisition settings of
    the reference's conf/File_input/Galileo/gnss-sdr_galileo_E1_extended_correlator_labsat.conf (N = 43 648 = 2^7 * 11 * 31)
    with a pfa instead of its bare threshold: without a pfa Acq_Conf selects the first/second-peak statistic, which
    chirp-z sizes do not support;
  * GPS L1 C/A at 16.368 Msps with make_two_steps=true (N = 16 368 = 2^4 * 3 * 11 * 31).

Both need the compiled reference blocks (oracle/Makefile `blocks`) and skip without them.
"""
import numpy as np
import pytest

import blocks_itf as bi
from gnss_synth import make_iq


@pytest.fixture(scope="module")
def reflib():
    lib = bi.ref_lib()
    if lib is None:
        pytest.skip("oracle/_ref/liboracle_ref_blocks.so not built (make -C oracle blocks; needs the reference tree)")
    return lib


@pytest.fixture(scope="module")
def b200lib():
    lib = bi.b200_lib()
    if lib is None:
        pytest.skip("oracle/_ref/libb200_blocks_check.so not built (make -C oracle blocks; needs the reference tree)")
    return lib


def acquire(lib, conf, impl, role, system, signal, prn, samples):
    ch = bi.Channel(lib, conf, impl, "", acq_role=role)
    ch.set_satellite(system, signal, prn)
    ch.acq_start()
    ch.acq_run(samples)
    s = ch.synchro()
    res = dict(delay=s.Acq_delay_samples, doppler=s.Acq_doppler_hz, stamp=s.Acq_samplestamp_samples, doppler_step=s.Acq_doppler_step,
               events=ch.events("acq"))
    ch.close()
    return res


@pytest.mark.gpu
def test_b200_galileo_e1_labsat_bit_transition_matches_reference(reflib, b200lib):
    """Galileo_E1_PCPS_Ambiguous_Acquisition(_B200) with the labsat configuration's acquisition settings: pilot (E1C)
    acquisition, 4 ms coherent integration, bit_transition_flag, doppler_max 5000 Hz, doppler_step 125 Hz; CFAR statistic
    (pfa 0.001).  Same decision, same code phase, Doppler and sample stamp."""
    fs, prn, delay = 5_456_000, 19, 9876
    rng = np.random.default_rng(19)
    e1b = bi.code_table(reflib, "E", "1B", prn)
    e1c = bi.code_table(reflib, "E", "1C", prn)
    data = rng.choice([-1.0, 1.0], 64)
    cp = (-delay * 2 * 1.023e6 / fs) % 8184
    svs = [dict(prn="b", doppler=1390.0, code_phase_chips=cp, cn0=45.0, symbols=data, periods_per_symbol=1),
           dict(prn="c", doppler=1390.0, code_phase_chips=cp, cn0=45.0, symbols=-np.ones(1), periods_per_symbol=1)]
    iq = make_iq({"b": e1b, "c": e1c}, float(fs), 4 * 43648, svs, seed=6, chips_per_table_chip=2.0)
    conf = {"GNSS-SDR.internal_fs_sps": fs, "Acquisition_1B.item_type": "gr_complex", "Acquisition_1B.coherent_integration_time_ms": 4,
            "Acquisition_1B.acquire_pilot": True, "Acquisition_1B.pfa": 0.001, "Acquisition_1B.doppler_max": 5000,
            "Acquisition_1B.doppler_step": 125, "Acquisition_1B.bit_transition_flag": True, "Acquisition_1B.blocking": True}
    ref = acquire(reflib, conf, "Galileo_E1_PCPS_Ambiguous_Acquisition", "Acquisition_1B", "E", "1B", prn, iq)
    got = acquire(b200lib, conf, "Galileo_E1_PCPS_Ambiguous_Acquisition_B200", "Acquisition_1B", "E", "1B", prn, iq)
    assert (got["delay"], got["doppler"], got["stamp"], got["events"]) == (ref["delay"], ref["doppler"], ref["stamp"], ref["events"]), (ref, got)
    assert ref["events"] == [1] and abs(ref["delay"] - delay) <= 1 and abs(ref["doppler"] - 1390.0) <= 125


@pytest.mark.gpu
def test_b200_gps_l1_two_step_at_16368_ksps_matches_reference(reflib, b200lib):
    """GPS_L1_CA_PCPS_Acquisition(_B200) at 16.368 Msps with make_two_steps: a positive first step on a 500 Hz grid, then
    the narrow 125 Hz search on the next buffer.  Same decision, code phase, Doppler, sample stamp and Acq_doppler_step."""
    fs, prn, delay = 16_368_000, 9, 7777
    code = bi.code_table(reflib, "G", "1C", prn)
    sv = dict(prn=prn, doppler=-2310.0, code_phase_chips=(-delay * 1.023e6 / fs) % 1023, cn0=47.0)
    iq = make_iq({prn: code}, float(fs), 6 * 16368, [sv], seed=12)
    conf = {"GNSS-SDR.internal_fs_sps": fs, "Acquisition_1C.item_type": "gr_complex", "Acquisition_1C.doppler_max": 5000,
            "Acquisition_1C.doppler_step": 500, "Acquisition_1C.pfa": 0.001, "Acquisition_1C.blocking": True,
            "Acquisition_1C.make_two_steps": True, "Acquisition_1C.second_nbins": 4, "Acquisition_1C.second_doppler_step": 125}
    ref = acquire(reflib, conf, "GPS_L1_CA_PCPS_Acquisition", "Acquisition_1C", "G", "1C", prn, iq)
    got = acquire(b200lib, conf, "GPS_L1_CA_PCPS_Acquisition_B200", "Acquisition_1C", "G", "1C", prn, iq)
    assert got == ref, (ref, got)
    assert ref["events"] == [1] and abs(ref["delay"] - delay) <= 1 and abs(ref["doppler"] + 2310.0) <= 125
    assert ref["doppler_step"] == 125
