"""One small acquisition on cuda:0 checked against the numpy oracle (used by __graft_entry__.smoke)."""


def run(eng):
    import gnss_sdr_b200.capi as capi
    import oracle
    import acq_rig as ar
    from gnss_synth import make_iq
    fs, prn = 4e6, 1
    code = oracle.port.gps_ca_code(prn)
    sv = dict(prn=prn, doppler=1680.0, code_phase_chips=(-524 / (fs / 1.023e6)) % 1023, cn0=47.0, phase0=0.4)
    iq = make_iq({prn: code}, fs, 4000, [sv], seed=1)
    p = ar.params(fs, doppler_max=5000, doppler_step=250)
    sampled = ar.ca_code(oracle.port, prn, fs)
    want = ar.oracle(p, sampled, pfa=0.001).acquisition_core(iq)
    acq = capi.PcpsAcquisition(eng, **p)
    acq.set_local_code(0, sampled)
    got = acq.search(iq, [0])[0]
    acq.close()
    ar.check(got, want, ("test_statistics",))
    print(f"smoke: acq PRN {prn}: delay {got['index_time']} samples, doppler {got['doppler']} Hz, "
          f"stat {got['test_statistics']:.2f} (oracle {want['test_statistics']:.2f})")
