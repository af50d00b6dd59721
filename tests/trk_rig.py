"""The rig of the tracking correlator tests (b200_trk_*): tap spacings, work items from tuples, ring bands fed with a
lead-in and the data, channels with their code table, and one b200_trk_batch_dev launch on device-resident items."""
import numpy as np

from gnss_sdr_b200.abi import TRK_ITEM_DTYPE

SENTINEL = -12345.0     # outputs a launch must not touch keep this value


def shifts(taps, spread=0.5):
    """taps tap shifts spread evenly over [-spread, spread] chips, rounded to float32; one tap is the prompt alone"""
    return [0.0] if taps == 1 else [float(s) for s in np.linspace(-spread, spread, taps).astype(np.float32)]


def items(rows, **fields):
    """b200_trk_item array from tuples in field order: (channel, n, sample_index, rem_carrier_phase_rad, phase_step_rad,
    phase_rate_step_rad, rem_code_phase_chips, code_phase_step_chips, code_phase_rate_step_chips).  Fields a tuple leaves
    off its end are zero; a keyword sets that field on every item."""
    width = len(TRK_ITEM_DTYPE.names)
    out = np.array([tuple(r) + (0,) * (width - len(r)) for r in rows], TRK_ITEM_DTYPE)
    for name, value in fields.items():
        out[name] = value
    return out


def ring(e, band, data, capacity=None, lead=None):
    """Create band `band` as a ring of `capacity` samples (default len(data)), push the complex64 lead-in, in pushes of
    at most one ring, then push data: complex64, or interleaved int16 / int8 I,Q through iq_push_int.  Returns the
    absolute index of data's first sample."""
    capacity = capacity or len(data)
    e.iq_create(band, capacity)
    if lead is not None:
        for k in range(0, len(lead), capacity):
            e.iq_push(band, lead[k:k + capacity])
    if data.dtype in (np.int16, np.int8):
        return e.iq_push_int(band, data)
    return e.iq_push(band, data)


def channel(e, band, code, shifts, hd=False):
    """a channel on `band` with one tap per shift and `code` as its float32 table; returns its id"""
    cid = e.channel_create(band, len(shifts))
    e.channel_set_code(cid, np.asarray(code, np.float32), shifts, hd)
    return cid


def run_dev(torch, e, items, stride, slices=1):
    """one b200_trk_batch_dev launch on `items` copied to the device -> float32 (items, stride, 2); the output starts as
    SENTINEL, so columns the launch leaves alone read SENTINEL"""
    items_t = torch.from_numpy(np.ascontiguousarray(items).view(np.uint8)).cuda()
    out_t = torch.full((len(items), stride, 2), SENTINEL, dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()        # the engine's stream does not wait for torch's
    e.trk_batch_dev(items_t.data_ptr(), len(items), out_t.data_ptr(), stride, slices)
    e.sync()
    return out_t.cpu().numpy()
