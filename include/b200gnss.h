/*
 * b200gnss.h -- C ABI of libb200gnss.so: the H100 (sm_90a) implementation of gnss-sdr's two
 * data-parallel hot paths, the multi-tap tracking correlator and the PCPS acquisition grid
 * search.  Plain pointers and sizes only; no C++/torch types cross this boundary.
 *
 * Every entry point cites the reference interface it replaces (paths relative to the
 * gnss-sdr tree; VG = src/algorithms/libs/volk_gnsssdr_module/volk_gnsssdr).
 *
 * Conventions
 *  - All functions return int: B200_OK (0) or a negative B200_ERR_* code; nothing calls
 *    exit() (contrast src/algorithms/tracking/libs/cuda_multicorrelator.cu:294-301).
 *    b200_last_error() returns a thread-local message for the last failure.
 *  - Complex samples are interleaved (re, im) float32 pairs == lv_32fc_t == gr_complex
 *    (VG include/volk_gnsssdr/volk_gnsssdr_complex.h).
 *  - "host" pointers are ordinary (optionally pinned) host memory; "dev" pointers are CUDA
 *    device pointers on the engine's device.  `stream` arguments are cudaStream_t passed as
 *    void* (NULL = the engine's own stream).
 *  - Handles are opaque.  Distinct handles may be used concurrently from different threads
 *    (one tracking block thread per channel, as in the reference's thread-per-block
 *    scheduler); calls on ONE handle must be serialised by the caller (the reference blocks
 *    do that with gr::block::d_setlock).
 */
#ifndef B200GNSS_H
#define B200GNSS_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C"
{
#endif

#define B200_OK 0
#define B200_ERR_ARG (-1)    /* bad argument / handle */
#define B200_ERR_CUDA (-2)   /* a CUDA call failed (message in b200_last_error) */
#define B200_ERR_NOMEM (-3)  /* host or device allocation failed */
#define B200_ERR_STATE (-4)  /* call sequence error (e.g. correlate before set_local_code) */
#define B200_ERR_RANGE (-5)  /* size outside what the engine was created for */
#define B200_ERR_NODEV (-6)  /* no usable sm_90 device */

#define B200_MAX_TAPS 8

    typedef struct b200_cf32
    {
        float re, im;
    } b200_cf32;

    typedef struct b200_engine b200_engine;
    typedef struct b200_trk b200_trk;
    typedef struct b200_acq b200_acq;

    /* ---- library / engine ------------------------------------------------------------- */
    int b200_version(void);
    const char* b200_last_error(void);
    int b200_device_count(int* count);

    /* One engine per (process, GPU): owns the device context, a compute stream, a copy
     * stream, the IQ band stores and the channel registry.  `stream` (cudaStream_t as void*)
     * makes the engine launch on a caller-owned stream instead of its own.
     * Precedent: the FPGA path's device-owned sample stream,
     * src/algorithms/tracking/libs/fpga_multicorrelator.cc:152-192. */
    int b200_engine_create(b200_engine** out, int device, void* stream);
    int b200_engine_destroy(b200_engine* e);
    int b200_engine_sync(b200_engine* e);
    /* device-side timing of work submitted to the engine stream (CUDA events) */
    int b200_engine_timer_start(b200_engine* e);
    int b200_engine_timer_stop_ms(b200_engine* e, float* ms);

    /* ---- IQ band store ---------------------------------------------------------------- */
    /* A band is one conditioned IQ stream (what gnss_flowgraph.cc:1227-1231 fans out to every
     * channel).  Samples are addressed by their absolute index in the stream
     * (== the reference's sample counter, Gnss_Synchro::Acq_samplestamp_samples).
     * capacity_samples is rounded up to a power of two; the store is a ring. */
    int b200_iq_create(b200_engine* e, int band, uint64_t capacity_samples);
    /* b200_iq_create with the band's sample type, item_type as b200_iq_push_file and the reference's
     * SignalSource.item_type: "gr_complex" (8 B per sample, what b200_iq_create makes), "ishort" (interleaved int16 I,Q
     * = lv_16sc_t, 4 B) or "ibyte" (interleaved int8 I,Q, 2 B); anything else is B200_ERR_ARG.  A narrow band holds its
     * samples at their own width: 2x (ishort) or 4x (ibyte) the samples of a gr_complex band in the same memory.  It takes
     * only pushes of its own type - b200_iq_push_i16 (ishort) or b200_iq_push_i8 (ibyte), and b200_iq_push_file with its
     * item type - which copy the integers into the ring as they are, with no conversion launch; every other push
     * (b200_iq_push, b200_iq_push_at, b200_iq_refill, the other integer width, a file of another type) is B200_ERR_STATE
     * and writes nothing.  The per-item tracking correlator and the band searches (b200_acq_search_band and its
     * variants) read a narrow band in place and widen each sample to float on load; int -> float is exact, so their
     * results equal those on a gr_complex band holding the same integers.  The shared-window correlator never runs a
     * batch while a channel with a code table sits on a narrow band (b200_trk_kernel_choice), and the device loops
     * refuse narrow bands (b200_trk_loop_create).  Re-creating a band with another type is allowed. */
    int b200_iq_create_typed(b200_engine* e, int band, uint64_t capacity_samples, const char* item_type);
    /* Append n host samples (async H2D on the copy stream, ordered before later launches).
     * *first_index receives the absolute index of host[0]. */
    int b200_iq_push(b200_engine* e, int band, const b200_cf32* host, uint64_t n, uint64_t* first_index);
    /* Idempotent push by ABSOLUTE index, for hosts where several threads hold the same stream: every tracking
     * block of a flowgraph receives the same conditioned samples in its own GNU Radio input buffer
     * (gnss_flowgraph.cc:1227-1231 fans one conditioner out to all channels).  Each block offers
     * [abs_index, abs_index + n); only the part beyond the band's write index is copied (*n_new samples), the
     * rest is already there.  abs_index beyond the write index opens a gap: the band restarts there
     * (b200_iq_window reports the new oldest valid sample).  Thread-safe. */
    int b200_iq_push_at(b200_engine* e, int band, uint64_t abs_index, const b200_cf32* host, uint64_t n, uint64_t* n_new);
    /* [valid_from, write_index): absolute indices of the samples a work item or a band search (b200_acq_search_band) may
     * address right now */
    int b200_iq_window(b200_engine* e, int band, uint64_t* valid_from, uint64_t* write_index);
    /* Declare what the band holds stale (the window becomes empty; the write index stays).  For hosts that start a new
     * stream whose indices overlap the previous one's (a flowgraph restarted inside one process): without this,
     * b200_iq_push_at would answer "already there" for indices the old stream had covered.  Launches already queued keep
     * reading what they were given. */
    int b200_iq_forget(b200_engine* e, int band);
    /* Same for front ends that deliver interleaved 16-bit / 8-bit (I,Q) integers (lv_16sc_t / lv_8sc_t):
     * the raw integers cross PCIe and are converted to float on the device, replacing the CPU
     * adapters src/algorithms/data_type_adapter/gnuradio_blocks/cshort_to_gr_complex.cc:48
     * (volk_gnsssdr_16ic_convert_32fc) and adapters/ibyte_to_complex.cc.  n counts complex samples;
     * host_iq holds 2*n integers.  Conversion is exact (int -> float).  Into a band of the push's own narrow type
     * (b200_iq_create_typed) the integers are copied as they are. */
    int b200_iq_push_i16(b200_engine* e, int band, const int16_t* host_iq, uint64_t n, uint64_t* first_index);
    int b200_iq_push_i8(b200_engine* e, int band, const int8_t* host_iq, uint64_t n, uint64_t* first_index);
    /* Stream a sample file into the band the way File_Signal_Source feeds the flowgraph
     * (src/algorithms/signal_source/adapters/file_source_base.cc: item types :340-378, header / seconds_to_skip
     * :385-414): item_type "gr_complex", "ishort" or "ibyte" (interleaved I,Q); header_bytes and skip_samples are
     * skipped; at most max_samples complex samples (0 = to the end of the file) are pushed in blocks of chunk_samples
     * (0 = 2^20) through two pinned staging buffers, so the disk read of one block overlaps the PCIe copy of the
     * previous one.  Integer types are converted on the device (b200_iq_push_i16 / _i8), or copied as they are into a
     * band of the same type. */
    int b200_iq_push_file(b200_engine* e, int band, const char* path, const char* item_type, uint64_t header_bytes,
        uint64_t skip_samples, uint64_t max_samples, uint64_t chunk_samples, uint64_t* first_index, uint64_t* samples_pushed);
    /* Use caller-owned device memory as the band (no copy): dev[0] is absolute index
     * first_index; n_samples need not be a power of two (no wrap).  The band's type becomes gr_complex. */
    int b200_iq_attach_dev(b200_engine* e, int band, const b200_cf32* dev, uint64_t n_samples, uint64_t first_index);

    /* Refill an attached band from host memory: host[0..n) becomes samples first_index .. first_index + n of the band
     * (asynchronous H2D on the copy stream, ordered before later launches like b200_iq_push).  For hosts that own the
     * device buffer because something else also touches it - e.g. rank 0 of a multi-GPU receiver pushes the band once
     * and NCCL broadcasts that buffer to the peers over NVLink (bench.py, SURVEY 8e). */
    int b200_iq_refill(b200_engine* e, int band, const b200_cf32* host, uint64_t n, uint64_t first_index);

    /* Copy samples [abs_index, abs_index + n) of a band to host memory in the band's own item format (8 B per gr_complex
     * sample, 4 B per ishort, 2 B per ibyte sample), after every write to the band queued so far; synchronous.  What the
     * reference's input filter writes to its dump file (freq_xlating_fir_filter.cc:171-176, 192-194), read back from a conditioned
     * band.  The samples must lie inside b200_iq_window, else B200_ERR_RANGE; an unused band is B200_ERR_STATE. */
    int b200_iq_read(b200_engine* e, int band, uint64_t abs_index, uint64_t n, void* host);

    /* ---- signal conditioner: frequency-translating decimating FIR on the device ------------------------------------
     * InputFilter.implementation = Freq_Xlating_Fir_Filter (src/algorithms/input_filter/adapters/freq_xlating_fir_filter.cc
     * :56-119), which instantiates gr::filter::freq_xlating_fir_filter_ccf(D, h, IF, fs) (:119): a receiver with a wideband
     * or IF front end moves the signal to baseband, low-pass filters and decimates it, and tracks at the filtered rate.
     *
     * b200_iq_set_conditioner links src_band to dst_band: every write into the source (b200_iq_push, _push_i16, _push_i8,
     * _push_at, _push_file) also fills the destination with, in absolute stream indices,
     *     y[j] = r(j) sum_{k=0}^{T-1} c[k] x[j D - k],   x[m < 0] = 0,
     *     c[k] = h[k] e^{+i k w},   r(j) = e^{-i w D j},   w = 2 pi IF / fs,
     * T = n_taps, D = decimation, h = taps.  The zero history below index 0 is the block's own at stream start, so
     * destination index j is the reference conditioner's j-th output and sample stamps line up with a reference flowgraph.
     *  - The composite taps c[k] are computed on the host in double and rounded once to float.  The sum runs k ascending
     *    from zero, every float product and sum rounded on its own: at IF = 0 (c = h, r = 1) the output is bit for bit that
     *    float32 loop.  Otherwise the sum is complex, (c.re x.re - c.im x.im) and (c.re x.im + c.im x.re) per tap, and y is
     *    the sum times r(j) in double, rounded once to float.
     *  - r(j) is computed per output from its absolute index j: D IF / fs mod 1 is taken exactly from the two doubles as a
     *    128-bit binary fraction q, phi(j) = j q mod 1 (top 64 bits, exact for every j < 2^64), r(j) = cos(2 pi phi) -
     *    i sin(2 pi phi) in double.  GNU Radio instead advances a float rotator output by output (gr::blocks::rotator),
     *    whose phase error grows with the stream; this one does not, so outputs past 2^32 are as accurate as the first.
     *  - The source may be a gr_complex, ishort or ibyte owned ring (integers are widened exactly at load); the
     *    destination must be a gr_complex owned ring whose capacity times D is at least the source's capacity.  One source
     *    may feed several destinations (GPS L1 and Galileo E1 at different IFs); a destination cannot also be a source,
     *    nor a source a destination.  Attached bands (b200_iq_attach_dev) are refused at either end.
     *  - After a push, each conditioner of the source launches once, on the engine's compute stream, for the outputs that
     *    became complete, [ceil(old_write / D), ceil(new_write / D)); a band search, batch or loop run issued after the
     *    push reads them, with no host synchronisation.  The next push's copy into the source waits for that launch.
     *  - The destination's window: write_index = ceil(src write_index / D); valid_from = 0 while the source's valid_from
     *    is 0 (stream start), else ceil((src valid_from + T - 1) / D), and never below where the conditioner was set or the
     *    destination was last b200_iq_forget-ed (an empty window while fewer outputs exist).  So a b200_iq_push_at gap or
     *    a b200_iq_forget on the source opens a gap in the destination, and the loops stall there as on any band.  Set on
     *    a source that already holds samples, the destination starts empty at ceil(src write_index / D).
     *  - While a conditioner is set, a direct push or push_at into its destination is B200_ERR_STATE, and a push into its
     *    source of more than capacity - (T - 1) samples is B200_ERR_RANGE (the filter's history must still be in the ring).
     *  - n_taps == 0 removes the destination's conditioner (src_band, taps and the rest are then not read); so does
     *    re-creating or attaching either band.  Setting a conditioner on a destination that has one replaces it.
     *  - Refused, with nothing launched and both windows unchanged: decimation < 1 or NULL taps (B200_ERR_ARG),
     *    decimation > B200_IQ_MAX_CONDITIONER_DECIMATION or n_taps > B200_IQ_MAX_CONDITIONER_TAPS (B200_ERR_RANGE),
     *    sampling_freq_hz <= 0 or a frequency that is not finite (B200_ERR_ARG), dst_band == src_band (B200_ERR_ARG),
     *    a band that is not an owned ring, a narrow destination, or a chain (B200_ERR_STATE), a destination too small
     *    (B200_ERR_RANGE).
     * The pm_remez band-pass design of the adapter's default filter_type is not restated: pass its taps. */
#define B200_IQ_MAX_CONDITIONER_TAPS 4096
#define B200_IQ_MAX_CONDITIONER_DECIMATION 4096
    int b200_iq_set_conditioner(b200_engine* e, int dst_band, int src_band, uint32_t decimation, const float* taps, uint32_t n_taps,
        double intermediate_freq_hz, double sampling_freq_hz);
    /* The adapter's filter_type = lowpass branch (freq_xlating_fir_filter.cc:103-110): gr::filter::firdes::low_pass(1, fs, bw,
     * tw) with the Hamming window, bw_hz <= 0 meaning the default (fs / decimation) / 2 and tw_hz <= 0 the default bw / 10.
     * The same design b200_acq_resampler_design computes: ntaps = int(53 fs / (22 tw)) made odd, windowed sinc scaled to unit
     * DC gain in double, each tap rounded once to float.  More taps than max_taps is B200_ERR_RANGE with the count needed in
     * *n_taps and b200_last_error(); taps may be NULL when max_taps is 0.  Host-only. */
    int b200_iq_conditioner_lowpass(double sampling_freq_hz, uint32_t decimation, double bw_hz, double tw_hz, uint32_t max_taps,
        float* taps, uint32_t* n_taps);

    /* ---- pulse blanking on the device ------------------------------------------------------------------------------
     * InputFilter.implementation = Pulse_Blanking_Filter (src/algorithms/input_filter/adapters/pulse_blanking_filter.cc:43-84),
     * which instantiates pulse_blanking_cc(pfa, length, segments_est, segments_reset)
     * (gnuradio_blocks/pulse_blanking_cc.cc:33-98): pulsed interference (DME/TACAN, radar, switching front ends) is removed
     * before acquisition and tracking see it.
     *
     * b200_iq_set_pulse_blanking links src_band to dst_band: every write into the source that completes segments fills the
     * destination with the block's output in absolute stream indices, dst[j] = src[j] widened, or 0 where j's segment is
     * blanked.  Segments are [o + k L, o + (k + 1) L), L = length, counted from the blanker's origin o.  For each, in order:
     *     e = sum_{i < L} (re_i re_i + im_i im_i)        (each square and sum rounded on its own, i ascending from 0.0)
     *     n < E and not last_filtered:  est = (float(n) est + e / float(2L)) / float(n + 1), copied        (estimation)
     *     else if e / est > thres:      zeroed, last_filtered = true                                         (detection)
     *     else:                         copied, last_filtered = false, and n = 0 if n > R
     *     n++
     * E = segments_est, R = segments_reset, thres = b200_iq_pulse_blanking_threshold(pfa, L); every float operation is
     * rounded on its own and e / est follows IEEE (E = 0: est stays 0, e / 0 is +inf and blanks, 0 / 0 is NaN and copies).
     *  - The energy sum is the generic VOLK order (volk_32f_accumulator_s32f_generic).  A VOLK dispatched to its AVX kernel
     *    sums in another order and can differ from this in the last bit of a segment energy.
     *  - The block keeps n in an int32; here it is 64-bit, which differs only after 2^31 segments without a reset (R near
     *    INT32_MAX), where the block's counter overflows.
     *  - The block processes a segment only once a sample past it has arrived (pulse_blanking_cc.cc:71); here every whole
     *    segment is published at once.  That delays the block's output and changes no value.
     *  - Origin and state: a blanker set on a fresh stream starts at index 0, one set on a source that already holds samples
     *    at the source's write index, with the block's initial state (n = 0, est = 0, last_filtered = false).  When the
     *    source's valid_from moves (a b200_iq_push_at gap or restart, b200_iq_forget on the source, or, chained, the
     *    conditioner's window moving), the blanker restarts at the new valid_from with its initial state.  So the
     *    destination always equals a reference block started on the stream at the origin.
     *  - The destination's window: write_index = o + floor((src write_index - o) / L) L (whole segments only);
     *    valid_from = o, never below where the destination was last b200_iq_forget-ed, nor above write_index.
     *  - The source may be a gr_complex, ishort or ibyte owned ring (integers are widened exactly, as Ishort_To_Complex and
     *    Ibyte_To_Complex do); the destination a gr_complex owned ring at least as large.  One source may feed several
     *    blankers.  The one chain allowed is a conditioner followed by a blanker: the source may be a conditioner's
     *    destination, which is the adapter's IF > 1 arm (pulse_blanking_filter.cc:73-84, freq_xlating_fir_filter_ccf(1,
     *    firdes::low_pass(1, fs, bw, tw), IF, fs) before the blanker): b200_iq_conditioner_lowpass, b200_iq_set_conditioner
     *    with decimation 1, then this.  A blanker or conditioner fed from a blanker's destination is refused.
     *  - After a push, the source's conditioners launch first, as before; then each blanker that reads the band or a
     *    destination just filled launches three kernels (segment energies, the state machine, copy or zero) on the compute
     *    stream when the write completed at least one segment, and none otherwise.  The state lives in device memory; a
     *    band search, batch or loop run issued after the push reads the blanked samples with no host synchronisation.  The
     *    next copy into a ring a blanker reads waits for its launches.
     *  - At most L - 1 source samples wait for their segment to complete, and they must stay in the ring: a push of more
     *    than capacity - (L - 1) samples into a blanker's source, or, chained, of more than D (capacity - (L - 1)) samples
     *    into the conditioner's source (capacity of the conditioner's destination, D its decimation), is B200_ERR_RANGE,
     *    refused before any byte is written; b200_iq_push_file cuts its blocks to fit.
     *  - While a blanker is set, a direct push or push_at into its destination is B200_ERR_STATE.  length == 0 removes the
     *    destination's blanker (the other arguments are then not read); so does re-creating or attaching either band.
     *    Setting a blanker on a destination that has one, or a notch, replaces it, restarting at the rule above.
     *  - Refused, with nothing launched and both windows unchanged: dst_band == src_band, length < 0, segments_est < 0,
     *    segments_reset < 0, or pfa outside (0, 1) (B200_ERR_ARG); length > B200_IQ_MAX_BLANKING_LENGTH or a destination
     *    smaller than the source or a source smaller than L (B200_ERR_RANGE); a band that is not an owned ring, a narrow
     *    destination, a destination that a conditioner fills or that feeds a stage, or a source that a blanker fills
     *    (B200_ERR_STATE). */
#define B200_IQ_MAX_BLANKING_LENGTH 4096
    int b200_iq_set_pulse_blanking(b200_engine* e, int dst_band, int src_band, float pfa, int32_t length, int32_t segments_est,
        int32_t segments_reset);
    /* thres of pulse_blanking_cc.cc:57-58, quantile(complement(chi_squared(2 length), pfa)): the x at which the chi-squared
     * upper tail with 2L degrees of freedom, e^{-x/2} sum_{k < L} (x/2)^k / k!, equals pfa, found in double and rounded once
     * to float.  pfa outside (0, 1) or length outside [1, B200_IQ_MAX_BLANKING_LENGTH] is B200_ERR_ARG.  Host-only. */
    int b200_iq_pulse_blanking_threshold(float pfa, int32_t length, float* thres);
    typedef struct
    {
        uint64_t origin;       /* absolute index of segment 0 */
        uint64_t segments;     /* segments processed since the origin */
        uint64_t blanked;      /* of them, zeroed */
        int64_t n;             /* the block's n_segments_ */
        float noise_power;     /* noise_power_estimation_ (est) */
        float threshold;       /* thres_ */
        int32_t last_filtered; /* last_filtered_ */
        int32_t length;        /* L */
    } b200_pulse_blanking_status;
    /* The state of dst_band's blanker after every push queued so far (synchronous): how much it blanks, and the state
     * machine it carries.  A band with no blanker is B200_ERR_STATE. */
    int b200_iq_pulse_blanking_status(b200_engine* e, int dst_band, b200_pulse_blanking_status* status);

    /* ---- notch filters on the device -------------------------------------------------------------------------------
     * InputFilter.implementation = Notch_Filter and Notch_Filter_Lite (src/core/receiver/gnss_block_factory.cc:835-841;
     * adapters/notch_filter.cc, adapters/notch_filter_lite.cc), which instantiate Notch(pfa, p_c_factor, length,
     * segments_est, segments_reset) (gnuradio_blocks/notch_cc.cc:63-121) and NotchLite(p_c_factor, pfa, length,
     * segments_est, segments_reset, segments_coeff) (notch_lite_cc.cc:71-138): continuous-wave and narrowband interference
     * is removed before acquisition and tracking see it.
     *
     * b200_iq_set_notch links src_band to dst_band: every write into the source that completes segments fills the
     * destination with the block's output in absolute stream indices.  Segment k is written to [o + k L, o + (k + 1) L),
     * L = length, o the notch's origin, and reads in[i] = src[o + k L + s + i], s = 0 for B200_NOTCH_LITE (the block's
     * set_history(2); in[-1] of the origin's segment is the zero history item, even when the ring holds a sample there) and
     * s = 1 for B200_NOTCH (the block's in++ without history: output j comes from input j + 1, so segment k is published
     * only once source index o + (k + 1) L exists).  For each segment, in order, every float operation rounded on its own:
     *     n < E and the filter off (estimation):  X[q] = sum_m in[m] W[m q mod L], W[m] = exp(-2 pi i m / L), in double
     *         (W made on the host in double, m ascending, each product and sum rounded); dB[q] = float(10 log10(|X[q]|^2 +
     *         1e-20)) in double; floor = volk_32f_s32f_calc_spectral_noise_floor_32f(dB, 15) in float (mean = sum / L + 15,
     *         then the mean of the dB[q] <= mean, or mean if none); sig2lin = float(10^(double(floor / 10))) / float(2L);
     *         est = (float(n) est + sig2lin) / float(n + 1); the segment is copied.
     *     else e = Re(volk_32fc_x2_conjugate_dot_prod_32fc(in, in, L)), in the generic order: even and odd samples into
     *         two sums of re re + im im, added, then + |in[L-1]|^2 when L is odd;
     *         e / est > thres (filtering): at the filter's switch-on last_out = 0 and (Lite) n_coeff = 0.
     *             Lite: when n_coeff == 0, z0 = exp(i float((a1 + a2) / 2)), a1 = atan2 of in[1] conj(in[0]), a2 of
     *             in[L-1] conj(in[L-2]); then n_coeff = (n_coeff + 1) mod segments_coeff.
     *             Notch: per sample, z0 = exp(i atan2 of in[i] conj(in[i-1])).
     *             out[i] = (in[i] - z0 in[i-1]) + (p z0) last_out, last_out = out[i]   (gr_complex products).
     *         else: copied, the filter off, and n = 0 if n > R.
     *     n++
     * E = segments_est, R = segments_reset, p = p_c_factor, thres = b200_iq_pulse_blanking_threshold(pfa, L) (the same
     * chi-squared quantile).  atan2, log10, pow, sin and cos are computed in double and rounded once to float.
     *  - The IIR is split-invariant: output samples are cut into blocks of 1024 on an absolute grid counted from the origin.
     *    Each block's affine map y -> A y + B is composed in double in sample order (a run start sets A = 0, B = b); y is
     *    carried from grid point to grid point in double, y_{g+1} = A_g y_g + B_g, and kept in the notch's state across
     *    pushes; inside a block the float recursion above runs serially from float(y_g).  So a filtered sample is within a
     *    float rounding bound (scaled by 1 / (1 - |p|)^2) of a float64 recursion with the same z0 and inputs, and the
     *    destination's bytes do not depend on how the source was pushed, which is why the device does not run the block's
     *    one serial float recursion per run: that recursion is as accurate (its rounding errors are damped by |p z0| <= |p|
     *    (1 + 2^-23), so they stay within the same 1 / (1 - |p|) form however long the run), but it cannot be split across
     *    threads.  Everything else (energies, est and every sig2lin, decisions, resets, runs, z0, copied and estimation
     *    samples) follows the statement above bit for bit.
     *  - Against the block itself: its spectrum comes from a float FFT and its transcendentals from the float libm
     *    functions, so est and z0 differ from the block's in the last few bits; a decision close to the threshold can
     *    then differ.  The reference's estimator compares a time-domain energy with a mean of dB values, which sits about
     *    2.5 dB under the mean power for noise, so the filter is on for much of a clean stream; this is reproduced.
     *  - Origin, window, chains, removal and replacement follow the pulse blanker above: the origin is 0 on a fresh stream
     *    and the source's write index when set mid-stream, the notch restarts with the block's initial state whenever the
     *    source's valid_from moves, and the destination holds whole segments only.  The source may be a conditioner's
     *    destination; nothing else chains (notch -> any stage, blanker -> notch and notch -> blanker are refused).
     *  - A push that completes segments launches six kernels on the compute stream (energies; the noise floor, which
     *    returns at once when no segment of the push can be in estimation; the state machine; the block maps; the carry;
     *    the output); none otherwise.  The state lives in device memory; a band search, batch or loop run issued after the
     *    push reads the notched samples with no host synchronisation.
     *  - A segment needs one sample beyond the L - 1 pending (Lite: the one before it, and at L = 1 also the one after it;
     *    Notch: the one after it): a push of more than capacity - L samples (Lite at L = 1: capacity - 2) into a notch's
     *    source, or D times that of the conditioner's destination through a chained conditioner, is B200_ERR_RANGE, refused
     *    before any byte is written; b200_iq_push_file cuts its blocks to fit.
     *  - Departures from the block: |p_c_factor| >= 1 or a non-finite one is refused (the block would run an unstable
     *    filter); n is 64-bit (the block's int32 overflows after 2^31 segments without a reset).
     *  - length == 0 removes the destination's notch (the other arguments are then not read); a pulse blanker there stays,
     *    and b200_iq_set_pulse_blanking with length 0 likewise leaves a notch in place.  Setting a notch on a destination
     *    that a blanker or notch fills replaces it, restarting with the block's initial state.  Refused, with nothing launched and both
     *    windows unchanged: an unknown variant, pfa outside (0, 1), a bad p_c_factor, length, segments_est or
     *    segments_reset < 0, dst_band == src_band, or Lite with segments_coeff < 1 (B200_ERR_ARG; Notch does not read
     *    segments_coeff); length > B200_IQ_MAX_NOTCH_LENGTH, a destination smaller than the source, or a source smaller than
     *    L + 1 (Lite at L = 1: 3), which could take no push (B200_ERR_RANGE); a band that is not an owned ring, a narrow destination, a destination a stage fills or
     *    that feeds one, or a forbidden chain (B200_ERR_STATE). */
#define B200_NOTCH 0      /* Notch_Filter: z0 per sample, output j from input j + 1 */
#define B200_NOTCH_LITE 1 /* Notch_Filter_Lite: z0 per coefficient period, output j from input j */
#define B200_IQ_MAX_NOTCH_LENGTH 1024
    int b200_iq_set_notch(b200_engine* e, int dst_band, int src_band, int variant, float pfa, float p_c_factor, int32_t length,
        int32_t segments_est, int32_t segments_reset, int32_t segments_coeff);
    typedef struct
    {
        uint64_t origin;       /* absolute index of segment 0 (destination indices) */
        uint64_t segments;     /* segments processed since the origin */
        uint64_t filtered;     /* of them, filtered */
        int64_t n;             /* n_segments_ */
        float noise_power;     /* noise_pow_est_ */
        float threshold;       /* thres_ */
        b200_cf32 z0;          /* z_0_ */
        b200_cf32 last_out;    /* last_out_ (the split-invariant recursion's) */
        int32_t filter_state;  /* filter_state_ */
        int32_t n_coeff;       /* n_segments_coeff_ (Lite; 0 for Notch) */
        int32_t length;        /* L */
        int32_t variant;       /* B200_NOTCH or B200_NOTCH_LITE */
    } b200_notch_status;
    /* The state of dst_band's notch after every push queued so far (synchronous).  A band with no notch is B200_ERR_STATE. */
    int b200_iq_notch_status(b200_engine* e, int dst_band, b200_notch_status* status);

    /* ---- tracking: single correlator, 1:1 with Cpu_Multicorrelator_Real_Codes ----------- */
    /* src/algorithms/tracking/libs/cpu_multicorrelator_real_codes.h:37-61 */
    /* init(max_signal_length_samples, n_correlators)                       (.cc:35-50) */
    int b200_trk_create(b200_engine* e, b200_trk** out, int max_signal_length_samples, int n_correlators);
    /* set_high_dynamics_resampler(bool)                                    (.cc:27-31 in .h:41) */
    int b200_trk_set_high_dynamics_resampler(b200_trk* t, int use_high_dynamics_resampler);
    /* set_local_code_and_taps(code_length_chips, local_code_in, shifts_chips) (.cc:53-63).
     * The table and shifts are COPIED.  The reference keeps the caller's shifts_chips POINTER and reads it on every
     * correlation, and dll_pll_veml_tracking mutates that array in place without calling this function again
     * (start_tracking :1045-1053, the narrow-correlator switch :2132-2146) - hosts that mirror the class must
     * therefore re-send the current values before each correlation with b200_trk_set_taps (a write into the
     * host-mapped control block: no copy, no synchronisation); B200_Multicorrelator_Real_Codes does. */
    int b200_trk_set_local_code_and_taps(b200_trk* t, int code_length_chips, const float* local_code_in, const float* shifts_chips);
    int b200_trk_set_taps(b200_trk* t, const float* shifts_chips);
    /* set_input_output_vectors + Carrier_wipeoff_multicorrelator_resampler (.cc:66-72,103-127):
     * corr_out[k] = sum_n sig_in[n] * exp(-j(rem_carrier + n*phase_step [+ rate term])) *
     *               code[ floor(step*n + shift_k - rem_code) mod L ].
     * Synchronous: copies sig_in to the device, correlates, copies n_correlators taps back.
     * Arithmetic contract: chip indices bit-exact with VG's a_avx/u_avx resampler
     * (..._32f_xn_resampler_32f_xn.h:362-435); taps within 1e-5*|prompt| of float64. */
    int b200_trk_correlate(b200_trk* t, const b200_cf32* sig_in_host,
        float rem_carrier_phase_in_rad, float phase_step_rad, float phase_rate_step_rad,
        float rem_code_phase_chips, float code_phase_step_chips, float code_phase_rate_step_chips,
        int signal_length_samples, b200_cf32* corr_out_host);
    /* ---- the reference's two other correlator classes (same handle type; one CTA per call, latency-oriented) ----------
     * Cpu_Multicorrelator - COMPLEX local code (src/algorithms/tracking/libs/cpu_multicorrelator.cc: set_local_code_and_taps
     * :53-63, Carrier_wipeoff_multicorrelator_resampler :86-100 = volk_gnsssdr_32fc_xn_resampler_32fc_xn +
     * volk_gnsssdr_32fc_x2_rotator_dot_prod_32fc_xn): corr_out[k] = sum_n sig[n] e^{-j(rem + n step)} code[idx_k(n)].
     * The class has no phase-rate / code-rate arguments. */
    int b200_trk_set_local_code_and_taps_cplx(b200_trk* t, int code_length_chips, const b200_cf32* local_code_in, const float* shifts_chips);
    int b200_trk_correlate_cplx(b200_trk* t, const b200_cf32* sig_in_host, float rem_carrier_phase_in_rad, float phase_step_rad,
        float rem_code_phase_chips, float code_phase_step_chips, int signal_length_samples, b200_cf32* corr_out_host);
    /* Cpu_Multicorrelator_16sc - 16-bit complex samples AND code (cpu_multicorrelator_16sc.cc:47-91 =
     * volk_gnsssdr_16ic_xn_resampler_16ic_xn + volk_gnsssdr_16ic_x2_rotator_dot_prod_16ic_xn): per sample the rotated
     * sample is rounded to int16, multiplied by the int16 code value (16-bit wrap of each product component, as
     * std::complex<int16_t> does) and accumulated; the reference saturates its 16-bit accumulator at every add, this sum is
     * exact and saturated once at the end (identical while the running sum stays inside int16, the class's operating range;
     * the reference's own QA tolerance between implementations is +-16 LSB, VG lib/kernel_tests.h).
     * Arrays are interleaved (I,Q) int16: 2 * code_length_chips, 2 * signal_length_samples, 2 * n_correlators values. */
    int b200_trk_set_local_code_and_taps_16sc(b200_trk* t, int code_length_chips, const int16_t* local_code_iq, const float* shifts_chips);
    int b200_trk_correlate_16sc(b200_trk* t, const int16_t* sig_in_iq_host, float rem_carrier_phase_in_rad, float phase_step_rad,
        float rem_code_phase_chips, float code_phase_step_chips, int signal_length_samples, int16_t* corr_out_iq_host);
    /* free()                                                               (.cc:147-160) */
    int b200_trk_destroy(b200_trk* t);

    /* ---- tracking: batched form (all channels in lock, many epochs, one launch) ---------- */
    /* A channel = one (band, code table, tap shifts) registration; the per-epoch scalars are
     * the seven arguments do_correlation_step passes
     * (src/algorithms/tracking/gnuradio_blocks/dll_pll_veml_tracking.cc:1232-1257). */
    typedef struct b200_trk_item
    {
        int32_t channel;       /* id returned by b200_trk_channel_create */
        int32_t n;             /* signal_length_samples (vector_length) */
        uint64_t sample_index; /* absolute index of the epoch's first sample in the band */
        float rem_carrier_phase_rad;
        float phase_step_rad;
        float phase_rate_step_rad;
        float rem_code_phase_chips;
        float code_phase_step_chips;
        float code_phase_rate_step_chips;
    } b200_trk_item; /* 40 bytes */

    int b200_trk_channel_create(b200_engine* e, int band, int n_correlators, int* channel_id);
    int b200_trk_channel_set_code(b200_engine* e, int channel_id, int code_length_chips, const float* local_code_in, const float* shifts_chips, int high_dynamics);
    /* tap shifts only (same reason as b200_trk_set_taps); takes effect, in stream order, from the next batch */
    int b200_trk_channel_set_taps(b200_engine* e, int channel_id, const float* shifts_chips);
    /* Correlate n_items (channel, epoch) work items.  out: n_items x out_stride complex taps
     * (out_stride >= the channel's n_correlators).  Host variant is synchronous (items H2D,
     * launch, taps D2H); the _dev variant takes device pointers and is asynchronous on the
     * engine stream. */
    int b200_trk_batch(b200_engine* e, const b200_trk_item* items_host, int n_items, b200_cf32* out_host, int out_stride);
    int b200_trk_batch_dev(b200_engine* e, const b200_trk_item* items_dev, int n_items, b200_cf32* out_dev, int out_stride, int slices);
    /* Asynchronous form of b200_trk_batch: submit returns at once with a ticket (items are copied;
     * the launch is ordered after every b200_iq_push made so far), wait blocks until that batch's
     * taps are in out_host.  Up to 16 batches may be in flight, so IQ pushes (copy engine) and
     * correlation (SMs) overlap.  These are the trk_submit / trk_wait of SURVEY 8b. */
    /* Which correlator kernel a batch runs on.  2 (default): the shared-window kernel (one TMA-staged sample window per group
     * of 8 items) for batches of >= 1024 items with C/A-sized code tables whose consecutive items overlap in the band -
     * known for b200_trk_submit, which sees the items; assumed for b200_trk_batch_dev - and the per-item kernel otherwise.
     * 1: shared-window whenever legal; 0: always per-item; -1: same as 2. */
    int b200_trk_kernel_choice(b200_engine* e, int mode);
    int b200_trk_submit(b200_engine* e, const b200_trk_item* items_host, int n_items, int out_stride, uint64_t* ticket);
    int b200_trk_wait(b200_engine* e, uint64_t ticket, b200_cf32* out_host);
    /* ---- tracking: free-running DLL/PLL loops on the device (SURVEY 8f N1) -------------------- */
    /* One loop = the per-epoch cycle of one dll_pll_veml_tracking block in its tracking state
     * (src/algorithms/tracking/gnuradio_blocks/dll_pll_veml_tracking.cc, general_work case 1 = pull-in
     * alignment :1948-1980 and case 2 :1982-2015: do_correlation_step :1232-1257,
     * cn0_and_tracking_lock_status :1167-1224, run_dll_pll :1260-1347, update_tracking_vars :1409-1483,
     * log_data :1599-1694), evaluated on the device between correlator launches, so that epoch k+1's
     * NCO commands never visit the host.  Types follow the reference member by member (float where it
     * is float, double where it is double).  A loop correlates its own channel (3 or 5 taps) and, when it
     * tracks a pilot and has a data channel (b200_trk_loop_set_data_channel), also the data code at the
     * prompt's shift with the same NCO values, as track_pilot does (:637-668, :1245-1256); both run on the
     * device.  Bit synchronisation, the secondary-code search, extended integration (states 3/4) and
     * telemetry stay with the host, which reads the per-epoch records (and, with a data channel, the pilot
     * prompts of b200_trk_loop_run_prompts).
     * Field names are Dll_Pll_Conf's (src/algorithms/tracking/libs/dll_pll_conf.h:32-89) or the
     * block's own members (dll_pll_veml_tracking.h:128-222). */
    typedef struct b200_trk_loop_conf
    {
        double fs_in;
        double code_chip_rate;       /* d_code_chip_rate */
        double signal_carrier_freq;  /* d_signal_carrier_freq */
        double code_period;          /* d_code_period [s] */
        double carrier_lock_th;
        uint32_t code_length_chips;  /* d_code_length_chips */
        uint32_t vector_length;      /* samples correlated per epoch (adapter: round(fs/(rate/length))) */
        uint32_t pull_in_time_s;
        uint32_t bit_synchronization_time_limit_s; /* fail-safe of :2001-2006; 0xFFFFFFFF disables it */
        uint32_t prn;
        int32_t code_samples_per_chip; /* d_code_samples_per_chip: 1, or 2 for Galileo E1 sinBOC */
        int32_t pll_filter_order;      /* 2 or 3 */
        int32_t dll_filter_order;      /* 1..3 */
        int32_t cn0_samples;           /* <= 64 */
        int32_t cn0_min;
        int32_t max_code_lock_fail;
        int32_t max_carrier_lock_fail;
        int32_t cn0_smoother_samples;
        int32_t carrier_lock_test_smoother_samples;
        int32_t veml;                  /* d_veml: 5 taps VE,E,P,L,VL instead of 3 taps E,P,L */
        int32_t cloop;                 /* d_cloop: Costas discriminator (true unless a pilot is tracked) */
        int32_t carrier_aiding;
        int32_t enable_fll_pull_in;
        int32_t enable_fll_steady_state;
        float pll_bw_hz;
        float dll_bw_hz;
        float fll_bw_hz;
        float early_late_space_chips;  /* becomes Dll_Pll_Conf::spc in state 2 (:1993) */
        float slope;
        float y_intercept;
        float cn0_smoother_alpha;
        float carrier_lock_test_smoother_alpha;
    } b200_trk_loop_conf; /* 152 bytes */

    /* One tracking dump record, byte for byte what log_data() writes per epoch
     * (dll_pll_veml_tracking.cc:1599-1694; read back by
     * tests/unit-tests/signal-processing-blocks/libs/tracking_dump_reader.cc:22-50).  108 bytes,
     * unpadded: the u64 and the double sit on 4-byte boundaries. */
#pragma pack(push, 1)
    typedef struct b200_trk_dump_record
    {
        float abs_VE, abs_E, abs_P, abs_L, abs_VL;
        float prompt_I, prompt_Q;
        uint64_t PRN_start_sample_count; /* nitems_read + d_current_prn_length_samples */
        float acc_carrier_phase_rad;
        float carrier_doppler_hz;
        float carrier_doppler_rate_hz_s;
        float code_freq_chips;
        float code_freq_rate_chips;
        float carr_error_hz;
        float carr_error_filt_hz;
        float code_error_chips;
        float code_error_filt_chips;
        float CN0_SNV_dB_Hz;
        float carrier_lock_test;
        float aux1; /* d_rem_code_phase_samples */
        double aux2;
        uint32_t PRN;
        uint64_t TOW_ms;
        uint32_t WN;
    } b200_trk_dump_record;
#pragma pack(pop)

    /* Loop status word returned by b200_trk_loop_status */
    typedef struct b200_trk_loop_status
    {
        int32_t state;              /* d_state: 0 standby (never started / loss of lock), 1 pull-in, 2 tracking */
        int32_t loss_of_lock;       /* 1 if the last cycle raised the reference's "events" message 3 */
        uint64_t sample_counter;    /* nitems_read(0): absolute index of the next epoch's first sample */
        uint64_t epochs;            /* valid DLL/PLL cycles (= records written) since start */
        double carrier_doppler_hz;
        double code_freq_chips;
        double rem_code_phase_samples;
        double acc_carrier_phase_rad;
        double CN0_SNV_dB_Hz;
        double carrier_lock_test;
    } b200_trk_loop_status;

    /* Create a loop over tracking channel `channel` (b200_trk_channel_create + b200_trk_channel_set_code
     * with the E,P,L / VE,E,P,L,VL shifts of start_tracking :1041-1054).  Filter coefficients are derived
     * here as Tracking_loop_filter::update_coefficients (tracking_loop_filter.cc:86-186) and
     * Tracking_FLL_PLL_filter::set_params (tracking_FLL_PLL_filter.cc:23-54) do.  The loops read gr_complex bands
     * only: a channel on an ishort or ibyte band (b200_iq_create_typed) is B200_ERR_STATE. */
    int b200_trk_loop_create(b200_engine* e, int channel, const b200_trk_loop_conf* conf, int* loop_id);
    /* start_tracking() (:791-1078): take the acquisition result; nitems_read = absolute index of the
     * first sample the tracking block would see next (state 1 then skips to the PRN start). */
    int b200_trk_loop_start(b200_engine* e, int loop_id, double acq_delay_samples, double acq_doppler_hz,
        uint64_t acq_samplestamp_samples, uint64_t nitems_read);
    /* Attach a data channel to a loop that tracks a pilot (track_pilot = true, :637-668, :820-903): every epoch
     * then also correlates data_channel - one correlator, at the pilot prompt's shift, on the loop's band, not
     * high-dynamics; anything else is refused with B200_ERR_ARG, and a channel on a narrow band with B200_ERR_STATE -
     * on the loop's item.  The records' prompt_I /
     * prompt_Q become the data prompt, as log_data writes it (:1614-1617); every other field and the whole loop
     * update keep using the pilot taps.  Accepted before b200_trk_loop_run or between runs; a second call
     * replaces the data channel.  Set cloop as a pilot loop needs it (b200_trk_loop_conf). */
    int b200_trk_loop_set_data_channel(b200_engine* e, int loop_id, int data_channel);
    /* Run up to max_epochs cycles of every started loop: per epoch the correlation of each loop's channel (and of
     * its data channel, if it has one) and the loop update, all on the device; a loop whose next vector_length
     * samples are not all inside its band's [valid_from, write_index) (the window b200_iq_window reports) stalls:
     * samples not pushed yet, overwritten, or left behind by a gap, a restart or b200_iq_forget are never correlated.
     * records_host: n_loops x max_epochs records (loop-major); n_records_host[loop] = cycles logged.
     * Either output may be NULL.  Same as b200_trk_loop_run_prompts with pilot_prompts_host = NULL.
     * B200_ERR_STATE, with nothing launched, while a started loop's channel or data channel sits on a narrow band (its
     * band was re-created with b200_iq_create_typed after the loop was made). */
    int b200_trk_loop_run(b200_engine* e, int max_epochs, b200_trk_dump_record* records_host, int* n_records_host);
    /* b200_trk_loop_run plus the complex pilot prompt of every logged record: pilot_prompts_host (NULL: not
     * returned) is n_loops x max_epochs, loop-major like the records.  With a data channel the record carries the
     * data prompt, and these are what the host's bit synchronisation and secondary-code search read (:2031, :2079). */
    int b200_trk_loop_run_prompts(b200_engine* e, int max_epochs, b200_trk_dump_record* records_host, int* n_records_host,
        b200_cf32* pilot_prompts_host);
    /* How b200_trk_loop_run schedules the work: 0 (default) one persistent kernel, one CTA per loop, free-running
     * for max_epochs cycles with no launch per epoch; 1 a correlator launch + a loop-update launch per epoch with
     * one CTA per loop (same integers as mode 0, floats within an ulp of atanf/log10f: the correlator sums in a different order); 2 the same with each epoch split over several CTAs
     * (lowest latency for a handful of channels). */
    int b200_trk_loop_set_mode(b200_engine* e, int mode);
    /* Prepare (if not already pending) and return the next work item of every loop: the seven scalars
     * do_correlation_step would pass, for hosts that correlate elsewhere.  n == 0 marks a loop in standby.
     * One item per loop: a loop's data item is that item with the data channel's id. */
    int b200_trk_loop_peek_items(b200_engine* e, b200_trk_item* items_host);
    /* One cycle with caller-supplied correlator outputs (taps_host: n_loops x taps of the loop's channel,
     * loop-major, stride = 8; a loop with a data channel takes its data tap in the slot after the pilot taps,
     * 3 after E,P,L or 5 after VE..VL): the loop arithmetic alone, for hosts that correlate elsewhere and for tests. */
    int b200_trk_loop_step_taps(b200_engine* e, const b200_cf32* taps_host, b200_trk_dump_record* records_host, int* logged_host);
    int b200_trk_loop_status_get(b200_engine* e, int loop_id, b200_trk_loop_status* out);
    /* Append records to a tracking dump file in the reference's format (d_dump_file, :1599-1694). */
    int b200_trk_dump_write(const char* filename, const b200_trk_dump_record* records, int n_records, int append);

    /* number of kernel launches issued by this engine so far (bench.py's gpu_launches) */
    int b200_engine_launch_count(b200_engine* e, uint64_t* n);

    /* ---- acquisition: PCPS grid search, 1:1 with the arithmetic of pcps_acquisition ------------- */
    /* src/algorithms/acquisition/gnuradio_blocks/pcps_acquisition.{h,cc}.  One b200_acq holds what one
     * pcps_acquisition block holds (FFT plan, Doppler wipe-off grid, local-code spectra, magnitude
     * grid) for up to n_code_slots PRNs, so that a cold-start sweep can search many PRNs on the
     * same samples while computing the wiped-off forward FFTs once. */
    typedef struct b200_acq_conf
    {
        uint32_t fft_size;            /* d_fft_size            (pcps_acquisition.cc:110) */
        uint32_t effective_fft_size;  /* d_effective_fft_size  (:111) */
        uint32_t consumed_samples;    /* d_consumed_samples    (:109) */
        uint32_t num_doppler_bins;    /* d_num_doppler_bins = ceil(2*doppler_max/doppler_step) (:112) */
        int32_t doppler_max;          /* Acq_Conf::doppler_max   */
        int32_t doppler_step;         /* Acq_Conf::doppler_step  */
        int64_t fs_in;                /* Acq_Conf::fs_in (or resampled_fs) used by update_local_carrier (:277) */
        uint32_t samples_per_chip;    /* Acq_Conf::samples_per_chip (second-peak exclusion window, :485) */
        uint32_t code_layout;         /* set_local_code placement: 0 front (:238-241), 1 bit-transition (:230-235), 2 zero-padded front (:243-246) */
        int32_t bit_transition_flag;  /* magnitudes taken from ifft_out + effective_fft_size (:544) */
        int32_t use_cfar;             /* d_use_CFAR_algorithm_flag: max/input-power (:409-449) else first/second peak (:452-519) */
        uint32_t max_dwells;          /* >1 allocates the magnitude grid so dwells can accumulate (:545-553) */
        uint32_t n_code_slots;        /* local-code spectra kept resident (PRNs searched per call <= this) */
        int32_t keep_grid;            /* 1: always materialise d_magnitude_grid (dump / mag()) */
    } b200_acq_conf;

    typedef struct b200_acq_result
    {
        uint32_t index_time;     /* AcquisitionResult::index_time (first maximum of the winning bin) */
        uint32_t index_doppler;  /* winning Doppler bin */
        int32_t doppler;         /* AcquisitionResult::doppler = -doppler_max + center + step*index_doppler (:432,:476) */
        float test_statistics;   /* AcquisitionResult::test_statistics */
        float grid_maximum;      /* peak |y|^2 */
        float input_power;       /* d_input_power (CFAR) */
        float second_peak;       /* secondPeak (non-CFAR) */
    } b200_acq_result;

    /* pcps_acquisition::pcps_acquisition(conf)  (:100-193): plan, buffers, wipe-off grid for center 0.
     * fft_size: prime factors 2, 3, 5, 7 up to 10 x 27 648 points run on the mixed-radix plans (in shared memory up to 27 648,
     * two-level beyond).  Any other size (16 368 points = 16.368 Msps x 1 ms, ...) runs through chirp-z (Bluestein) on the
     * same kernels, with every code layout, bit_transition_flag, consumed_samples < fft_size, dwells, keep_grid, the assisted
     * Doppler centre and two-step acquisition.  Two limits remain there: use_cfar = 1 is required, and fft_size <= 5 x 27 648.
     * Everything else is B200_ERR_RANGE with the reason in b200_last_error(). */
    int b200_acq_create(b200_engine* e, const b200_acq_conf* conf, b200_acq** out);
    /* set_local_code(code)  (:218-251): code_host holds consumed_samples (layout 0/2) or fft_size/2
     * (layout 1) complex samples; stores conj(FFT(padded code)) in slot `slot`. */
    int b200_acq_set_local_code(b200_acq* a, uint32_t slot, const b200_cf32* code_host);
    /* set_doppler_center / is_fdma bias + update_grid_doppler_wipeoffs  (:254-291) */
    int b200_acq_set_doppler_center(b200_acq* a, int32_t doppler_center, int32_t doppler_bias);
    /* acquisition_core's arithmetic (:648-683): doppler_grid + compute_statistics for n_slots PRNs on
     * the same consumed_samples input.  dwell_counter = d_num_noncoherent_integrations_counter AFTER
     * its increment (1 for the first dwell; >1 accumulates into the magnitude grid).
     * results[i] belongs to slots[i].  Synchronous (input H2D, kernels, results D2H). */
    int b200_acq_search(b200_acq* a, const b200_cf32* in_host, const uint32_t* slots, uint32_t n_slots,
        uint32_t dwell_counter, b200_acq_result* results_host);
    /* Two-step acquisition (Acq_Conf::make_2_steps, pcps_acquisition.cc:294-301,:609-625): after a
     * positive first step the block re-searches num_doppler_bins_step2 bins spaced doppler_step2 around
     * the step-one Doppler on the NEXT buffer of samples.  set_step_two = d_doppler_center_step_two +
     * update_grid_doppler_wipeoffs_step2(); search_step_two = doppler_grid + compute_statistics with
     * d_step_two == true (Doppler from the float formula :436/:480, CFAR input power carried over from
     * step one :428-438).  One PRN slot per call. */
    int b200_acq_set_step_two(b200_acq* a, float doppler_center_step_two, float doppler_step2, uint32_t num_doppler_bins_step2);
    int b200_acq_search_step_two(b200_acq* a, const b200_cf32* in_host, uint32_t slot, uint32_t dwell_counter,
        float prev_input_power, b200_acq_result* result_host);
    /* cshort input (Acq_Conf::it_size == sizeof(lv_16sc_t); the reference converts on the host with
     * volk_gnsssdr_16ic_convert_32fc, pcps_acquisition.cc:653-656): in_host_iq holds 2 * consumed_samples int16
     * (I,Q interleaved); half the PCIe bytes, exact int -> float conversion on the device, then the float path. */
    int b200_acq_search_i16(b200_acq* a, const int16_t* in_host_iq, const uint32_t* slots, uint32_t n_slots,
        uint32_t dwell_counter, b200_acq_result* results_host);
    int b200_acq_search_step_two_i16(b200_acq* a, const int16_t* in_host_iq, uint32_t slot, uint32_t dwell_counter,
        float prev_input_power, b200_acq_result* result_host);
    /* Asynchronous form: submit returns once the sweep is queued (the input is copied first, the caller's buffer
     * is free again), wait blocks for its results.  One sweep may be in flight per acquisition object; objects own
     * their stream, so the sweeps of different channels' blocks overlap on the device as the reference's
     * acquisition threads overlap on the host.  While a sweep is in flight, every search that returns results to the
     * host (b200_acq_search, _i16, _step_two, _step_two_i16, _submit and the band forms below) is refused with
     * B200_ERR_STATE and queues nothing; b200_acq_search_dev is not refused. */
    int b200_acq_search_submit(b200_acq* a, const b200_cf32* in_host, const uint32_t* slots_host, uint32_t n_slots, uint32_t dwell_counter);
    int b200_acq_search_wait(b200_acq* a, b200_acq_result* results_host);
    /* same with the input already on the device and results left on the device (asynchronous) */
    int b200_acq_search_dev(b200_acq* a, const b200_cf32* in_dev, const uint32_t* slots_host, uint32_t n_slots,
        uint32_t dwell_counter, b200_acq_result* results_dev);
    /* Search straight from a band of the acquisition object's engine: the input is samples [abs_index, abs_index +
     * consumed_samples) of `band`, the buffer the reference's block copies its d_consumed_samples from
     * (pcps_acquisition.cc:790-815).  The same samples a host would otherwise keep a second copy of, in host memory, for
     * b200_acq_search; the forward stage reads them where they lie in the ring (a window may wrap around the ring's end),
     * with no extra copy or launch, so a band search issues exactly the kernels b200_acq_search_dev does and computes
     * bit for bit what b200_acq_search computes on the same samples.
     *  - The window must lie inside [valid_from, write_index) as b200_iq_window reports it (the rule b200_trk_submit
     *    applies to work items); attached bands are linear from their first_index.  Otherwise B200_ERR_RANGE, with the
     *    window and the band's window in b200_last_error(), and nothing is launched.  An unused band is B200_ERR_STATE.
     *  - The search is ordered after every b200_iq_push* / b200_iq_refill of the band made before the call, without a host
     *    synchronisation and without waiting for tracking work queued on the engine.
     *  - A later push that laps the ring over a window still queued for a search overwrites what it reads: sizing the
     *    ring so that this cannot happen is the caller's responsibility, as for tracking.
     *  - Successive dwells and step two take the following windows (abs_index + k * consumed_samples), as the block's
     *    successive input buffers.
     *  - The result's sample stamp (Acq_samplestamp_samples, :594) for b200_trk_loop_start is abs_index + consumed_samples.
     *  - The window is resolved when the call is made: these calls are not meant for CUDA-graph capture (that is what
     *    b200_acq_search_dev is for).
     * b200_acq_search_band replaces b200_acq_search (synchronous); b200_acq_search_band_submit replaces
     * b200_acq_search_submit (results through b200_acq_search_wait, one search in flight per object);
     * b200_acq_search_step_two_band replaces b200_acq_search_step_two.
     * With a band resampler set (b200_acq_set_band_resampler below), the window, the dwells and the sample stamp are
     * those given there. */
    int b200_acq_search_band(b200_acq* a, int band, uint64_t abs_index, const uint32_t* slots, uint32_t n_slots,
        uint32_t dwell_counter, b200_acq_result* results_host);
    int b200_acq_search_band_submit(b200_acq* a, int band, uint64_t abs_index, const uint32_t* slots, uint32_t n_slots,
        uint32_t dwell_counter);
    int b200_acq_search_step_two_band(b200_acq* a, int band, uint64_t abs_index, uint32_t slot, uint32_t dwell_counter,
        float prev_input_power, b200_acq_result* result_host);
    /* The acquisition resampler of GNSS-SDR.use_acquisition_resampler = true (gnss_flowgraph.cc:1117-1212): the reference
     * acquires a signal from a full-rate stream at its optimal acquisition rate (2 Msps for GPS L1 C/A, Galileo E1 and L2C,
     * 10 Msps for L5, E5a and E5b) through a decimating low-pass FIR, while tracking stays at the full rate.
     *
     * b200_acq_resampler_design: that filter for a stream at fs_in and a signal whose optimal rate is opt_acq_fs.  Host-only.
     *  - *decimation = floor(fs_in / opt_acq_fs), lowered until it divides fs_in (:1164-1170).  When opt_acq_fs >= fs_in or
     *    the decimation comes out as 1 the reference inserts nothing: *decimation = 1, *n_taps = 0, B200_OK.
     *  - Otherwise the taps of gr::filter::firdes::low_pass(1.0, fs_in, fs_d / 2.1, fs_d / 2) with fs_d = fs_in / decimation:
     *    Hamming window, ntaps = int(53 fs_in / (22 transition)) made odd, windowed sinc scaled to unit DC gain.  Computed
     *    in double, returned as float.  The taps are symmetric; the filter's latency is (n_taps - 1) / 2 full-rate samples.
     *  - More taps than max_taps is B200_ERR_RANGE with the count needed in b200_last_error() and in *n_taps (*decimation
     *    is set too); taps may be NULL when max_taps is 0.
     * The acquisition object for that signal is created at fs_in / decimation, with the sizes Acq_Conf::SetDerivedParams
     * derives from that rate (acq_conf.cc:98-124). */
#define B200_ACQ_MAX_RESAMPLER_TAPS 1024
    int b200_acq_resampler_design(int64_t fs_in, int64_t opt_acq_fs, uint32_t max_taps, uint32_t* decimation, float* taps,
        uint32_t* n_taps);
    /* b200_acq_set_band_resampler: put the decimating filter taps[0..n_taps) in front of this object's band searches
     * (b200_acq_search_band, _band_submit, _step_two_band).  The object works at the decimated rate; its bands hold the full
     * rate.  Input sample j < consumed_samples of a band search becomes y[j] = sum_{k < n_taps} taps[k] x[abs_index + j D - k]
     * (x: the band, D: decimation; k ascending from 0, every product and sum rounded to float on its own), so the search
     * computes bit for bit what b200_acq_search computes on that float32 vector.  The filter runs once per search ahead of
     * the forward stage: a decimated band search issues the kernels of b200_acq_search_dev plus one.
     *  - The span read is [abs_index - (n_taps - 1), abs_index + (consumed_samples - 1) D + 1).  It must lie inside the
     *    band's [valid_from, write_index), or the search is B200_ERR_RANGE with the span and the window in
     *    b200_last_error() and nothing launched.  Samples before a band's first index are not zeros: start at
     *    abs_index >= n_taps - 1.  Every band type works, and a span may wrap around the ring's end.
     *  - Dwell k and step two take abs_index + k consumed_samples D.
     *  - Mapping the result to the full rate is the host's (pcps_acquisition.cc:583-597): the sample stamp for
     *    b200_trk_loop_start is abs_index + consumed_samples D, and the full-rate delay is
     *    fmod(index_time, samples_per_code) D - (n_taps - 1) / 2.
     *  - The host-input searches (b200_acq_search, _i16, _submit, _step_two*) and b200_acq_search_dev ignore the resampler:
     *    their input is already at the object's rate.
     * decimation == 1 turns the resampler off (taps and n_taps are then not read).  decimation == 0, n_taps == 0 or NULL
     * taps is B200_ERR_ARG; n_taps > B200_ACQ_MAX_RESAMPLER_TAPS is B200_ERR_RANGE; a call while a sweep is in flight is
     * B200_ERR_STATE.  The taps are copied to the device before the call returns. */
    int b200_acq_set_band_resampler(b200_acq* a, uint32_t decimation, const float* taps, uint32_t n_taps);
    /* Multi-GPU cold start (SURVEY 8e): the PRN x Doppler grid is sharded by PRN; each rank reduces its sweep to ONE
     * 16-byte record on the device and the ranks exchange the records (an all-gather of N x 16 bytes over NVLink; the
     * host or a peer then takes the best, ties to the lowest PRN / bin / code phase as the reference's strict '>' scans).
     * results_dev: what b200_acq_search_dev left on the device; prn_of_result_dev[i] = PRN searched in results_dev[i].
     * Asynchronous on the acquisition object's stream; no host synchronisation (CUDA-graph capturable). */
    typedef struct b200_acq_peak
    {
        float test_statistics;
        uint32_t prn;
        uint32_t index_doppler;
        uint32_t index_time;
    } b200_acq_peak;
    int b200_acq_sweep_best_dev(b200_acq* a, const b200_acq_result* results_dev, const uint32_t* prn_of_result_dev, uint32_t n_results,
        b200_acq_peak* peak_dev);
    /* d_magnitude_grid of one slot (bins x effective_fft_size floats); needs keep_grid or max_dwells>1.
     * Replaces the grid copy in doppler_grid (:555-558) / dump_results (:354-406). */
    int b200_acq_read_grid(b200_acq* a, uint32_t slot, float* grid_host);
    /* Self-test hook of the transform under the search: out = DFT_fft_size(in) in natural order, computed the way this
     * object computes its spectra (chirp-z objects only; B200_ERR_STATE otherwise).  No reference counterpart: the
     * reference calls gr::fft, whose outputs no reference test holds either. */
    int b200_acq_selftest_dft(b200_acq* a, const b200_cf32* in_host, b200_cf32* out_host);
    /* the wipe-off grid (bins x fft_size complex), for parity tests against volk_gnsssdr_s32f_sincos_32fc */
    int b200_acq_read_wipeoffs(b200_acq* a, b200_cf32* wipe_host);
    int b200_acq_destroy(b200_acq* a);

    /* ---- acquisition: fine Doppler estimate of pcps_acquisition_fine_doppler_cc (SURVEY 8f N4) -------- */
    /* estimate_Doppler() (src/algorithms/acquisition/gnuradio_blocks/pcps_acquisition_fine_doppler_cc.cc:316-389):
     * 10 ms of samples x 10 replicas of the aligned local code, zero-padded 8x, FFT, first maximum of |X[k]|^2.
     * The 80 x fft_size transform is computed as eight (10 x fft_size)-point transforms of the code-wiped signal
     * modulated by eight sub-bin phasors, so the zero padding costs nothing.  fft_size = samples per ms
     * (prime factors 2,3,5,7; <= 27 648).  code_replica_host: fft_size values of
     * gps_l1_ca_code_gen_complex_sampled already rotated as :336-340 do.  *index_freq = tmp_index_freq of :357
     * (0 .. 80 fft_size - 1); the mapping to Hz and the 1 kHz plausibility check (:360-386) are the host's
     * (b200::Pcps_Acquisition_Fine_Doppler_Core).  The coarse grid of the same block is b200_acq with
     * use_cfar = 0, max_dwells and doppler_max = doppler_step (its wipe-offs start at -doppler_step, :172). */
    typedef struct b200_acq_fine b200_acq_fine;
    int b200_acq_fine_create(b200_engine* e, uint32_t fft_size, b200_acq_fine** out);
    int b200_acq_fine_estimate(b200_acq_fine* f, const b200_cf32* buffer_10ms_host, const b200_cf32* code_replica_host,
        uint32_t* index_freq, float* peak);
    /* |X[k]|^2, k = 0 .. 80 fft_size - 1, of the last estimate (parity tests) */
    int b200_acq_fine_read_spectrum(b200_acq_fine* f, float* mag_host);
    int b200_acq_fine_destroy(b200_acq_fine* f);

    /* Acquisition dump (SURVEY 8f N2): the variables pcps_acquisition::dump_results writes
     * (pcps_acquisition.cc:354-406), same names, classes and shapes.  The reference writes them through matio
     * as MAT 7.3 (HDF5); this library writes a Level-5 MAT-file, which matio (hence the reference's
     * acquisition_dump_reader.cc), MATLAB/Octave and scipy read alike; utils/python/plot_acq_grid.py uses h5py
     * and needs the 7.3 container.  Host-only. */
    typedef struct b200_acq_dump
    {
        const float* acq_grid;        /* num_doppler_bins x effective_fft_size, as b200_acq_read_grid returns it */
        const float* acq_grid_narrow; /* make_2_steps only (else NULL): num_doppler_bins_step2 x effective_fft_size */
        uint32_t effective_fft_size;
        uint32_t num_doppler_bins;
        uint32_t num_doppler_bins_step2;
        int32_t doppler_max;
        int32_t doppler_step;
        int32_t positive_acq;
        int32_t num_dwells;
        uint32_t prn;
        float acq_doppler_hz;
        float acq_delay_samples;
        float test_statistic;
        float threshold;
        float input_power;
        float doppler_step_narrow;     /* d_acq_parameters.doppler_step2 */
        float doppler_grid_narrow_min; /* d_doppler_center_step_two - floor(bins2 / 2) * doppler_step2 (:397) */
        uint64_t sample_counter;
    } b200_acq_dump;
    int b200_acq_dump_write(const char* filename, const b200_acq_dump* dump);
    /* <base>_<System>_<Signal>_ch_<channel>_<dump_number>_sat_<PRN>.mat (:357-370) */
    int b200_acq_dump_filename(const char* base, char system, const char* signal2, uint32_t channel, uint32_t dump_number,
        uint32_t prn, char* out, size_t out_size);

#ifdef __cplusplus
}
#endif
#endif /* B200GNSS_H */
