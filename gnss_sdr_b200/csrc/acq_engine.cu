// Host side of the acquisition C ABI (include/b200gnss.h, b200_acq_*): owns what one
// pcps_acquisition block owns (src/algorithms/acquisition/gnuradio_blocks/pcps_acquisition.h:
// FFT plans, d_grid_doppler_wipeoffs, d_fft_codes, d_magnitude_grid) as device buffers.

#include "acq_fft.cuh"
#include "engine.cuh"

#include <cmath>
#include <cstring>
#include <memory>
#include <new>
#include <vector>

using namespace b200;

struct b200_acq
{
    CudaStream stream;  // own, or the engine's; declared first, so released after the buffers used on it
    b200_engine* e{nullptr};
    b200_acq_conf c{};
    FftPlan plan{};
    int doppler_center{0};
    int doppler_bias{0};
    DevBuf<float2> tw;
    DevBuf<float2> wipe;        // bins x n
    DevBuf<float2> X;           // bins x n   forward spectra (digit-reversed)
    DevBuf<float2> codes;       // slots x n  conj(FFT(code)) (digit-reversed)
    DevBuf<float2> in_dev;      // consumed
    DevBuf<short> raw_dev;      // 2 x consumed int16 (cshort input, converted on the device)
    DevBuf<float2> code_stage;
    DevBuf<float> grid;         // slots x bins x ne (optional)
    DevBuf<float2> wipe2;       // step-two wipe-offs (bins2 x n)
    DevBuf<float2> Z;           // two-level FFT only: rows x fft_size inverse-transformed blocks
    DevBuf<AcqRowStat> partial;
    float center2{0.f}, step2{0.f};
    uint32_t bins2{0};
    DevBuf<AcqRowStat> rowstat;
    DevBuf<int> slot_list;
    DevBuf<AcqBest> best;
    DevBuf<float> second_peak;
    DevBuf<b200_acq_result> results_dev;
    PinBuf<b200_acq_result> results_pin;
    PinBuf<int> slot_pin;
    std::vector<char> slot_set;
    // asynchronous search (b200_acq_search_submit / _wait): one sweep in flight per object
    PinBuf<float2> in_pin;
    CudaEvent done;
    uint32_t pending_slots{0};
    bool pending{false};
    std::vector<int> slots_on_device;  // slot list last uploaded (sweeps usually repeat it)
    // band-search resampler (b200_acq_set_band_resampler): band searches read a full-rate span and decimate it into in_dev
    uint32_t decimation{1};            // 1: off
    uint32_t n_taps{0};
    DevBuf<float> resampler_taps;      // B200_ACQ_MAX_RESAMPLER_TAPS
    // Bluestein (chirp-z) path for transform sizes the mixed-radix planner cannot factor (e.g. 16 368 = 2^4 * 3 * 11 * 31):
    // every N-point DFT is a circular convolution with a chirp, done with M-point transforms (M >= 2N-1, two-level plan).
    struct Bluestein
    {
        int M{0};
        FftPlan plM{};
        DevBuf<float2> twM;
        DevBuf<float2> chirp;         // w[k] = exp(+j pi k^2 / N), k < N
        DevBuf<float2> chirp_conj_M;  // conj(w[k]) / M
        DevBuf<float2> chirp_M;       // w[k] / M
        DevBuf<float2> chirp_conj;    // conj(w[k])
        DevBuf<float2> filt;          // 2 x M: FFT_M(h), FFT_M(conj h), h = w extended symmetrically
        DevBuf<float2> mult;          // bins x N: wipe-off . conj(w)
        DevBuf<float2> mult2;         // bins2 x N: step-two wipe-off . conj(w)
        DevBuf<float2> A;             // bins x M spectra of the padded, chirped rows
        DevBuf<float2> Zw;            // bins x M inverse workspace
        DevBuf<float2> Xs;            // bins x N: DFT_N(signal . wipe-off)
        DevBuf<float2> CW;            // slots x N: conj(DFT_N(code)) . w / M
        DevBuf<int> slot_ids;         // device {0, 1}
        DevBuf<AcqRowStat> partial;
    };
    std::unique_ptr<Bluestein> bl;

    ~b200_acq()
    {
        if (stream) cudaStreamSynchronize(stream);
    }
};

namespace
{
// smallest M >= 2N - 1 that the two-level planner accepts
int bluestein_size(int n, FftPlan* pl)
{
    for (long long m = 2LL * n - 1; m <= 10LL * kAcqMaxSmemPoints; m++)
        {
            long long r = m;
            for (int p : {2, 3, 5, 7})
                while (r % p == 0) r /= p;
            if (r != 1) continue;
            if (acq_plan_make_two_level(static_cast<int>(m), pl) == B200_OK) return static_cast<int>(m);
        }
    return 0;
}

// The Doppler rows a search multiplies its input by: the wipe-off rows (wipe, or wipe2 for step two) from the object's
// Doppler settings, and on a chirp-z object their chirped copy, mult[d][i] = wipe[d][i] * conj(w[i]) (mult2 from wipe2):
// the wipe-off grid keeps the reference's float32 sincos values, the chirp is extra.  The chirped copy reads chirp_conj,
// so it needs bluestein_setup first.
int build_rows(b200_acq* a, bool step_two)
{
    const b200_acq_conf& c = a->c;
    const int n = static_cast<int>(c.fft_size);
    const int bins = step_two ? static_cast<int>(a->bins2) : static_cast<int>(c.num_doppler_bins);
    float2* wipe = step_two ? a->wipe2 : a->wipe;
    const int rc = step_two ? acq_launch_wipeoff(wipe, n, bins, 0, 0, 0, a->doppler_bias, c.fs_in, 1, a->center2, a->step2, a->stream)
                            : acq_launch_wipeoff(wipe, n, bins, c.doppler_max, a->doppler_center, c.doppler_step, a->doppler_bias, c.fs_in,
                                  0, 0.f, 0.f, a->stream);
    if (rc || !a->bl) return rc;
    return acq_launch_rows_times_vector(wipe, n, a->bl->chirp_conj, n, 0, step_two ? a->bl->mult2 : a->bl->mult, n, bins, a->stream);
}

int bluestein_setup_queue(b200_acq* a, std::vector<float2> (&host)[6]);

int bluestein_setup(b200_acq* a)
{
    // the host tables must outlive the asynchronous copies queued from them, on the error paths too
    std::vector<float2> host[6];
    const int rc = bluestein_setup_queue(a, host);
    if (a->stream) cudaStreamSynchronize(a->stream);
    return rc;
}

int bluestein_setup_queue(b200_acq* a, std::vector<float2> (&host)[6])
{
    const b200_acq_conf& c = a->c;
    const int n = static_cast<int>(c.fft_size);
    a->bl.reset(new (std::nothrow) b200_acq::Bluestein());
    if (!a->bl) return B200_ERR_NOMEM;
    b200_acq::Bluestein* b = a->bl.get();
    b->M = bluestein_size(n, &b->plM);
    if (b->M == 0)
        {
            set_error("fft_size %d: no chirp-z size M >= 2N-1 within %d points", n, 10 * kAcqMaxSmemPoints);
            return B200_ERR_RANGE;
        }
    const size_t M = static_cast<size_t>(b->M), bins = c.num_doppler_bins, slots = c.n_code_slots;
    B200_CUDA_TRY(b->twM.alloc(M));
    B200_CUDA_TRY(b->chirp.alloc(n));
    B200_CUDA_TRY(b->chirp_conj.alloc(n));
    B200_CUDA_TRY(b->chirp_conj_M.alloc(n));
    B200_CUDA_TRY(b->chirp_M.alloc(n));
    B200_CUDA_TRY(b->filt.alloc(2 * M));
    B200_CUDA_TRY(b->mult.alloc(bins * n));
    B200_CUDA_TRY(b->A.alloc(bins * M));
    B200_CUDA_TRY(b->Zw.alloc(bins * M));
    B200_CUDA_TRY(b->Xs.alloc(bins * n));
    B200_CUDA_TRY(b->CW.alloc(slots * n));
    B200_CUDA_TRY(b->slot_ids.alloc(2));
    B200_CUDA_TRY(b->partial.alloc(bins * acq_final_chunks(b->plM)));
    // every copy below goes through a->stream: a synchronous cudaMemcpy from pageable memory may return before its DMA has
    // landed and is ordered only against the legacy default stream, which a->stream (non-blocking) does not wait for - the
    // filter kernels launched right after it read a half-written chirp (found on sizes with M > 32768)
    static const int ids[2] = {0, 1};
    B200_CUDA_TRY(cudaMemcpyAsync(b->slot_ids, ids, sizeof(ids), cudaMemcpyHostToDevice, a->stream));
    int rc = acq_launch_twiddles(b->twM, b->plM, a->stream);
    if (rc) return rc;
    // chirp tables in double: w[k] = exp(j pi k^2 / N) with k^2 reduced mod 2N
    std::vector<float2>&w = host[0], &wc = host[1], &wcm = host[2], &wm = host[3], &h = host[4], &hc = host[5];
    w.resize(n);
    wc.resize(n);
    wcm.resize(n);
    wm.resize(n);
    h.resize(M);
    hc.resize(M);
    const double inv_m = 1.0 / static_cast<double>(M);
    for (size_t i = 0; i < M; i++) h[i] = hc[i] = make_float2(0.f, 0.f);
    for (int k = 0; k < n; k++)
        {
            const long long k2 = (static_cast<long long>(k) * k) % (2LL * n);
            const double ang = 3.14159265358979323846 * static_cast<double>(k2) / static_cast<double>(n);
            const double cr = std::cos(ang), ci = std::sin(ang);
            w[k] = make_float2(static_cast<float>(cr), static_cast<float>(ci));
            wc[k] = make_float2(static_cast<float>(cr), static_cast<float>(-ci));
            wcm[k] = make_float2(static_cast<float>(cr * inv_m), static_cast<float>(-ci * inv_m));
            wm[k] = make_float2(static_cast<float>(cr * inv_m), static_cast<float>(ci * inv_m));
            h[k] = w[k];
            hc[k] = wc[k];
            if (k > 0)
                {
                    h[M - k] = w[k];
                    hc[M - k] = wc[k];
                }
        }
    B200_CUDA_TRY(cudaMemcpyAsync(b->chirp, w.data(), sizeof(float2) * n, cudaMemcpyHostToDevice, a->stream));
    B200_CUDA_TRY(cudaMemcpyAsync(b->chirp_conj, wc.data(), sizeof(float2) * n, cudaMemcpyHostToDevice, a->stream));
    B200_CUDA_TRY(cudaMemcpyAsync(b->chirp_conj_M, wcm.data(), sizeof(float2) * n, cudaMemcpyHostToDevice, a->stream));
    B200_CUDA_TRY(cudaMemcpyAsync(b->chirp_M, wm.data(), sizeof(float2) * n, cudaMemcpyHostToDevice, a->stream));
    // filter spectra through the code-spectrum kernel, which stores conj(FFT(.)): for a symmetric h, conj(FFT(conj h)) = FFT(h)
    B200_CUDA_TRY(cudaMemcpyAsync(b->A, hc.data(), sizeof(float2) * M, cudaMemcpyHostToDevice, a->stream));
    rc = acq_launch_code_fft(b->A, b->M, 0, b->filt, b->plM, b->twM, a->stream);
    if (rc) return rc;
    B200_CUDA_TRY(cudaMemcpyAsync(b->Zw, h.data(), sizeof(float2) * M, cudaMemcpyHostToDevice, a->stream));
    rc = acq_launch_code_fft(b->Zw, b->M, 0, b->filt + M, b->plM, b->twM, a->stream);
    return rc;
}

// rows x N: out[r] = DFT_N(in[r * in_stride .. ] . mult[r * mult_stride ..])   (forward chirp-z, natural order); inputs past
// `consumed` count as zeros (acquisition_core zero-pads the consumed samples to fft_size, :657-664)
int bluestein_forward_rows(b200_acq* a, AcqInput in, size_t in_stride, int consumed, const float2* mult, size_t mult_stride, int rows,
    float2* out, uint64_t& launched)
{
    b200_acq::Bluestein* b = a->bl.get();
    const int n = static_cast<int>(a->c.fft_size);
    int rc = acq_launch_fwd_rows(in, in_stride, consumed, mult, mult_stride, b->A, rows, b->plM, b->twM, launched, a->stream);
    if (rc) return rc;
    return acq_launch_inverse_store_rows(b->A, b->filt, b->slot_ids, rows, b->plM, b->twM, b->Zw, b->chirp_conj_M, n, out, n, launched,
        a->stream);
}

// One sweep over n_slots code slots on the samples `in`, records into results_dev; launches counted on success only
int search_impl(b200_acq* a, AcqInput in, const uint32_t* slots, uint32_t n_slots, uint32_t dwell_counter,
    b200_acq_result* results_dev, int step_two = 0, float prev_input_power = 0.f)
{
    const b200_acq_conf& c = a->c;
    if (n_slots == 0) return B200_OK;
    if (n_slots > c.n_code_slots || !slots) return B200_ERR_ARG;
    if (dwell_counter < 1) dwell_counter = 1;
    if (dwell_counter > 1 && !a->grid)
        {
            set_error("dwell_counter %u needs the magnitude grid (create with max_dwells > 1 or keep_grid)", dwell_counter);
            return B200_ERR_STATE;
        }
    for (uint32_t i = 0; i < n_slots; i++)
        {
            if (slots[i] >= c.n_code_slots || !a->slot_set[slots[i]])
                {
                    set_error("slot %u has no local code", slots[i]);
                    return B200_ERR_STATE;
                }
        }
    b200_acq::Bluestein* b = a->bl.get();
    const float2* rows = b ? (step_two ? b->mult2 : b->mult) : (step_two ? a->wipe2 : a->wipe);  // what build_rows built
    if (step_two && (a->bins2 == 0 || !rows || n_slots != 1))
        {
            set_error("step two needs b200_acq_set_step_two first and exactly one slot");
            return B200_ERR_STATE;
        }
    const int bins = step_two ? static_cast<int>(a->bins2) : static_cast<int>(c.num_doppler_bins);
    const int ne = static_cast<int>(c.effective_fft_size);
    const int off = c.bit_transition_flag ? ne : 0;
    const int accumulate = dwell_counter > 1 ? 1 : 0;
    cudaStream_t st = a->stream;
    uint64_t launched = 0;
    int rc;
    if (b)
        {
            // X_d = DFT_N(x . wipe_d) for every Doppler bin, once per sweep (x: the consumed samples, zero-padded to N)
            const int n = static_cast<int>(c.fft_size);
            rc = bluestein_forward_rows(a, in, 0, static_cast<int>(c.consumed_samples), rows, n, bins, b->Xs, launched);
            if (rc) return rc;
            for (uint32_t i = 0; i < n_slots; i++)
                {
                    // rows of this PRN: y = IDFT_N(X_d . C) = w . IFFT_M(FFT_M(pad(X_d . C . w)) . FFT_M(conj h)) / M ; |w| = 1
                    rc = acq_launch_fwd_rows(AcqInput::linear(b->Xs), n, n, b->CW + static_cast<size_t>(slots[i]) * n, 0, b->A, bins, b->plM, b->twM, launched, st);
                    if (rc) return rc;
                    // the correlation kernel addresses the grid by code-slot id, and the "code" here is filter slot 1; the grid rows are
                    // [off, off + ne) of y, so slot s lands where the mixed-radix search puts it: (s * bins + bin) * ne
                    float* grid = a->grid ? a->grid + (static_cast<ptrdiff_t>(slots[i]) - 1) * static_cast<ptrdiff_t>(bins) * ne : nullptr;
                    rc = acq_launch_row_stats(b->A, b->filt, b->slot_ids + 1, 1, bins, b->plM, b->twM, off, ne, grid, accumulate,
                        a->rowstat + static_cast<size_t>(i) * bins, b->Zw, b->partial, launched, st);
                    if (rc) return rc;
                }
        }
    else
        {
            bool same = a->slots_on_device.size() == n_slots;
            for (uint32_t i = 0; same && i < n_slots; i++) same = a->slots_on_device[i] == static_cast<int>(slots[i]);
            if (!same)
                {
                    // slot_pin is read by the asynchronous copy: wait for a previous upload's reader before rewriting it
                    B200_CUDA_TRY(cudaStreamSynchronize(st));
                    for (uint32_t i = 0; i < n_slots; i++) a->slot_pin[i] = static_cast<int>(slots[i]);
                    B200_CUDA_TRY(cudaMemcpyAsync(a->slot_list, a->slot_pin, sizeof(int) * n_slots, cudaMemcpyHostToDevice, st));
                    a->slots_on_device.assign(a->slot_pin.get(), a->slot_pin.get() + n_slots);
                }
            rc = acq_launch_fwd(in, static_cast<int>(c.consumed_samples), rows, a->X, bins, a->plan, a->tw, launched, st);
            if (rc) return rc;
            rc = acq_launch_row_stats(a->X, a->codes, a->slot_list, static_cast<int>(n_slots), bins, a->plan, a->tw, off, ne, a->grid,
                accumulate, a->rowstat, a->Z, a->partial, launched, st);
            if (rc) return rc;
        }
    rc = acq_launch_stats(a->rowstat, static_cast<int>(n_slots), bins, ne, c.doppler_max, a->doppler_center, c.doppler_step, dwell_counter,
        c.use_cfar, a->best, results_dev, step_two, a->center2, a->step2, prev_input_power, launched, st);
    if (rc) return rc;
    if (!c.use_cfar)  // mixed radix only: b200_acq_create takes the chirp-z path with use_cfar only
        {
            rc = acq_launch_second_peak(a->X, a->codes, a->slot_list, static_cast<int>(n_slots), bins, a->plan, a->tw, off, ne, a->grid,
                a->best, static_cast<int>(c.samples_per_chip), a->second_peak, a->Z, a->partial, launched, st);
            if (rc) return rc;
            rc = acq_launch_finish_second_peak(a->second_peak, static_cast<int>(n_slots), results_dev, launched, st);
            if (rc) return rc;
        }
    a->e->launches += launched;
    return B200_OK;
}

// The samples of one search that returns its records to the host: consumed_samples complex values in the caller's memory,
// as b200_cf32 or as I,Q-interleaved int16, or samples [abs_index, abs_index + consumed_samples) of one of the engine's bands
// (with a band resampler set, the span decimate_band reads)
struct SearchSource
{
    enum Kind { kHostF32, kHostI16, kBand } kind;
    const void* host;
    int band;
    uint64_t abs_index;
};
}  // namespace

extern "C"
{
    int b200_acq_create(b200_engine* e, const b200_acq_conf* conf, b200_acq** out)
    {
        if (!e || !conf || !out) return B200_ERR_ARG;
        *out = nullptr;
        const b200_acq_conf& c = *conf;
        if (c.fft_size < 2 || c.effective_fft_size < 1 || c.effective_fft_size > c.fft_size || c.consumed_samples < 1 ||
            c.consumed_samples > c.fft_size || c.num_doppler_bins < 1 || c.n_code_slots < 1 || c.code_layout > 2 || c.fs_in <= 0)
            {
                set_error("b200_acq_create: inconsistent configuration");
                return B200_ERR_ARG;
            }
        if (c.bit_transition_flag && 2 * c.effective_fft_size > c.fft_size) return B200_ERR_ARG;
        FftPlan pl{};
        int rc = acq_plan_make(static_cast<int>(c.fft_size), &pl);
        bool use_bluestein = false;
        if (rc)
            {
                // sizes with prime factors > 7 (16 368 = 16.368 Msps x 1 ms, a standard front-end rate): chirp-z through M-point
                // transforms, every code layout; the CFAR statistic only, and N <= 5 x 27 648 (M <= 10 x 27 648, two-level plan)
                FftPlan probe{};
                if (c.use_cfar && bluestein_size(static_cast<int>(c.fft_size), &probe) != 0)
                    {
                        use_bluestein = true;
                        pl = FftPlan{};
                        pl.n = static_cast<int>(c.fft_size);
                        pl.n_total = pl.n;
                        pl.n1 = 1;
                    }
                else
                    {
                        set_error("fft_size %u unsupported: prime factors must be 2,3,5,7 and fft_size <= 10 x %d (sizes with larger prime "
                                  "factors need use_cfar = 1 and fft_size <= %d)",
                            c.fft_size, kAcqMaxSmemPoints, 5 * kAcqMaxSmemPoints);
                        return rc;
                    }
            }
        B200_ENTER_DEVICE(e->device);
        std::unique_ptr<b200_acq> a(new (std::nothrow) b200_acq());
        if (!a) return B200_ERR_NOMEM;
        a->e = e;
        a->c = c;
        a->plan = pl;
        a->slot_set.assign(c.n_code_slots, 0);
        const size_t n = c.fft_size, bins = c.num_doppler_bins, slots = c.n_code_slots, ne = c.effective_fft_size;
        if (e->stream.owned())
            B200_CUDA_TRY(a->stream.create(cudaStreamNonBlocking));  // one private stream per acquisition object: blocks of different channels overlap
        else
            a->stream.borrow(e->stream);  // caller-owned stream (e.g. for event timing on that stream)
        B200_CUDA_TRY(a->tw.alloc(n));
        B200_CUDA_TRY(a->wipe.alloc(n * bins));
        B200_CUDA_TRY(a->X.alloc(n * bins));
        B200_CUDA_TRY(a->codes.alloc(n * slots));
        B200_CUDA_TRY(a->in_dev.alloc(n));
        B200_CUDA_TRY(a->code_stage.alloc(n));
        B200_CUDA_TRY(a->rowstat.alloc(bins * slots));
        B200_CUDA_TRY(a->slot_list.alloc(slots));
        B200_CUDA_TRY(a->best.alloc(slots));
        B200_CUDA_TRY(a->second_peak.alloc(slots));
        B200_CUDA_TRY(a->results_dev.alloc(slots));
        B200_CUDA_TRY(a->results_pin.alloc(slots));
        B200_CUDA_TRY(a->slot_pin.alloc(slots));
        if (pl.n1 > 1)
            {
                const size_t rows = bins * slots;
                cudaError_t zerr = a->Z.alloc(n * rows);
                if (zerr != cudaSuccess)
                    {
                        set_error("two-level FFT workspace (%zu bytes): %s", sizeof(float2) * n * rows, cudaGetErrorString(zerr));
                        return B200_ERR_NOMEM;
                    }
                B200_CUDA_TRY(a->partial.alloc(rows * acq_final_chunks(pl)));
            }
        if (c.max_dwells > 1 || c.keep_grid)
            {
                cudaError_t err = a->grid.alloc(ne * bins * slots);
                if (err != cudaSuccess)
                    {
                        set_error("magnitude grid (%zu bytes): %s", sizeof(float) * ne * bins * slots, cudaGetErrorString(err));
                        return B200_ERR_NOMEM;
                    }
                B200_CUDA_TRY(cudaMemsetAsync(a->grid, 0, sizeof(float) * ne * bins * slots, a->stream));
            }
        rc = use_bluestein ? bluestein_setup(a.get()) : acq_launch_twiddles(a->tw, a->plan, a->stream);
        if (rc) return rc;
        rc = build_rows(a.get(), false);
        if (rc) return rc;
        B200_CUDA_TRY(cudaStreamSynchronize(a->stream));
        *out = a.release();
        return B200_OK;
    }


    int b200_acq_set_local_code(b200_acq* a, uint32_t slot, const b200_cf32* code_host)
    {
        if (!a || !code_host || slot >= a->c.n_code_slots) return B200_ERR_ARG;
        B200_ENTER_DEVICE(a->e->device);
        const b200_acq_conf& c = a->c;
        const size_t need = (c.code_layout == 1) ? c.fft_size / 2 : c.consumed_samples;
        if (a->bl)
            {
                // the code staged in an N-point buffer where set_local_code places it (acq_code_offset), zeros elsewhere
                b200_acq::Bluestein* b = a->bl.get();
                const int n = static_cast<int>(c.fft_size);
                const int place = acq_code_offset(static_cast<int>(c.code_layout), n, static_cast<int>(c.consumed_samples));
                if (need < c.fft_size) B200_CUDA_TRY(cudaMemsetAsync(a->code_stage, 0, sizeof(float2) * c.fft_size, a->stream));
                B200_CUDA_TRY(cudaMemcpyAsync(a->code_stage + place, code_host, sizeof(float2) * need, cudaMemcpyHostToDevice, a->stream));
                // CW = conj(DFT_N(code)) . w / M  (volk_32fc_conjugate_32fc of set_local_code :250, then the inverse chirp-z pre-multiplier)
                uint64_t setup_launches = 0;  // set-up, not counted
                int rcb = bluestein_forward_rows(a, AcqInput::linear(a->code_stage), 0, n, b->chirp_conj, 0, 1, b->Xs, setup_launches);
                if (rcb) return rcb;
                rcb = acq_launch_rows_times_vector(b->Xs, n, b->chirp_M, n, 1, b->CW + static_cast<size_t>(slot) * n, n, 1, a->stream);
                if (rcb) return rcb;
                B200_CUDA_TRY(cudaStreamSynchronize(a->stream));
                a->slot_set[slot] = 1;
                return B200_OK;
            }
        B200_CUDA_TRY(cudaMemcpyAsync(a->code_stage, code_host, sizeof(float2) * need, cudaMemcpyHostToDevice, a->stream));
        int rc = acq_launch_code_fft(a->code_stage, static_cast<int>(c.consumed_samples), static_cast<int>(c.code_layout),
            a->codes + static_cast<size_t>(slot) * c.fft_size, a->plan, a->tw, a->stream);
        if (rc) return rc;
        B200_CUDA_TRY(cudaStreamSynchronize(a->stream));
        a->slot_set[slot] = 1;
        return B200_OK;
    }

    int b200_acq_set_doppler_center(b200_acq* a, int32_t doppler_center, int32_t doppler_bias)
    {
        if (!a) return B200_ERR_ARG;
        B200_ENTER_DEVICE(a->e->device);
        a->doppler_center = doppler_center;
        a->doppler_bias = doppler_bias;
        const int rc = build_rows(a, false);
        if (rc) return rc;
        B200_CUDA_TRY(cudaStreamSynchronize(a->stream));
        return B200_OK;
    }

    // B200_ERR_STATE while a submitted search still has results to collect
    static int check_no_search_in_flight(const b200_acq* a)
    {
        if (!a->pending) return B200_OK;
        set_error("a search is already in flight on this acquisition object: call b200_acq_search_wait");
        return B200_ERR_STATE;
    }

    // Host input of either format crosses the same way: into pinned memory (the caller's buffer is free as soon as the call
    // returns, and the copy is truly asynchronous), then one copy on a->stream.  cshort input (pcps_acquisition.cc:653-656
    // converts with volk_gnsssdr_16ic_convert_32fc on the host): the raw 16-bit pairs cross PCIe (half the bytes) and become
    // float2 on the device; int -> float is exact, so results are those of the float path on the converted samples.
    static int stage_host(b200_acq* a, const SearchSource& src)
    {
        const size_t n = a->c.consumed_samples;
        const bool i16 = src.kind == SearchSource::kHostI16;
        const size_t bytes = i16 ? sizeof(int16_t) * 2 * n : sizeof(float2) * n;
        if (!a->in_pin) B200_CUDA_TRY(a->in_pin.alloc(a->c.fft_size));
        if (i16 && !a->raw_dev) B200_CUDA_TRY(a->raw_dev.alloc(2 * a->c.fft_size));
        std::memcpy(a->in_pin, src.host, bytes);
        void* dst = i16 ? static_cast<void*>(a->raw_dev.get()) : static_cast<void*>(a->in_dev.get());
        B200_CUDA_TRY(cudaMemcpyAsync(dst, a->in_pin, bytes, cudaMemcpyHostToDevice, a->stream));
        if (!i16) return B200_OK;
        const int rc = launch_convert_i16(a->raw_dev, a->in_dev, ~0ULL, 0ULL, n, a->stream);
        if (rc == B200_OK) a->e->launches++;
        return rc;
    }

    // The view of samples [abs_index, abs_index + n) of one of the engine's bands, with a->stream made to wait for every
    // write to the band queued so far.  The window check and the waits share one critical section of e->mu, so no
    // push can be queued between them.  Float pushes and refills are copies on the copy stream (copy_done marks the latest);
    // integer pushes are converted on the compute stream, and raw_free[raw_last] follows the band's latest conversion; a band
    // a conditioner fills is written on the compute stream too, and cond_done follows its latest launch.  The search waits
    // for those events only, not for the whole compute stream, so it never queues behind tracking batches.
    static int band_input(b200_acq* a, int band, unsigned long long abs_index, unsigned long long n, AcqInput* in)
    {
        if (band < 0 || band >= kMaxBands) return B200_ERR_ARG;
        b200_engine* e = a->e;
        std::lock_guard<std::mutex> lk(e->mu);
        const Band& b = e->bands[band];
        if (!b.in_use)
            {
                set_error("band %d holds no samples (call b200_iq_create or b200_iq_attach_dev)", band);
                return B200_ERR_STATE;
            }
        if (!b.holds(abs_index, n))
            {
                set_error("band %d: samples [%llu, %llu) are outside the band's window [%llu, %llu)", band, (unsigned long long)abs_index,
                    (unsigned long long)abs_index + n, b.window_lo(), b.write_index);
                return B200_ERR_RANGE;
            }
        B200_CUDA_TRY(cudaStreamWaitEvent(a->stream, e->copy_done, 0));
        if (b.raw_last >= 0) B200_CUDA_TRY(cudaStreamWaitEvent(a->stream, b.raw_free[b.raw_last], 0));
        if (b.cond_recorded) B200_CUDA_TRY(cudaStreamWaitEvent(a->stream, b.cond_done, 0));
        // a ring window may wrap around the ring's end; an attached buffer is linear from first_index (mask ~0), and the
        // window check keeps the window inside it.  A narrow band is read at its own width (AcqInput::at widens on load).
        const unsigned long long off = (abs_index - b.first_index) & b.mask;
        const unsigned long long run = b.capacity - off;
        *in = AcqInput{static_cast<const char*>(b.base) + off * 2ULL * b.fmt, static_cast<int>(n < run ? n : run), b.base, b.fmt};
        return B200_OK;
    }

    // A band search through the resampler: the span [abs_index - (T - 1), abs_index + (consumed - 1) D + 1) of the band,
    // filtered and decimated into in_dev, in_dev[j] = sum_k h[k] x[abs_index + j D - k]; one launch more than a plain band
    // search, and a refused span launches nothing.
    static int decimate_band(b200_acq* a, int band, uint64_t abs_index)
    {
        const uint64_t history = a->n_taps - 1, n_out = a->c.consumed_samples;
        const uint64_t count = history + (n_out - 1) * a->decimation + 1;
        if (abs_index < history)
            {
                set_error("band %d: the resampler's span of sample %llu starts %llu samples before index 0 (start at index >= %llu)", band,
                    (unsigned long long)abs_index, (unsigned long long)(history - abs_index), (unsigned long long)history);
                return B200_ERR_RANGE;
            }
        if (count > 0x7fffffffULL)
            {
                set_error("band %d: the resampler's span of %llu samples exceeds 2^31 - 1", band, (unsigned long long)count);
                return B200_ERR_RANGE;
            }
        AcqInput span{};
        int rc = band_input(a, band, abs_index - history, count, &span);
        if (rc) return rc;
        uint64_t launched = 0;
        rc = acq_launch_decimate(span, a->resampler_taps, static_cast<int>(a->n_taps), static_cast<int>(a->decimation), static_cast<int>(n_out),
            a->in_dev, launched, a->stream);
        if (rc) return rc;
        a->e->launches += launched;
        return B200_OK;
    }

    // Every search that returns its records to the host goes through here: refused while a sweep is in flight, it stages
    // the input, queues the search on a->stream and its n_slots records into results_pin, and records `done` for
    // b200_acq_search_wait.
    static int submit_search(b200_acq* a, const SearchSource& src, const uint32_t* slots, uint32_t n_slots, uint32_t dwell_counter,
        int step_two, float prev_input_power)
    {
        if (!a || (src.kind != SearchSource::kBand && !src.host)) return B200_ERR_ARG;
        if (const int rc = check_no_search_in_flight(a)) return rc;
        B200_ENTER_DEVICE(a->e->device);
        AcqInput in = AcqInput::linear(a->in_dev);
        int rc = src.kind != SearchSource::kBand ? stage_host(a, src)
                 : a->decimation > 1              ? decimate_band(a, src.band, src.abs_index)
                                                  : band_input(a, src.band, src.abs_index, a->c.consumed_samples, &in);
        if (rc) return rc;
        rc = search_impl(a, in, slots, n_slots, dwell_counter, a->results_dev, step_two, prev_input_power);
        if (rc) return rc;
        if (!a->done) B200_CUDA_TRY(a->done.create(cudaEventDisableTiming));
        B200_CUDA_TRY(cudaMemcpyAsync(a->results_pin, a->results_dev, sizeof(b200_acq_result) * n_slots, cudaMemcpyDeviceToHost, a->stream));
        B200_CUDA_TRY(cudaEventRecord(a->done, a->stream));
        a->pending = true;
        a->pending_slots = n_slots;
        return B200_OK;
    }

    // the synchronous searches: submit_search, then b200_acq_search_wait
    static int search_and_wait(b200_acq* a, const SearchSource& src, const uint32_t* slots, uint32_t n_slots, uint32_t dwell_counter,
        int step_two, float prev_input_power, b200_acq_result* results_host)
    {
        if (!results_host) return B200_ERR_ARG;
        const int rc = submit_search(a, src, slots, n_slots, dwell_counter, step_two, prev_input_power);
        return rc ? rc : b200_acq_search_wait(a, results_host);
    }

    int b200_acq_search_submit(b200_acq* a, const b200_cf32* in_host, const uint32_t* slots, uint32_t n_slots, uint32_t dwell_counter)
    {
        return submit_search(a, SearchSource{SearchSource::kHostF32, in_host}, slots, n_slots, dwell_counter, 0, 0.f);
    }

    int b200_acq_search_wait(b200_acq* a, b200_acq_result* results_host)
    {
        if (!a || !results_host) return B200_ERR_ARG;
        if (!a->pending)
            {
                set_error("no search in flight on this acquisition object");
                return B200_ERR_STATE;
            }
        B200_ENTER_DEVICE(a->e->device);
        B200_CUDA_TRY(cudaEventSynchronize(a->done));
        std::memcpy(results_host, a->results_pin, sizeof(b200_acq_result) * a->pending_slots);
        a->pending = false;
        return B200_OK;
    }

    int b200_acq_search(b200_acq* a, const b200_cf32* in_host, const uint32_t* slots, uint32_t n_slots,
        uint32_t dwell_counter, b200_acq_result* results_host)
    {
        return search_and_wait(a, SearchSource{SearchSource::kHostF32, in_host}, slots, n_slots, dwell_counter, 0, 0.f, results_host);
    }

    int b200_acq_search_i16(b200_acq* a, const int16_t* in_host_iq, const uint32_t* slots, uint32_t n_slots, uint32_t dwell_counter,
        b200_acq_result* results_host)
    {
        return search_and_wait(a, SearchSource{SearchSource::kHostI16, in_host_iq}, slots, n_slots, dwell_counter, 0, 0.f, results_host);
    }

    int b200_acq_search_step_two_i16(b200_acq* a, const int16_t* in_host_iq, uint32_t slot, uint32_t dwell_counter, float prev_input_power,
        b200_acq_result* result_host)
    {
        return search_and_wait(a, SearchSource{SearchSource::kHostI16, in_host_iq}, &slot, 1, dwell_counter, 1, prev_input_power, result_host);
    }

    int b200_acq_set_step_two(b200_acq* a, float doppler_center_step_two, float doppler_step2, uint32_t num_doppler_bins_step2)
    {
        if (!a || num_doppler_bins_step2 < 1) return B200_ERR_ARG;
        if (num_doppler_bins_step2 > a->c.num_doppler_bins)
            {
                set_error("step-two bins %u exceed the grid's %u rows", num_doppler_bins_step2, a->c.num_doppler_bins);
                return B200_ERR_RANGE;
            }
        B200_ENTER_DEVICE(a->e->device);
        if (!a->wipe2 || a->bins2 < num_doppler_bins_step2)
            {
                B200_CUDA_TRY(cudaStreamSynchronize(a->stream));
                B200_CUDA_TRY(a->wipe2.alloc(a->c.fft_size * num_doppler_bins_step2));
            }
        if (a->bl && !a->bl->mult2.fits(a->c.fft_size * num_doppler_bins_step2))
            {
                B200_CUDA_TRY(cudaStreamSynchronize(a->stream));
                B200_CUDA_TRY(a->bl->mult2.alloc(a->c.fft_size * num_doppler_bins_step2));
            }
        a->bins2 = num_doppler_bins_step2;
        a->center2 = doppler_center_step_two;
        a->step2 = doppler_step2;
        const int rc = build_rows(a, true);
        if (rc) return rc;
        B200_CUDA_TRY(cudaStreamSynchronize(a->stream));
        return B200_OK;
    }

    int b200_acq_search_step_two(b200_acq* a, const b200_cf32* in_host, uint32_t slot, uint32_t dwell_counter, float prev_input_power,
        b200_acq_result* result_host)
    {
        return search_and_wait(a, SearchSource{SearchSource::kHostF32, in_host}, &slot, 1, dwell_counter, 1, prev_input_power, result_host);
    }

    // Not a submit_search path, and not refused while a sweep is in flight: the input is on the device and the records stay
    // there, so it touches neither in_pin nor results_pin, and it must stay capturable in a CUDA graph.  (search_impl
    // synchronises by itself when - and only when - the slot list changed and slot_pin must be rewritten; a repeated sweep
    // over the same slots issues no host synchronisation.)
    int b200_acq_search_dev(b200_acq* a, const b200_cf32* in_dev, const uint32_t* slots_host, uint32_t n_slots,
        uint32_t dwell_counter, b200_acq_result* results_dev)
    {
        if (!a || !in_dev || !results_dev) return B200_ERR_ARG;
        B200_ENTER_DEVICE(a->e->device);
        return search_impl(a, AcqInput::linear(reinterpret_cast<const float2*>(in_dev)), slots_host, n_slots, dwell_counter, results_dev);
    }

    int b200_acq_search_band_submit(b200_acq* a, int band, uint64_t abs_index, const uint32_t* slots, uint32_t n_slots, uint32_t dwell_counter)
    {
        return submit_search(a, SearchSource{SearchSource::kBand, nullptr, band, abs_index}, slots, n_slots, dwell_counter, 0, 0.f);
    }

    int b200_acq_search_band(b200_acq* a, int band, uint64_t abs_index, const uint32_t* slots, uint32_t n_slots, uint32_t dwell_counter,
        b200_acq_result* results_host)
    {
        return search_and_wait(a, SearchSource{SearchSource::kBand, nullptr, band, abs_index}, slots, n_slots, dwell_counter, 0, 0.f,
            results_host);
    }

    int b200_acq_search_step_two_band(b200_acq* a, int band, uint64_t abs_index, uint32_t slot, uint32_t dwell_counter, float prev_input_power,
        b200_acq_result* result_host)
    {
        return search_and_wait(a, SearchSource{SearchSource::kBand, nullptr, band, abs_index}, &slot, 1, dwell_counter, 1, prev_input_power,
            result_host);
    }

    int b200_acq_set_band_resampler(b200_acq* a, uint32_t decimation, const float* taps, uint32_t n_taps)
    {
        if (!a) return B200_ERR_ARG;
        if (const int rc = check_no_search_in_flight(a)) return rc;
        if (decimation == 1)
            {
                a->decimation = 1;
                a->n_taps = 0;
                return B200_OK;
            }
        if (decimation == 0 || n_taps == 0 || !taps)
            {
                set_error("b200_acq_set_band_resampler: decimation %u with %u taps at %p", decimation, n_taps, static_cast<const void*>(taps));
                return B200_ERR_ARG;
            }
        if (n_taps > B200_ACQ_MAX_RESAMPLER_TAPS)
            {
                set_error("b200_acq_set_band_resampler: %u taps, at most %d", n_taps, B200_ACQ_MAX_RESAMPLER_TAPS);
                return B200_ERR_RANGE;
            }
        B200_ENTER_DEVICE(a->e->device);
        if (!a->resampler_taps) B200_CUDA_TRY(a->resampler_taps.alloc(B200_ACQ_MAX_RESAMPLER_TAPS));
        // synchronised: the caller's taps are free again on return, and no earlier search on the stream still reads the old ones
        B200_CUDA_TRY(cudaStreamSynchronize(a->stream));
        B200_CUDA_TRY(cudaMemcpyAsync(a->resampler_taps, taps, sizeof(float) * n_taps, cudaMemcpyHostToDevice, a->stream));
        B200_CUDA_TRY(cudaStreamSynchronize(a->stream));
        a->decimation = decimation;
        a->n_taps = n_taps;
        return B200_OK;
    }

    int b200_acq_sweep_best_dev(b200_acq* a, const b200_acq_result* results_dev, const uint32_t* prn_of_result_dev, uint32_t n_results,
        b200_acq_peak* peak_dev)
    {
        if (!a || !results_dev || !prn_of_result_dev || !peak_dev) return B200_ERR_ARG;
        uint64_t launched = 0;
        const int rc = acq_launch_sweep_best(results_dev, prn_of_result_dev, static_cast<int>(n_results), peak_dev, launched, a->stream);
        if (rc) return rc;
        a->e->launches += launched;
        return B200_OK;
    }

    int b200_acq_selftest_dft(b200_acq* a, const b200_cf32* in_host, b200_cf32* out_host)
    {
        if (!a || !in_host || !out_host) return B200_ERR_ARG;
        if (!a->bl)
            {
                set_error("selftest_dft: not a chirp-z object");
                return B200_ERR_STATE;
            }
        B200_ENTER_DEVICE(a->e->device);
        const size_t n = a->c.fft_size;
        B200_CUDA_TRY(cudaMemcpyAsync(a->code_stage, in_host, sizeof(float2) * n, cudaMemcpyHostToDevice, a->stream));
        uint64_t selftest_launches = 0;  // a self-test, not a search: not counted
        const int rc = bluestein_forward_rows(a, AcqInput::linear(a->code_stage), 0, static_cast<int>(n), a->bl->chirp_conj, 0, 1, a->bl->Xs, selftest_launches);
        if (rc) return rc;
        B200_CUDA_TRY(cudaMemcpyAsync(out_host, a->bl->Xs, sizeof(float2) * n, cudaMemcpyDeviceToHost, a->stream));
        B200_CUDA_TRY(cudaStreamSynchronize(a->stream));
        return B200_OK;
    }

    int b200_acq_read_grid(b200_acq* a, uint32_t slot, float* grid_host)
    {
        if (!a || !grid_host || slot >= a->c.n_code_slots) return B200_ERR_ARG;
        if (!a->grid)
            {
                set_error("no magnitude grid: create with keep_grid or max_dwells > 1");
                return B200_ERR_STATE;
            }
        B200_ENTER_DEVICE(a->e->device);
        const size_t row = static_cast<size_t>(a->c.num_doppler_bins) * a->c.effective_fft_size;
        B200_CUDA_TRY(cudaMemcpyAsync(grid_host, a->grid + row * slot, sizeof(float) * row, cudaMemcpyDeviceToHost, a->stream));
        B200_CUDA_TRY(cudaStreamSynchronize(a->stream));
        return B200_OK;
    }

    int b200_acq_read_wipeoffs(b200_acq* a, b200_cf32* wipe_host)
    {
        if (!a || !wipe_host) return B200_ERR_ARG;
        B200_ENTER_DEVICE(a->e->device);
        B200_CUDA_TRY(cudaMemcpyAsync(wipe_host, a->wipe, sizeof(float2) * a->c.fft_size * a->c.num_doppler_bins, cudaMemcpyDeviceToHost, a->stream));
        B200_CUDA_TRY(cudaStreamSynchronize(a->stream));
        return B200_OK;
    }

    int b200_acq_destroy(b200_acq* a)
    {
        if (!a) return B200_ERR_ARG;
        cudaSetDevice(a->e->device);
        delete a;
        return B200_OK;
    }
}
