// Host side of the free-running DLL/PLL loops (include/b200gnss.h, "tracking: free-running DLL/PLL loops").
// Configuration-time arithmetic only: filter coefficients and start-of-tracking state; the per-epoch cycle is
// loop_kernels_nofma.cu.
//
//   Tracking_loop_filter::update_coefficients   src/algorithms/tracking/libs/tracking_loop_filter.cc:99-196
//   Tracking_FLL_PLL_filter::set_params         src/algorithms/tracking/libs/tracking_FLL_PLL_filter.cc:23-54
//   Tracking_FLL_PLL_filter::initialize         :57-69
//   dll_pll_veml_tracking ctor / start_tracking src/algorithms/tracking/gnuradio_blocks/dll_pll_veml_tracking.cc:97-146,601-605,680-694,791-1078
//   Exponential_Smoother defaults               src/algorithms/tracking/libs/exponential_smoother.h:54-62
#include "engine.cuh"

#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <utility>
#include <vector>

using namespace b200;

static_assert(sizeof(b200_trk_dump_record) == 108, "dump record must match log_data()");
static_assert(sizeof(b200_trk_loop_conf) == 152, "b200_trk_loop_conf layout");

namespace
{
constexpr double kTwoPi = 6.283185307179586;

void code_filter_coefficients(LoopDev& L, float update_interval, float noise_bandwidth, int order)
{
    // include_last_integrator = false (dll_pll_veml_tracking.cc:604)
    float g1, g2, g3, wn;
    const float T = update_interval;
    const float zeta = 1.0F / std::sqrt(2.0F);
    switch (order)
        {
        case 1:
            wn = noise_bandwidth * 4.0F;
            g1 = wn;
            L.dll_n_in = 1;
            L.dll_in_c[0] = g1;
            L.dll_n_out = 0;
            break;
        case 2:
            wn = noise_bandwidth * (8.0F * zeta) / (4.0F * zeta * zeta + 1.0F);
            g1 = wn * wn;
            g2 = wn * 2.0F * zeta;
            L.dll_n_in = 2;
            L.dll_in_c[0] = static_cast<float>(g1 * T / 2.0 + g2);
            L.dll_in_c[1] = static_cast<float>(g1 * T / 2.0 - g2);
            L.dll_n_out = 1;
            L.dll_out_c[0] = 1.0F;
            break;
        default:
            {
                wn = noise_bandwidth / 0.7845F;
                const float a3 = 1.1;
                const float b3 = 2.4;
                g1 = wn * wn * wn;
                g2 = a3 * wn * wn;
                g3 = b3 * wn;
                L.dll_n_in = 3;
                L.dll_in_c[0] = static_cast<float>(g3 + T / 2.0 * (g2 + T / 2.0 * g1));
                L.dll_in_c[1] = static_cast<float>(g1 * T * T / 2.0 - 2.0 * g3);
                L.dll_in_c[2] = static_cast<float>(g3 + T / 2.0 * (-g2 + T / 2.0 * g1));
                L.dll_n_out = 2;
                L.dll_out_c[0] = 2.0F;
                L.dll_out_c[1] = -1.0F;
            }
        }
}

void carrier_filter_params(LoopDev& L, float fll_bw_hz, float pll_bw_hz, int order)
{
    L.pll_order = order;
    if (order == 3)
        {
            L.pll_b3 = 2.400;
            L.pll_a3 = 1.100;
            L.pll_a2 = 1.414;
            L.pll_w0p = pll_bw_hz / 0.7845F;
            L.pll_w0p2 = L.pll_w0p * L.pll_w0p;
            L.pll_w0p3 = L.pll_w0p2 * L.pll_w0p;
            L.pll_w0f = fll_bw_hz / 0.53F;
            L.pll_w0f2 = L.pll_w0f * L.pll_w0f;
        }
    else
        {
            L.pll_a2 = 1.414;
            L.pll_w0p = pll_bw_hz / 0.53F;
            L.pll_w0p2 = L.pll_w0p * L.pll_w0p;
            L.pll_w0f = fll_bw_hz / 0.25F;
        }
}

void smoother_init(LoopSmoother& s, float alpha, float min_value, float offset, int samples)
{
    s.alpha = alpha;
    if (s.alpha < 0) s.alpha = 0;
    if (s.alpha > 1) s.alpha = 1;
    s.one_minus_alpha = 1.0F - s.alpha;
    s.old_value = 0.0F;
    s.min_value = min_value;
    s.offset = offset;
    s.init_sum = 0.0F;
    s.samples_for_initialization = samples <= 0 ? 1 : samples;
    s.init_counter = 0;
    s.init_n = 0;
    s.initializing = 1;
}

int ensure_loop_buffers(b200_engine* e, int rec_capacity)
{
    const int n = static_cast<int>(e->loops.size());
    if (!e->loops_dev.fits(n))
        {
            // the loop states are kept; loops_dev is replaced last, so after a failure its capacity still asks for all the others
            const int cap = n + 32;
            DevBuf<LoopDev> nd;
            B200_CUDA_TRY(nd.alloc(cap));
            B200_CUDA_TRY(cudaMemsetAsync(nd, 0, sizeof(LoopDev) * cap, e->stream));
            if (e->loops_dev)
                B200_CUDA_TRY(cudaMemcpyAsync(nd, e->loops_dev, sizeof(LoopDev) * e->loops_dev.capacity(), cudaMemcpyDeviceToDevice, e->stream));
            B200_CUDA_TRY(cudaStreamSynchronize(e->stream));
            // items and taps: one row per loop, then one per data channel (modes 1 and 2)
            B200_CUDA_TRY(e->loop_items_dev.alloc(2 * cap));
            B200_CUDA_TRY(e->loop_taps_dev.alloc(kLoopTapStride * 2 * cap));
            B200_CUDA_TRY(e->loop_nrec_dev.alloc(cap));
            B200_CUDA_TRY(e->loop_data_dev.alloc(cap));
            B200_CUDA_TRY(cudaMemsetAsync(e->loop_items_dev, 0, sizeof(b200_trk_item) * 2 * cap, e->stream));
            B200_CUDA_TRY(cudaMemsetAsync(e->loop_taps_dev, 0, sizeof(float2) * kLoopTapStride * 2 * cap, e->stream));
            e->loops_dev = std::move(nd);
        }
    const size_t words = static_cast<size_t>(n) * static_cast<size_t>(rec_capacity > 0 ? rec_capacity : 1) * kLoopRecordWords;
    B200_CUDA_TRY(e->loop_rec_dev.grow(words, words + words / 4));
    return B200_OK;
}

// what the bands hold right now: [window_lo, write_index), the window b200_iq_window reports (ring slots below valid_from
// still hold the stream from before a gap, restart or forget; an attached buffer refilled with fewer samples than it
// holds still has the previous fill's past write_index)
LoopAvail snapshot_avail(const b200_engine* e)
{
    LoopAvail a{};
    for (int i = 0; i < kMaxBands; i++)
        {
            const Band& b = e->bands[i];
            if (!b.in_use) continue;
            a.lo[i] = b.window_lo();
            a.hi[i] = b.write_index;
        }
    return a;
}

// numbers the data items (rows n_loops, n_loops + 1, ... in loop order) and uploads the table
int upload_loop_data(b200_engine* e)
{
    const int n = static_cast<int>(e->loops.size());
    int row = n;
    for (LoopData& d : e->loop_data) d.item = d.channel >= 0 ? row++ : 0;
    e->loop_n_data = row - n;
    B200_CUDA_TRY(cudaMemcpyAsync(e->loop_data_dev, e->loop_data.data(), sizeof(LoopData) * n, cudaMemcpyHostToDevice, e->stream));
    B200_CUDA_TRY(cudaStreamSynchronize(e->stream));
    return B200_OK;
}

// the kernels' view: nullptr while no loop has a data channel
const LoopData* loop_data_dev(const b200_engine* e) { return e->loop_n_data ? e->loop_data_dev.get() : nullptr; }

// the loops read float bands only (narrow_band_refusal keeps them there), so only the float instantiations run
int correlate_loop_items(b200_engine* e, int n, int slices, uint64_t& launched)
{
    return launch_trk_batch(e->loop_items_dev, n, e->chans_dev, e->bands_dev, e->loop_taps_dev, kLoopTapStride, slices, e->partial,
        e->counters, e->max_code_len, e->taps_mask, 1u << kCf32, e->stream, launched);
}

// B200_ERR_STATE with the error text when channel sits on a narrow band: the loop kernels read their bands as float2, so a
// narrow ring would be read past its end
int narrow_band_refusal(const b200_engine* e, int channel, const char* caller)
{
    const int band = e->chans[channel].desc.band;
    if (e->bands[band].fmt == kCf32) return B200_OK;
    set_error("%s: channel %d is on band %d, which holds narrow (integer) samples; the device loops read gr_complex bands only",
        caller, channel, band);
    return B200_ERR_STATE;
}
}  // namespace

extern "C"
{
    int b200_trk_loop_create(b200_engine* e, int channel, const b200_trk_loop_conf* conf, int* loop_id)
    {
        if (!e || !conf || !loop_id) return B200_ERR_ARG;
        std::lock_guard<std::mutex> lk(e->mu);
        if (channel < 0 || channel >= static_cast<int>(e->chans.size()) || e->chans[channel].desc.code == nullptr)
            {
                set_error("loop_create: channel %d has no code table", channel);
                return B200_ERR_STATE;
            }
        if (const int rc = narrow_band_refusal(e, channel, "loop_create")) return rc;
        const int need_taps = conf->veml ? 5 : 3;
        if (e->chans[channel].desc.taps != need_taps)
            {
                set_error("loop_create: channel %d has %d correlators, the loop needs %d", channel, e->chans[channel].desc.taps, need_taps);
                return B200_ERR_ARG;
            }
        if (e->chans[channel].desc.high_dyn)
            {
                set_error("loop_create: high-dynamics channels are not supported by the device loop");
                return B200_ERR_ARG;
            }
        if (conf->cn0_samples < 1 || conf->cn0_samples > kLoopMaxCn0Samples || conf->fs_in < 1.0 || conf->vector_length < 1 ||
            conf->code_length_chips < 1 || conf->code_chip_rate <= 0.0 || conf->pll_filter_order < 2 || conf->pll_filter_order > 3 ||
            conf->dll_filter_order < 1 || conf->dll_filter_order > 3 || conf->code_samples_per_chip < 1 || conf->slope == 0.0F)
            {
                set_error("loop_create: configuration out of range");
                return B200_ERR_RANGE;
            }
        LoopDev L;
        std::memset(&L, 0, sizeof(L));
        L.c = *conf;
        L.channel = channel;
        L.taps = need_taps;
        L.band = e->chans[channel].desc.band;
        L.carrier_lock_threshold = conf->carrier_lock_th;
        L.code_freq_chips = conf->code_chip_rate;
        code_filter_coefficients(L, static_cast<float>(conf->code_period), conf->dll_bw_hz, conf->dll_filter_order);
        carrier_filter_params(L, conf->fll_bw_hz, conf->pll_bw_hz, conf->pll_filter_order);
        int cn0_init = 200;
        if (conf->code_period > 0.0)
            {
                const int ms = static_cast<int>(conf->code_period * 1000.0);
                if (ms < 1)
                    {
                        set_error("loop_create: code_period below 1 ms");
                        return B200_ERR_RANGE;
                    }
                cn0_init = conf->cn0_smoother_samples / ms;
            }
        smoother_init(L.cn0_smoother, conf->cn0_smoother_alpha, 25.0F, 12.0F, cn0_init);
        smoother_init(L.carrier_lock_test_smoother, conf->carrier_lock_test_smoother_alpha, -1.0F, 0.0F, conf->carrier_lock_test_smoother_samples);
        L.spc = conf->early_late_space_chips;
        L.pull_in_transitory = 1;
        L.cloop = 1;
        L.state = 0;
        e->loops.push_back(L);
        e->loop_data.push_back(LoopData{-1, 0});
        *loop_id = static_cast<int>(e->loops.size()) - 1;
        B200_ENTER_DEVICE(e->device);
        int rc = ensure_loop_buffers(e, 1);
        if (rc) return rc;
        B200_CUDA_TRY(cudaMemcpyAsync(e->loops_dev + *loop_id, &e->loops[*loop_id], sizeof(LoopDev), cudaMemcpyHostToDevice, e->stream));
        B200_CUDA_TRY(cudaStreamSynchronize(e->stream));
        return upload_loop_data(e);
    }

    int b200_trk_loop_set_data_channel(b200_engine* e, int loop_id, int data_channel)
    {
        if (!e) return B200_ERR_ARG;
        std::lock_guard<std::mutex> lk(e->mu);
        if (loop_id < 0 || loop_id >= static_cast<int>(e->loops.size()))
            {
                set_error("loop_set_data_channel: no loop %d", loop_id);
                return B200_ERR_ARG;
            }
        if (data_channel < 0 || data_channel >= static_cast<int>(e->chans.size()) || e->chans[data_channel].desc.code == nullptr)
            {
                set_error("loop_set_data_channel: channel %d has no code table", data_channel);
                return B200_ERR_ARG;
            }
        if (const int rc = narrow_band_refusal(e, data_channel, "loop_set_data_channel")) return rc;
        const ChanDesc& d = e->chans[data_channel].desc;
        if (d.taps != 1)
            {
                set_error("loop_set_data_channel: channel %d has %d correlators, the data channel needs 1", data_channel, d.taps);
                return B200_ERR_ARG;
            }
        if (d.band != e->loops[loop_id].band)
            {
                set_error("loop_set_data_channel: channel %d is on band %d, loop %d on band %d", data_channel, d.band, loop_id, e->loops[loop_id].band);
                return B200_ERR_ARG;
            }
        if (d.high_dyn)
            {
                set_error("loop_set_data_channel: high-dynamics channels are not supported by the device loop");
                return B200_ERR_ARG;
            }
        e->loop_data[loop_id].channel = data_channel;
        B200_ENTER_DEVICE(e->device);
        return upload_loop_data(e);
    }

    int b200_trk_loop_start(b200_engine* e, int loop_id, double acq_delay_samples, double acq_doppler_hz, uint64_t acq_samplestamp_samples,
        uint64_t nitems_read)
    {
        if (!e) return B200_ERR_ARG;
        std::lock_guard<std::mutex> lk(e->mu);
        if (loop_id < 0 || loop_id >= static_cast<int>(e->loops.size())) return B200_ERR_ARG;
        LoopDev& L = e->loops[loop_id];
        const b200_trk_loop_conf& c = L.c;
        L.acq_code_phase_samples = acq_delay_samples;
        L.acq_carrier_doppler_hz = acq_doppler_hz;
        L.acq_sample_stamp = acq_samplestamp_samples;
        L.nitems_read = nitems_read;
        L.carrier_doppler_hz = L.acq_carrier_doppler_hz;
        L.carrier_phase_step_rad = kTwoPi * L.carrier_doppler_hz / c.fs_in;
        L.carrier_phase_rate_step_rad = 0.0;
        L.carrier_lock_fail_counter = 0;
        L.code_lock_fail_counter = 0;
        L.rem_code_phase_samples = 0.0;
        L.rem_carr_phase_rad = 0.0F;
        L.rem_code_phase_chips = 0.0;
        L.acc_carrier_phase_rad = 0.0;
        L.cn0_estimation_counter = 0;
        L.carrier_lock_test = 1.0;
        L.CN0_SNV_dB_Hz = 0.0;
        L.current_correlation_time_s = c.code_period;
        carrier_filter_params(L, c.fll_bw_hz, c.pll_bw_hz, c.pll_filter_order);
        code_filter_coefficients(L, static_cast<float>(c.code_period), c.dll_bw_hz, c.dll_filter_order);
        // d_carrier_loop_filter.initialize(acq doppler); d_code_loop_filter.initialize()
        if (L.pll_order == 3)
            {
                L.pll_x = 2.0F * static_cast<float>(L.acq_carrier_doppler_hz);
                L.pll_w = 0;
            }
        else
            {
                L.pll_w = static_cast<float>(L.acq_carrier_doppler_hz);
                L.pll_x = 0;
            }
        for (int i = 0; i < 4; i++)
            {
                L.dll_inputs[i] = 0.0F;
                L.dll_outputs[i] = 0.0F;
            }
        L.dll_index = 3;
        L.state = 1;
        L.cloop = c.cloop ? 1 : 0;
        L.pull_in_transitory = 1;
        L.loss_of_lock = 0;
        L.epochs = 0;
        L.pending = 0;
        // the device copy is replaced by the start-of-tracking state (what start_tracking leaves alone -
        // d_P_accu_old, the error terms - was zeroed by clear_tracking_vars when the previous run ended)
        B200_ENTER_DEVICE(e->device);
        int rc = ensure_loop_buffers(e, 1);
        if (rc) return rc;
        B200_CUDA_TRY(cudaMemcpyAsync(e->loops_dev + loop_id, &L, sizeof(LoopDev), cudaMemcpyHostToDevice, e->stream));
        B200_CUDA_TRY(cudaStreamSynchronize(e->stream));
        return B200_OK;
    }

    int b200_trk_loop_run(b200_engine* e, int max_epochs, b200_trk_dump_record* records_host, int* n_records_host)
    {
        return b200_trk_loop_run_prompts(e, max_epochs, records_host, n_records_host, nullptr);
    }

    int b200_trk_loop_run_prompts(b200_engine* e, int max_epochs, b200_trk_dump_record* records_host, int* n_records_host,
        b200_cf32* pilot_prompts_host)
    {
        if (!e || max_epochs < 0) return B200_ERR_ARG;
        std::lock_guard<std::mutex> lk(e->mu);
        const int n = static_cast<int>(e->loops.size());
        if (n == 0 || max_epochs == 0) return B200_OK;
        // a band may have been re-created narrow after its loops were made
        for (int i = 0; i < n; i++)
            {
                if (e->loops[i].state == 0) continue;
                if (const int rc = narrow_band_refusal(e, e->loops[i].channel, "loop_run")) return rc;
                if (e->loop_data[i].channel >= 0)
                    if (const int rc = narrow_band_refusal(e, e->loop_data[i].channel, "loop_run")) return rc;
            }
        B200_ENTER_DEVICE(e->device);
        int rc = upload_tables(e);
        if (rc) return rc;
        rc = ensure_loop_buffers(e, max_epochs);
        if (rc) return rc;
        float2* prompts = nullptr;
        if (pilot_prompts_host)
            {
                const size_t elems = static_cast<size_t>(n) * static_cast<size_t>(max_epochs);
                B200_CUDA_TRY(e->loop_prm_dev.grow(elems, elems + elems / 4));
                prompts = e->loop_prm_dev;
            }
        const LoopData* data = loop_data_dev(e);
        const LoopAvail avail = snapshot_avail(e);
        B200_CUDA_TRY(cudaMemsetAsync(e->loop_nrec_dev, 0, sizeof(int) * n, e->stream));
        uint64_t launched = 0;
        if (e->loop_mode == 0)
            {
                rc = launch_loop_persistent(e->loops_dev, n, max_epochs, avail, e->chans_dev, e->bands_dev, data, e->loop_rec_dev, max_epochs,
                    e->loop_nrec_dev, prompts, e->max_code_len, e->stream, launched);
                if (rc) return rc;
            }
        else
            {
                // the data items follow the loops' items in the same correlator launch (the mixed-tap path), split like them:
                // the slice count follows the loops alone, so a data channel leaves the pilot taps bit for bit as they were
                const int n_items = n + e->loop_n_data;
                const int slices = e->loop_mode == 1 ? 1 : batch_slices(n);
                const int data_items = data ? kLoopDataItems : 0;
                rc = ensure_partials(e, n_items, slices);
                if (rc) return rc;
                rc = launch_loop_cycle(e->loops_dev, n, kLoopPrepare | kLoopCheckAvail | data_items, avail, e->loop_items_dev, e->loop_taps_dev, data,
                    nullptr, 0, nullptr, nullptr, e->stream, launched);
                if (rc) return rc;
                for (int k = 0; k < max_epochs; k++)
                    {
                        rc = correlate_loop_items(e, n_items, slices, launched);
                        if (rc) return rc;
                        rc = launch_loop_cycle(e->loops_dev, n, kLoopUpdate | kLoopPrepare | kLoopCheckAvail | data_items, avail, e->loop_items_dev,
                            e->loop_taps_dev, data, e->loop_rec_dev, max_epochs, e->loop_nrec_dev, prompts, e->stream, launched);
                        if (rc) return rc;
                    }
            }
        e->launches += launched;
        std::vector<int> nrec(n);
        B200_CUDA_TRY(cudaMemcpyAsync(nrec.data(), e->loop_nrec_dev, sizeof(int) * n, cudaMemcpyDeviceToHost, e->stream));
        if (records_host)
            B200_CUDA_TRY(cudaMemcpyAsync(records_host, e->loop_rec_dev, sizeof(b200_trk_dump_record) * static_cast<size_t>(n) * max_epochs,
                cudaMemcpyDeviceToHost, e->stream));
        if (pilot_prompts_host)
            B200_CUDA_TRY(cudaMemcpyAsync(pilot_prompts_host, prompts, sizeof(float2) * static_cast<size_t>(n) * max_epochs, cudaMemcpyDeviceToHost,
                e->stream));
        B200_CUDA_TRY(cudaStreamSynchronize(e->stream));
        if (n_records_host)
            for (int i = 0; i < n; i++) n_records_host[i] = nrec[i] < max_epochs ? nrec[i] : max_epochs;
        return B200_OK;
    }

    int b200_trk_loop_set_mode(b200_engine* e, int mode)
    {
        if (!e || mode < 0 || mode > 2) return B200_ERR_ARG;
        std::lock_guard<std::mutex> lk(e->mu);
        e->loop_mode = mode;
        return B200_OK;
    }

    int b200_trk_loop_peek_items(b200_engine* e, b200_trk_item* items_host)
    {
        if (!e || !items_host) return B200_ERR_ARG;
        std::lock_guard<std::mutex> lk(e->mu);
        const int n = static_cast<int>(e->loops.size());
        if (n == 0) return B200_OK;
        B200_ENTER_DEVICE(e->device);
        int rc = ensure_loop_buffers(e, 1);
        if (rc) return rc;
        const LoopAvail avail{};
        uint64_t launched = 0;
        rc = launch_loop_cycle(e->loops_dev, n, kLoopPrepare, avail, e->loop_items_dev, e->loop_taps_dev, loop_data_dev(e), nullptr, 0, nullptr,
            nullptr, e->stream, launched);
        if (rc) return rc;
        e->launches += launched;
        B200_CUDA_TRY(cudaMemcpyAsync(items_host, e->loop_items_dev, sizeof(b200_trk_item) * n, cudaMemcpyDeviceToHost, e->stream));
        B200_CUDA_TRY(cudaStreamSynchronize(e->stream));
        return B200_OK;
    }

    int b200_trk_loop_step_taps(b200_engine* e, const b200_cf32* taps_host, b200_trk_dump_record* records_host, int* logged_host)
    {
        if (!e || !taps_host) return B200_ERR_ARG;
        std::lock_guard<std::mutex> lk(e->mu);
        const int n = static_cast<int>(e->loops.size());
        if (n == 0) return B200_OK;
        B200_ENTER_DEVICE(e->device);
        int rc = ensure_loop_buffers(e, 1);
        if (rc) return rc;
        const LoopAvail avail{};
        B200_CUDA_TRY(cudaMemsetAsync(e->loop_nrec_dev, 0, sizeof(int) * n, e->stream));
        const LoopData* data = loop_data_dev(e);
        uint64_t launched = 0;
        rc = launch_loop_cycle(e->loops_dev, n, kLoopPrepare, avail, e->loop_items_dev, e->loop_taps_dev, data, nullptr, 0, nullptr, nullptr, e->stream,
            launched);
        if (rc) return rc;
        B200_CUDA_TRY(cudaMemcpyAsync(e->loop_taps_dev, taps_host, sizeof(float2) * kLoopTapStride * n, cudaMemcpyHostToDevice, e->stream));
        rc = launch_loop_cycle(e->loops_dev, n, kLoopUpdate, avail, e->loop_items_dev, e->loop_taps_dev, data, e->loop_rec_dev, 1, e->loop_nrec_dev,
            nullptr, e->stream, launched);
        if (rc) return rc;
        e->launches += launched;
        if (records_host)
            B200_CUDA_TRY(cudaMemcpyAsync(records_host, e->loop_rec_dev, sizeof(b200_trk_dump_record) * n, cudaMemcpyDeviceToHost, e->stream));
        if (logged_host) B200_CUDA_TRY(cudaMemcpyAsync(logged_host, e->loop_nrec_dev, sizeof(int) * n, cudaMemcpyDeviceToHost, e->stream));
        B200_CUDA_TRY(cudaStreamSynchronize(e->stream));
        return B200_OK;
    }

    int b200_trk_loop_status_get(b200_engine* e, int loop_id, b200_trk_loop_status* out)
    {
        if (!e || !out) return B200_ERR_ARG;
        std::lock_guard<std::mutex> lk(e->mu);
        if (loop_id < 0 || loop_id >= static_cast<int>(e->loops.size())) return B200_ERR_ARG;
        B200_ENTER_DEVICE(e->device);
        LoopDev L;
        B200_CUDA_TRY(cudaMemcpyAsync(&L, e->loops_dev + loop_id, sizeof(LoopDev), cudaMemcpyDeviceToHost, e->stream));
        B200_CUDA_TRY(cudaStreamSynchronize(e->stream));
        out->state = L.state;
        out->loss_of_lock = L.loss_of_lock;
        out->sample_counter = L.nitems_read;
        out->epochs = L.epochs;
        out->carrier_doppler_hz = L.carrier_doppler_hz;
        out->code_freq_chips = L.code_freq_chips;
        out->rem_code_phase_samples = L.rem_code_phase_samples;
        out->acc_carrier_phase_rad = L.acc_carrier_phase_rad;
        out->CN0_SNV_dB_Hz = L.CN0_SNV_dB_Hz;
        out->carrier_lock_test = L.carrier_lock_test;
        return B200_OK;
    }

    int b200_trk_dump_write(const char* filename, const b200_trk_dump_record* records, int n_records, int append)
    {
        if (!filename || n_records < 0 || (n_records && !records)) return B200_ERR_ARG;
        FILE* f = std::fopen(filename, append ? "ab" : "wb");
        if (!f)
            {
                set_error("dump_write: cannot open %s", filename);
                return B200_ERR_STATE;
            }
        const size_t w = std::fwrite(records, sizeof(b200_trk_dump_record), static_cast<size_t>(n_records), f);
        const int bad = std::fclose(f);
        if (w != static_cast<size_t>(n_records) || bad)
            {
                set_error("dump_write: short write to %s", filename);
                return B200_ERR_STATE;
            }
        return B200_OK;
    }
}
