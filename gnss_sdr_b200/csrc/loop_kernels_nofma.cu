// Per-epoch DLL/PLL loop arithmetic on the device (SURVEY 8f N1): one thread per tracking loop, run between
// correlator launches so that epoch k+1's NCO commands are produced where epoch k's taps land.
//
// This file is compiled with --fmad=false (see build.py: *_nofma.cu): the reference evaluates every
// expression below with separately rounded IEEE multiplies and adds (x86-64, no FMA contraction), in the
// float / double types of its members, and so does this kernel.  The only operations that are not IEEE-exact
// on both sides are atanf, atan2f and log10f: the device evaluates them in double and rounds once (correctly
// rounded float), glibc's are <= 1 ulp.  hypotf = sqrt of the exact double sum of squares on both sides.
//
// Reference, statement by statement:
//   general_work head, cases 1-2, tail   tracking/gnuradio_blocks/dll_pll_veml_tracking.cc:1898-2015, :2292
//   cn0_and_tracking_lock_status         :1167-1224        run_dll_pll   :1260-1347
//   update_tracking_vars                 :1409-1483        log_data      :1599-1694
//   clear_tracking_vars                  :1359-1383
//   tracking_discriminators.cc:26-39,69-77,86-89,100-107,119-129,142-153
//   tracking_FLL_PLL_filter.cc:72-104    tracking_loop_filter.cc:62-96
//   lock_detectors.cc:99-147,160-181     exponential_smoother.cc:86-115
#include "loop.cuh"
#include "trk_item.cuh"

namespace b200
{
namespace
{
constexpr double kTwoPi = 6.283185307179586;   // MATH_CONSTANTS.h TWO_PI
constexpr double kGnssPi = 3.1415926535898;    // GNSS_PI
constexpr double kHalfPi = 1.570796326794897;  // HALF_PI

__device__ __forceinline__ float atanf_cr(float x) { return static_cast<float>(atan(static_cast<double>(x))); }
__device__ __forceinline__ float atan2f_cr(float y, float x) { return static_cast<float>(atan2(static_cast<double>(y), static_cast<double>(x))); }
__device__ __forceinline__ float log10f_cr(float x) { return static_cast<float>(log10(static_cast<double>(x))); }
__device__ __forceinline__ float hypotf_cr(float x, float y)
{
    return static_cast<float>(sqrt(static_cast<double>(x) * static_cast<double>(x) + static_cast<double>(y) * static_cast<double>(y)));
}

__device__ float smoother_smooth(LoopSmoother& s, float raw)
{
    float smoothed_value;
    if (s.initializing)
        {
            s.init_counter++;
            smoothed_value = raw;
            s.init_sum = s.init_sum + smoothed_value;
            s.init_n++;
            if (s.init_counter == s.samples_for_initialization)
                {
                    s.old_value = s.init_sum / static_cast<float>(s.init_n);
                    if (s.old_value < (s.min_value + s.offset))
                        {
                            s.init_counter = 0;
                            s.init_sum = 0.0f;
                            s.init_n = 0;
                        }
                    else
                        {
                            s.initializing = 0;
                        }
                }
        }
    else
        {
            smoothed_value = s.alpha * raw + s.one_minus_alpha * s.old_value;
            s.old_value = smoothed_value;
        }
    return smoothed_value;
}

__device__ void smoother_reset(LoopSmoother& s)
{
    s.initializing = 1;
    s.init_counter = 0;
    s.init_sum = 0.0f;
    s.init_n = 0;
}

__device__ float code_filter_apply(LoopDev& L, float current_input)
{
    float result = 0.0f;
    for (int ii = 0; ii < L.dll_n_out; ++ii) result += L.dll_out_c[ii] * L.dll_outputs[(L.dll_index + ii) % 4];
    L.dll_index--;
    if (L.dll_index < 0) L.dll_index += 4;
    L.dll_inputs[L.dll_index] = current_input;
    for (int ii = 0; ii < L.dll_n_in; ++ii) result += L.dll_in_c[ii] * L.dll_inputs[(L.dll_index + ii) % 4];
    L.dll_outputs[L.dll_index] = result;
    return result;
}

__device__ float carrier_filter(LoopDev& L, float FLL_discriminator, float PLL_discriminator, float correlation_time_s)
{
    float carrier_error_hz;
    if (L.pll_order == 3)
        {
            L.pll_w = L.pll_w + correlation_time_s * (L.pll_w0p3 * PLL_discriminator + L.pll_w0f2 * FLL_discriminator);
            L.pll_x = L.pll_x + correlation_time_s * (0.5f * L.pll_w + L.pll_a2 * L.pll_w0f * FLL_discriminator + L.pll_a3 * L.pll_w0p2 * PLL_discriminator);
            carrier_error_hz = 0.5f * L.pll_x + L.pll_b3 * L.pll_w0p * PLL_discriminator;
        }
    else
        {
            const float pll_w_new = L.pll_w + PLL_discriminator * L.pll_w0p2 * correlation_time_s + FLL_discriminator * L.pll_w0f * correlation_time_s;
            carrier_error_hz = 0.5f * (pll_w_new + L.pll_w) + L.pll_a2 * L.pll_w0p * PLL_discriminator;
            L.pll_w = pll_w_new;
        }
    return carrier_error_hz;
}

__device__ double phase_unwrap(double phase_rad)
{
    if (phase_rad >= kHalfPi) return phase_rad - kGnssPi;
    if (phase_rad <= -kHalfPi) return phase_rad + kGnssPi;
    return phase_rad;
}

__device__ float cn0_m2m4_estimator(const float2* buf, int length, float coh_integration_time_s)
{
    float SNR_aux = 0.0f, Psig = 0.0f, m_2 = 0.0f, m_4 = 0.0f, aux;
    const float n = static_cast<float>(length);
    if (length == 0 || coh_integration_time_s == 0.0f) return -100.0f;
    for (int i = 0; i < length; i++)
        {
            Psig += fabsf(buf[i].x);
            aux = buf[i].y * buf[i].y + buf[i].x * buf[i].x;
            m_2 += aux;
            m_4 += (aux * aux);
        }
    Psig /= n;
    Psig = Psig * Psig;
    m_2 /= n;
    m_4 /= n;
    aux = sqrtf(2.0f * m_2 * m_2 - m_4);
    float denominator;
    if (isnan(aux))
        {
            denominator = m_2 - Psig;
            if (denominator == 0) return -100.0f;
            SNR_aux = Psig / denominator;
        }
    else
        {
            denominator = m_2 - aux;
            if (denominator == 0) return -100.0f;
            SNR_aux = aux / denominator;
        }
    if (SNR_aux == 0) return -100.0f;
    return 10.0f * log10f_cr(SNR_aux) - 10.0f * log10f_cr(coh_integration_time_s);
}

__device__ float carrier_lock_detector(const float2* buf, int length)
{
    float tmp_sum_I = 0.0f, tmp_sum_Q = 0.0f;
    for (int i = 0; i < length; i++)
        {
            tmp_sum_I += buf[i].x;
            tmp_sum_Q += buf[i].y;
        }
    const float NBP = tmp_sum_I * tmp_sum_I + tmp_sum_Q * tmp_sum_Q;
    const float NBD = tmp_sum_I * tmp_sum_I - tmp_sum_Q * tmp_sum_Q;
    if (NBP == 0) return 0.0f;
    return NBD / NBP;
}

__device__ void clear_tracking_vars(LoopDev& L)
{
    L.P_accu_old = make_float2(0.f, 0.f);
    L.carr_phase_error_hz = 0.0;
    L.carr_freq_error_hz = 0.0;
    L.carr_error_filt_hz = 0.0;
    L.code_error_chips = 0.0;
    L.code_error_filt_chips = 0.0;
    L.carrier_phase_rate_step_rad = 0.0;
    L.code_phase_rate_step_chips = 0.0;
}

__device__ void pull_in_check(LoopDev& L)
{
    if (L.pull_in_transitory)
        {
            if (L.c.pull_in_time_s < (L.nitems_read - L.acq_sample_stamp) / static_cast<unsigned long long>(static_cast<int>(L.c.fs_in)))
                {
                    L.pull_in_transitory = 0;
                    L.carrier_lock_fail_counter = 0;
                    L.code_lock_fail_counter = 0;
                }
        }
}

// general_work up to do_correlation_step: returns true when an item was produced
__device__ bool loop_prepare(LoopDev& L, b200_trk_item& it, bool check_avail, unsigned long long lo, unsigned long long hi)
{
    const b200_trk_loop_conf& c = L.c;
    it.channel = L.channel;
    it.n = 0;
    if (L.state == 0) return false;
    pull_in_check(L);
    if (L.state == 1)
        {
            const long long acq_trk_diff_samples = static_cast<long long>(L.nitems_read) - static_cast<long long>(L.acq_sample_stamp);
            const double delta_trk_to_acq_prn_start_samples = static_cast<double>(acq_trk_diff_samples) - L.acq_code_phase_samples;
            L.code_freq_chips = c.code_chip_rate;
            L.code_phase_step_chips = L.code_freq_chips / c.fs_in;
            L.code_phase_rate_step_chips = 0.0;
            const double T_chip_mod_seconds = 1.0 / L.code_freq_chips;
            const double T_prn_mod_seconds = T_chip_mod_seconds * static_cast<double>(c.code_length_chips);
            const double T_prn_mod_samples = T_prn_mod_seconds * c.fs_in;
            L.acq_code_phase_samples = T_prn_mod_samples - fmod(delta_trk_to_acq_prn_start_samples, T_prn_mod_samples);
            L.current_prn_length_samples = static_cast<int>(round(T_prn_mod_samples));
            const int samples_offset = static_cast<int>(round(L.acq_code_phase_samples));
            L.acc_carrier_phase_rad -= L.carrier_phase_step_rad * static_cast<double>(samples_offset);
            L.state = 2;
            smoother_reset(L.cn0_smoother);
            smoother_reset(L.carrier_lock_test_smoother);
            L.nitems_read += static_cast<unsigned long long>(static_cast<long long>(samples_offset));
            pull_in_check(L);
        }
    if (check_avail && (L.nitems_read < lo || L.nitems_read + c.vector_length > hi)) return false;  // stall: samples not resident
    it.n = static_cast<int>(c.vector_length);
    it.sample_index = L.nitems_read;
    it.rem_carrier_phase_rad = L.rem_carr_phase_rad;
    it.phase_step_rad = static_cast<float>(L.carrier_phase_step_rad);
    it.phase_rate_step_rad = static_cast<float>(L.carrier_phase_rate_step_rad);
    it.rem_code_phase_chips = static_cast<float>(L.rem_code_phase_chips) * static_cast<float>(c.code_samples_per_chip);
    it.code_phase_step_chips = static_cast<float>(L.code_phase_step_chips) * static_cast<float>(c.code_samples_per_chip);
    it.code_phase_rate_step_chips = static_cast<float>(L.code_phase_rate_step_chips) * static_cast<float>(c.code_samples_per_chip);
    return true;
}

__device__ bool lock_status(LoopDev& L, float2 P_accu, double coh_integration_time_s)
{
    const b200_trk_loop_conf& c = L.c;
    if (L.cn0_estimation_counter < c.cn0_samples)
        {
            L.Prompt_buffer[L.cn0_estimation_counter] = P_accu;
            L.cn0_estimation_counter++;
            return true;
        }
    L.Prompt_buffer[L.cn0_estimation_counter % c.cn0_samples] = P_accu;
    L.cn0_estimation_counter++;
    const float raw = cn0_m2m4_estimator(L.Prompt_buffer, c.cn0_samples, static_cast<float>(coh_integration_time_s));
    L.CN0_SNV_dB_Hz = smoother_smooth(L.cn0_smoother, raw);
    L.carrier_lock_test = smoother_smooth(L.carrier_lock_test_smoother, carrier_lock_detector(L.Prompt_buffer, 1));
    if (!L.pull_in_transitory)
        {
            if (L.carrier_lock_test < L.carrier_lock_threshold)
                L.carrier_lock_fail_counter++;
            else if (L.carrier_lock_fail_counter > 0)
                L.carrier_lock_fail_counter--;
            if (L.CN0_SNV_dB_Hz < c.cn0_min)
                L.code_lock_fail_counter++;
            else if (L.code_lock_fail_counter > 0)
                L.code_lock_fail_counter--;
        }
    if (L.carrier_lock_fail_counter > c.max_carrier_lock_fail || L.code_lock_fail_counter > c.max_code_lock_fail)
        {
            L.carrier_lock_fail_counter = 0;
            L.code_lock_fail_counter = 0;
            return false;
        }
    return true;
}

// general_work case 2 after do_correlation_step, then consume_each, in three parts that touch DISJOINT members of LoopDev so
// that the persistent kernel can run them on different warps at the same time (the serial double-precision chain of one
// thread was 40 % of an epoch):
//   loop_lock_part    the bit-synchronisation time limit and cn0_and_tracking_lock_status (:1167-1224): Prompt_buffer,
//                     cn0_estimation_counter, the two smoothers, CN0_SNV_dB_Hz, carrier_lock_test, the fail counters;
//   loop_track_part   run_dll_pll (:1260-1347) and update_tracking_vars (:1409-1483): discriminators, loop filters, NCO and
//                     remnant-phase members, current_prn_length_samples, epochs;
//   loop_record_part  log_data (:1599-1694) from the members the other two left behind.
// loop_update() is their sequential composition in the reference's order and is what every other caller uses.
__device__ __forceinline__ void loop_taps(const b200_trk_loop_conf& c, const float2* t, float2& VE, float2& E, float2& P, float2& Lt, float2& VL)
{
    VE = make_float2(0.f, 0.f);
    VL = make_float2(0.f, 0.f);
    if (c.veml)
        {
            VE = t[0];
            E = t[1];
            P = t[2];
            Lt = t[3];
            VL = t[4];
        }
    else
        {
            E = t[0];
            P = t[1];
            Lt = t[2];
        }
}

__device__ bool loop_lock_part(LoopDev& L, const float2* t)
{
    const b200_trk_loop_conf& c = L.c;
    float2 VE, E, P, Lt, VL;
    loop_taps(c, t, VE, E, P, Lt, VL);
    L.spc = c.early_late_space_chips;   // (nobody reads the member: the DLL discriminator takes the value from the configuration)
    if (c.bit_synchronization_time_limit_s < (L.nitems_read - L.acq_sample_stamp) / static_cast<unsigned long long>(static_cast<int>(c.fs_in)))
        L.carrier_lock_fail_counter = 300000;
    return lock_status(L, P, c.code_period);
}

__device__ void loop_lost_lock(LoopDev& L)
{
    clear_tracking_vars(L);
    L.state = 0;
    L.loss_of_lock = 1;
}

__device__ void loop_track_part(LoopDev& L, const float2* t)
{
    const b200_trk_loop_conf& c = L.c;
    float2 VE, E, P, Lt, VL;
    loop_taps(c, t, VE, E, P, Lt, VL);
    const float spc = c.early_late_space_chips;
    // ---- run_dll_pll
    if (L.cloop)
        L.carr_phase_error_hz = (P.x != 0.0f ? static_cast<double>(atanf_cr(P.y / P.x)) : 0.0) / kTwoPi;
    else
        L.carr_phase_error_hz = static_cast<double>(atan2f_cr(P.y, P.x)) / kTwoPi;
    const float T = static_cast<float>(L.current_correlation_time_s);
    if ((L.pull_in_transitory && c.enable_fll_pull_in) || c.enable_fll_steady_state)
        {
            double diff_atan = atanf_cr(P.y / P.x) - atanf_cr(L.P_accu_old.y / L.P_accu_old.x);
            if (isnan(diff_atan)) diff_atan = 0;
            L.carr_freq_error_hz = phase_unwrap(diff_atan) / (L.current_correlation_time_s - 0.0) / kTwoPi;
            L.P_accu_old = P;
            if (L.pull_in_transitory && c.enable_fll_pull_in)
                L.carr_error_filt_hz = carrier_filter(L, static_cast<float>(L.carr_freq_error_hz), 0.0f, T);
            else
                L.carr_error_filt_hz = carrier_filter(L, static_cast<float>(L.carr_freq_error_hz), static_cast<float>(L.carr_phase_error_hz), T);
        }
    else
        {
            L.carr_error_filt_hz = carrier_filter(L, 0.0f, static_cast<float>(L.carr_phase_error_hz), T);
        }
    L.carrier_doppler_hz = L.carr_error_filt_hz;
    if (c.veml)
        {
            const double Early = sqrtf(VE.x * VE.x + VE.y * VE.y + E.x * E.x + E.y * E.y);
            const double Late = sqrtf(Lt.x * Lt.x + Lt.y * Lt.y + VL.x * VL.x + VL.y * VL.y);
            const double E_plus_L = Early + Late;
            L.code_error_chips = (E_plus_L == 0.0) ? 0.0 : (Early - Late) / E_plus_L;
        }
    else
        {
            const double P_early = hypotf_cr(E.x, E.y);
            const double P_late = hypotf_cr(Lt.x, Lt.y);
            const double E_plus_L = P_early + P_late;
            L.code_error_chips = (E_plus_L == 0.0) ? 0.0 : ((c.y_intercept - c.slope * spc) / c.slope) * (P_early - P_late) / E_plus_L;
        }
    L.code_error_filt_chips = code_filter_apply(L, static_cast<float>(L.code_error_chips));
    L.code_freq_chips = c.code_chip_rate - L.code_error_filt_chips;
    if (c.carrier_aiding) L.code_freq_chips += L.carrier_doppler_hz * c.code_chip_rate / c.signal_carrier_freq;
    // ---- update_tracking_vars
    const double T_chip_seconds = 1.0 / L.code_freq_chips;
    const double T_prn_seconds = T_chip_seconds * static_cast<double>(static_cast<int>(c.code_length_chips));
    const double T_prn_samples = T_prn_seconds * c.fs_in;
    const double K_blk_samples = T_prn_samples + L.rem_code_phase_samples;
    L.current_prn_length_samples = static_cast<int>(floor(K_blk_samples));
    const double len = static_cast<double>(L.current_prn_length_samples);
    L.carrier_phase_step_rad = kTwoPi * (L.carrier_doppler_hz + 0.0) / c.fs_in;
    const double adv = L.carrier_phase_step_rad * len + 0.5 * L.carrier_phase_rate_step_rad * len * len;
    L.rem_carr_phase_rad += static_cast<float>(adv);
    L.rem_carr_phase_rad = static_cast<float>(fmod(static_cast<double>(L.rem_carr_phase_rad), kTwoPi));
    L.acc_carrier_phase_rad -= adv;
    L.code_phase_step_chips = L.code_freq_chips / c.fs_in;
    L.rem_code_phase_samples = K_blk_samples - len;
    L.rem_code_phase_chips = L.code_freq_chips * L.rem_code_phase_samples / c.fs_in;
    L.epochs++;
}

// the five correlator magnitudes of the dump record (abs_VE, abs_E, abs_P, abs_L, abs_VL)
__device__ __forceinline__ float loop_record_magnitude(const b200_trk_loop_conf& c, const float2* t, int which)
{
    float2 VE, E, P, Lt, VL;
    loop_taps(c, t, VE, E, P, Lt, VL);
    switch (which)
        {
        case 0: return c.veml ? hypotf_cr(VE.x, VE.y) : 0.0f;
        case 1: return hypotf_cr(E.x, E.y);
        case 2: return hypotf_cr(P.x, P.y);
        case 3: return hypotf_cr(Lt.x, Lt.y);
        default: return c.veml ? hypotf_cr(VL.x, VL.y) : 0.0f;
        }
}

__device__ __forceinline__ unsigned long long loop_record_stamp(const LoopDev& L)
{
    return L.nitems_read + static_cast<unsigned long long>(static_cast<long long>(L.current_prn_length_samples));
}

// mags: the five magnitudes (computed here when nullptr); stamp: loop_record_stamp() taken BEFORE loop_consume().
// data: the data prompt of a loop with a data channel (d_correlator_data_cpu, :1245-1256), nullptr without one; log_data
// writes it as prompt_I/prompt_Q (:1614-1617), every other field comes from the pilot taps.  pilot_out (may be nullptr):
// receives the pilot prompt.
__device__ void loop_record_part(const LoopDev& L, const float2* t, const float2* data, const float* mags, unsigned long long stamp,
    unsigned int* rec, float2* pilot_out)
{
    const b200_trk_loop_conf& c = L.c;
    float2 VE, E, P, Lt, VL;
    loop_taps(c, t, VE, E, P, Lt, VL);
    for (int q = 0; q < 5; q++) rec[q] = __float_as_uint(mags ? mags[q] : loop_record_magnitude(c, t, q));
    const float2 Pr = data ? *data : P;
    rec[5] = __float_as_uint(Pr.x);
    rec[6] = __float_as_uint(Pr.y);
    if (pilot_out) *pilot_out = P;
    rec[7] = static_cast<unsigned int>(stamp);
    rec[8] = static_cast<unsigned int>(stamp >> 32);
    rec[9] = __float_as_uint(static_cast<float>(L.acc_carrier_phase_rad));
    rec[10] = __float_as_uint(static_cast<float>(L.carrier_doppler_hz));
    rec[11] = __float_as_uint(static_cast<float>(L.carrier_phase_rate_step_rad * c.fs_in * c.fs_in / kTwoPi));
    rec[12] = __float_as_uint(static_cast<float>(L.code_freq_chips));
    rec[13] = __float_as_uint(static_cast<float>(L.code_phase_rate_step_chips * c.fs_in * c.fs_in));
    rec[14] = __float_as_uint(static_cast<float>(L.carr_phase_error_hz));
    rec[15] = __float_as_uint(static_cast<float>(L.carr_error_filt_hz));
    rec[16] = __float_as_uint(static_cast<float>(L.code_error_chips));
    rec[17] = __float_as_uint(static_cast<float>(L.code_error_filt_chips));
    rec[18] = __float_as_uint(static_cast<float>(L.CN0_SNV_dB_Hz));
    rec[19] = __float_as_uint(static_cast<float>(L.carrier_lock_test));
    rec[20] = __float_as_uint(static_cast<float>(L.rem_code_phase_samples));
    const unsigned long long aux2 = static_cast<unsigned long long>(__double_as_longlong(static_cast<double>(stamp)));
    rec[21] = static_cast<unsigned int>(aux2);
    rec[22] = static_cast<unsigned int>(aux2 >> 32);
    rec[23] = c.prn;
    rec[24] = 0u;  // TOW (telemetry stays on the host)
    rec[25] = 0u;
    rec[26] = 0u;  // WN
}

__device__ __forceinline__ void loop_consume(LoopDev& L)
{
    L.nitems_read += static_cast<unsigned long long>(static_cast<long long>(L.current_prn_length_samples));  // consume_each
}

// Returns true when a record was logged.
__device__ bool loop_update(LoopDev& L, const float2* t, const float2* data, unsigned int* rec, float2* pilot_out)
{
    bool logged = false;
    if (!loop_lock_part(L, t))
        {
            loop_lost_lock(L);
        }
    else
        {
            loop_track_part(L, t);
            if (rec) loop_record_part(L, t, data, nullptr, loop_record_stamp(L), rec, pilot_out);
            logged = true;
        }
    loop_consume(L);
    return logged;
}

// The record slot k of loop i (nullptr when records is nullptr or the loop's capacity is used up) and its pilot prompt (nullptr
// also without prompts).
__device__ __forceinline__ unsigned int* record_slot(unsigned int* records, float2* prompts, int rec_capacity, int i, int k, float2*& prompt)
{
    prompt = nullptr;
    if (!records || k >= rec_capacity) return nullptr;
    if (prompts) prompt = prompts + static_cast<size_t>(i) * rec_capacity + k;
    return records + (static_cast<size_t>(i) * rec_capacity + k) * kLoopRecordWords;
}

__global__ void trk_loop_cycle_kernel(LoopDev* loops, int n_loops, int mode, LoopAvail avail, b200_trk_item* items,
    const float2* __restrict__ taps, const LoopData* __restrict__ data, unsigned int* records, int rec_capacity, int* n_records,
    float2* prompts)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_loops) return;
    LoopDev& L = loops[i];
    const bool check = (mode & kLoopCheckAvail) != 0;
    const unsigned long long lo = avail.lo[L.band & 15], hi = avail.hi[L.band & 15];
    const LoopData d = data ? data[i] : LoopData{-1, 0};
    if ((mode & kLoopUpdate) && L.pending)
        {
            const int k = n_records ? n_records[i] : 0;
            float2* prm;
            unsigned int* rec = record_slot(records, prompts, rec_capacity, i, k, prm);
            const float2* t = taps + static_cast<size_t>(i) * kLoopTapStride;
            // the data tap: row d.item of the correlator output, or the slot after the pilot taps (b200_trk_loop_step_taps)
            const float2* pd = nullptr;
            if (d.channel >= 0) pd = (mode & kLoopDataItems) ? taps + static_cast<size_t>(d.item) * kLoopTapStride : t + L.taps;
            const bool logged = loop_update(L, t, pd, rec, prm);
            if (logged && n_records) n_records[i] = k + 1;
            L.pending = 0;
        }
    // A prepare-only call opens every API entry (run / peek / step): it always re-derives the item from the state
    // (idempotent once the loop is in state 2), so an item buffer that was reallocated since cannot be stale.
    const bool force = (mode & kLoopPrepare) && !(mode & kLoopUpdate);
    if ((mode & kLoopPrepare) && (force || !L.pending))
        {
            b200_trk_item it;
            L.pending = loop_prepare(L, it, check, lo, hi) ? 1 : 0;
            items[i] = it;
            if (d.channel >= 0 && (mode & kLoopDataItems))
                {
                    it.channel = d.channel;   // the same epoch against the data code (n == 0 when the loop stalls)
                    items[d.item] = it;
                }
        }
}
// Persistent free-running tracker: one CTA per loop runs epoch after epoch without leaving the SM - loop update of the
// previous epoch + prepare of the next (thread 0, one serial section, one barrier) -> correlate vector_length samples (all
// kLoopThreads threads with the batch kernel's per-item templates, slices = 1).  Loops are independent, so there is no
// grid-wide dependency and no launch per epoch; a CTA ends when its loop has run max_epochs cycles, loses lock, or
// finds its next vector_length samples not resident (stall).
// Each channel is a latency chain (epoch k+1's NCO commands need epoch k's taps).  The serial double-precision loop update,
// not the correlation, dominates the epoch time, and wider CTAs cost residency when many loops run.
constexpr int kLoopThreadsMany = 256;   // CTA width when loops outnumber the SMs (two CTAs per SM)
constexpr int kLoopThreadsFew = 512;    // one loop per SM at most: wider CTAs shorten the correlation

// The data pass of a loop with a data channel: its own function, not inlined, so that the pilot's code in the persistent
// kernel stays laid out as without it (inlined, the 1-tap correlation made every epoch of a loop without a data channel about
// 1 us slower on an H100).
template <int kLoopThreads>
__device__ __noinline__ float2 loop_correlate_data(const b200_trk_item& it, const ChanDesc& ch, const BandDesc& bd, float* smem_tbl, int tbl_cap,
    float2* smem_red, int* tbl_cache)
{
    float2 r[1];
    process_item<1, true, kLoopThreads>(it, ch, bd, smem_tbl, tbl_cap, smem_red, 0, 1, r, tbl_cache);
    return r[0];
}

// the persistent kernel's copies of a LoopDev between global and shared memory, word by word over the CTA (tid, stride)
__device__ __forceinline__ void copy_words(LoopDev* dst, const LoopDev* src, int tid, int stride)
{
    unsigned int* d = reinterpret_cast<unsigned int*>(dst);
    const unsigned int* s = reinterpret_cast<const unsigned int*>(src);
    for (int w = tid; w < static_cast<int>(sizeof(LoopDev) / 4); w += stride) d[w] = s[w];
}

// data: nullptr when no loop of the launch has a data channel; otherwise the data channel of every loop (-1: none), and the
// dynamic shared memory holds a second code table of tbl_cap entries for it, right after the pilot's.
template <int kLoopThreads>
__global__ void __launch_bounds__(kLoopThreads, 512 / kLoopThreads) trk_loop_persistent_kernel(LoopDev* loops, int n_loops, int max_epochs, LoopAvail avail,
    const ChanDesc* __restrict__ chans, const BandDesc* __restrict__ bands, const LoopData* __restrict__ data, unsigned int* records,
    int rec_capacity, int* n_records, float2* prompts, int tbl_cap)
{
    extern __shared__ __align__(16) float smem[];
    float* smem_tbl = smem;
    float* smem_tbl_data = data ? smem + tbl_cap : nullptr;
    float2* smem_red = reinterpret_cast<float2*>(smem + (data ? 2 * tbl_cap : tbl_cap));
    LoopDev* sL = reinterpret_cast<LoopDev*>(smem_red + (kLoopThreads / 32) * B200_MAX_TAPS);
    LoopDev* sBackup = sL + 1;   // the state before the current update (see the loop)
    __shared__ b200_trk_item s_item;
    __shared__ int s_lock_ok;
    __shared__ float s_mags[5];
    __shared__ unsigned long long s_stamp;
    __shared__ unsigned int* s_rec;
    __shared__ float2* s_prm;
    __shared__ int s_go;
    __shared__ int s_tbl_cache[2];       // chip-index window held in smem_tbl (process_item<.., REUSE>)
    __shared__ int s_tbl_cache_data[2];  // the same for the data table in smem_tbl_data: the two never evict each other
    __shared__ int s_data_channel;       // -1: none
    __shared__ float2 s_data_tap;        // data prompt of the last epoch (kept here, not in registers across the correlation)

    const int i = blockIdx.x;
    const int tid = threadIdx.x;
    if (i >= n_loops) return;
    copy_words(sL, loops + i, tid, kLoopThreads);
    if (tid == 0)
        {
            s_tbl_cache[0] = s_tbl_cache[1] = s_tbl_cache_data[0] = s_tbl_cache_data[1] = 0;
            s_data_channel = data ? data[i].channel : -1;
        }
    __syncthreads();
    const ChanDesc& ch = chans[sL->channel];
    const BandDesc bd = bands[ch.band];
    const int taps = sL->taps;
    const unsigned long long lo = avail.lo[sL->band & 15], hi = avail.hi[sL->band & 15];
    int k_rec = 0;
    bool have_taps = false;
    float2 t[B200_MAX_TAPS];

    for (int k = 0; k <= max_epochs; k++)
        {
            if (have_taps)
                {
                    // Loop update of epoch k-1 on three warps at once (every thread holds the taps t[]):
                    //   warp 0 / lane 0   run_dll_pll + update_tracking_vars, speculating that lock holds
                    //   warp 1 / lane 0   the lock detectors (C/N0 estimator, carrier lock test, counters)
                    //   warp 2 / lanes<5  the five magnitudes of the dump record
                    // The parts write disjoint members of the state.  When the lock verdict is "lost" (once per run at most) the
                    // state is put back from the copy taken below and the update is replayed in the reference's order.
                    copy_words(sBackup, sL, tid, kLoopThreads);
                    __syncthreads();
                    if (tid == 0)
                        {
                            loop_track_part(*sL, t);
                            s_stamp = loop_record_stamp(*sL);
                            float2* prm;
                            s_rec = record_slot(records, prompts, rec_capacity, i, k_rec, prm);
                            s_prm = prm;
                        }
                    else if (tid == 32)
                        s_lock_ok = loop_lock_part(*sL, t) ? 1 : 0;
                    else if (tid >= 64 && tid < 69)
                        s_mags[tid - 64] = loop_record_magnitude(sL->c, t, tid - 64);
                    __syncthreads();
                    // the dump record goes out from warp 1 while thread 0 consumes the epoch and prepares the next one: in the
                    // tracking state neither of those writes a member the record reads (the sample stamp was taken above)
                    if (tid == 32 && s_lock_ok > 0 && s_rec != nullptr) loop_record_part(*sL, t, s_data_channel >= 0 ? &s_data_tap : nullptr, s_mags, s_stamp, s_rec,
                                                                                          s_prm);
                }
            if (tid == 0)
                {
                    if (have_taps)
                        {
                            float2* prm;
                            unsigned int* rec = record_slot(records, prompts, rec_capacity, i, k_rec, prm);
                            if (s_lock_ok < 0)
                                {
                                    if (loop_update(*sL, t, s_data_channel >= 0 ? &s_data_tap : nullptr, rec, prm)) k_rec++;
                                }
                            else if (s_lock_ok)
                                {
                                    loop_consume(*sL);
                                    k_rec++;
                                }
                            else
                                {
                                    copy_words(sL, sBackup, 0, 1);
                                    if (loop_update(*sL, t, s_data_channel >= 0 ? &s_data_tap : nullptr, rec, prm)) k_rec++;
                                }
                        }
                    int go = 0;
                    if (k < max_epochs)
                        {
                            b200_trk_item it;
                            // in state 2 preparing is a pure function of the state, so an item left pending by the
                            // per-launch path is simply recomputed
                            go = loop_prepare(*sL, it, true, lo, hi) ? 1 : 0;
                            s_item = it;
                        }
                    s_go = go;
                }
            __syncthreads();
            if (!s_go) break;
            if (taps == 3)
                {
                    float2 r[3];
                    process_item<3, true, kLoopThreads>(s_item, ch, bd, smem_tbl, tbl_cap, smem_red, 0, 1, r, s_tbl_cache);
#pragma unroll
                    for (int q = 0; q < 3; q++) t[q] = r[q];
                }
            else
                {
                    float2 r[5];
                    process_item<5, true, kLoopThreads>(s_item, ch, bd, smem_tbl, tbl_cap, smem_red, 0, 1, r, s_tbl_cache);
#pragma unroll
                    for (int q = 0; q < 5; q++) t[q] = r[q];
                }
            if (s_data_channel >= 0)
                {
                    // the same epoch against the data code: a second pass over the samples (the next iteration's barriers order
                    // thread 0's store before any read)
                    const float2 r = loop_correlate_data<kLoopThreads>(s_item, chans[s_data_channel], bd, smem_tbl_data, tbl_cap, smem_red, s_tbl_cache_data);
                    if (tid == 0) s_data_tap = r;
                }
            have_taps = true;
        }
    __syncthreads();
    if (tid == 0) sL->pending = 0;
    __syncthreads();
    copy_words(loops + i, sL, tid, kLoopThreads);
    if (tid == 0 && n_records) n_records[i] = k_rec;
}
}  // namespace

template <int THREADS>
static int launch_loop_persistent_width(LoopDev* loops, int n_loops, int max_epochs, const LoopAvail& avail, const ChanDesc* chans, const BandDesc* bands,
    const LoopData* data, unsigned int* records, int rec_capacity, int* n_records, float2* prompts, int tbl_cap, cudaStream_t st)
{
    const size_t tables = data ? 2 : 1;
    const size_t smem_bytes = tables * tbl_cap * 4 + (THREADS / 32) * B200_MAX_TAPS * sizeof(float2) + 2 * sizeof(LoopDev);
    static DeviceOnce once;
    const int once_dev = once.begin();
    if (once_dev >= 0)
        {
            B200_CUDA_TRY(cudaFuncSetAttribute(trk_loop_persistent_kernel<THREADS>, cudaFuncAttributeMaxDynamicSharedMemorySize, kTrkSmemMax));
            once.done(once_dev);
        }
    trk_loop_persistent_kernel<THREADS><<<n_loops, THREADS, smem_bytes, st>>>(loops, n_loops, max_epochs, avail, chans, bands, data, records,
        rec_capacity, n_records, prompts, tbl_cap);
    B200_CUDA_TRY(cudaGetLastError());
    return B200_OK;
}

int launch_loop_persistent(LoopDev* loops, int n_loops, int max_epochs, const LoopAvail& avail, const ChanDesc* chans, const BandDesc* bands,
    const LoopData* data, unsigned int* records, int rec_capacity, int* n_records, float2* prompts, int max_code_len, cudaStream_t st,
    uint64_t& launched)
{
    if (n_loops <= 0 || max_epochs <= 0) return B200_OK;
    const int tbl_cap = trk_table_cap(max_code_len, data ? 2 : 1, 4096);   // one table, or two with the data channels'
    // width: each loop is a latency chain, so with no more loops than SMs a wide CTA is the faster one; beyond that two narrow
    // CTAs per SM overlap each other's serial sections.  On an H100 (400 W), us per epoch: 32 loops 10.1-10.5 at 512 threads,
    // 11.2 at 256; 256 loops 29.5-30.0 at 256 threads, 33.6-34.0 at 512.
    int sms = 0, dev = 0;
    B200_CUDA_TRY(cudaGetDevice(&dev));
    B200_CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    const int rc = n_loops <= sms
                       ? launch_loop_persistent_width<kLoopThreadsFew>(loops, n_loops, max_epochs, avail, chans, bands, data, records, rec_capacity,
                             n_records, prompts, tbl_cap, st)
                       : launch_loop_persistent_width<kLoopThreadsMany>(loops, n_loops, max_epochs, avail, chans, bands, data, records, rec_capacity,
                             n_records, prompts, tbl_cap, st);
    if (rc == B200_OK) launched++;
    return rc;
}

int launch_loop_cycle(LoopDev* loops, int n_loops, int mode, const LoopAvail& avail, b200_trk_item* items, const float2* taps,
    const LoopData* data, unsigned int* records, int rec_capacity, int* n_records, float2* prompts, cudaStream_t st, uint64_t& launched)
{
    if (n_loops <= 0) return B200_OK;
    const int threads = 32;  // one loop per thread, spread over SMs: the per-loop chain is latency-bound
    trk_loop_cycle_kernel<<<(n_loops + threads - 1) / threads, threads, 0, st>>>(loops, n_loops, mode, avail, items, taps, data, records,
        rec_capacity, n_records, prompts);
    B200_CUDA_TRY(cudaGetLastError());
    launched++;
    return B200_OK;
}
}  // namespace b200
