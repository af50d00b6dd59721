// Shared host/device declarations for libb200gnss.so (sm_90a only).
#pragma once

#include "../../include/b200gnss.h"

#include <cuda_runtime.h>
#include <atomic>
#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <type_traits>

namespace b200
{
// thread-local last-error text behind b200_last_error()
void set_error(const char* fmt, ...);
const char* get_error();

#define B200_CUDA_TRY(expr)                                                                            \
    do                                                                                                 \
        {                                                                                              \
            cudaError_t _e = (expr);                                                                   \
            if (_e != cudaSuccess)                                                                     \
                {                                                                                      \
                    ::b200::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
                    (void)cudaGetLastError(); /* reported here: must not surface again after a later launch */ \
                    return B200_ERR_CUDA;                                                              \
                }                                                                                      \
        }                                                                                              \
    while (0)

// First statement of every entry point that touches the device.  The runtime keeps ONE last-error slot per host thread,
// shared with every other CUDA user in the process (torch leaves "invalid device ordinal" there while it initialises): an
// error somebody else left must not be reported by the cudaGetLastError() after our next launch.
#define B200_ENTER_DEVICE(dev)              \
    do                                      \
        {                                   \
            (void)cudaGetLastError();       \
            B200_CUDA_TRY(cudaSetDevice(dev)); \
        }                                   \
    while (0)

// Function attributes (opt-in dynamic shared memory) are per device: remember per device, thread-safe, which
// kernels have been prepared.  Usage:
//   static DeviceOnce once;  const int d = once.begin();  if (d >= 0) { cudaFuncSetAttribute(...); once.done(d); }
struct DeviceOnce
{
    std::atomic<unsigned long long> mask{0ULL};
    // current device index when its attributes still have to be set (64 = unknown device: set them again,
    // the call is idempotent), -1 when nothing is left to do
    int begin()
    {
        int d = -1;
        if (cudaGetDevice(&d) != cudaSuccess || d < 0 || d >= 64) return 64;
        return (mask.load(std::memory_order_acquire) & (1ULL << d)) ? -1 : d;
    }
    void done(int d)
    {
        if (d >= 0 && d < 64) mask.fetch_or(1ULL << d, std::memory_order_release);
    }
};

// A band's sample type, by bytes per component: gr_complex (float I, Q), and interleaved (I, Q) int16 (lv_16sc_t, the
// reference's "ishort") and int8 ("ibyte") pairs.  A sample takes 2 * format bytes.
enum SampleFormat
{
    kI8 = 1,
    kI16 = 2,
    kCf32 = 4,
};

// f(std::integral_constant<int, F>{}) for the SampleFormat F that equals fmt; B200_ERR_ARG when there is none
template <class F>
int with_format(int fmt, const F& f)
{
    switch (fmt)
        {
        case kCf32: return f(std::integral_constant<int, kCf32>{});
        case kI16: return f(std::integral_constant<int, kI16>{});
        case kI8: return f(std::integral_constant<int, kI8>{});
        default: set_error("unknown sample format %d", fmt); return B200_ERR_ARG;
        }
}

// int -> float of narrow sample components (I2F; exact for every int16 and int8).  w holds (I, Q) of one int16 sample, or of
// int8 samples in bytes (2K, 2K + 1).  The exact I2F-free alternative (the biased component permuted into the mantissa of
// 2^23, then one FADD) was measured against it on an H100 80GB HBM3 (700 W), per-item kernel, ms per step: C2 distinct-IQ
// ishort 0.707 vs 0.689 (I2F), ibyte 0.638 vs 0.648; C2 shared layout ishort 1.224 vs 1.186, ibyte 1.214 vs 1.223.  Neither
// wins on both widths, and only I2F keeps every instantiation spill-free (the permute form spilled at 8 taps on ishort).
__device__ __forceinline__ float2 widen_i16(unsigned int w)
{
    return make_float2(static_cast<float>(static_cast<short>(w & 0xffffu)), static_cast<float>(static_cast<short>(w >> 16)));
}
template <int K>
__device__ __forceinline__ float2 widen_i8(unsigned int w)
{
    return make_float2(static_cast<float>(static_cast<signed char>((w >> (16 * K)) & 0xffu)),
        static_cast<float>(static_cast<signed char>((w >> (16 * K + 8)) & 0xffu)));
}

// the raw element of one sample of SampleFormat FMT, and that element widened to float
template <int FMT>
using SampleRaw = std::conditional_t<FMT == kCf32, float2, std::conditional_t<FMT == kI16, unsigned int, unsigned short>>;
template <int FMT>
__device__ __forceinline__ float2 widen(SampleRaw<FMT> v)
{
    if constexpr (FMT == kCf32)
        return v;
    else if constexpr (FMT == kI16)
        return widen_i16(v);
    else
        return widen_i8<0>(v);
}

// One conditioned IQ stream resident in HBM.  Sample with absolute index i lives at sample slot (i - first_index) & mask
// from base, each slot 2 * fmt bytes; attach-mode (linear) bands use mask = ~0.
struct BandDesc
{
    const void* base;
    unsigned long long mask;
    unsigned long long first_index;
    unsigned long long limit;  // samples addressable from base (ring capacity or attached length)
    int fmt;                   // SampleFormat
};

// The samples an acquisition forward stage reads: x(i) = a[i] for i < na, b[i - na] from there on, in format fmt.  A window
// of a band is at most two linear runs (it may wrap around the ring's end); a linear buffer is one run of float2, with na
// past every index.
struct AcqInput
{
    const void* a;
    int na;
    const void* b;
    int fmt;  // SampleFormat
    static AcqInput linear(const float2* p) { return AcqInput{p, 0x7fffffff, nullptr, kCf32}; }
    // x(i) for an input of format FMT (== fmt), widened to float on load
    template <int FMT>
    __device__ __forceinline__ float2 at(int i) const
    {
        using Raw = SampleRaw<FMT>;
        return widen<FMT>(__ldg(i < na ? static_cast<const Raw*>(a) + i : static_cast<const Raw*>(b) + (i - na)));
    }
};

// One tracking channel registration: code table (device), its length, taps and shifts.
struct ChanDesc
{
    const float* code;
    int code_len;
    int taps;
    int band;
    int high_dyn;
    float shifts[B200_MAX_TAPS];
};

constexpr int kTrkThreads = 256;            // threads per CTA
constexpr int kTrkTile = 2 * kTrkThreads;   // samples per CTA iteration (one LDG.128 per thread)
constexpr int kTrkReseed = 16;              // tiles between exact phasor re-seeds
constexpr int kTrkTablePad = 64;            // extra entries of the extended code table
constexpr int kTrkSmemMax = 200 * 1024;     // dynamic shared memory the per-item and loop kernels opt in to

// entries of each extended code table in a CTA's shared memory: the longest code + padding, limited so that `tables` of them
// and reserved_bytes of other data fit, rounded up to 4
inline int trk_table_cap(int max_code_len, int tables, int reserved_bytes)
{
    const int cap_limit = (kTrkSmemMax - reserved_bytes) / (4 * tables);
    const int cap = max_code_len + kTrkTablePad;
    return ((cap < cap_limit ? cap : cap_limit) + 3) & ~3;
}

// f(std::integral_constant<int, T>{}) for the T of Ts that equals taps; B200_ERR_ARG when there is none
template <int... Ts, class F>
int with_taps(int taps, const F& f)
{
    int rc = B200_ERR_ARG;
    (void)((taps == Ts ? (rc = f(std::integral_constant<int, Ts>{}), true) : false) || ...);
    return rc;
}

// Launchers (trk_kernels.cu).  All pointers are device-accessible.  Each adds the number of kernels it issued to `launched`.
// taps_mask: bit t set when some channel with a code table has t taps; fmt_mask: bit f set when some such channel is on a band
// of SampleFormat f.  One launch per (tap count, format) pair; an empty mask is an error.
int launch_trk_batch(const b200_trk_item* items, int n_items, const ChanDesc* chans, const BandDesc* bands,
    float2* out, int out_stride, int slices, float2* partial, unsigned int* counters,
    int max_code_len, unsigned int taps_mask, unsigned int fmt_mask, cudaStream_t stream, uint64_t& launched);
size_t trk_partial_elems(int n_items, int slices);
// shared-window kernel (trk_shared_kernel.cu): groups of 8 items share one copy of the samples; every channel has `taps` taps
// and sits on a float band (it reads samples as float2)
int launch_trk_shared(const b200_trk_item* items, int n_items, const ChanDesc* chans, const BandDesc* bands, float2* out,
    int out_stride, int taps, cudaStream_t stream, uint64_t& launched);
int trk_shared_max_code_len();
// legacy correlator variants (trk_variants.cu): complex local code, 16-bit samples and code
int launch_trk_cplx_code(const float2* x, const float2* code, int n, int L, int taps, const float* shifts, float rem_carr, float dphi, float rem_code,
    float step, float2* out, cudaStream_t st, uint64_t& launched);
int launch_trk_16sc(const short* x_iq, const short* code_iq, int n, int L, int taps, const float* shifts, float rem_carr, float dphi, float rem_code,
    float step, short* out_iq, cudaStream_t st, uint64_t& launched);

}  // namespace b200

namespace b200
{
// sample-type adapters (ingest_kernels.cu)
int launch_convert_i16(const short* raw, float2* ring, unsigned long long mask, unsigned long long dst_off, unsigned long long n, cudaStream_t st);
int launch_convert_i8(const signed char* raw, float2* ring, unsigned long long mask, unsigned long long dst_off, unsigned long long n, cudaStream_t st);

// signal conditioner (iq_conditioner.cu): outputs [j0, j0 + n_out) of b200_iq_set_conditioner's filter from the ring src (slot
// mask src_mask, SampleFormat src_fmt) into the float ring dst.  taps: the n_taps composite taps c[k]; real_taps: IF = 0 (c[k]
// real, no rotator); (rot_hi, rot_lo): cond_rotator_step's phase step per output.  n_out == 0 launches nothing.
int launch_iq_condition(const void* src, int src_fmt, unsigned long long src_mask, const float2* taps, int n_taps, int decimation,
    unsigned long long j0, unsigned long long n_out, int real_taps, unsigned long long rot_hi, unsigned long long rot_lo, float2* dst,
    unsigned long long dst_mask, cudaStream_t st);
// decimation * intermediate_freq_hz / sampling_freq_hz mod 1 (cycles per output) as a 128-bit binary fraction, computed exactly
// from the two doubles; sampling_freq_hz > 0
void cond_rotator_step(double intermediate_freq_hz, double sampling_freq_hz, unsigned decimation, unsigned long long* hi,
    unsigned long long* lo);
// gr::filter::firdes::low_pass(1.0, fs, cutoff, transition) with the Hamming window, in double (acq_resampler.cu): returns the
// tap count int(53 fs / (22 transition)) made odd, and writes the taps, each rounded once to float, only when that count is
// <= max_taps
long long firdes_low_pass(double fs, double cutoff, double transition, long long max_taps, float* taps);

// pulse blanker (iq_blanker.cu).  The state pulse_blanking_cc carries from one segment to the next (n_segments_,
// noise_power_estimation_, last_filtered_), kept in device memory, and the segments it has zeroed.
struct BlankState
{
    long long n;
    float est;
    int last_filtered;
    unsigned long long blanked;
};
// energies[k] of the n_seg segments of L samples from absolute index s0 of the ring src (slot mask src_mask, SampleFormat src_fmt)
int launch_blank_energy(const void* src, int src_fmt, unsigned long long src_mask, unsigned long long s0, int L, int n_seg, float* energy,
    cudaStream_t st);
// the block's state machine over those energies: flags[k] = 1 where segment k is zeroed; *state carried (fresh: initial state)
int launch_blank_scan(const float* energy, int n_seg, int fresh, int L, long long n_est, long long n_reset, float thres, BlankState* state,
    unsigned char* flags, cudaStream_t st);
// the n_seg L samples from s0: copied from src (widened) or zeroed by flags, into the float ring dst.  Each launcher issues one
// kernel, none for n_seg == 0.
int launch_blank_apply(const void* src, int src_fmt, unsigned long long src_mask, unsigned long long s0, int L, int n_seg,
    const unsigned char* flags, float2* dst, unsigned long long dst_mask, cudaStream_t st);

// notch filters (iq_notch.cu).  The state Notch / NotchLite carry from one segment to the next, kept in device memory, with
// the IIR's double carry on the absolute grid of kNotchGrid output samples counted from the origin.
constexpr int kNotchGrid = 1024;
struct NotchState
{
    long long n;                    // n_segments_
    float est;                      // noise_pow_est_
    int filter_state;               // filter_state_
    int n_coeff;                    // n_segments_coeff_ (Lite)
    int last_seg;                   // the last filtered segment of the latest push (-1: none)
    float2 z0;                      // z_0_
    float2 last_out, last_in;       // last_out_ after the latest push; and before it (read by the apply pass)
    double2 y_grid;                 // y entering the grid block in progress
    double2 pa, pb;                 // that block's map y -> pa y + pb over its samples so far
    unsigned long long filtered;    // segments filtered
};
// the resources of one notch: flags[k] bit 0 filtered, bit 1 a run starts; zsrc[k] the segment (push index) whose z0
// segment k uses (Lite; < 0: the carried one); zseg[k] that z0; zs[i] the per-sample z0 of the push (Notch)
struct NotchBufs
{
    NotchState* state;
    const double2* twiddle;  // exp(-2 pi i m / L), m < L, made on the host
    float* energy;
    float* sig2lin;
    unsigned char* flags;
    int* zsrc;
    float2* zseg;
    float2* zs;
    double2* block_ab;       // (A, B) of each grid block of the push
    double2* y_grid;         // y entering each grid block of the push
};
struct NotchParams
{
    int variant;  // B200_NOTCH or B200_NOTCH_LITE
    int L;
    long long n_est, n_reset;
    int n_coeff;
    float thres, p;
    unsigned long long origin;
};
// the six launches of a push that completes n_seg >= 1 segments, from segment seg0 (counted from the origin), on st
int launch_notch(const void* src, int src_fmt, unsigned long long src_mask, const NotchParams& prm, unsigned long long seg0, int n_seg,
    int fresh, const NotchBufs& b, float2* dst, unsigned long long dst_mask, cudaStream_t st);
}  // namespace b200

// ---- acquisition launchers (acq_kernels.cu) ----------------------------------------------------------
namespace b200
{
struct FftPlan;

// (max, first arg-max, sum) of |y|^2 over one correlation row
struct AcqRowStat
{
    float max;
    unsigned int argmax;
    float sum;
    float pad;
};

// winning cell of one searched slot, as acq_stats_kernel found it
struct AcqBest
{
    unsigned int index_time;
    unsigned int index_doppler;
};

// set_local_code (pcps_acquisition.cc:230-246): where the local code starts in the n-point buffer.  Layout 0: code[0..consumed)
// at the front (sampled_ms == ms_per_code); 1: bit_transition_flag, code[0..n/2) in the second half; 2: zero-padded front,
// code[0..consumed) at [n - consumed, n).  Zeros elsewhere.
__host__ __device__ inline int acq_code_offset(int layout, int n, int consumed)
{
    return (layout == 1) ? n / 2 : (layout == 2) ? n - consumed : 0;
}

// CTA "first maximum" of (value, index) plus the sum of the values: xor-shuffle 16 -> 1 in each warp, then thread 0 combines
// warps 1..WARPS-1 in ascending order.  The result is valid in thread 0 only.
template <int WARPS>
__device__ __forceinline__ void acq_cta_first_max(float& bv, unsigned int& bi, float& sm)
{
    __shared__ float red_v[WARPS];
    __shared__ unsigned int red_i[WARPS];
    __shared__ float red_s[WARPS];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1)
        {
            const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
            const unsigned int oi = __shfl_xor_sync(0xffffffffu, bi, o);
            sm += __shfl_xor_sync(0xffffffffu, sm, o);
            if (ov > bv || (ov == bv && oi < bi))
                {
                    bv = ov;
                    bi = oi;
                }
        }
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0)
        {
            red_v[warp] = bv;
            red_i[warp] = bi;
            red_s[warp] = sm;
        }
    __syncthreads();
    if (threadIdx.x == 0)
        {
            for (int w = 1; w < WARPS; w++)
                {
                    if (red_v[w] > bv || (red_v[w] == bv && red_i[w] < bi))
                        {
                            bv = red_v[w];
                            bi = red_i[w];
                        }
                    sm += red_s[w];
                }
        }
}

// Acquisition launchers (acq_kernels.cu).  Those on the search path add the number of kernels they issued to `launched`.
int acq_plan_make(int n, FftPlan* pl);
int acq_plan_make_two_level(int m, FftPlan* pl);
int acq_final_chunks(const FftPlan& pl);
int acq_launch_twiddles(float2* tw, const FftPlan& pl, cudaStream_t st);
int acq_launch_wipeoff(float2* wipe, int n, int bins, int doppler_max, int doppler_center, int doppler_step,
    int doppler_bias, long long fs_in, int step_two, float center2, float step2, cudaStream_t st);
int acq_launch_code_fft(const float2* code, int consumed, int layout, float2* out, const FftPlan& pl, const float2* tw, cudaStream_t st);
int acq_launch_fwd(AcqInput in, int consumed, const float2* wipe, float2* X, int bins, const FftPlan& pl, const float2* tw,
    uint64_t& launched, cudaStream_t st);
// rowstat[slot_pos * bins + bin] for every (slot, bin) row over [off, off + ne) of the correlation; grid != nullptr: each row's
// |y|^2 is stored there (accumulate: added to what is there)
int acq_launch_row_stats(const float2* X, const float2* codes, const int* slot_list, int n_slots, int bins, const FftPlan& pl,
    const float2* tw, int off, int ne, float* grid, int accumulate, AcqRowStat* rowstat, float2* Z, AcqRowStat* partial,
    uint64_t& launched, cudaStream_t st);
// second_peak[slot_pos]: maximum of the winning row best[slot_pos] with +-samples_per_chip around its peak zeroed, read from the
// grid when there is one, else recomputed
int acq_launch_second_peak(const float2* X, const float2* codes, const int* slot_list, int n_slots, int bins, const FftPlan& pl,
    const float2* tw, int off, int ne, float* grid, const AcqBest* best, int samples_per_chip, float* second_peak, float2* Z,
    AcqRowStat* partial, uint64_t& launched, cudaStream_t st);
int acq_launch_stats(const AcqRowStat* rowstat, int n_slots, int bins, int ne, int doppler_max, int doppler_center,
    int doppler_step, unsigned int dwell_counter, int use_cfar, AcqBest* best, b200_acq_result* results, int step_two, float center2,
    float step2, float prev_input_power, uint64_t& launched, cudaStream_t st);
int acq_launch_finish_second_peak(const float* second_peak, int n_slots, b200_acq_result* results, uint64_t& launched, cudaStream_t st);
// in_stride > 0 (rows of one linear buffer) needs a linear view
int acq_launch_fwd_rows(AcqInput in, size_t in_stride, int consumed, const float2* mult, size_t mult_stride, float2* X, int rows,
    const FftPlan& pl, const float2* tw, uint64_t& launched, cudaStream_t st);
int acq_launch_inverse_store_rows(const float2* X, const float2* filt, const int* one_slot_dev, int rows, const FftPlan& pl, const float2* tw,
    float2* Z, const float2* post, int n_out, float2* out, size_t out_stride, uint64_t& launched, cudaStream_t st);
int acq_launch_rows_times_vector(const float2* a, size_t a_stride, const float2* b, int n, int conj_a, float2* out, size_t out_stride, int rows,
    cudaStream_t st);
int acq_launch_sweep_best(const b200_acq_result* results, const unsigned int* prn_of_result, int n, b200_acq_peak* out, uint64_t& launched,
    cudaStream_t st);
// acquisition resampler (acq_resampler.cu): out[j] = sum_{k < n_taps} taps[k] * x(j * decimation + n_taps - 1 - k), j < n_out, for
// the span x = in; every product and sum rounded on its own, k ascending.  n_taps <= B200_ACQ_MAX_RESAMPLER_TAPS.
int acq_launch_decimate(AcqInput in, const float* taps, int n_taps, int decimation, int n_out, float2* out, uint64_t& launched,
    cudaStream_t st);
}  // namespace b200
