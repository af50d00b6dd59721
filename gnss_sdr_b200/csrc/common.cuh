// Shared host/device declarations for libb200gnss.so (sm_90a only).
#pragma once

#include "../../include/b200gnss.h"

#include <cuda_runtime.h>
#include <atomic>
#include <cstdarg>
#include <cstdint>
#include <cstdio>

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

// One conditioned IQ stream resident in HBM.  Sample with absolute index i lives at
// base[(i - first_index) & mask]; attach-mode (linear) bands use mask = ~0.
struct BandDesc
{
    const float2* base;
    unsigned long long mask;
    unsigned long long first_index;
    unsigned long long limit;  // samples addressable from base (ring capacity or attached length)
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

// Launchers (trk_kernels.cu).  All pointers are device-accessible.
int launch_trk_batch(const b200_trk_item* items, int n_items, const ChanDesc* chans, const BandDesc* bands,
    float2* out, int out_stride, int slices, float2* partial, unsigned int* counters,
    int max_code_len, int taps_uniform, cudaStream_t stream, unsigned int taps_mask = 0u);
size_t trk_partial_elems(int n_items, int slices);
// shared-window kernel (trk_shared_kernel.cu): groups of 8 items share one copy of the samples
int launch_trk_shared(const b200_trk_item* items, int n_items, const ChanDesc* chans, const BandDesc* bands, float2* out,
    int out_stride, int taps_uniform, cudaStream_t stream);
int trk_shared_max_code_len();
// legacy correlator variants (trk_variants.cu): complex local code, 16-bit samples and code
int launch_trk_cplx_code(const float2* x, const float2* code, int n, int L, int taps, const float* shifts, float rem_carr, float dphi, float rem_code,
    float step, float2* out, cudaStream_t st);
int launch_trk_16sc(const short* x_iq, const short* code_iq, int n, int L, int taps, const float* shifts, float rem_carr, float dphi, float rem_code,
    float step, short* out_iq, cudaStream_t st);

}  // namespace b200

namespace b200
{
// sample-type adapters (ingest_kernels.cu)
int launch_convert_i16(const short* raw, float2* ring, unsigned long long mask, unsigned long long dst_off, unsigned long long n, cudaStream_t st);
int launch_convert_i8(const signed char* raw, float2* ring, unsigned long long mask, unsigned long long dst_off, unsigned long long n, cudaStream_t st);
}  // namespace b200

// ---- acquisition launchers (acq_kernels.cu) ----------------------------------------------------------
namespace b200
{
struct FftPlan;
struct AcqRowStat;
int acq_plan_make(int n, FftPlan* pl);
int acq_launch_twiddles(float2* tw, const FftPlan& pl, cudaStream_t st);
int acq_launch_wipeoff(float2* wipe, int n, int bins, int doppler_max, int doppler_center, int doppler_step,
    int doppler_bias, long long fs_in, int step_two, float center2, float step2, cudaStream_t st);
int acq_launch_code_fft(const float2* code, int consumed, int layout, float2* out, const FftPlan& pl, const float2* tw, cudaStream_t st);
int acq_launch_fwd(const float2* in, int consumed, const float2* wipe, float2* X, int bins, const FftPlan& pl, const float2* tw, cudaStream_t st);
int acq_launch_corr(const float2* X, const float2* codes, const int* slot_list, int n_slots, int bins, const FftPlan& pl,
    const float2* tw, int off, int ne, AcqRowStat* rowstat, float* grid, int accumulate, int mode, const void* best,
    int samples_per_chip, float* second_peak, float2* Z, AcqRowStat* partial, cudaStream_t st);
int acq_final_chunks(const FftPlan& pl);
int acq_launch_stats(const AcqRowStat* rowstat, int n_slots, int bins, int ne, int doppler_max, int doppler_center,
    int doppler_step, unsigned int dwell_counter, int use_cfar, void* best, b200_acq_result* results, int step_two, float center2,
    float step2, float prev_input_power, cudaStream_t st);
int acq_launch_finish_second_peak(const float* second_peak, int n_slots, b200_acq_result* results, cudaStream_t st);
int acq_plan_make_two_level(int m, FftPlan* pl);
int acq_launch_fwd_rows(const float2* in, size_t in_stride, int consumed, const float2* mult, size_t mult_stride, float2* X, int rows,
    const FftPlan& pl, const float2* tw, cudaStream_t st);
int acq_launch_inverse_store_rows(const float2* X, const float2* filt, const int* one_slot_dev, int rows, const FftPlan& pl, const float2* tw,
    float2* Z, const float2* post, int n_out, float2* out, size_t out_stride, cudaStream_t st);
int acq_launch_rows_times_vector(const float2* a, size_t a_stride, const float2* b, int n, int conj_a, float2* out, size_t out_stride, int rows,
    cudaStream_t st);
int acq_launch_sweep_best(const b200_acq_result* results, const unsigned int* prn_of_result, int n, b200_acq_peak* out, cudaStream_t st);
}  // namespace b200
