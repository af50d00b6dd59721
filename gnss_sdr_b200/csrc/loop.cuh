// Device-resident state of one free-running DLL/PLL loop (SURVEY 8f N1): the members of dll_pll_veml_tracking
// (src/algorithms/tracking/gnuradio_blocks/dll_pll_veml_tracking.h:128-222) that its per-epoch cycle reads or
// writes, with the reference's types (double / float / int32), plus the flattened state of its
// Tracking_loop_filter, Tracking_FLL_PLL_filter and two Exponential_Smoother members.
#pragma once

#include "common.cuh"

namespace b200
{
constexpr int kLoopMaxCn0Samples = 64;
constexpr int kLoopTapStride = B200_MAX_TAPS;  // taps buffer stride (complex values per loop)
constexpr int kLoopRecordWords = 27;           // sizeof(b200_trk_dump_record) / 4

// Exponential_Smoother (tracking/libs/exponential_smoother.h:54-62); init_buffer_ is only ever summed in
// push order from 0.0F, so a running float sum stands for it.
struct LoopSmoother
{
    float alpha, one_minus_alpha, old_value, min_value, offset, init_sum;
    int samples_for_initialization, init_counter, init_n, initializing;
};

struct LoopDev
{
    b200_trk_loop_conf c;
    int channel;  // engine tracking channel (code table, shifts, band)
    int taps;     // 3 (E,P,L) or 5 (VE,E,P,L,VL)
    int band;
    int pending;  // an item has been prepared for this loop and not yet consumed by an update
    // Tracking_loop_filter d_code_loop_filter (tracking_loop_filter.h:62-75)
    float dll_in_c[4], dll_out_c[3];
    int dll_n_in, dll_n_out, dll_index;
    float dll_inputs[4], dll_outputs[4];
    // Tracking_FLL_PLL_filter d_carrier_loop_filter (tracking_FLL_PLL_filter.h:40-50)
    float pll_w, pll_w0p3, pll_w0f2, pll_x, pll_a2, pll_w0f, pll_a3, pll_w0p2, pll_b3, pll_w0p;
    int pll_order;
    LoopSmoother cn0_smoother, carrier_lock_test_smoother;
    float2 Prompt_buffer[kLoopMaxCn0Samples];
    // block members
    double acq_code_phase_samples, acq_carrier_doppler_hz, current_correlation_time_s;
    double carr_phase_error_hz, carr_freq_error_hz, carr_error_filt_hz, code_error_chips, code_error_filt_chips;
    double code_freq_chips, carrier_doppler_hz, acc_carrier_phase_rad, rem_code_phase_chips;
    double carrier_lock_test, CN0_SNV_dB_Hz, carrier_lock_threshold;
    double carrier_phase_step_rad, carrier_phase_rate_step_rad, code_phase_step_chips, code_phase_rate_step_chips;
    double rem_code_phase_samples;
    float2 P_accu_old;
    unsigned long long acq_sample_stamp, nitems_read, epochs;
    float rem_carr_phase_rad, spc;
    int state, current_prn_length_samples, cn0_estimation_counter, carrier_lock_fail_counter, code_lock_fail_counter;
    int pull_in_transitory, cloop, loss_of_lock;
};

// absolute sample range currently resident in each band (host snapshot taken when a run is enqueued)
struct LoopAvail
{
    unsigned long long lo[16];
    unsigned long long hi[16];
};

// The data correlator of a loop that tracks a pilot (track_pilot: d_correlator_data_cpu, dll_pll_veml_tracking.cc:637-668):
// a 1-tap channel correlated on the loop's items with the pilot's NCO values.
struct LoopData
{
    int channel;  // data channel, -1: none
    int item;     // row of its item and tap in the batch buffers (kLoopDataItems): n_loops + its rank among the data loops
};

constexpr int kLoopPrepare = 1;     // prepare an item for loops that have none pending
constexpr int kLoopUpdate = 2;      // consume taps for loops with a pending item
constexpr int kLoopCheckAvail = 4;  // stall loops whose next vector_length samples are not resident
constexpr int kLoopDataItems = 8;   // prepare writes the data items to their rows, and the update takes the data tap from there
                                    // (without it the data tap is slot `taps` of the loop's own row, as b200_trk_loop_step_taps passes it)

// loop_kernels_nofma.cu.  data: per loop (may be nullptr: no data channels); prompts: n_loops x rec_capacity pilot prompts
// beside the records (may be nullptr).  Both launchers add the number of kernels they issued to `launched`.
int launch_loop_cycle(LoopDev* loops, int n_loops, int mode, const LoopAvail& avail, b200_trk_item* items, const float2* taps,
    const LoopData* data, unsigned int* records, int rec_capacity, int* n_records, float2* prompts, cudaStream_t st, uint64_t& launched);
// persistent free-running tracker: one CTA per loop, up to max_epochs cycles without leaving the SM; data == nullptr when no
// loop of the launch has a data channel (one code table in shared memory instead of two)
int launch_loop_persistent(LoopDev* loops, int n_loops, int max_epochs, const LoopAvail& avail, const ChanDesc* chans, const BandDesc* bands,
    const LoopData* data, unsigned int* records, int rec_capacity, int* n_records, float2* prompts, int max_code_len, cudaStream_t st,
    uint64_t& launched);
}  // namespace b200
