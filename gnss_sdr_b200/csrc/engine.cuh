// Host-side engine state shared by engine.cu (tracking) and acq_engine.cu (acquisition).
#pragma once

#include "common.cuh"
#include "cuda_owned.cuh"
#include "loop.cuh"

#include <algorithm>
#include <atomic>
#include <mutex>
#include <vector>

namespace b200
{
constexpr int kMaxBands = 16;

struct Band
{
    DevBuf<unsigned char> dev;  // owned ring (empty when attached)
    const void* base{nullptr};
    SampleFormat fmt{kCf32};    // what the ring holds (b200_iq_create_typed); attached buffers are float
    unsigned long long mask{0};
    unsigned long long first_index{0};
    unsigned long long capacity{0};
    unsigned long long write_index{0};  // absolute index of the next pushed sample
    unsigned long long valid_from{0};   // oldest absolute index whose sample is meaningful (after a gap push)
    bool attached{false};
    bool in_use{false};
    // device staging for integer sample pushes: two buffers, so that the next raw copy runs while the previous
    // block is being converted on the compute stream
    DevBuf<unsigned char> raw_stage[2];
    CudaEvent raw_free[2];  // conversion that read the buffer has finished
    int raw_next{0};
    int raw_last{-1};       // raw_free[raw_last] is recorded right after the band's latest conversion (-1: none yet)
    // the signal conditioner that fills this band from another (b200_iq_set_conditioner); src < 0: none
    struct Conditioner
    {
        int src{-1};
        unsigned decimation{1};
        unsigned n_taps{0};
        bool real_taps{true};                // IF = 0: real taps, no rotator
        unsigned long long rot_hi{0}, rot_lo{0};  // cond_rotator_step
        unsigned long long floor{0};         // no output below this is valid: where the conditioner was set or the band forgotten
        DevBuf<float2> taps;                 // composite taps c[k]
    } cond;
    // the segment stage that fills this band from another: a pulse blanker (b200_iq_set_pulse_blanking) or a notch
    // (b200_iq_set_notch); src < 0: none.  Both share the origin, restart, window, push-limit and chain rules.
    enum StageKind
    {
        kBlanker,
        kNotch,
    };
    struct SegStage
    {
        int src{-1};
        StageKind kind{kBlanker};
        int length{0};                       // L
        long long n_est{0}, n_reset{0};      // E, R
        float thres{0.f};
        unsigned long long origin{0};        // absolute index of segment 0
        unsigned long long segments{0};      // processed since origin
        unsigned long long seen_valid_from{0};  // the source's valid_from the origin follows: a move restarts the stage
        unsigned long long floor{0};         // no output below this is valid: where the band was last forgotten
        bool fresh{true};                    // the next scan starts from the block's initial state
        DevBuf<BlankState> state;
        DevBuf<float> energy;                // one per segment of a push
        DevBuf<unsigned char> flags;
        // notch only
        int variant{0};
        int n_coeff{1};
        float p{0.f};
        DevBuf<NotchState> notch_state;
        DevBuf<double2> twiddle, block_ab, y_grid;
        DevBuf<float> sig2lin;
        DevBuf<int> zsrc;
        DevBuf<float2> zseg, zs;
    } stage;
    CudaEvent cond_done;        // recorded on the compute stream after the latest conditioner or stage launch that read or wrote the band
    bool cond_recorded{false};  // cond_done has been recorded

    // B200_OK, or B200_ERR_STATE with the error text when this is not a ring made by b200_iq_create
    int check_owned_ring(int band) const
    {
        if (in_use && !attached && dev) return B200_OK;
        set_error("band %d is not an owned ring (call b200_iq_create)", band);
        return B200_ERR_STATE;
    }
    // oldest absolute index still held: an owned ring (first_index 0) keeps the last `capacity` samples pushed
    unsigned long long oldest() const { return (!attached && write_index > capacity) ? write_index - capacity : first_index; }
    // the band's readable window is [window_lo(), write_index) (what b200_iq_window reports)
    unsigned long long window_lo() const { return std::max(valid_from, oldest()); }
    // samples [s0, s0 + n) all lie inside that window; the test cannot wrap around 2^64
    bool holds(unsigned long long s0, unsigned long long n) const { return s0 >= window_lo() && s0 <= write_index && n <= write_index - s0; }
};

struct Channel
{
    DevBuf<float> code_dev;
    ChanDesc desc{};
};
}  // namespace b200

struct b200_engine
{
    // declared first, so released last: every buffer and event below was used on these streams
    b200::CudaStream stream;  // the caller's (borrowed) or the engine's own
    b200::CudaStream copy_stream;
    int device{0};
    b200::CudaEvent copy_done;
    b200::CudaEvent t0, t1;
    std::mutex mu;
    std::mutex push_mu[b200::kMaxBands];  // serialises competing producers of one band (b200_iq_push_at)
    b200::Band bands[b200::kMaxBands];
    std::vector<b200::Channel> chans;
    // device mirrors
    b200::DevBuf<b200::BandDesc> bands_dev;
    b200::DevBuf<b200::ChanDesc> chans_dev;
    bool tables_dirty{true};
    int max_code_len{0};
    unsigned int taps_mask{0};   // bit t set: some channel with a code table has t taps (a batch runs one launch per tap count)
    unsigned int fmt_mask{0};    // bit f set: some channel with a code table is on a band of SampleFormat f (and one per format)
    bool any_high_dyn{false};
    int shared_mode{2};    // shared-window kernel: 2 auto, 0 never, 1 always-when-legal (b200_trk_kernel_choice)
    b200::DevBuf<float2> partial;
    b200::DevBuf<unsigned int> counters;
    std::atomic<uint64_t> launches{0};  // kernels issued (b200_engine_launch_count); counted without e->mu
    // asynchronous batches (b200_trk_submit / b200_trk_wait)
    struct Slot
    {
        b200::PinBuf<b200_trk_item> items_pin;
        b200::DevBuf<b200_trk_item> items_dev;
        b200::DevBuf<float2> out_dev;
        b200::PinBuf<float2> out_pin;
        int n_items{0};
        int out_stride{0};
        b200::CudaEvent done;
        b200::CudaEvent items_ready;  // work items have arrived (copy stream)
        bool busy{false};
        bool zero_copy{false};  // items read from / taps written to the pinned host buffers directly (small batches)
        uint64_t ticket{0};
        std::vector<int> perm;  // results k belong to the caller's item perm[k] (empty = identity)
    };
    static constexpr int kSlots = 16;
    Slot slots[kSlots];
    uint64_t next_ticket{1};
    // free-running DLL/PLL loops (loop_engine.cu)
    std::vector<b200::LoopDev> loops;  // host mirror: configuration and start-of-tracking state
    b200::DevBuf<b200::LoopDev> loops_dev;
    b200::DevBuf<b200_trk_item> loop_items_dev;
    b200::DevBuf<float2> loop_taps_dev;
    b200::DevBuf<int> loop_nrec_dev;
    b200::DevBuf<unsigned int> loop_rec_dev;
    b200::DevBuf<float2> loop_prm_dev;          // pilot prompts beside the records (b200_trk_loop_run_prompts)
    std::vector<b200::LoopData> loop_data;      // data channel of each loop (b200_trk_loop_set_data_channel)
    int loop_n_data{0};                         // loops that have one
    b200::DevBuf<b200::LoopData> loop_data_dev;
    int loop_mode{0};        // 0 persistent kernel (default), 1 one launch pair per epoch with slices = 1, 2 same with automatic slices

    ~b200_engine()
    {
        if (stream) cudaStreamSynchronize(stream);
        if (copy_stream) cudaStreamSynchronize(copy_stream);
    }
};

namespace b200
{
// engine.cu
int upload_tables(b200_engine* e);
int ensure_partials(b200_engine* e, int n_items, int slices);
int batch_slices(int n_items);
}  // namespace b200
