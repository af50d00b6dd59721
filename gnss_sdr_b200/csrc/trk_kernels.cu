// Multi-tap tracking correlator for sm_90a.
//
// One CTA per (work item, slice).  A work item is one (channel, epoch): N complex samples of the
// band store, one code table, up to 8 taps.  The kernel fuses what the reference does in three
// passes over memory (VG = src/algorithms/libs/volk_gnsssdr_module/volk_gnsssdr):
//   a1  VG kernels/volk_gnsssdr/volk_gnsssdr_32f_xn_resampler_32f_xn.h:362-435  (code resampling,
//       never materialised here: the chip index is computed per sample in registers with the
//       SAME float32 operation order as the a_avx/u_avx kernel, so indices are bit-identical),
//   a2  VG kernels/volk_gnsssdr/volk_gnsssdr_32fc_32f_rotator_dot_prod_32fc_xn.h:155-314 (carrier
//       rotation + E/P/L dot products),
//   a3  src/algorithms/tracking/libs/cpu_multicorrelator_real_codes.cc:103-127 (phase set-up).
//
// Data movement: each sample is read exactly once per channel with coalesced 16-byte loads
// (LDG.128 = 2 samples per lane; 8 or 4 bytes for the same 2 samples of an int16 or int8 band); the code table is staged once per CTA in shared memory as an
// "extended" table that already contains the wrap-around, so the inner loop has no modulo.
// Reductions: registers -> warp shuffles -> shared memory -> (optionally) a deterministic
// cross-CTA combine when an epoch is split into slices for latency.
//
// Carrier: phase(n) = -(rem + n*step) is kept as a 64-bit fixed-point fraction of a turn.  The
// scalar path (correlate_range) re-seeds every group of kTrkReseed tiles exactly from it, to 2^-32
// turn regardless of n.  The fast path (correlate_tiles_fast) seeds each thread's two phasors
// exactly once per slice, advances them by the rounded phasor D of one tile inside a group and
// carries the group seed forward by the rounded phasor G of kTrkReseed tiles (8192 samples), so its
// phase error grows with the length of the slice.  On 20 ms GPS L2 CM-like epochs at one slice
// (tests/test_trk_paths_gpu.py) the worst measured error on an H100 80GB HBM3 (700 W) was
// 5.8e-6 |P| at 2 000 000 samples, against the suite's bound of 1e-5 |P|.
// No tensor cores: there is no dense contraction here.

#include "trk_item.cuh"

namespace b200
{
namespace
{
template <int TAPS, int FMT>
__device__ __forceinline__ void run_item(const b200_trk_item& it, const ChanDesc& ch, const BandDesc& bd,
    float* smem_tbl, int tbl_cap, float2* smem_red, int* smem_flag, int item_id, int slice, int slices,
    float2* out, int out_stride, float2* partial, unsigned int* counters)
{
    float2 result[TAPS];
    process_item<TAPS, false, kTrkThreads, FMT>(it, ch, bd, smem_tbl, tbl_cap, smem_red, slice, slices, result);
    const int tid = threadIdx.x;
    if (slices == 1)
        {
            if (tid < TAPS) out[static_cast<size_t>(item_id) * out_stride + tid] = result[tid];
            return;
        }
    // deterministic cross-CTA combine: every slice publishes its partial; the last one to arrive
    // adds them in slice order.
    float2* my = partial + (static_cast<size_t>(item_id) * slices + slice) * B200_MAX_TAPS;
    if (tid < TAPS) my[tid] = result[tid];
    __threadfence();
    __syncthreads();
    if (tid == 0)
        {
            const unsigned int prev = atomicAdd(&counters[item_id], 1u);
            *smem_flag = (prev == static_cast<unsigned int>(slices - 1));
        }
    __syncthreads();
    if (*smem_flag)
        {
            __threadfence();
            if (tid < TAPS)
                {
                    float2 s = make_float2(0.f, 0.f);
                    const volatile float2* p = partial + static_cast<size_t>(item_id) * slices * B200_MAX_TAPS;
                    for (int k = 0; k < slices; k++)
                        {
                            s.x += p[k * B200_MAX_TAPS + tid].x;
                            s.y += p[k * B200_MAX_TAPS + tid].y;
                        }
                    out[static_cast<size_t>(item_id) * out_stride + tid] = s;
                }
            if (tid == 0) counters[item_id] = 0u;  // ready for the next launch
        }
}

// One instantiation per tap count 1..8 (registers specialised to it).
// No minimum-blocks hint for 1, 3 and 5 taps.  sm_90a, no spills: <3> 64 registers (4 CTAs per SM), <1> 60, <5> 80 (3 CTAs).
// On an H100 (400 W), ms per step: a minimum of 4 blocks (everything at 64 registers; the generic kernel then in use spilled
// 3.3 KB) C3 5.43-5.46 vs 5.52-5.53, but C3 + pilot 9.12-9.14 vs 8.93-8.98 and the C5 share 2.73-2.80 vs 2.60-2.64; a minimum
// of 3 blocks slower on all four legs.
// Other tap counts keep the register budget of two CTAs per SM (128) that the kernel which read the tap count per item had:
// left to ptxas, <4>, <6> and <7> settle at 64-80 registers and spill.
// One instantiation per SampleFormat FMT of the band as well: each reads only the items whose band has its format (a float
// read of a narrow ring would run past its end) and leaves the others to the launch of theirs.
template <int TAPS, int FMT>
__global__ void __launch_bounds__(kTrkThreads, (TAPS == 1 || TAPS == 3 || TAPS == 5) ? 0 : 2)
    trk_correlate_kernel(const b200_trk_item* __restrict__ items, int n_items, const ChanDesc* __restrict__ chans, const BandDesc* __restrict__ bands, float2* __restrict__ out, int out_stride,
    int slices, float2* partial, unsigned int* counters, int tbl_cap, unsigned int only_mask)
{
    // only_mask != 0: a batch with several tap counts runs as one launch per tap count; this launch serves the items whose
    // channel has (1 << taps) in the mask and leaves the others to their own launch
    extern __shared__ __align__(16) float smem[];
    float* smem_tbl = smem;
    float2* smem_red = reinterpret_cast<float2*>(smem + tbl_cap);
    int* smem_flag = reinterpret_cast<int*>(smem_red + (kTrkThreads / 32) * B200_MAX_TAPS);

    for (int w = blockIdx.x; w < n_items * slices; w += gridDim.x)
        {
            const int item_id = w / slices;
            const int slice = w - item_id * slices;
            const b200_trk_item it = items[item_id];
            const ChanDesc& ch = chans[it.channel];
            if (only_mask != 0u && ((1u << ch.taps) & only_mask) == 0u) continue;   // uniform per CTA iteration
            const BandDesc bd = bands[ch.band];
            if (bd.fmt != FMT) continue;   // uniform per CTA iteration
            if (w != static_cast<int>(blockIdx.x)) __syncthreads();  // smem reuse across items
            if (it.n <= 0)
                {
                    if (slice == 0 && threadIdx.x < ch.taps) out[static_cast<size_t>(item_id) * out_stride + threadIdx.x] = make_float2(0.f, 0.f);
                    continue;
                }
            run_item<TAPS, FMT>(it, ch, bd, smem_tbl, tbl_cap, smem_red, smem_flag, item_id, slice, slices, out, out_stride, partial, counters);
        }
}

template <int T, int FMT>
int launch_one(const b200_trk_item* items, int n_items, const ChanDesc* chans, const BandDesc* bands, float2* out,
    int out_stride, int slices, float2* partial, unsigned int* counters, int tbl_cap, size_t smem_bytes, cudaStream_t stream, unsigned int only_mask)
{
    static DeviceOnce once;
    const int once_dev = once.begin();
    if (once_dev >= 0)
        {
            B200_CUDA_TRY(cudaFuncSetAttribute(trk_correlate_kernel<T, FMT>, cudaFuncAttributeMaxDynamicSharedMemorySize, kTrkSmemMax));
            once.done(once_dev);
        }
    const long long work = static_cast<long long>(n_items) * slices;
    // plain grid for moderate sizes, grid-stride beyond (keeps blockIdx math in int)
    const int grid = static_cast<int>(work < (1LL << 20) ? work : (1LL << 20));
    trk_correlate_kernel<T, FMT><<<grid, kTrkThreads, smem_bytes, stream>>>(items, n_items, chans, bands, out, out_stride, slices, partial, counters, tbl_cap,
        only_mask);
    B200_CUDA_TRY(cudaGetLastError());
    return B200_OK;
}
}  // namespace

size_t trk_partial_elems(int n_items, int slices)
{
    return static_cast<size_t>(n_items) * static_cast<size_t>(slices) * B200_MAX_TAPS;
}

int launch_trk_batch(const b200_trk_item* items, int n_items, const ChanDesc* chans, const BandDesc* bands,
    float2* out, int out_stride, int slices, float2* partial, unsigned int* counters,
    int max_code_len, unsigned int taps_mask, unsigned int fmt_mask, cudaStream_t stream, uint64_t& launched)
{
    if (n_items <= 0) return B200_OK;
    if (taps_mask == 0u || fmt_mask == 0u)
        {
            set_error("tracking batch: no channel has a code table");
            return B200_ERR_STATE;
        }
    if (slices < 1) slices = 1;
    const int tbl_cap = trk_table_cap(max_code_len, 1, 1024);
    const size_t smem_bytes = static_cast<size_t>(tbl_cap) * 4 + (kTrkThreads / 32) * B200_MAX_TAPS * sizeof(float2) + 16;
    // Several tap counts in one batch (a tracked pilot's 5 + 1 taps, a multi-signal receiver): one launch per tap count, each
    // serving its own items.  A kernel that read the tap count per item needed 128 registers and halved the occupancy.  Bands
    // of several sample formats: one launch per format as well.
    const bool mixed = (taps_mask & (taps_mask - 1u)) != 0u;
    for (int taps = 1; taps <= B200_MAX_TAPS; taps++)
        {
            if (!(taps_mask & (1u << taps))) continue;
            const unsigned int only_mask = mixed ? 1u << taps : 0u;
            for (const int fmt : {kCf32, kI16, kI8})
                {
                    if (!(fmt_mask & (1u << fmt))) continue;
                    const int rc = with_taps<1, 2, 3, 4, 5, 6, 7, 8>(taps, [&](auto tc) {
                        return with_format(fmt, [&](auto fc) {
                            return launch_one<decltype(tc)::value, decltype(fc)::value>(items, n_items, chans, bands, out, out_stride, slices,
                                partial, counters, tbl_cap, smem_bytes, stream, only_mask);
                        });
                    });
                    if (rc) return rc;
                    launched++;
                }
        }
    return B200_OK;
}

}  // namespace b200
