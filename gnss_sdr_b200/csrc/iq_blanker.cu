// The pulse-blanking input filter of InputFilter.implementation = Pulse_Blanking_Filter
// (src/algorithms/input_filter/gnuradio_blocks/pulse_blanking_cc.cc:33-98, adapters/pulse_blanking_filter.cc:43-84): every
// push into a source band fills a destination band with the source's samples, zeroed over each L-sample segment whose
// energy exceeds the chi-squared threshold times the noise estimate (b200_iq_set_pulse_blanking, engine.cu).  A push that
// completes K segments launches three kernels: the K segment energies, one CTA that runs the block's state machine over
// them, and the copy-or-zero pass into the destination.  This file holds the kernels and the host threshold.
#include "common.cuh"

#include <algorithm>
#include <cmath>

using namespace b200;

namespace
{
constexpr int kEnergyThreads = 128;   // one segment energy per thread
constexpr int kEnergyStage = 4096;    // samples a CTA stages (at most kEnergyThreads segments of them)
constexpr int kScanThreads = 1024;    // the scan's one CTA decides up to this many detection segments per step
constexpr int kApplyThreads = 256;

// e[k] = sum_{i < L} (re_i re_i + im_i im_i) over samples s0 + k L + i of the ring src, for k < n_seg: each square and sum
// rounded on its own, i ascending from 0.0 (volk_32fc_magnitude_squared_32f, then the generic volk_32f_accumulator_s32f).
// A CTA stages its segments in shared memory with coalesced loads, segment q at q * pitch, pitch = L | 1 (odd, so the
// threads of a warp, each reading its own segment, hit different banks).
template <int FMT>
__global__ void __launch_bounds__(kEnergyThreads) blank_energy_kernel(const void* __restrict__ src, unsigned long long src_mask,
    unsigned long long s0, int L, int per_cta, int n_seg, float* __restrict__ energy)
{
    extern __shared__ float2 x[];
    const int pitch = L | 1;
    const int seg0 = blockIdx.x * per_cta;
    const int here = min(per_cta, n_seg - seg0);
    const unsigned long long m0 = s0 + static_cast<unsigned long long>(seg0) * L;
    const SampleRaw<FMT>* const ring = static_cast<const SampleRaw<FMT>*>(src);
    const int span = here * L;
    for (int s = threadIdx.x; s < span; s += blockDim.x)
        {
            const int q = s / L;
            x[q * pitch + (s - q * L)] = widen<FMT>(__ldg(ring + ((m0 + s) & src_mask)));
        }
    __syncthreads();
    const int t = threadIdx.x;
    if (t >= here) return;
    const float2* const xs = x + t * pitch;
    float acc = 0.f;
    for (int i = 0; i < L; i++)
        {
            const float2 v = xs[i];
            acc = __fadd_rn(acc, __fadd_rn(__fmul_rn(v.x, v.x), __fmul_rn(v.y, v.y)));
        }
    energy[seg0 + t] = acc;
}

// pulse_blanking_cc::general_work's loop over n_seg segment energies (:71-95), writing flags[k] = 1 where segment k is
// zeroed, and carrying (n, est, last_filtered) and the blanked count in *state from one push to the next (fresh: start from
// the block's initial state instead).  Estimation (n < E and not last_filtered) is a serial recurrence and runs on thread 0,
// every operation rounded on its own.  In detection est is fixed, so every segment's decision e / est > thres is
// independent: the threads decide a step of up to kScanThreads segments at once, and the step ends at its first reset (a
// copied segment whose running n exceeds R), after which n = 1 and the state machine goes on from there.
__global__ void __launch_bounds__(kScanThreads) blank_scan_kernel(const float* __restrict__ energy, int n_seg, int fresh, float two_l,
    long long n_est, long long n_reset, float thres, BlankState* __restrict__ state, unsigned char* __restrict__ flags)
{
    __shared__ float e_sh[kScanThreads];
    __shared__ unsigned char f_sh[kScanThreads];
    __shared__ int warp_first[kScanThreads / 32];
    __shared__ long long n_sh;
    __shared__ float est_sh;
    __shared__ int lf_sh, i_sh, first_sh;
    __shared__ unsigned long long blanked_sh;
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    if (t == 0)
        {
            const BlankState s = fresh ? BlankState{} : *state;
            n_sh = s.n;
            est_sh = s.est;
            lf_sh = s.last_filtered;
            blanked_sh = s.blanked;
        }
    for (int base = 0; base < n_seg; base += kScanThreads)
        {
            const int c = min(kScanThreads, n_seg - base);
            if (t < c) e_sh[t] = energy[base + t];
            if (t == 0) i_sh = 0;
            __syncthreads();
            for (;;)
                {
                    const int i = i_sh;
                    const long long n = n_sh;
                    const int lf = lf_sh;
                    const float est = est_sh;
                    __syncthreads();  // every thread holds the step's state before thread 0 moves it on
                    if (i >= c) break;
                    if (n < n_est && !lf)
                        {
                            if (t == 0)
                                {
                                    float v = est;
                                    long long m = n;
                                    int k = i;
                                    for (; k < c && m < n_est; k++, m++)
                                        {
                                            v = __fdiv_rn(__fadd_rn(__fmul_rn(__ll2float_rn(m), v), __fdiv_rn(e_sh[k], two_l)), __ll2float_rn(m + 1));
                                            f_sh[k] = 0;
                                        }
                                    est_sh = v;
                                    n_sh = m;
                                    i_sh = k;
                                }
                        }
                    else
                        {
                            const int k = i + t;
                            const bool valid = k < c;
                            const bool blank = valid && __fdiv_rn(e_sh[k], est) > thres;
                            const bool reset = valid && !blank && n + t > n_reset;
                            const unsigned b = __ballot_sync(0xffffffffu, reset);
                            if (lane == 0) warp_first[warp] = b ? warp * 32 + __ffs(b) - 1 : kScanThreads;
                            __syncthreads();
                            if (warp == 0)
                                {
                                    int v = warp_first[lane];
                                    for (int o = 16; o > 0; o >>= 1) v = min(v, __shfl_xor_sync(0xffffffffu, v, o));
                                    if (lane == 0) first_sh = v;
                                }
                            __syncthreads();
                            const int first = first_sh;  // step index of the first reset, kScanThreads if none
                            const int end = min(first + 1, c - i);
                            if (t < end) f_sh[k] = blank;
                            const int nb = __syncthreads_count(t < end && blank);
                            if (t == 0)
                                {
                                    blanked_sh += static_cast<unsigned long long>(nb);
                                    if (first < kScanThreads)
                                        {
                                            n_sh = 1;  // n = 0 at the reset, then n++
                                            lf_sh = 0;
                                        }
                                    else
                                        {
                                            n_sh = n + end;
                                            lf_sh = f_sh[i + end - 1];
                                        }
                                    i_sh = i + end;
                                }
                        }
                    __syncthreads();
                }
            if (t < c) flags[base + t] = f_sh[t];
            __syncthreads();  // before the next step overwrites e_sh and f_sh
        }
    if (t == 0) *state = BlankState{n_sh, est_sh, lf_sh, blanked_sh};
}

// dst[m] = 0 where m's segment is flagged, else src[m] widened, for m = s0 + i, i < n_seg L; both rings wrap by their masks
template <int FMT>
__global__ void __launch_bounds__(kApplyThreads) blank_apply_kernel(const void* __restrict__ src, unsigned long long src_mask,
    unsigned long long s0, unsigned L, unsigned long long n, const unsigned char* __restrict__ flags, float2* __restrict__ dst,
    unsigned long long dst_mask)
{
    const SampleRaw<FMT>* const ring = static_cast<const SampleRaw<FMT>*>(src);
    for (unsigned long long i = static_cast<unsigned long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
         i += static_cast<unsigned long long>(gridDim.x) * blockDim.x)
        {
            const unsigned long long m = s0 + i;
            dst[m & dst_mask] = flags[i / L] ? make_float2(0.f, 0.f) : widen<FMT>(__ldg(ring + (m & src_mask)));
        }
}
}  // namespace

namespace b200
{
int launch_blank_energy(const void* src, int src_fmt, unsigned long long src_mask, unsigned long long s0, int L, int n_seg, float* energy,
    cudaStream_t st)
{
    if (n_seg <= 0) return B200_OK;
    const int per_cta = std::min(kEnergyThreads, std::max(1, kEnergyStage / L));
    const size_t smem = sizeof(float2) * static_cast<size_t>(per_cta) * static_cast<size_t>(L | 1);
    const unsigned blocks = static_cast<unsigned>((n_seg + per_cta - 1) / per_cta);
    const int rc = with_format(src_fmt, [&](auto F) {
        constexpr int FMT = decltype(F)::value;
        blank_energy_kernel<FMT><<<blocks, kEnergyThreads, smem, st>>>(src, src_mask, s0, L, per_cta, n_seg, energy);
        return B200_OK;
    });
    if (rc) return rc;
    B200_CUDA_TRY(cudaGetLastError());
    return B200_OK;
}

int launch_blank_scan(const float* energy, int n_seg, int fresh, int L, long long n_est, long long n_reset, float thres, BlankState* state,
    unsigned char* flags, cudaStream_t st)
{
    if (n_seg <= 0) return B200_OK;
    blank_scan_kernel<<<1, kScanThreads, 0, st>>>(energy, n_seg, fresh, static_cast<float>(2 * L), n_est, n_reset, thres, state, flags);
    B200_CUDA_TRY(cudaGetLastError());
    return B200_OK;
}

int launch_blank_apply(const void* src, int src_fmt, unsigned long long src_mask, unsigned long long s0, int L, int n_seg,
    const unsigned char* flags, float2* dst, unsigned long long dst_mask, cudaStream_t st)
{
    if (n_seg <= 0) return B200_OK;
    const unsigned long long n = static_cast<unsigned long long>(n_seg) * L;
    const unsigned long long want = (n + kApplyThreads - 1) / kApplyThreads;
    const unsigned blocks = static_cast<unsigned>(std::min<unsigned long long>(want, 132ULL * 64));
    const int rc = with_format(src_fmt, [&](auto F) {
        constexpr int FMT = decltype(F)::value;
        blank_apply_kernel<FMT><<<blocks, kApplyThreads, 0, st>>>(src, src_mask, s0, static_cast<unsigned>(L), n, flags, dst, dst_mask);
        return B200_OK;
    });
    if (rc) return rc;
    B200_CUDA_TRY(cudaGetLastError());
    return B200_OK;
}
}  // namespace b200

namespace
{
// log of the chi-squared upper tail with 2L degrees of freedom at x: Q = e^{-y} sum_{k < L} y^k / k!, y = x / 2, summed in
// log space so that neither e^{-y} nor y^k under- or overflows
double log_erlang_tail(double x, int L)
{
    const double y = 0.5 * x;
    if (y <= 0.0) return 0.0;
    const double ly = std::log(y);
    double lt = -y, m = -y;  // log of term k, and the largest so far
    double sum = 1.0;        // sum of exp(log term - m)
    for (int k = 1; k < L; k++)
        {
            lt += ly - std::log(static_cast<double>(k));
            if (lt > m)
                {
                    sum = sum * std::exp(m - lt) + 1.0;
                    m = lt;
                }
            else
                sum += std::exp(lt - m);
        }
    return m + std::log(sum);
}
}  // namespace

extern "C"
{
    int b200_iq_pulse_blanking_threshold(float pfa, int32_t length, float* thres)
    {
        if (!thres || !(pfa > 0.f && pfa < 1.f) || length < 1 || length > B200_IQ_MAX_BLANKING_LENGTH)
            {
                set_error("iq_pulse_blanking_threshold: pfa %g must lie in (0, 1) and length %d in [1, %d]", static_cast<double>(pfa), length,
                    B200_IQ_MAX_BLANKING_LENGTH);
                return B200_ERR_ARG;
            }
        // the tail falls monotonically in x: bisect in double until the bracket cannot shrink
        const double lp = std::log(static_cast<double>(pfa));
        double lo = 0.0, hi = 2.0 * length + 16.0;
        while (log_erlang_tail(hi, length) > lp) hi *= 2.0;
        for (int it = 0; it < 4096; it++)
            {
                const double mid = 0.5 * (lo + hi);
                if (mid <= lo || mid >= hi) break;
                if (log_erlang_tail(mid, length) > lp)
                    lo = mid;
                else
                    hi = mid;
            }
        *thres = static_cast<float>(hi);
        return B200_OK;
    }
}
