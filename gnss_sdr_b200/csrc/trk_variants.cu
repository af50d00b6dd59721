// Legacy correlator variants of the reference (SURVEY 2.1 / 8f N3), one CTA per call, latency-oriented:
//
//   complex local code   Cpu_Multicorrelator (src/algorithms/tracking/libs/cpu_multicorrelator.cc:73-100):
//                        volk_gnsssdr_32fc_xn_resampler_32fc_xn + volk_gnsssdr_32fc_x2_rotator_dot_prod_32fc_xn
//                        (VG kernels/volk_gnsssdr/...32fc_xn_resampler_32fc_xn.h:60-80, ...32fc_x2_rotator_dot_prod_32fc_xn.h:67-101)
//   16-bit samples       Cpu_Multicorrelator_16sc (cpu_multicorrelator_16sc.cc:64-91):
//                        volk_gnsssdr_16ic_xn_resampler_16ic_xn + volk_gnsssdr_16ic_x2_rotator_dot_prod_16ic_xn
//                        (...16ic_xn_resampler_16ic_xn.h:60-80, ...16ic_x2_rotator_dot_prod_16ic_xn.h:66-104)
//
// In the reference only the legacy TCP-connector tracking blocks use the former and no block uses the latter; they are
// here for completeness of the engine seam, not for throughput: every sample gets an exact phasor from the 64-bit
// fixed-point phase (no recurrence), the chip index is the same float32 sequence as everywhere else (AVX association
// below 8*floor(N/8), generic in the tail) with an integer modulo.
#include "common.cuh"
#include "trk_device.cuh"

namespace b200
{
namespace
{
constexpr int kVarThreads = 256;

struct VarArgs
{
    int n;
    int L;
    int taps;
    float rem_carrier_phase_rad, phase_step_rad, rem_code_phase_chips, code_phase_step_chips;
    float shifts[B200_MAX_TAPS];
};

__device__ __forceinline__ int chip_of(const VarArgs& a, int n, int body, int t)
{
    return mod_pos(chip_index_at(a.code_phase_step_chips, n, body, a.shifts[t], a.rem_code_phase_chips), a.L);
}

// result[t] = sum_n (x[n] * exp(-j(phi0 + n dphi))) * code[idx_t(n)]   (complex code)
__global__ void __launch_bounds__(kVarThreads) trk_cplx_code_kernel(const float2* __restrict__ x, const float2* __restrict__ code, VarArgs a,
    float2* __restrict__ out)
{
    __shared__ float2 red[kVarThreads / 32][B200_MAX_TAPS];
    const ItemPhase ph = item_phase(a.rem_carrier_phase_rad, a.phase_step_rad, a.n);
    float2 acc[B200_MAX_TAPS];
#pragma unroll
    for (int t = 0; t < B200_MAX_TAPS; t++) acc[t] = make_float2(0.f, 0.f);
    for (int n = threadIdx.x; n < a.n; n += kVarThreads)
        {
            const float2 w = cmulf(x[n], phasor_from_turns(ph.T0 + ph.DT * static_cast<unsigned long long>(n)));
#pragma unroll
            for (int t = 0; t < B200_MAX_TAPS; t++)
                {
                    if (t < a.taps)
                        {
                            const float2 c = __ldg(code + chip_of(a, n, ph.body, t));
                            acc[t].x += fmaf(w.x, c.x, -w.y * c.y);
                            acc[t].y += fmaf(w.x, c.y, w.y * c.x);
                        }
                }
        }
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
    for (int t = 0; t < B200_MAX_TAPS; t++)
        {
            const float2 s = warp_sum(acc[t]);
            if (lane == 0) red[warp][t] = s;
        }
    __syncthreads();
    if (threadIdx.x < a.taps)
        {
            float2 s = make_float2(0.f, 0.f);
            for (int w = 0; w < kVarThreads / 32; w++)
                {
                    s.x += red[w][threadIdx.x].x;
                    s.y += red[w][threadIdx.x].y;
                }
            out[threadIdx.x] = s;
        }
}

// 16-bit path: per sample the rotated sample is rounded to int16 (rintf), multiplied with the int16 complex code value
// with 16-bit wrap-around of each product component (std::complex<int16_t> multiplication truncates to 16 bits), and
// accumulated.  The reference accumulates with a saturating 16-bit add per sample; the sum here is exact in 64 bits and
// saturated once at the end - identical whenever the running sum never leaves [-32768, 32767], which is the operating
// range of that class (its own QA compares implementations to +-16 LSB, VG lib/kernel_tests.h).
__global__ void __launch_bounds__(kVarThreads) trk_16sc_kernel(const short2* __restrict__ x, const short2* __restrict__ code, VarArgs a,
    short2* __restrict__ out)
{
    __shared__ long long red[kVarThreads / 32][B200_MAX_TAPS][2];
    // the 16-bit resamplers have no AVX float association of their own in the tail; index sequence as for the float kernels
    const ItemPhase ph = item_phase(a.rem_carrier_phase_rad, a.phase_step_rad, a.n);
    long long ar[B200_MAX_TAPS], ai[B200_MAX_TAPS];
#pragma unroll
    for (int t = 0; t < B200_MAX_TAPS; t++) ar[t] = ai[t] = 0;
    for (int n = threadIdx.x; n < a.n; n += kVarThreads)
        {
            const short2 s = x[n];
            const float2 w = cmulf(make_float2(static_cast<float>(s.x), static_cast<float>(s.y)), phasor_from_turns(ph.T0 + ph.DT * static_cast<unsigned long long>(n)));
            const int wr = static_cast<short>(__float2int_rn(w.x)), wi = static_cast<short>(__float2int_rn(w.y));
#pragma unroll
            for (int t = 0; t < B200_MAX_TAPS; t++)
                {
                    if (t < a.taps)
                        {
                            const short2 c = code[chip_of(a, n, ph.body, t)];
                            const short pr = static_cast<short>(wr * c.x - wi * c.y);
                            const short pi = static_cast<short>(wr * c.y + wi * c.x);
                            ar[t] += pr;
                            ai[t] += pi;
                        }
                }
        }
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
    for (int t = 0; t < B200_MAX_TAPS; t++)
        {
            const long long sr = warp_sum(ar[t]), si = warp_sum(ai[t]);
            if (lane == 0)
                {
                    red[warp][t][0] = sr;
                    red[warp][t][1] = si;
                }
        }
    __syncthreads();
    if (threadIdx.x < a.taps)
        {
            long long sr = 0, si = 0;
            for (int w = 0; w < kVarThreads / 32; w++)
                {
                    sr += red[w][threadIdx.x][0];
                    si += red[w][threadIdx.x][1];
                }
            sr = sr > 32767 ? 32767 : (sr < -32768 ? -32768 : sr);
            si = si > 32767 ? 32767 : (si < -32768 ? -32768 : si);
            out[threadIdx.x] = make_short2(static_cast<short>(sr), static_cast<short>(si));
        }
}

VarArgs var_args(int n, int L, int taps, const float* shifts, float rem_carr, float dphi, float rem_code, float step)
{
    VarArgs a{};
    a.n = n;
    a.L = L;
    a.taps = taps;
    a.rem_carrier_phase_rad = rem_carr;
    a.phase_step_rad = dphi;
    a.rem_code_phase_chips = rem_code;
    a.code_phase_step_chips = step;
    for (int t = 0; t < taps; t++) a.shifts[t] = shifts[t];
    return a;
}
}  // namespace

int launch_trk_cplx_code(const float2* x, const float2* code, int n, int L, int taps, const float* shifts, float rem_carr, float dphi, float rem_code,
    float step, float2* out, cudaStream_t st, uint64_t& launched)
{
    trk_cplx_code_kernel<<<1, kVarThreads, 0, st>>>(x, code, var_args(n, L, taps, shifts, rem_carr, dphi, rem_code, step), out);
    B200_CUDA_TRY(cudaGetLastError());
    launched++;
    return B200_OK;
}

int launch_trk_16sc(const short* x_iq, const short* code_iq, int n, int L, int taps, const float* shifts, float rem_carr, float dphi, float rem_code,
    float step, short* out_iq, cudaStream_t st, uint64_t& launched)
{
    trk_16sc_kernel<<<1, kVarThreads, 0, st>>>(reinterpret_cast<const short2*>(x_iq), reinterpret_cast<const short2*>(code_iq),
        var_args(n, L, taps, shifts, rem_carr, dphi, rem_code, step), reinterpret_cast<short2*>(out_iq));
    B200_CUDA_TRY(cudaGetLastError());
    launched++;
    return B200_OK;
}
}  // namespace b200
