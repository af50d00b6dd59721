// The signal conditioner's input filter of InputFilter.implementation = Freq_Xlating_Fir_Filter
// (src/algorithms/input_filter/adapters/freq_xlating_fir_filter.cc:56-119, gr::filter::freq_xlating_fir_filter_ccf): every
// push into a source band fills a destination band with the frequency-translated, low-pass filtered and decimated stream
// (b200_iq_set_conditioner, engine.cu).  This file holds the filter kernel and the host arithmetic of its rotator.
#include "common.cuh"

#include <cmath>

using namespace b200;

namespace
{
constexpr int kCondThreads = 128;               // threads per CTA; a CTA makes at most this many consecutive outputs
constexpr int kCondSmemBytes = 99 * 1024;       // dynamic shared memory a CTA may take (two CTAs fit in one SM)

// Outputs j = j0 + blockIdx.x * per_cta + t, t < per_cta, of
//   y[j] = r(j) * sum_{k < n_taps} c[k] x[j D - k],  x[m < 0] = 0,
// x read from the ring `src` (slot m & src_mask) and widened to float at load, y written to slot j & dst_mask of `dst`.
// The CTA stages its span x[j_first D - (T - 1) .. j_last D] ((per_cta - 1) D + T samples) and the taps in shared memory.
// Arithmetic order is fixed: k ascends from a zero accumulator and every float product and sum rounds on its own (the
// intrinsics are never contracted into an FMA).  real_taps (IF = 0: c = h, r = 1): re += h x.re, im += h x.im and y is the
// accumulator itself.  Otherwise re += (c.re x.re - c.im x.im), im += (c.re x.im + c.im x.re), and y is the accumulator
// times r(j) = e^{-i 2 pi phi(j)} in double, rounded to float once per component.  phi(j) in cycles is the top 64 bits of
// j * rot mod 2^128, rot = (rot_hi, rot_lo) being D * IF / fs mod 1 as a 128-bit binary fraction (cond_rotator_step), so
// the phase of every output is reduced exactly from its absolute index.
template <int FMT>
__global__ void __launch_bounds__(kCondThreads) iq_condition_kernel(const void* __restrict__ src, unsigned long long src_mask,
    const float2* __restrict__ taps, int n_taps, int decimation, int per_cta, unsigned long long j0, unsigned long long n_out,
    int real_taps, unsigned long long rot_hi, unsigned long long rot_lo, float2* __restrict__ dst, unsigned long long dst_mask)
{
    extern __shared__ float2 sh[];
    float2* const h = sh;
    float2* const x = sh + n_taps;
    const unsigned long long first = static_cast<unsigned long long>(blockIdx.x) * per_cta;
    const int here = static_cast<int>(n_out - first < static_cast<unsigned long long>(per_cta) ? n_out - first : per_cta);
    const unsigned long long jc = j0 + first;
    const int span = (here - 1) * decimation + n_taps;
    const long long m0 = static_cast<long long>(jc * decimation) - (n_taps - 1);
    const SampleRaw<FMT>* const ring = static_cast<const SampleRaw<FMT>*>(src);
    for (int k = threadIdx.x; k < n_taps; k += blockDim.x) h[k] = taps[k];
    for (int s = threadIdx.x; s < span; s += blockDim.x)
        {
            const long long m = m0 + s;
            x[s] = m < 0 ? make_float2(0.f, 0.f) : widen<FMT>(__ldg(ring + (static_cast<unsigned long long>(m) & src_mask)));
        }
    __syncthreads();
    const int t = threadIdx.x;
    if (t >= here) return;
    const float2* const xj = x + t * decimation + (n_taps - 1);  // x[j D]
    float re = 0.f, im = 0.f;
    if (real_taps)
        {
            for (int k = 0; k < n_taps; k++)
                {
                    const float c = h[k].x;
                    const float2 v = xj[-k];
                    re = __fadd_rn(re, __fmul_rn(c, v.x));
                    im = __fadd_rn(im, __fmul_rn(c, v.y));
                }
            dst[(jc + t) & dst_mask] = make_float2(re, im);
            return;
        }
    for (int k = 0; k < n_taps; k++)
        {
            const float2 c = h[k];
            const float2 v = xj[-k];
            re = __fadd_rn(re, __fadd_rn(__fmul_rn(c.x, v.x), -__fmul_rn(c.y, v.y)));
            im = __fadd_rn(im, __fadd_rn(__fmul_rn(c.x, v.y), __fmul_rn(c.y, v.x)));
        }
    const unsigned long long j = jc + t;
    const unsigned long long top = j * rot_hi + __umul64hi(j, rot_lo);  // top 64 bits of j * rot mod 2^128
    const double phi = static_cast<double>(static_cast<long long>(top)) * 0x1p-64;  // cycles, in [-1/2, 1/2)
    double s, c;
    sincospi(2.0 * phi, &s, &c);
    // (re + i im) (c - i s)
    const double yr = __dadd_rn(__dmul_rn(re, c), __dmul_rn(im, s));
    const double yi = __dadd_rn(__dmul_rn(im, c), -__dmul_rn(re, s));
    dst[j & dst_mask] = make_float2(static_cast<float>(yr), static_cast<float>(yi));
}
}  // namespace

namespace b200
{
void cond_rotator_step(double intermediate_freq_hz, double sampling_freq_hz, unsigned decimation, unsigned long long* hi,
    unsigned long long* lo)
{
    // |IF| = mi 2^ei and fs = mf 2^ef with integer mantissas: |IF| D / fs = (D mi / mf) 2^s.  Bit i (weight 2^-i) of its
    // fraction is bit -i - s of D mi / mf: from the integer quotient for non-negative weights, from the remainder's long
    // division for negative ones.
    int ei = 0, ef = 0;
    const double fi = std::frexp(std::fabs(intermediate_freq_hz), &ei), ff = std::frexp(sampling_freq_hz, &ef);
    const unsigned long long mi = static_cast<unsigned long long>(std::ldexp(fi, 53)), mf = static_cast<unsigned long long>(std::ldexp(ff, 53));
    const int s = ei - ef;
    unsigned __int128 frac = 0;
    if (mi != 0)
        {
            const unsigned __int128 num = static_cast<unsigned __int128>(mi) * decimation;
            const unsigned __int128 quot = num / mf;
            unsigned long long rem = static_cast<unsigned long long>(num % mf);
            int pos = 0;  // weight of the last remainder bit generated (0: none yet)
            int last = 0;
            for (int i = 1; i <= 128; i++)
                {
                    const int w = -i - s;
                    int bit;
                    if (w >= 0)
                        bit = w < 128 ? static_cast<int>((quot >> w) & 1u) : 0;
                    else
                        {
                            while (pos > w)
                                {
                                    rem <<= 1;
                                    last = rem >= mf;
                                    if (last) rem -= mf;
                                    pos--;
                                }
                            bit = last;
                        }
                    frac |= static_cast<unsigned __int128>(bit) << (128 - i);
                }
        }
    if (intermediate_freq_hz < 0) frac = ~frac + 1;  // -x mod 1
    *hi = static_cast<unsigned long long>(frac >> 64);
    *lo = static_cast<unsigned long long>(frac);
}

int launch_iq_condition(const void* src, int src_fmt, unsigned long long src_mask, const float2* taps, int n_taps, int decimation,
    unsigned long long j0, unsigned long long n_out, int real_taps, unsigned long long rot_hi, unsigned long long rot_lo, float2* dst,
    unsigned long long dst_mask, cudaStream_t st)
{
    if (n_out == 0) return B200_OK;
    // as many consecutive outputs per CTA as the shared-memory budget stages (taps + span), at most one per thread
    const long long fit = (kCondSmemBytes / static_cast<long long>(sizeof(float2)) - 2LL * n_taps) / decimation + 1;
    const int per_cta = static_cast<int>(fit < kCondThreads ? (fit < 1 ? 1 : fit) : kCondThreads);
    const size_t smem = sizeof(float2) * (static_cast<size_t>(n_taps) + static_cast<size_t>(per_cta - 1) * decimation + n_taps);
    const unsigned long long blocks = (n_out + per_cta - 1) / per_cta;
    if (blocks > 0x7fffffffULL)
        {
            set_error("iq conditioner: %llu outputs in one launch", n_out);
            return B200_ERR_RANGE;
        }
    const int rc = with_format(src_fmt, [&](auto F) {
        constexpr int FMT = decltype(F)::value;
        static DeviceOnce once;
        const int d = once.begin();
        if (d >= 0)
            {
                B200_CUDA_TRY(cudaFuncSetAttribute(iq_condition_kernel<FMT>, cudaFuncAttributeMaxDynamicSharedMemorySize, kCondSmemBytes));
                once.done(d);
            }
        iq_condition_kernel<FMT><<<static_cast<unsigned>(blocks), kCondThreads, smem, st>>>(src, src_mask, taps, n_taps, decimation, per_cta,
            j0, n_out, real_taps, rot_hi, rot_lo, dst, dst_mask);
        return B200_OK;
    });
    if (rc) return rc;
    B200_CUDA_TRY(cudaGetLastError());
    return B200_OK;
}
}  // namespace b200

extern "C"
{
    int b200_iq_conditioner_lowpass(double sampling_freq_hz, uint32_t decimation, double bw_hz, double tw_hz, uint32_t max_taps,
        float* taps, uint32_t* n_taps)
    {
        if (!n_taps || (max_taps > 0 && !taps) || decimation < 1 || !(sampling_freq_hz > 0.0) || !std::isfinite(sampling_freq_hz) ||
            !std::isfinite(bw_hz) || !std::isfinite(tw_hz))
            return B200_ERR_ARG;
        *n_taps = 0;
        // freq_xlating_fir_filter.cc:103-110: bw defaults to (fs / decimation) / 2, tw to bw / 10
        const double bw = bw_hz > 0.0 ? bw_hz : (sampling_freq_hz / decimation) / 2;
        const double tw = tw_hz > 0.0 ? tw_hz : bw / 10.0;
        const long long nt = firdes_low_pass(sampling_freq_hz, bw, tw, max_taps, taps);
        *n_taps = static_cast<uint32_t>(nt < UINT32_MAX ? nt : UINT32_MAX);
        if (nt > static_cast<long long>(max_taps))
            {
                set_error("b200_iq_conditioner_lowpass: %lld taps needed, max_taps is %u", nt, max_taps);
                return B200_ERR_RANGE;
            }
        return B200_OK;
    }
}
