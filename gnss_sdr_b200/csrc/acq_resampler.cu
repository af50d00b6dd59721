// The acquisition resampler of GNSS-SDR.use_acquisition_resampler (src/core/receiver/gnss_flowgraph.cc:1117-1212): a
// decimating low-pass FIR between the signal conditioner and a signal's acquisition blocks, so acquisition runs at the
// signal's optimal acquisition rate while tracking keeps the full rate.  b200_acq_resampler_design restates the filter
// design (host only) through firdes_low_pass, which b200_iq_conditioner_lowpass shares; acq_launch_decimate is the filter itself, run once per band search ahead of its forward stage.
#include "common.cuh"

#include <climits>
#include <cmath>

using namespace b200;

namespace
{
// Hamming, the default window of gr::filter::firdes::low_pass: its stop-band attenuation in dB (window::max_attenuation)
constexpr double kHammingAttenuationDb = 53.0;

// y[j] = sum_{k < n_taps} h[k] * x(j * D + (n_taps - 1) - k), j < n_out, where x(i) is sample i of the span (`in`, whose
// sample 0 is the oldest one the filter's history reaches).  k ascends from a zero accumulator and every multiply and add
// rounds on its own (__fmul_rn / __fadd_rn are never contracted into an FMA), so y is bit for bit the same loop in float32
// on the host.  One thread per output, the taps in shared memory.
template <int FMT>
__global__ void __launch_bounds__(256) acq_decimate_kernel(AcqInput in, const float* __restrict__ taps, int n_taps, int decimation,
    int n_out, float2* __restrict__ out)
{
    extern __shared__ float h[];
    for (int k = threadIdx.x; k < n_taps; k += blockDim.x) h[k] = taps[k];
    __syncthreads();
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n_out) return;
    const int newest = j * decimation + n_taps - 1;
    float re = 0.f, im = 0.f;
    for (int k = 0; k < n_taps; k++)
        {
            const float2 x = in.at<FMT>(newest - k);
            re = __fadd_rn(re, __fmul_rn(h[k], x.x));
            im = __fadd_rn(im, __fmul_rn(h[k], x.y));
        }
    out[j] = make_float2(re, im);
}
}  // namespace

namespace b200
{
long long firdes_low_pass(double fs, double cutoff, double transition, long long max_taps, float* taps)
{
    const double count = kHammingAttenuationDb * fs / (22.0 * transition);
    if (!(count < 0x1p62)) return LLONG_MAX;  // no buffer holds that many
    long long nt = static_cast<long long>(count);
    if ((nt & 1) == 0) nt++;
    if (nt > max_taps) return nt;
    const long long m = (nt - 1) / 2;
    const double pi = 3.14159265358979323846;
    const double fwT0 = 2.0 * pi * cutoff / fs;
    // taps[M + n] = w[M + n] sin(n fwT0) / (n pi), taps[M] = w[M] fwT0 / pi; Hamming w[i] = 0.54 - 0.46 cos(2 pi i / (ntaps - 1))
    const auto windowed_sinc = [&](long long n) {
        const double w = 0.54 - 0.46 * std::cos(2.0 * pi * static_cast<double>(n + m) / static_cast<double>(nt - 1));
        return w * (n == 0 ? fwT0 / pi : std::sin(static_cast<double>(n) * fwT0) / (static_cast<double>(n) * pi));
    };
    double dc_gain = 0.0;
    for (long long n = -m; n <= m; n++) dc_gain += windowed_sinc(n);
    // scaled to unit DC gain in double, each tap rounded once to float
    for (long long n = -m; n <= m; n++) taps[n + m] = static_cast<float>(windowed_sinc(n) / dc_gain);
    return nt;
}

int acq_launch_decimate(AcqInput in, const float* taps, int n_taps, int decimation, int n_out, float2* out, uint64_t& launched,
    cudaStream_t st)
{
    const int threads = 256;
    const int rc = with_format(in.fmt, [&](auto F) {
        acq_decimate_kernel<decltype(F)::value><<<(n_out + threads - 1) / threads, threads, sizeof(float) * n_taps, st>>>(in, taps, n_taps,
            decimation, n_out, out);
        return B200_OK;
    });
    if (rc) return rc;
    B200_CUDA_TRY(cudaGetLastError());
    launched++;
    return B200_OK;
}
}  // namespace b200

extern "C"
{
    int b200_acq_resampler_design(int64_t fs_in, int64_t opt_acq_fs, uint32_t max_taps, uint32_t* decimation, float* taps, uint32_t* n_taps)
    {
        if (fs_in <= 0 || opt_acq_fs <= 0 || !decimation || !n_taps || (max_taps > 0 && !taps)) return B200_ERR_ARG;
        *decimation = 1;
        *n_taps = 0;
        // gnss_flowgraph.cc:1164-1172: nothing is inserted when the optimal rate is not below the input rate, or when the
        // largest decimation that divides fs_in is 1
        if (opt_acq_fs >= fs_in) return B200_OK;
        int64_t d = static_cast<int64_t>(std::floor(static_cast<double>(fs_in) / static_cast<double>(opt_acq_fs)));
        while (fs_in % d > 0) d--;
        if (d <= 1) return B200_OK;
        // firdes::low_pass(1.0, fs, acq_fs_dec / 2.1, acq_fs_dec / 2) with the Hamming window, in double
        const double fs = static_cast<double>(fs_in);
        const double acq_fs_dec = fs / static_cast<double>(d);
        const int64_t nt = firdes_low_pass(fs, acq_fs_dec / 2.1, acq_fs_dec / 2.0, max_taps, taps);
        if (d > UINT32_MAX || nt > UINT32_MAX)
            {
                set_error("b200_acq_resampler_design: decimation %lld with %lld taps is out of range", (long long)d, (long long)nt);
                return B200_ERR_RANGE;
            }
        *decimation = static_cast<uint32_t>(d);
        *n_taps = static_cast<uint32_t>(nt);
        if (nt > static_cast<int64_t>(max_taps))
            {
                set_error("b200_acq_resampler_design: %lld taps needed (decimation %lld), max_taps is %u", (long long)nt, (long long)d, max_taps);
                return B200_ERR_RANGE;
            }
        return B200_OK;
    }
}
