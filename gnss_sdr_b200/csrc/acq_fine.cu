// Fine Doppler estimate of pcps_acquisition_fine_doppler_cc::estimate_Doppler
// (src/algorithms/acquisition/gnuradio_blocks/pcps_acquisition_fine_doppler_cc.cc:316-389): the 10 ms buffer is
// wiped off with 10 replicas of the aligned local code, zero-padded 8x, transformed, and the frequency of the
// largest |X[k]|^2 (first maximum) is the refined Doppler.
//
// The reference runs one FFT of 80 N points over a vector that is 7/8 zeros.  Here the zeros are never touched:
// with M = 10 N and k = 8 r + s,
//     X[8 r + s] = sum_{n < M} (x[n] c[n] e^{-2 pi j n s / (8 M)}) e^{-2 pi j n r / M} = FFT_M(x . c . phasor_s)[r],
// i.e. eight M-point transforms of the code-wiped signal modulated by eight sub-bin phasors.  They run through the
// acquisition's own forward path (acq_launch_fwd: "input x wipe-off row" -> FFT, rows = the 8 modulated code
// replicas), and one reduction kernel maps storage positions back to k and takes the first maximum of
// volk_32fc_magnitude_squared_32f / volk_gnsssdr_32f_index_max_32u (:352-357).
#include "acq_fft.cuh"
#include "engine.cuh"

#include <memory>
#include <new>
#include <vector>

using namespace b200;

namespace
{
constexpr int kZeroPadding = 8;   // zero_padding_factor (:319)
constexpr int kPrnReplicas = 10;  // prn_replicas (:320)

// rows s = 0..7 of (aligned code replica, repeated) x e^{-2 pi j n s / (8 M)}
__global__ void acq_fine_modulate_kernel(const float2* __restrict__ code, int n1ms, int m, float2* __restrict__ rows)
{
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    const int s = blockIdx.y;
    if (n >= m) return;
    const float2 c = code[n % n1ms];
    // phase = -2 pi (n s mod 8M) / (8M), reduced exactly in integers
    const long long t = (static_cast<long long>(n) * s) % (static_cast<long long>(kZeroPadding) * m);
    double sn, cs;
    sincospi(-2.0 * static_cast<double>(t) / (static_cast<double>(kZeroPadding) * m), &sn, &cs);
    const float pr = static_cast<float>(cs), pi = static_cast<float>(sn);
    rows[static_cast<size_t>(s) * m + n] = make_float2(fmaf(c.x, pr, -c.y * pi), fmaf(c.x, pi, c.y * pr));
}

// frequency index of the value stored at position g of a forward spectrum (see FftPlan: two-level block order,
// permuted storage of single-level plans, digit reversal of the in-shared-memory stages)
__host__ __device__ int storage_to_freq(const FftPlan& pl, int g)
{
    int blk = 0, p = g;
    if (pl.n1 > 1)
        {
            blk = g / pl.n;
            p = g - blk * pl.n;
        }
    else if (pl.perm_r > 1)
        {
            const int q = p / pl.perm_nb;
            const int b = p - q * pl.perm_nb;
            p = b * pl.perm_r + q;
        }
    int M = pl.n, mult = 1, r = 0;
    for (int st = 0; st < pl.n_stages; st++)
        {
            const int m = M / pl.radix[st];
            const int q = p / m;
            p -= q * m;
            r += q * mult;
            mult *= pl.radix[st];
            M = m;
        }
    return (pl.n1 > 1) ? blk + pl.n1 * r : r;
}

struct FineBest
{
    float peak;
    unsigned int index;
};

constexpr int kArgmaxThreads = 1024;

__global__ void __launch_bounds__(kArgmaxThreads) acq_fine_argmax_kernel(const float2* __restrict__ X, FftPlan pl, FineBest* __restrict__ out)
{
    const int m = pl.n_total;
    float bv = -1.0f;
    unsigned int bi = 0xffffffffu;
    for (int s = 0; s < kZeroPadding; s++)
        {
            const float2* row = X + static_cast<size_t>(s) * m;
            for (int g = threadIdx.x; g < m; g += blockDim.x)
                {
                    const float2 v = row[g];
                    const float mag = __fadd_rn(__fmul_rn(v.x, v.x), __fmul_rn(v.y, v.y));
                    const unsigned int k = static_cast<unsigned int>(kZeroPadding) * static_cast<unsigned int>(storage_to_freq(pl, g)) + s;
                    if (mag > bv || (mag == bv && k < bi))
                        {
                            bv = mag;
                            bi = k;
                        }
                }
        }
    float no_sum = 0.0f;
    acq_cta_first_max<kArgmaxThreads / 32>(bv, bi, no_sum);
    if (threadIdx.x == 0)
        {
            out->peak = bv;
            out->index = bi;
        }
}
}  // namespace

struct b200_acq_fine
{
    CudaStream stream;  // own, or the engine's; declared first, so released after the buffers used on it
    b200_engine* e{nullptr};
    int n1ms{0};
    int m{0};
    FftPlan plan{};
    DevBuf<float2> tw;
    DevBuf<float2> code_dev;  // n1ms
    DevBuf<float2> rows;      // 8 x m modulated code replicas
    DevBuf<float2> in_dev;    // m
    DevBuf<float2> X;         // 8 x m
    DevBuf<FineBest> best_dev;
    PinBuf<FineBest> best_pin;

    ~b200_acq_fine() { cudaStreamSynchronize(stream); }
};

extern "C"
{
    int b200_acq_fine_destroy(b200_acq_fine* f)
    {
        if (!f) return B200_ERR_ARG;
        cudaSetDevice(f->e->device);
        delete f;
        return B200_OK;
    }

    int b200_acq_fine_create(b200_engine* e, uint32_t fft_size, b200_acq_fine** out)
    {
        if (!e || !out || fft_size < 2) return B200_ERR_ARG;
        *out = nullptr;
        const long long m = static_cast<long long>(kPrnReplicas) * fft_size;
        FftPlan pl{};
        if (m > (1LL << 30) || acq_plan_make(static_cast<int>(m), &pl) != B200_OK)
            {
                set_error("fine Doppler: 10 x %u points unsupported (prime factors 2,3,5,7; 10 x fft_size <= 10 x %d)", fft_size, kAcqMaxSmemPoints);
                return B200_ERR_RANGE;
            }
        B200_ENTER_DEVICE(e->device);
        std::unique_ptr<b200_acq_fine> f(new (std::nothrow) b200_acq_fine());
        if (!f) return B200_ERR_NOMEM;
        f->e = e;
        f->n1ms = static_cast<int>(fft_size);
        f->m = static_cast<int>(m);
        f->plan = pl;
        cudaError_t err = cudaSuccess;
        if (e->stream.owned())
            err = f->stream.create(cudaStreamNonBlocking);
        else
            f->stream.borrow(e->stream);
        if (err == cudaSuccess) err = f->tw.alloc(m);
        if (err == cudaSuccess) err = f->code_dev.alloc(fft_size);
        if (err == cudaSuccess) err = f->rows.alloc(m * kZeroPadding);
        if (err == cudaSuccess) err = f->in_dev.alloc(m);
        if (err == cudaSuccess) err = f->X.alloc(m * kZeroPadding);
        if (err == cudaSuccess) err = f->best_dev.alloc(1);
        if (err == cudaSuccess) err = f->best_pin.alloc(1);
        if (err != cudaSuccess)
            {
                set_error("fine Doppler buffers: %s", cudaGetErrorString(err));
                return err == cudaErrorMemoryAllocation ? B200_ERR_NOMEM : B200_ERR_CUDA;
            }
        const int rc = acq_launch_twiddles(f->tw, f->plan, f->stream);
        if (rc) return rc;
        B200_CUDA_TRY(cudaStreamSynchronize(f->stream));
        *out = f.release();
        return B200_OK;
    }

    int b200_acq_fine_estimate(b200_acq_fine* f, const b200_cf32* buffer_10ms_host, const b200_cf32* code_replica_host, uint32_t* index_freq,
        float* peak)
    {
        if (!f || !buffer_10ms_host || !code_replica_host || !index_freq) return B200_ERR_ARG;
        std::lock_guard<std::mutex> lk(f->e->mu);
        B200_ENTER_DEVICE(f->e->device);
        B200_CUDA_TRY(cudaMemcpyAsync(f->in_dev, buffer_10ms_host, sizeof(float2) * f->m, cudaMemcpyHostToDevice, f->stream));
        B200_CUDA_TRY(cudaMemcpyAsync(f->code_dev, code_replica_host, sizeof(float2) * f->n1ms, cudaMemcpyHostToDevice, f->stream));
        const dim3 g((f->m + 255) / 256, kZeroPadding);
        acq_fine_modulate_kernel<<<g, 256, 0, f->stream>>>(f->code_dev, f->n1ms, f->m, f->rows);
        B200_CUDA_TRY(cudaGetLastError());
        uint64_t launched = 1;  // acq_fine_modulate_kernel
        // volk_32fc_x2_multiply_32fc (:347) fused into the transform's load, then the 8 M-point FFTs
        int rc = acq_launch_fwd(AcqInput::linear(f->in_dev), f->m, f->rows, f->X, kZeroPadding, f->plan, f->tw, launched, f->stream);
        if (rc) return rc;
        acq_fine_argmax_kernel<<<1, kArgmaxThreads, 0, f->stream>>>(f->X, f->plan, f->best_dev);
        B200_CUDA_TRY(cudaGetLastError());
        launched += 1;
        B200_CUDA_TRY(cudaMemcpyAsync(f->best_pin, f->best_dev, sizeof(FineBest), cudaMemcpyDeviceToHost, f->stream));
        B200_CUDA_TRY(cudaStreamSynchronize(f->stream));
        f->e->launches += launched;
        *index_freq = f->best_pin->index;
        if (peak) *peak = f->best_pin->peak;
        return B200_OK;
    }

    // debug / parity: |X[k]|^2 for all k of the zero-padded transform (8 x 10 x fft_size floats, natural order)
    int b200_acq_fine_read_spectrum(b200_acq_fine* f, float* mag_host)
    {
        if (!f || !mag_host) return B200_ERR_ARG;
        std::lock_guard<std::mutex> lk(f->e->mu);
        B200_ENTER_DEVICE(f->e->device);
        std::vector<float2> x(static_cast<size_t>(f->m) * kZeroPadding);
        B200_CUDA_TRY(cudaMemcpyAsync(x.data(), f->X, sizeof(float2) * x.size(), cudaMemcpyDeviceToHost, f->stream));
        B200_CUDA_TRY(cudaStreamSynchronize(f->stream));
        const FftPlan& pl = f->plan;
        for (int s = 0; s < kZeroPadding; s++)
            for (int g = 0; g < f->m; g++)
                {
                    const int freq = storage_to_freq(pl, g);
                    const float2 v = x[static_cast<size_t>(s) * f->m + g];
                    mag_host[static_cast<size_t>(kZeroPadding) * freq + s] = v.x * v.x + v.y * v.y;
                }
        return B200_OK;
    }
}
