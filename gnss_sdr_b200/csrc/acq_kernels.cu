// PCPS acquisition grid search for sm_90a.  Reference: src/algorithms/acquisition/
// gnuradio_blocks/pcps_acquisition.cc (doppler_grid :522-560, statistics :409-519,
// set_local_code :218-251, wipe-off grid :275-291).
//
// Kernels (all FFT work in shared memory, acq_fft.cuh; no cuFFT):
//   acq_wipeoff_kernel   Doppler wipe-off carriers, bit-compatible with the AVX2 variant of
//                        volk_gnsssdr_s32f_sincos_32fc (what runs on an x86-64 host).
//   acq_code_fft_kernel  set_local_code: FFT of the (padded) local code, conjugated, stored in
//                        digit-reversed order.
//   acq_fwd_kernel       one CTA per Doppler bin: x = in * wipe[d]; X_d = FFT(x), stored
//                        digit-reversed.  Computed ONCE per bin and shared by every PRN searched
//                        on the same samples (the reference recomputes it per channel).
//   acq_corr_kernel      one CTA per (PRN, bin) row: Y = X_d . conj(FFT(code)); y = IFFT(Y); the
//                        last inverse stage feeds |y|^2 straight into (max, first arg-max, sum)
//                        so the N-point row never leaves the SM (optionally accumulated into the
//                        magnitude grid for non-coherent dwells / dumps).
//   acq_stats_kernel     per PRN: arg-max over bins (strict '>' in ascending bin order) and the
//                        CFAR statistic, or hands the winning row to acq_corr_kernel in
//                        "second peak" mode.
#include "acq_fft.cuh"
#include "common.cuh"

#include <type_traits>

namespace b200
{
namespace
{
// ---- wipe-off carrier, reference float32 semantics --------------------------------------------
// One lane of VG kernels/volk_gnsssdr/volk_gnsssdr_s32f_sincos_32fc.h:448-633 (Cephes-style
// polynomial); every operation separately rounded, in the upstream order.
__device__ __forceinline__ float2 cephes_sincos(float p)
{
    const float FOPI = 1.27323954473516f;
    const float DP1 = -0.78515625f, DP2 = -2.4187564849853515625e-4f, DP3 = -3.77489497744594108e-8f;
    const float cc0 = 2.443315711809948E-005f, cc1 = -1.388731625493765E-003f, cc2 = 4.166664568298827E-002f;
    const float sc0 = -1.9515295891E-4f, sc1 = 8.3321608736E-3f, sc2 = -1.6666654611E-1f;
    float x = fabsf(p);
    unsigned int sign_bit_sin = __float_as_uint(p) & 0x80000000u;
    float y = __fmul_rn(x, FOPI);
    int emm2 = __float2int_rz(y);
    emm2 = (emm2 + 1) & ~1;
    y = __int2float_rn(emm2);
    int emm4 = emm2;
    const unsigned int swap_sign_bit_sin = (static_cast<unsigned int>(emm2 & 4)) << 29;
    const bool poly_sel = (emm2 & 2) == 0;
    const float xmm1 = __fmul_rn(y, DP1), xmm2 = __fmul_rn(y, DP2), xmm3 = __fmul_rn(y, DP3);
    x = __fadd_rn(x, xmm1);
    x = __fadd_rn(x, xmm2);
    x = __fadd_rn(x, xmm3);
    emm4 = emm4 - 2;
    const unsigned int sign_bit_cos = (static_cast<unsigned int>((~emm4) & 4)) << 29;
    sign_bit_sin ^= swap_sign_bit_sin;
    const float z = __fmul_rn(x, x);
    y = cc0;
    y = __fmul_rn(y, z);
    y = __fadd_rn(y, cc1);
    y = __fmul_rn(y, z);
    y = __fadd_rn(y, cc2);
    y = __fmul_rn(y, z);
    y = __fmul_rn(y, z);
    const float tmp = __fmul_rn(z, 0.5f);
    y = __fsub_rn(y, tmp);
    y = __fadd_rn(y, 1.0f);
    float y2 = sc0;
    y2 = __fmul_rn(y2, z);
    y2 = __fadd_rn(y2, sc1);
    y2 = __fmul_rn(y2, z);
    y2 = __fadd_rn(y2, sc2);
    y2 = __fmul_rn(y2, z);
    y2 = __fmul_rn(y2, x);
    y2 = __fadd_rn(y2, x);
    // select: sine takes y2 where poly_sel, else y; cosine the other one
    const float sm = poly_sel ? y2 : y;
    const float cm = poly_sel ? y : y2;
    const float s = __uint_as_float(__float_as_uint(sm) ^ sign_bit_sin);
    const float c = __uint_as_float(__float_as_uint(cm) ^ sign_bit_cos);
    return make_float2(c, s);
}

// grid: bins blocks of 32 threads; lanes 0..7 carry the eight float32 phase accumulators of the
// AVX2 kernel (p_l = phase + l*inc, advanced by fl(8*inc) per iteration); lane 0 does the tail.
__global__ void acq_wipeoff_kernel(float2* __restrict__ wipe, int n, int bins, int doppler_max, int doppler_center,
    int doppler_step, int doppler_bias, long long fs_in, int step_two, float center2, float step2)
{
    const int d = blockIdx.x;
    const int lane = threadIdx.x;
    if (d >= bins || lane >= 8) return;
    float freq;
    if (!step_two)
        {
            // pcps_acquisition.cc:288-289 and :277-278
            const int doppler = -doppler_max + doppler_center + doppler_step * d;
            freq = static_cast<float>(doppler_bias + doppler);
        }
    else
        {
            // update_grid_doppler_wipeoffs_step2 (:294-301): float Doppler around the step-one estimate
            const float doppler = __fmul_rn(__fsub_rn(static_cast<float>(d), static_cast<float>(floor(bins / 2.0))), step2);
            freq = __fadd_rn(center2, doppler);
        }
    const float phase_step_rad = __fdiv_rn(__fmul_rn(static_cast<float>(6.283185307179586), freq), static_cast<float>(fs_in));
    const float inc = -phase_step_rad;
    const int iters = n / 8;
    float p = (lane == 0) ? 0.0f : __fadd_rn(0.0f, __fmul_rn(static_cast<float>(lane), inc));
    if (lane == 1) p = __fadd_rn(0.0f, inc);
    const float inc8 = __fmul_rn(8.0f, inc);
    float2* row = wipe + static_cast<size_t>(d) * n;
    for (int it = 0; it < iters; it++)
        {
            row[8 * it + lane] = cephes_sincos(p);
            p = __fadd_rn(p, inc8);
        }
    if (lane == 0)
        {
            // scalar tail (n % 8 samples): cosf/sinf of the float-accumulated phase (:616-620);
            // CUDA's sinf/cosf are not glibc's, so these <8 samples are within 1 ulp, not bit-exact.
            float ph = __fadd_rn(0.0f, __fmul_rn(inc, static_cast<float>(static_cast<unsigned int>(iters * 8))));
            for (int i = iters * 8; i < n; i++)
                {
                    row[i] = make_float2(cosf(ph), sinf(ph));
                    ph = __fadd_rn(ph, inc);
                }
        }
}

// ---- set_local_code ------------------------------------------------------------------------------
// sample i of the n-point buffer that set_local_code fills from `code` (acq_code_offset)
__device__ __forceinline__ float2 acq_code_sample(const float2* __restrict__ code, int i, int n, int consumed, int layout)
{
    const int off = acq_code_offset(layout, n, consumed);
    const int end = (layout == 0) ? consumed : n;
    return (i >= off && i < end) ? code[i - off] : make_float2(0.f, 0.f);
}

template <int THREADS>
__global__ void __launch_bounds__(THREADS, 1) acq_code_fft_kernel(const float2* __restrict__ code, int consumed, int layout,
    float2* __restrict__ out, FftPlan pl, const float2* __restrict__ tw)
{
    extern __shared__ __align__(16) float2 s[];
    for (int i = threadIdx.x; i < pl.n; i += blockDim.x) s[i] = acq_code_sample(code, i, pl.n, consumed, layout);
    // forward FFT, then volk_32fc_conjugate_32fc (:250) fused into the store
    fft_forward_to_global<true, THREADS == kAcqThreads25>(s, pl, tw, out);
}

// ---- forward: wipe-off + FFT, one CTA per Doppler bin ------------------------------------------------
// FMT: the SampleFormat of the input (in.fmt); narrow samples are widened to float on load, exactly
template <int THREADS, int FMT>
__global__ void __launch_bounds__(THREADS, 1) acq_fwd_kernel(AcqInput in, int consumed,
    const float2* __restrict__ wipe, float2* __restrict__ X, FftPlan pl, const float2* __restrict__ tw)
{
    extern __shared__ __align__(16) float2 s[];
    const int n = pl.n;
    const int d = blockIdx.x;
    const float2* w = wipe + static_cast<size_t>(d) * n;
#pragma unroll 4
    for (int i = threadIdx.x; i < n; i += blockDim.x)
        {
            // acquisition_core zero-pads beyond consumed samples (:657-664); volk_32fc_x2_multiply_32fc (:531)
            s[i] = (i < consumed) ? cmul_rn(in.at<FMT>(i), w[i]) : make_float2(0.f, 0.f);
        }
    fft_forward_to_global<false, THREADS == kAcqThreads25>(s, pl, tw, X + static_cast<size_t>(d) * n);
}

// ---- correlation rows ---------------------------------------------------------------------------------
// Row r of a correlation launch.  best == nullptr: every (slot, bin) row, r = slot_pos * bins + bin.  Otherwise the
// second-peak pass: r = slot_pos, its winning bin from best[r], and the window of +-samples_per_chip around the winning
// index_time excluded (pcps_acquisition.cc:485-497).
struct AcqRow
{
    int slot_pos, bin;
    int ex1, ex2;  // excluded window [ex1, ex2) with wrap-around; ex1 < 0: none
    __device__ __forceinline__ AcqRow(int r, int bins, const AcqBest* __restrict__ best, int samples_per_chip, int ne)
    {
        if (best == nullptr)
            {
                slot_pos = r / bins;
                bin = r - slot_pos * bins;
                ex1 = ex2 = -1;
                return;
            }
        slot_pos = r;
        bin = static_cast<int>(best[r].index_doppler);
        ex1 = static_cast<int>(best[r].index_time) - samples_per_chip;
        ex2 = static_cast<int>(best[r].index_time) + samples_per_chip;
        if (ex1 < 0)
            ex1 = ne + ex1;
        else if (ex2 >= ne)
            ex2 = ex2 - ne;
    }
    __device__ __forceinline__ bool in_window(int t) const { return (ex1 <= ex2) ? (t >= ex1 && t < ex2) : (t >= ex1 || t < ex2); }
};

struct RowSink
{
    // natural-order outputs of the last inverse stage -> |y|^2 -> running statistics
    int off;        // first output index that counts (bit_transition: effective_fft_size, else 0)
    int ne;         // effective_fft_size
    AcqRow row;
    float* grid;    // optional magnitude row (ne floats): store or accumulate
    int accumulate;
    float best;
    unsigned int best_t;
    float sum;
    __device__ __forceinline__ RowSink(int off_, int ne_, const AcqRow& row_, float* grid_, int accumulate_)
        : off(off_), ne(ne_), row(row_), grid(grid_), accumulate(accumulate_), best(-1.0f), best_t(0xffffffffu), sum(0.0f)
    {
    }
    __device__ __forceinline__ void keep_first_max(float mag, int t)
    {
        if (mag > best || (mag == best && static_cast<unsigned int>(t) < best_t))
            {
                best = mag;
                best_t = static_cast<unsigned int>(t);
            }
    }
    __device__ __forceinline__ void operator()(float2* /*p*/, int pos, float2 v)
    {
        const int t = pos - off;
        if (t < 0 || t >= ne) return;
        // volk_32fc_magnitude_squared_32f (:547/:551)
        float mag = __fadd_rn(__fmul_rn(v.x, v.x), __fmul_rn(v.y, v.y));
        if (grid)
            {
                if (accumulate) mag = __fadd_rn(grid[t], mag);  // volk_32f_x2_add_32f (:552)
                grid[t] = mag;
            }
        // the reference zeroes the window before its second arg-max (:499-509)
        if (row.ex1 >= 0 && row.in_window(t)) mag = 0.0f;
        sum += mag;
        keep_first_max(mag, t);
    }
};

// best == nullptr: one CTA per (slot, bin) row, writes rowstat.  Otherwise one CTA per slot over its winning row (AcqRow),
// writes second_peak[slot_pos].
template <int THREADS>
__global__ void __launch_bounds__(THREADS, 1) acq_corr_kernel(const float2* __restrict__ X, const float2* __restrict__ codes,
    const int* __restrict__ slot_list, int bins, FftPlan pl, const float2* __restrict__ tw, int off, int ne,
    AcqRowStat* __restrict__ rowstat, float* __restrict__ grid, int accumulate,
    const AcqBest* __restrict__ best, int samples_per_chip, float* __restrict__ second_peak)
{
    extern __shared__ __align__(16) float2 s[];
    const int n = pl.n;
    const AcqRow row(blockIdx.x, bins, best, samples_per_chip, ne);
    const int slot = slot_list[row.slot_pos];
    float* g = (grid != nullptr) ? grid + (static_cast<size_t>(slot) * bins + row.bin) * ne : nullptr;
    // the second-peak pass reads an already accumulated grid row and does not touch it
    RowSink sink(off, ne, row, best ? nullptr : g, accumulate);

    if (best != nullptr && g != nullptr)
        {
            // dwell-accumulated grids: statistics come from the stored row, not from a recomputation
            for (int t = threadIdx.x; t < ne; t += blockDim.x) sink.keep_first_max(row.in_window(t) ? 0.0f : g[t], t);
        }
    else
        {
            const float2* x = X + static_cast<size_t>(row.bin) * n;
            const float2* c = codes + static_cast<size_t>(slot) * n;
            if (pl.perm_r > 1)
                {
                    // product (volk_32fc_x2_multiply_32fc, :538) and first inverse stage straight from global memory
                    fft_inverse_from_global<THREADS == kAcqThreads25>(x, c, s, pl, tw, sink);
                }
            else
                {
#pragma unroll 4
                    for (int i = threadIdx.x; i < n; i += blockDim.x) s[i] = cmul_rn(__ldg(x + i), __ldg(c + i));  // (:538)
                    fft_inverse_smem(s, pl, tw, sink);
                }
        }

    float bv = sink.best;
    unsigned int bi = sink.best_t;
    float sm = sink.sum;
    acq_cta_first_max<THREADS / 32>(bv, bi, sm);
    if (threadIdx.x == 0)
        {
            if (best == nullptr)
                rowstat[static_cast<size_t>(row.slot_pos) * bins + row.bin] = AcqRowStat{bv, bi, sm, 0.f};
            else
                second_peak[row.slot_pos] = bv;
        }
}

// ---- two-level transforms (fft_size > kAcqMaxSmemPoints): n_total = n1 * n ----------------------------------
// Forward: one radix-n1 DIF stage through global memory (block length n_total, sub-length n), then the
// in-shared-memory plan on each of the n1 blocks.  Inverse: the blocks first, then the radix-n1 DIT stage,
// whose natural-order outputs feed the statistics directly.  Layout stays "digit reversed" end to end.
template <int FMT>
__device__ __forceinline__ float2 acq_source(const AcqInput& in, const float2* __restrict__ wipe, int i, int consumed,
    int layout, int n_total)
{
    // wipe != nullptr: signal * wipe-off, zero-padded beyond consumed (acquisition_core :657-664, :531)
    // wipe == nullptr: local code placed by `layout`, from the linear float buffer in.a
    if (wipe != nullptr) return (i < consumed) ? cmul_rn(in.at<FMT>(i), wipe[i]) : make_float2(0.f, 0.f);
    return acq_code_sample(static_cast<const float2*>(in.a), i, n_total, consumed, layout);
}

// in_stride / wipe_stride: elements between the inputs / multiplier tables of consecutive rows (0 = one shared by all rows;
// in_stride > 0 only with a linear float input); FMT: the SampleFormat of the input (in.fmt)
template <int R, int FMT>
__global__ void acq_global_fwd_stage(AcqInput in, int consumed, int layout, const float2* __restrict__ wipe,
    float2* __restrict__ X, FftPlan pl, const float2* __restrict__ tw, size_t in_stride, size_t wipe_stride)
{
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    const int n2 = pl.n;
    if (j >= n2) return;
    const int d = blockIdx.y;
    const float2* w = wipe ? wipe + static_cast<size_t>(d) * wipe_stride : nullptr;
    in.a = static_cast<const float2*>(in.a) + static_cast<size_t>(d) * in_stride;
    float2 v[R];
#pragma unroll
    for (int q = 0; q < R; q++) v[q] = acq_source<FMT>(in, w, j + q * n2, consumed, layout, pl.n_total);
    Bfly<R>::fwd(v);
    const float2 w1 = __ldg(tw + pl.tw_goff + j);
    float2 wp = w1;
    float2* o = X + static_cast<size_t>(d) * pl.n_total;
    o[j] = v[0];
#pragma unroll
    for (int q = 1; q < R; q++)
        {
            o[q * n2 + j] = cmul(v[q], wp);
            if (q + 1 < R) wp = cmul(wp, w1);
        }
}

// forward in-smem FFT of block p of row d, in place; conj_out for the local code
__global__ void __launch_bounds__(kAcqThreads, 1) acq_block_fft_kernel(float2* __restrict__ X, FftPlan pl, const float2* __restrict__ tw, int conj_out)
{
    extern __shared__ __align__(16) float2 s[];
    const int n = pl.n;
    float2* blk = X + static_cast<size_t>(blockIdx.y) * pl.n_total + static_cast<size_t>(blockIdx.x) * n;
#pragma unroll 4
    for (int i = threadIdx.x; i < n; i += blockDim.x) s[i] = blk[i];
    fft_forward_smem(s, pl, tw);
    for (int i = threadIdx.x; i < n; i += blockDim.x) blk[i] = conj_out ? make_float2(s[i].x, -s[i].y) : s[i];
}

// block p of row r (AcqRow; the exclusion window is the final stage's)
__global__ void __launch_bounds__(kAcqThreads, 1) acq_corr_block_kernel(const float2* __restrict__ X, const float2* __restrict__ codes,
    const int* __restrict__ slot_list, int bins, FftPlan pl, const float2* __restrict__ tw, float2* __restrict__ Z,
    const AcqBest* __restrict__ best)
{
    extern __shared__ __align__(16) float2 s[];
    const int n = pl.n;
    const int p = blockIdx.x;
    const int r = blockIdx.y;
    const AcqRow row(r, bins, best, 0, 0);
    const int slot = slot_list[row.slot_pos];
    const float2* x = X + static_cast<size_t>(row.bin) * pl.n_total + static_cast<size_t>(p) * n;
    const float2* c = codes + static_cast<size_t>(slot) * pl.n_total + static_cast<size_t>(p) * n;
#pragma unroll 4
    for (int i = threadIdx.x; i < n; i += blockDim.x) s[i] = cmul_rn(__ldg(x + i), __ldg(c + i));
    fft_inverse_smem_inplace(s, pl, tw);
    float2* z = Z + static_cast<size_t>(r) * pl.n_total + static_cast<size_t>(p) * n;
    for (int i = threadIdx.x; i < n; i += blockDim.x) z[i] = s[i];
}

// final radix-n1 DIT stage of row z over the CTAs of grid.x: natural-order output k goes to sink(nullptr, k, y[k])
template <int R, class Sink>
__device__ __forceinline__ void acq_global_final_dit(const float2* __restrict__ z, const FftPlan& pl, const float2* __restrict__ tw, Sink& sink)
{
    const int n2 = pl.n;
    for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n2; j += gridDim.x * blockDim.x)
        {
            float2 v[R];
#pragma unroll
            for (int q = 0; q < R; q++) v[q] = z[q * n2 + j];
            const float2 w1 = __ldg(tw + pl.tw_goff + j);
            float2 wp = w1;
#pragma unroll
            for (int q = 1; q < R; q++)
                {
                    v[q] = cmul_conj(v[q], wp);
                    if (q + 1 < R) wp = cmul(wp, w1);
                }
#pragma unroll
            for (int q = 0; q < R; q++) v[q] = swap_ri(v[q]);
            Bfly<R>::fwd(v);
#pragma unroll
            for (int q = 0; q < R; q++) sink(nullptr, j + q * n2, swap_ri(v[q]));
        }
}

// final radix-n1 DIT stage + |.|^2 + statistics; grid (chunks, rows); partial[r * chunks + chunk]
template <int R>
__global__ void __launch_bounds__(256) acq_global_final_stage(const float2* __restrict__ Z, FftPlan pl, const float2* __restrict__ tw,
    const int* __restrict__ slot_list, int bins, int off, int ne, float* __restrict__ grid, int accumulate,
    const AcqBest* __restrict__ best, int samples_per_chip, AcqRowStat* __restrict__ partial)
{
    const int r = blockIdx.y;
    const AcqRow row(r, bins, best, samples_per_chip, ne);
    float* g = (grid != nullptr && best == nullptr) ? grid + (static_cast<size_t>(slot_list[row.slot_pos]) * bins + row.bin) * ne : nullptr;
    RowSink sink(off, ne, row, g, accumulate);
    acq_global_final_dit<R>(Z + static_cast<size_t>(r) * pl.n_total, pl, tw, sink);
    float bv = sink.best;
    unsigned int bi = sink.best_t;
    float sm = sink.sum;
    acq_cta_first_max<256 / 32>(bv, bi, sm);
    if (threadIdx.x == 0) partial[static_cast<size_t>(r) * gridDim.x + blockIdx.x] = AcqRowStat{bv, bi, sm, 0.f};
}

// ---- Bluestein (chirp-z) support: sizes the mixed-radix planner cannot factor (prime factors > 7, e.g. 16 368) --------
// The first n_out natural-order outputs of a final stage, multiplied by post[k] and STORED (complex) instead of being
// reduced to statistics: out[k] = y[k] * post[k], k < n_out.
struct PostMulStoreSink
{
    const float2* __restrict__ post;
    int n_out;
    float2* __restrict__ out;
    __device__ __forceinline__ void operator()(float2* /*p*/, int k, float2 v) const
    {
        if (k < n_out) out[k] = cmul(v, __ldg(post + k));
    }
};

template <int R>
__global__ void __launch_bounds__(256) acq_global_final_store_stage(const float2* __restrict__ Z, FftPlan pl, const float2* __restrict__ tw,
    const float2* __restrict__ post, int n_out, float2* __restrict__ out, size_t out_stride)
{
    const int r = blockIdx.y;
    const float2* z = Z + static_cast<size_t>(r) * pl.n_total;
    PostMulStoreSink sink{post, n_out, out + static_cast<size_t>(r) * out_stride};
    acq_global_final_dit<R>(z, pl, tw, sink);
}

// out[r][i] = a[r][i] * b[i] (conj_a: conj(a[r][i]) * b[i]), i < n; rows r < rows
__global__ void acq_rows_times_vector_kernel(const float2* __restrict__ a, size_t a_stride, const float2* __restrict__ b, int n, int conj_a,
    float2* __restrict__ out, size_t out_stride)
{
    const int r = blockIdx.y;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
        {
            float2 x = a[static_cast<size_t>(r) * a_stride + i];
            if (conj_a) x.y = -x.y;
            out[static_cast<size_t>(r) * out_stride + i] = cmul(x, __ldg(b + i));
        }
}

// writes rowstat[r], or only the maximum to second_peak[r] when second_peak != nullptr
__global__ void acq_row_reduce_kernel(const AcqRowStat* __restrict__ partial, int chunks, int rows, AcqRowStat* __restrict__ rowstat,
    float* __restrict__ second_peak)
{
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= rows) return;
    AcqRowStat a = partial[static_cast<size_t>(r) * chunks];
    for (int k = 1; k < chunks; k++)
        {
            const AcqRowStat b = partial[static_cast<size_t>(r) * chunks + k];
            if (b.max > a.max || (b.max == a.max && b.argmax < a.argmax))
                {
                    a.max = b.max;
                    a.argmax = b.argmax;
                }
            a.sum += b.sum;
        }
    if (second_peak == nullptr)
        rowstat[r] = a;
    else
        second_peak[r] = a.max;
}

// ---- statistics ---------------------------------------------------------------------------------------
// one thread per searched PRN (bins <= a few hundred): pcps_acquisition.cc:417-449 / :464-482
__global__ void acq_stats_kernel(const AcqRowStat* __restrict__ rowstat, int n_slots, int bins, int ne, int doppler_max,
    int doppler_center, int doppler_step, unsigned int dwell_counter, int use_cfar, AcqBest* __restrict__ best,
    b200_acq_result* __restrict__ results, int step_two, float center2, float step2, float prev_input_power)
{
    // one warp per PRN slot.  The reference scans the bins in ascending order with a strict '>' from 0.0
    // (:417-426 / :464-473): the winner is the largest per-bin maximum, the lowest bin among equals, and (0, 0)
    // when nothing exceeds 0.  Lanes scan bins lane, lane+32, ... in ascending order, then combine.
    const int sp = blockIdx.x;
    if (sp >= n_slots) return;
    const int lane = threadIdx.x;
    const AcqRowStat* rs = rowstat + static_cast<size_t>(sp) * bins;
    float grid_maximum = 0.0f;
    unsigned int index_doppler = 0xffffffffu, index_time = 0;
    for (int i = lane; i < bins; i += 32)
        {
            const AcqRowStat v = rs[i];
            if (v.max > grid_maximum)
                {
                    grid_maximum = v.max;
                    index_doppler = static_cast<unsigned int>(i);
                    index_time = v.argmax;
                }
        }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1)
        {
            const float ov = __shfl_xor_sync(0xffffffffu, grid_maximum, o);
            const unsigned int od = __shfl_xor_sync(0xffffffffu, index_doppler, o);
            const unsigned int ot = __shfl_xor_sync(0xffffffffu, index_time, o);
            if (ov > grid_maximum || (ov == grid_maximum && od < index_doppler))
                {
                    grid_maximum = ov;
                    index_doppler = od;
                    index_time = ot;
                }
        }
    if (lane != 0) return;
    if (index_doppler == 0xffffffffu)
        {
            index_doppler = 0;
            index_time = 0;
        }
    b200_acq_result r;
    r.index_time = index_time;
    r.index_doppler = index_doppler;
    if (!step_two)
        r.doppler = -doppler_max + doppler_center + doppler_step * static_cast<int>(index_doppler);
    else  // (:436, :480) static_cast<int32_t>(center2 + (float(index) - float(floor(bins2 / 2.0))) * step2)
        r.doppler = static_cast<int>(__fadd_rn(center2, __fmul_rn(__fsub_rn(static_cast<float>(index_doppler), static_cast<float>(floor(bins / 2.0))), step2)));
    r.grid_maximum = grid_maximum;
    r.test_statistics = 0.0f;
    r.input_power = 0.0f;
    r.second_peak = 0.0f;
    if (use_cfar && step_two)
        {
            // the second step keeps d_input_power from the first one (:428-438)
            r.input_power = prev_input_power;
            r.test_statistics = (prev_input_power < 1.1920929e-07f) ? 0.0f : __fdiv_rn(grid_maximum, prev_input_power);
        }
    else if (use_cfar)
        {
            const unsigned int index_opp = (index_doppler + static_cast<unsigned int>(bins) / 2u) % static_cast<unsigned int>(bins);
            // static_cast<float>(accumulate(...) / N_eff / 2.0 / counter)   (:431)
            const float a = __fdiv_rn(rs[index_opp].sum, static_cast<float>(static_cast<unsigned int>(ne)));
            const double ip = static_cast<double>(a) / 2.0 / static_cast<double>(dwell_counter);
            const float input_power = static_cast<float>(ip);
            r.input_power = input_power;
            r.test_statistics = (input_power < 1.1920929e-07f) ? 0.0f : __fdiv_rn(grid_maximum, input_power);
        }
    best[sp].index_time = index_time;
    best[sp].index_doppler = index_doppler;
    results[sp] = r;
}

__global__ void acq_finish_second_peak_kernel(const float* __restrict__ second_peak, int n_slots, b200_acq_result* __restrict__ results)
{
    const int sp = blockIdx.x * blockDim.x + threadIdx.x;
    if (sp >= n_slots) return;
    const float sec = second_peak[sp];
    results[sp].second_peak = sec;
    results[sp].test_statistics = __fdiv_rn(results[sp].grid_maximum, sec);  // (:517)
}

// per-stage compact twiddle tables exp(-2 pi j k / M_stage), k < m_stage, in double, rounded once
__global__ void acq_twiddle_kernel(float2* __restrict__ tw, FftPlan pl)
{
    int M = pl.n;
    for (int st = 0; st < pl.n_stages; st++)
        {
            const int m = M / pl.radix[st];
            for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < m; k += gridDim.x * blockDim.x)
                {
                    double s, c;
                    sincospi(-2.0 * static_cast<double>(k) / static_cast<double>(M), &s, &c);
                    tw[pl.tw_off[st] + k] = make_float2(static_cast<float>(c), static_cast<float>(s));
                }
            M = m;
        }
    if (pl.n1 > 1)
        {
            for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < pl.n; k += gridDim.x * blockDim.x)
                {
                    double s, c;
                    sincospi(-2.0 * static_cast<double>(k) / static_cast<double>(pl.n_total), &s, &c);
                    tw[pl.tw_goff + k] = make_float2(static_cast<float>(c), static_cast<float>(s));
                }
        }
}

// (statistic, PRN, bin, code phase) a comes before b: the larger statistic, then the lower PRN, bin and code phase
__device__ __forceinline__ bool acq_peak_before(const b200_acq_peak& a, const b200_acq_peak& b)
{
    if (a.test_statistics != b.test_statistics) return a.test_statistics > b.test_statistics;
    if (a.prn != b.prn) return a.prn < b.prn;
    if (a.index_doppler != b.index_doppler) return a.index_doppler < b.index_doppler;
    return a.index_time < b.index_time;
}

// Best satellite of one sweep as ONE 16-byte record {test statistic, PRN, Doppler bin, code phase}: what a rank
// contributes to the multi-GPU peak exchange (an all-gather of N records; SURVEY 8e).  Ties go to the lowest
// (PRN, bin, code phase), the rule of dist.best_peak and of the reference's strict '>' scans (pcps_acquisition.cc:417-426),
// whatever order prn_of_result lists the PRNs in.
__global__ void acq_sweep_best_kernel(const b200_acq_result* __restrict__ results, const unsigned int* __restrict__ prn_of_result, int n,
    b200_acq_peak* __restrict__ out)
{
    const int lane = threadIdx.x;
    // statistic -1 with the lowest keys: only a record with a statistic above -1 replaces it
    b200_acq_peak best{-1.0f, 0u, 0u, 0u};
    for (int i = lane; i < n; i += 32)
        {
            const b200_acq_peak v{results[i].test_statistics, prn_of_result[i], results[i].index_doppler, results[i].index_time};
            if (acq_peak_before(v, best)) best = v;
        }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1)
        {
            const b200_acq_peak ov{__shfl_xor_sync(0xffffffffu, best.test_statistics, o), __shfl_xor_sync(0xffffffffu, best.prn, o),
                __shfl_xor_sync(0xffffffffu, best.index_doppler, o), __shfl_xor_sync(0xffffffffu, best.index_time, o)};
            if (acq_peak_before(ov, best)) best = ov;
        }
    if (lane == 0) *out = (best.test_statistics > -1.0f) ? best : b200_acq_peak{0.0f, 0u, 0u, 0u};
}

DeviceOnce g_attr_once;  // per device (a second engine on another GPU needs its own opt-in), thread-safe
int set_attrs()
{
    const int once_dev = g_attr_once.begin();
    if (once_dev < 0) return B200_OK;
    const int bytes = kAcqMaxSmemPoints * static_cast<int>(sizeof(float2));
    B200_CUDA_TRY(cudaFuncSetAttribute(acq_code_fft_kernel<kAcqThreads>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
    B200_CUDA_TRY(cudaFuncSetAttribute(acq_fwd_kernel<kAcqThreads, kCf32>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
    B200_CUDA_TRY(cudaFuncSetAttribute(acq_fwd_kernel<kAcqThreads, kI16>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
    B200_CUDA_TRY(cudaFuncSetAttribute(acq_fwd_kernel<kAcqThreads, kI8>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
    B200_CUDA_TRY(cudaFuncSetAttribute(acq_corr_kernel<kAcqThreads>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
    B200_CUDA_TRY(cudaFuncSetAttribute(acq_code_fft_kernel<kAcqThreads25>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
    B200_CUDA_TRY(cudaFuncSetAttribute(acq_fwd_kernel<kAcqThreads25, kCf32>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
    B200_CUDA_TRY(cudaFuncSetAttribute(acq_fwd_kernel<kAcqThreads25, kI16>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
    B200_CUDA_TRY(cudaFuncSetAttribute(acq_fwd_kernel<kAcqThreads25, kI8>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
    B200_CUDA_TRY(cudaFuncSetAttribute(acq_corr_kernel<kAcqThreads25>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
    B200_CUDA_TRY(cudaFuncSetAttribute(acq_block_fft_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
    B200_CUDA_TRY(cudaFuncSetAttribute(acq_corr_block_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
    g_attr_once.done(once_dev);
    return B200_OK;
}
}  // namespace

// ---- launchers (called from acq_engine.cu) --------------------------------------------------------------
static int acq_plan_make_smem(int n, FftPlan* pl, bool allow25);

// two-level plan: the first global radix n1 of `cand` that divides n_total and leaves blocks the in-shared-memory planner takes
static int acq_plan_make_global(int n_total, const int (&cand)[7], FftPlan* pl)
{
    for (int n1 : cand)
        {
            if (n_total % n1) continue;
            const int n2 = n_total / n1;
            if (n2 > kAcqMaxSmemPoints) continue;
            if (acq_plan_make_smem(n2, pl, false) != B200_OK) continue;
            pl->n1 = n1;
            pl->n_total = n_total;
            int off = 0, M = n2;
            for (int st = 0; st < pl->n_stages; st++)
                {
                    M /= pl->radix[st];
                    off += M;
                }
            pl->tw_goff = off;  // after the per-stage tables; n2 entries follow
            return B200_OK;
        }
    return B200_ERR_RANGE;
}

int acq_plan_make(int n_total, FftPlan* pl)
{
    if (n_total < 2) return B200_ERR_RANGE;
    if (n_total <= kAcqMaxSmemPoints)
        {
            // radix-25 stages (one shared-memory pass instead of two radix-5 passes) on 512-thread CTAs wherever
            // acq_plan_make_smem can place them; every other size keeps the radix <= 8 plan on 1024 threads
            const int rc = acq_plan_make_smem(n_total, pl, true);
            pl->n1 = 1;
            pl->n_total = n_total;
            pl->tw_goff = 0;
            if (rc == B200_OK && pl->n_stages >= 2)
                {
                    pl->perm_r = pl->radix[pl->n_stages - 1];
                    pl->perm_nb = pl->n / pl->perm_r;
                }
            return rc;
        }
    // two-level: smallest supported radix n1 that brings the blocks into shared memory
    return acq_plan_make_global(n_total, {2, 3, 4, 5, 7, 8, 10}, pl);
}

// two-level plan for EXACTLY m points with a global radix n1 >= 2 even when m would fit shared memory (the chirp-z path is
// written on the through-global-memory kernels only); powers of two first
int acq_plan_make_two_level(int m, FftPlan* pl) { return acq_plan_make_global(m, {2, 4, 8, 3, 5, 7, 10}, pl); }

static int acq_plan_make_smem(int n, FftPlan* pl, bool allow25)
{
    if (n < 2 || n > kAcqMaxSmemPoints) return B200_ERR_RANGE;
    int rem = n;
    int cnt[8] = {0};
    const int primes[4] = {7, 5, 3, 2};
    for (int p : primes)
        while (rem % p == 0)
            {
                cnt[p]++;
                rem /= p;
            }
    if (rem != 1) return B200_ERR_RANGE;  // unsupported prime factor
    pl->n = n;
    pl->perm_r = 1;
    pl->perm_nb = n;
    pl->threads = kAcqThreads;
    int k = 0;
    // Powers of two first (large sub-block stride m, conflict-free stride-1 accesses), odd radices
    // last: in the final stages consecutive threads are R*m apart and an ODD stride spreads over
    // all shared-memory banks, while an even one would serialise.
    int twos = cnt[2];
    while (twos >= 3)
        {
            pl->radix[k++] = 8;
            twos -= 3;
        }
    if (twos == 2) pl->radix[k++] = 4;
    if (twos == 1) pl->radix[k++] = 2;
    for (int i = 0; i < cnt[3]; i++) pl->radix[k++] = 3;
    for (int i = 0; i < cnt[7]; i++) pl->radix[k++] = 7;
    int fives = cnt[5];
    // pairs of 5 become radix-25 stages as long as at least two stages remain (the fused first/last stage
    // paths take the final radix from the plan and are not instantiated for 25)
    if (allow25 && fives >= 2 && (k + fives / 2 + (fives & 1)) >= 2 && ((fives & 1) || k >= 1))
        {
            const bool odd = (fives & 1) != 0;
            int pairs = fives / 2;
            if (!odd)
                {
                    // the last stage must be a radix the fused paths support: keep one pair as 5, 5
                    pairs -= 1;
                }
            for (int i = 0; i < pairs; i++) pl->radix[k++] = 25;
            if (pairs > 0) pl->threads = kAcqThreads25;
            fives -= 2 * pairs;
        }
    for (int i = 0; i < fives; i++) pl->radix[k++] = 5;
    if (k > kAcqMaxStages) return B200_ERR_RANGE;
    pl->n_stages = k;
    int M = n;
    int off = 0;
    for (int st = 0; st < k; st++)
        {
            const int m = M / pl->radix[st];
            pl->mdiv[st] = (m <= 1) ? 0u : static_cast<unsigned int>((1ULL << 32) / static_cast<unsigned long long>(m)) + 1u;
            pl->tw_off[st] = off;
            off += m;   // sum of m over the stages < n
            M = m;
        }
    return B200_OK;
}

int acq_launch_twiddles(float2* tw, const FftPlan& pl, cudaStream_t st)
{
    acq_twiddle_kernel<<<32, 256, 0, st>>>(tw, pl);
    B200_CUDA_TRY(cudaGetLastError());
    return B200_OK;
}

int acq_launch_wipeoff(float2* wipe, int n, int bins, int doppler_max, int doppler_center, int doppler_step,
    int doppler_bias, long long fs_in, int step_two, float center2, float step2, cudaStream_t st)
{
    acq_wipeoff_kernel<<<bins, 32, 0, st>>>(wipe, n, bins, doppler_max, doppler_center, doppler_step, doppler_bias, fs_in, step_two, center2, step2);
    B200_CUDA_TRY(cudaGetLastError());
    return B200_OK;
}

template <typename F>
static int dispatch_radix(int r, F&& f)
{
    switch (r)
        {
        case 2: f(std::integral_constant<int, 2>{}); return B200_OK;
        case 3: f(std::integral_constant<int, 3>{}); return B200_OK;
        case 4: f(std::integral_constant<int, 4>{}); return B200_OK;
        case 5: f(std::integral_constant<int, 5>{}); return B200_OK;
        case 7: f(std::integral_constant<int, 7>{}); return B200_OK;
        case 8: f(std::integral_constant<int, 8>{}); return B200_OK;
        case 10: f(std::integral_constant<int, 10>{}); return B200_OK;
        default: return B200_ERR_RANGE;
        }
}

// the single-CTA kernels at the plan's CTA width
template <typename F>
static void dispatch_threads(const FftPlan& pl, F&& f)
{
    if (pl.threads == kAcqThreads25)
        f(std::integral_constant<int, kAcqThreads25>{});
    else
        f(std::integral_constant<int, kAcqThreads>{});
}

int acq_final_chunks(const FftPlan& pl) { return pl.n1 > 1 ? (pl.n + 1023) / 1024 : 0; }

int acq_launch_code_fft(const float2* code, int consumed, int layout, float2* out, const FftPlan& pl, const float2* tw, cudaStream_t st)
{
    int rc = set_attrs();
    if (rc) return rc;
    if (pl.n1 == 1)
        {
            dispatch_threads(pl, [&](auto T) {
                acq_code_fft_kernel<decltype(T)::value><<<1, decltype(T)::value, pl.n * sizeof(float2), st>>>(code, consumed, layout, out, pl, tw);
            });
        }
    else
        {
            const dim3 g((pl.n + 255) / 256, 1);
            rc = dispatch_radix(pl.n1, [&](auto R) { acq_global_fwd_stage<decltype(R)::value, kCf32><<<g, 256, 0, st>>>(AcqInput::linear(code), consumed, layout, nullptr, out, pl, tw, 0, 0); });
            if (rc) return rc;
            acq_block_fft_kernel<<<dim3(pl.n1, 1), kAcqThreads, pl.n * sizeof(float2), st>>>(out, pl, tw, 1);
        }
    B200_CUDA_TRY(cudaGetLastError());
    return B200_OK;
}

int acq_launch_fwd(AcqInput in, int consumed, const float2* wipe, float2* X, int bins, const FftPlan& pl, const float2* tw,
    uint64_t& launched, cudaStream_t st)
{
    int rc = set_attrs();
    if (rc) return rc;
    if (pl.n1 == 1)
        {
            rc = with_format(in.fmt, [&](auto F) {
                dispatch_threads(pl, [&](auto T) {
                    acq_fwd_kernel<decltype(T)::value, decltype(F)::value><<<bins, decltype(T)::value, pl.n * sizeof(float2), st>>>(in, consumed, wipe,
                        X, pl, tw);
                });
                return B200_OK;
            });
            if (rc) return rc;
        }
    else
        {
            const dim3 g((pl.n + 255) / 256, bins);
            rc = with_format(in.fmt, [&](auto F) {
                return dispatch_radix(pl.n1, [&](auto R) {
                    acq_global_fwd_stage<decltype(R)::value, decltype(F)::value><<<g, 256, 0, st>>>(in, consumed, 0, wipe, X, pl, tw, 0,
                        static_cast<size_t>(pl.n_total));
                });
            });
            if (rc) return rc;
            acq_block_fft_kernel<<<dim3(pl.n1, bins), kAcqThreads, pl.n * sizeof(float2), st>>>(X, pl, tw, 0);
        }
    B200_CUDA_TRY(cudaGetLastError());
    launched += (pl.n1 == 1) ? 1 : 2;
    return B200_OK;
}

// best == nullptr: statistics of every (slot, bin) row into rowstat; otherwise the second-peak pass into second_peak
static int launch_corr(const float2* X, const float2* codes, const int* slot_list, int n_slots, int bins, const FftPlan& pl,
    const float2* tw, int off, int ne, float* grid, int accumulate, const AcqBest* best, int samples_per_chip, AcqRowStat* rowstat,
    float* second_peak, float2* Z, AcqRowStat* partial, uint64_t& launched, cudaStream_t st)
{
    int rc = set_attrs();
    if (rc) return rc;
    const int rows = (best == nullptr) ? n_slots * bins : n_slots;
    const bool one_kernel = pl.n1 == 1 || (best != nullptr && grid != nullptr);
    if (one_kernel)
        {
            const size_t smem = (pl.n1 == 1) ? pl.n * sizeof(float2) : 16;
            dispatch_threads(pl, [&](auto T) {
                acq_corr_kernel<decltype(T)::value><<<rows, decltype(T)::value, smem, st>>>(X, codes, slot_list, bins, pl, tw, off, ne, rowstat,
                    grid, accumulate, best, samples_per_chip, second_peak);
            });
        }
    else
        {
            acq_corr_block_kernel<<<dim3(pl.n1, rows), kAcqThreads, pl.n * sizeof(float2), st>>>(X, codes, slot_list, bins, pl, tw, Z, best);
            const int chunks = acq_final_chunks(pl);
            rc = dispatch_radix(pl.n1, [&](auto R) {
                acq_global_final_stage<decltype(R)::value><<<dim3(chunks, rows), 256, 0, st>>>(Z, pl, tw, slot_list, bins, off, ne, grid, accumulate,
                    best, samples_per_chip, partial);
            });
            if (rc) return rc;
            acq_row_reduce_kernel<<<(rows + 127) / 128, 128, 0, st>>>(partial, chunks, rows, rowstat, second_peak);
        }
    B200_CUDA_TRY(cudaGetLastError());
    launched += one_kernel ? 1 : 3;
    return B200_OK;
}

int acq_launch_row_stats(const float2* X, const float2* codes, const int* slot_list, int n_slots, int bins, const FftPlan& pl,
    const float2* tw, int off, int ne, float* grid, int accumulate, AcqRowStat* rowstat, float2* Z, AcqRowStat* partial,
    uint64_t& launched, cudaStream_t st)
{
    return launch_corr(X, codes, slot_list, n_slots, bins, pl, tw, off, ne, grid, accumulate, nullptr, 0, rowstat, nullptr, Z, partial,
        launched, st);
}

int acq_launch_second_peak(const float2* X, const float2* codes, const int* slot_list, int n_slots, int bins, const FftPlan& pl,
    const float2* tw, int off, int ne, float* grid, const AcqBest* best, int samples_per_chip, float* second_peak, float2* Z,
    AcqRowStat* partial, uint64_t& launched, cudaStream_t st)
{
    return launch_corr(X, codes, slot_list, n_slots, bins, pl, tw, off, ne, grid, 0, best, samples_per_chip, nullptr, second_peak, Z,
        partial, launched, st);
}

int acq_launch_stats(const AcqRowStat* rowstat, int n_slots, int bins, int ne, int doppler_max, int doppler_center,
    int doppler_step, unsigned int dwell_counter, int use_cfar, AcqBest* best, b200_acq_result* results, int step_two, float center2,
    float step2, float prev_input_power, uint64_t& launched, cudaStream_t st)
{
    acq_stats_kernel<<<n_slots, 32, 0, st>>>(rowstat, n_slots, bins, ne, doppler_max, doppler_center, doppler_step,
        dwell_counter, use_cfar, best, results, step_two, center2, step2, prev_input_power);
    B200_CUDA_TRY(cudaGetLastError());
    launched += 1;
    return B200_OK;
}

int acq_launch_finish_second_peak(const float* second_peak, int n_slots, b200_acq_result* results, uint64_t& launched, cudaStream_t st)
{
    acq_finish_second_peak_kernel<<<(n_slots + 63) / 64, 64, 0, st>>>(second_peak, n_slots, results);
    B200_CUDA_TRY(cudaGetLastError());
    launched += 1;
    return B200_OK;
}

int acq_launch_sweep_best(const b200_acq_result* results, const unsigned int* prn_of_result, int n, b200_acq_peak* out, uint64_t& launched,
    cudaStream_t st)
{
    acq_sweep_best_kernel<<<1, 32, 0, st>>>(results, prn_of_result, n, out);
    B200_CUDA_TRY(cudaGetLastError());
    launched += 1;
    return B200_OK;
}

// ---- Bluestein building blocks (acq_engine.cu composes them) --------------------------------------------------------
// X[r] = FFT_M( pad( in(r * in_stride + i) * mult[r * mult_stride + i], i < consumed ) ), rows r < rows (two-level plan)
int acq_launch_fwd_rows(AcqInput in, size_t in_stride, int consumed, const float2* mult, size_t mult_stride, float2* X, int rows,
    const FftPlan& pl, const float2* tw, uint64_t& launched, cudaStream_t st)
{
    int rc = set_attrs();
    if (rc) return rc;
    if (pl.n1 < 2) return B200_ERR_ARG;
    const dim3 g((pl.n + 255) / 256, rows);
    rc = with_format(in.fmt, [&](auto F) {
        return dispatch_radix(pl.n1, [&](auto R) {
            acq_global_fwd_stage<decltype(R)::value, decltype(F)::value><<<g, 256, 0, st>>>(in, consumed, 0, mult, X, pl, tw, in_stride,
                mult_stride);
        });
    });
    if (rc) return rc;
    acq_block_fft_kernel<<<dim3(pl.n1, rows), kAcqThreads, pl.n * sizeof(float2), st>>>(X, pl, tw, 0);
    B200_CUDA_TRY(cudaGetLastError());
    launched += 2;
    return B200_OK;
}

// out[r][k] = IFFT_M( X[r] . filt )[k] * post[k], k < n_out   (Z: rows x M workspace; one_slot_dev: device int == 0)
int acq_launch_inverse_store_rows(const float2* X, const float2* filt, const int* one_slot_dev, int rows, const FftPlan& pl, const float2* tw,
    float2* Z, const float2* post, int n_out, float2* out, size_t out_stride, uint64_t& launched, cudaStream_t st)
{
    int rc = set_attrs();
    if (rc) return rc;
    if (pl.n1 < 2) return B200_ERR_ARG;
    acq_corr_block_kernel<<<dim3(pl.n1, rows), kAcqThreads, pl.n * sizeof(float2), st>>>(X, filt, one_slot_dev, rows, pl, tw, Z, nullptr);
    const int chunks = acq_final_chunks(pl);
    rc = dispatch_radix(pl.n1, [&](auto R) {
        acq_global_final_store_stage<decltype(R)::value><<<dim3(chunks, rows), 256, 0, st>>>(Z, pl, tw, post, n_out, out, out_stride);
    });
    if (rc) return rc;
    B200_CUDA_TRY(cudaGetLastError());
    launched += 2;
    return B200_OK;
}

int acq_launch_rows_times_vector(const float2* a, size_t a_stride, const float2* b, int n, int conj_a, float2* out, size_t out_stride, int rows,
    cudaStream_t st)
{
    acq_rows_times_vector_kernel<<<dim3((n + 255) / 256, rows), 256, 0, st>>>(a, a_stride, b, n, conj_a, out, out_stride);
    B200_CUDA_TRY(cudaGetLastError());
    return B200_OK;
}

}  // namespace b200
