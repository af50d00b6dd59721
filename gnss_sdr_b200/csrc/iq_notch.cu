// The notch input filters of InputFilter.implementation = Notch_Filter and Notch_Filter_Lite
// (src/algorithms/input_filter/gnuradio_blocks/notch_cc.cc:63-121, notch_lite_cc.cc:71-138): every push into a source band
// fills a destination band with the block's output, CW interference removed by a first-order complex IIR notch over each
// L-sample segment whose energy exceeds the chi-squared threshold times the noise estimate (b200_iq_set_notch, engine.cu).
// A push that completes K segments launches six kernels: the K segment energies, the spectral noise floor of the segments
// that can be in estimation, one CTA that runs the block's state machine, then the IIR as a split-invariant chunked scan
// (each grid block's affine map in double, the double carry from grid point to grid point, and the float pass that writes
// the destination).  The header states the arithmetic.
#include "common.cuh"

#include <algorithm>
#include <cmath>

using namespace b200;

namespace
{
constexpr int kEnergyThreads = 128;  // one segment per thread
constexpr int kScanThreads = 1024;   // the scan's one CTA decides up to this many detection segments per step
constexpr int kGridThreads = 128;    // one grid block per thread in the compose and apply passes

// the block's gr_complex product a * b, each product and sum rounded on its own
__device__ __forceinline__ float2 cmul(float2 a, float2 b)
{
    return make_float2(__fsub_rn(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)), __fadd_rn(__fmul_rn(a.x, b.y), __fmul_rn(a.y, b.x)));
}
__device__ __forceinline__ float2 conjf2(float2 a) { return make_float2(a.x, -a.y); }
__device__ __forceinline__ double2 dmul(double2 a, double2 b)
{
    return make_double2(__dsub_rn(__dmul_rn(a.x, b.x), __dmul_rn(a.y, b.y)), __dadd_rn(__dmul_rn(a.x, b.y), __dmul_rn(a.y, b.x)));
}
__device__ __forceinline__ double2 dadd(double2 a, double2 b) { return make_double2(__dadd_rn(a.x, b.x), __dadd_rn(a.y, b.y)); }
__device__ __forceinline__ double2 f2d(float2 a) { return make_double2(a.x, a.y); }

// z0 = exp(i angle): cos and sin in double, each rounded once to float
__device__ __forceinline__ float2 unit(float angle)
{
    double s, c;
    sincos(static_cast<double>(angle), &s, &c);
    return make_float2(__double2float_rn(c), __double2float_rn(s));
}
// volk_32fc_s32f_atan2_32f of a * conj(b) with factor 1, atan2 in double rounded once to float
__device__ __forceinline__ float angle_of(float2 a, float2 b)
{
    const float2 c = cmul(a, conjf2(b));
    return __double2float_rn(atan2(static_cast<double>(c.y), static_cast<double>(c.x)));
}

// the block's in[]: output j of segment k reads input j + shift (Notch 1, Lite 0).  For Lite the sample before the origin is
// the zero history item.
template <int FMT>
struct Input
{
    const SampleRaw<FMT>* ring;
    unsigned long long mask;
    unsigned long long zero_at;  // the index read as 0 (Lite: origin - 1); ~0: none
    __device__ __forceinline__ float2 operator()(unsigned long long i) const
    {
        return i == zero_at ? make_float2(0.f, 0.f) : widen<FMT>(__ldg(ring + (i & mask)));
    }
};
template <int FMT>
__device__ __forceinline__ Input<FMT> input_of(const void* src, unsigned long long mask, const NotchParams& p)
{
    return Input<FMT>{static_cast<const SampleRaw<FMT>*>(src), mask, p.variant == B200_NOTCH_LITE ? p.origin - 1 : ~0ULL};
}
__device__ __forceinline__ unsigned long long shift_of(const NotchParams& p) { return p.variant == B200_NOTCH ? 1ULL : 0ULL; }

// e[k] = Re(volk_32fc_x2_conjugate_dot_prod_32fc(in, in, L)) of segment seg0 + k, in the generic kernel's order: even
// samples into one sum, odd into another, each |x|^2 = re re + im im; e = sum0 + sum1, then + |x_{L-1}|^2 when L is odd
template <int FMT>
__global__ void __launch_bounds__(kEnergyThreads) notch_energy_kernel(const void* __restrict__ src, unsigned long long src_mask,
    NotchParams prm, unsigned long long seg0, int n_seg, float* __restrict__ energy)
{
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n_seg) return;
    const Input<FMT> in = input_of<FMT>(src, src_mask, prm);
    const unsigned long long b = prm.origin + (seg0 + k) * static_cast<unsigned long long>(prm.L) + shift_of(prm);
    const int L = prm.L;
    float s0 = 0.f, s1 = 0.f;
    int i = 0;
    for (; i + 1 < L; i += 2)
        {
            const float2 u = in(b + i), v = in(b + i + 1);
            s0 = __fadd_rn(s0, __fadd_rn(__fmul_rn(u.x, u.x), __fmul_rn(u.y, u.y)));
            s1 = __fadd_rn(s1, __fadd_rn(__fmul_rn(v.x, v.x), __fmul_rn(v.y, v.y)));
        }
    float e = __fadd_rn(s0, s1);
    if (i < L)
        {
            const float2 u = in(b + i);
            e = __fadd_rn(e, __fadd_rn(__fmul_rn(u.x, u.x), __fmul_rn(u.y, u.y)));
        }
    energy[k] = e;
}

// sig2lin of segment seg0 + blockIdx.x, only where the segment can be in estimation: n_k = n0 + k while no reset can have
// happened (n0 + k - 1 <= R), and such a segment with n_k >= E cannot be.  The spectrum is a direct DFT in double,
// X[q] = sum_m x[m] W[m q mod L] (m ascending, each product and sum rounded), dB[q] = float(10 log10(|X[q]|^2 + 1e-20));
// then volk_32f_s32f_calc_spectral_noise_floor_32f (exclusion 15 dB) in float, and sig2lin = float(10^(dB / 10)) / 2L.
template <int FMT>
__global__ void notch_floor_kernel(const void* __restrict__ src, unsigned long long src_mask, NotchParams prm, unsigned long long seg0,
    int fresh, const NotchState* __restrict__ state, const double2* __restrict__ twiddle, float* __restrict__ sig2lin)
{
    __shared__ float2 x[B200_IQ_MAX_NOTCH_LENGTH];
    __shared__ float db[B200_IQ_MAX_NOTCH_LENGTH];
    const long long k = blockIdx.x;
    const long long n0 = fresh ? 0 : state->n;
    if (n0 + k >= prm.n_est && n0 + k - 1 <= prm.n_reset) return;
    const Input<FMT> in = input_of<FMT>(src, src_mask, prm);
    const int L = prm.L;
    const unsigned long long b = prm.origin + (seg0 + k) * static_cast<unsigned long long>(L) + shift_of(prm);
    for (int m = threadIdx.x; m < L; m += blockDim.x) x[m] = in(b + m);
    __syncthreads();
    for (int q = threadIdx.x; q < L; q += blockDim.x)
        {
            double2 acc = make_double2(0.0, 0.0);
            int w = 0;
            for (int m = 0; m < L; m++)
                {
                    acc = dadd(acc, dmul(f2d(x[m]), __ldg(twiddle + w)));
                    w += q;
                    if (w >= L) w -= L;
                }
            const double pw = __dadd_rn(__dmul_rn(acc.x, acc.x), __dmul_rn(acc.y, acc.y));
            db[q] = __double2float_rn(__dmul_rn(10.0, log10(__dadd_rn(pw, 1e-20))));
        }
    __syncthreads();
    if (threadIdx.x != 0) return;
    const float nf = static_cast<float>(static_cast<unsigned>(L));
    float sum = 0.f;
    for (int q = 0; q < L; q++) sum = __fadd_rn(sum, db[q]);
    const float mean = __fadd_rn(__fdiv_rn(sum, nf), 15.f);
    sum = 0.f;
    unsigned cnt = static_cast<unsigned>(L);
    for (int q = 0; q < L; q++)
        if (db[q] <= mean)
            sum = __fadd_rn(sum, db[q]);
        else
            cnt--;
    const float floor_db = cnt == 0 ? mean : __fdiv_rn(sum, static_cast<float>(cnt));
    const float lin = __double2float_rn(pow(10.0, static_cast<double>(__fdiv_rn(floor_db, 10.f))));
    sig2lin[k] = __fdiv_rn(lin, static_cast<float>(2 * L));
}

// the block's segment loop over the push's n_seg segments: flags[k] bit 0 filtered, bit 1 a run starts there (last_out_ =
// 0).  Estimation (n < E and the filter off) is a serial recurrence on thread 0.  In detection est is fixed, so every
// decision e / est > thres is independent: a step decides up to kScanThreads segments at once and ends at its first reset
// (found by ballot).  Runs and Lite coefficient epochs come from a max-scan of the last unfiltered segment: a filtered
// segment q places into its run has n_segments_coeff_ = q mod Nc, and takes z0 from segment k - (q mod Nc).  Lite: the
// epoch starts then compute z0 from the ring, and every filtered segment copies its epoch's.
template <int FMT>
__global__ void __launch_bounds__(kScanThreads) notch_scan_kernel(const void* __restrict__ src, unsigned long long src_mask, NotchParams prm,
    unsigned long long seg0, int n_seg, int fresh, const float* __restrict__ energy, const float* __restrict__ sig2lin,
    NotchState* __restrict__ state, unsigned char* __restrict__ flags, int* __restrict__ zsrc, float2* __restrict__ zseg)
{
    __shared__ int warp_v[kScanThreads / 32];
    __shared__ long long n_sh;
    __shared__ float est_sh;
    __shared__ int fs_sh, nc_sh, i_sh, first_sh, lastf_sh, qlast_sh, last_seg_sh;
    __shared__ float2 z0_sh;
    __shared__ unsigned long long filtered_sh;
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    const bool lite = prm.variant == B200_NOTCH_LITE;
    if (t == 0)
        {
            if (fresh)
                {
                    NotchState s{};
                    s.last_seg = -1;
                    s.pa = make_double2(1.0, 0.0);
                    *state = s;
                }
            const NotchState s = *state;
            n_sh = s.n;
            est_sh = s.est;
            fs_sh = s.filter_state;
            nc_sh = s.n_coeff;
            z0_sh = s.z0;
            filtered_sh = s.filtered;
            last_seg_sh = -1;
        }
    for (int base = 0; base < n_seg; base += kScanThreads)
        {
            const int c = min(kScanThreads, n_seg - base);
            if (t == 0) i_sh = 0;
            __syncthreads();
            for (;;)
                {
                    const int i = i_sh;
                    const long long n = n_sh;
                    const int fs = fs_sh, nc = nc_sh;
                    const float est = est_sh;
                    __syncthreads();  // every thread holds the step's state before thread 0 moves it on
                    if (i >= c) break;
                    if (n < prm.n_est && !fs)
                        {
                            if (t == 0)
                                {
                                    float v = est;
                                    long long m = n;
                                    int k = i;
                                    for (; k < c && m < prm.n_est; k++, m++)
                                        {
                                            v = __fdiv_rn(__fadd_rn(__fmul_rn(__ll2float_rn(m), v), sig2lin[base + k]), __ll2float_rn(m + 1));
                                            flags[base + k] = 0;
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
                            const bool filt = valid && __fdiv_rn(energy[base + k], est) > prm.thres;
                            const bool reset = valid && !filt && n + t > prm.n_reset;
                            unsigned b = __ballot_sync(0xffffffffu, reset);
                            if (lane == 0) warp_v[warp] = b ? warp * 32 + __ffs(b) - 1 : kScanThreads;
                            if (t == 0) lastf_sh = -1;
                            __syncthreads();
                            if (warp == 0)
                                {
                                    int v = warp_v[lane];
                                    for (int o = 16; o > 0; o >>= 1) v = min(v, __shfl_xor_sync(0xffffffffu, v, o));
                                    if (lane == 0) first_sh = v;
                                }
                            __syncthreads();
                            const int first = first_sh;  // step index of the first reset, kScanThreads if none
                            const int end = min(first + 1, c - i);
                            const bool in = t < end;
                            // inclusive max-scan of the last unfiltered step index (-1: none yet in this step)
                            int v = (in && !filt) ? t : -1;
                            for (int o = 1; o < 32; o <<= 1)
                                {
                                    const int u = __shfl_up_sync(0xffffffffu, v, o);
                                    if (lane >= o) v = max(v, u);
                                }
                            if (lane == 31) warp_v[warp] = v;
                            __syncthreads();
                            if (warp == 0)
                                {
                                    int w = warp_v[lane];
                                    for (int o = 1; o < 32; o <<= 1)
                                        {
                                            const int u = __shfl_up_sync(0xffffffffu, w, o);
                                            if (lane >= o) w = max(w, u);
                                        }
                                    warp_v[lane] = w;
                                }
                            __syncthreads();
                            const int lnf = warp > 0 ? max(v, warp_v[warp - 1]) : v;
                            const int q = lnf >= 0 ? t - lnf - 1 : t + (fs ? nc : 0);
                            if (in)
                                {
                                    const bool start = filt && q == 0 && !(lnf < 0 && fs);
                                    flags[base + k] = static_cast<unsigned char>((filt ? 1 : 0) | (start ? 2 : 0));
                                    if (filt && lite) zsrc[base + k] = base + k - q % prm.n_coeff;
                                    if (filt) atomicMax(&lastf_sh, t);
                                }
                            const int nf = __syncthreads_count(in && filt);
                            if (t == lastf_sh) qlast_sh = q;
                            if (t == end - 1) fs_sh = filt ? 1 : 0;
                            __syncthreads();
                            if (t == 0)
                                {
                                    filtered_sh += static_cast<unsigned long long>(nf);
                                    if (lastf_sh >= 0)
                                        {
                                            nc_sh = lite ? (qlast_sh + 1) % prm.n_coeff : 0;
                                            last_seg_sh = base + i + lastf_sh;
                                        }
                                    n_sh = first < kScanThreads ? 1 : n + end;  // a reset: n = 0, then n++
                                    i_sh = i + end;
                                }
                        }
                    __syncthreads();
                }
            __syncthreads();  // before the next step resets i_sh
        }
    if (lite)
        {
            const Input<FMT> in = input_of<FMT>(src, src_mask, prm);
            const int L = prm.L;
            for (int k = t; k < n_seg; k += blockDim.x)
                if ((flags[k] & 1) && zsrc[k] == k)
                    {
                        const unsigned long long b = prm.origin + (seg0 + k) * static_cast<unsigned long long>(L);
                        const float a1 = angle_of(in(b + 1), in(b));
                        const float a2 = angle_of(in(b + L - 1), in(b + L - 2));
                        zseg[k] = unit(__fdiv_rn(__fadd_rn(a1, a2), 2.f));
                    }
            __syncthreads();
            for (int k = t; k < n_seg; k += blockDim.x)
                if ((flags[k] & 1) && zsrc[k] != k) zseg[k] = zsrc[k] >= 0 ? zseg[zsrc[k]] : z0_sh;
            __syncthreads();
        }
    if (t == 0)
        {
            state->n = n_sh;
            state->est = est_sh;
            state->filter_state = fs_sh;
            state->n_coeff = nc_sh;
            state->filtered = filtered_sh;
            state->last_seg = last_seg_sh;
            if (lite && last_seg_sh >= 0) state->z0 = zseg[last_seg_sh];
        }
}

// the terms of output r (counted from the origin) of a filtered segment: b = x - z0 x_prev and a = p z0, as the block rounds them
template <int FMT, int VAR>
__device__ __forceinline__ void notch_terms(const Input<FMT>& in, const NotchParams& prm, unsigned long long r, int kp, unsigned long long ri,
    const float2* __restrict__ zseg, float2* __restrict__ zs, bool store_z0, float2& a, float2& b)
{
    const unsigned long long i = prm.origin + r + (VAR == B200_NOTCH ? 1ULL : 0ULL);
    const float2 x = in(i), xp = in(i - 1);
    float2 z0;
    if (VAR == B200_NOTCH_LITE)
        z0 = zseg[kp];
    else if (store_z0)
        {
            z0 = unit(angle_of(x, xp));
            zs[ri] = z0;
        }
    else
        z0 = zs[ri];
    const float2 t = cmul(z0, xp);
    b = make_float2(__fsub_rn(x.x, t.x), __fsub_rn(x.y, t.y));
    a = cmul(make_float2(prm.p, 0.f), z0);
}

// one thread per grid block of the push: the block's map y -> A y + B in double over its samples in the push, in sample
// order: a run start sets (0, b), a filtered sample (a A, a B + b), an unfiltered one (0, 0).  The block in progress at the
// push's start continues from the stored partial map.  Notch: the per-sample z0 are computed here and kept for the apply pass.
template <int FMT, int VAR>
__global__ void __launch_bounds__(kGridThreads) notch_compose_kernel(const void* __restrict__ src, unsigned long long src_mask, NotchParams prm,
    unsigned long long seg0, int n_seg, const unsigned char* __restrict__ flags, const float2* __restrict__ zseg, float2* __restrict__ zs,
    const NotchState* __restrict__ state, double2* __restrict__ block_ab)
{
    const unsigned long long L = static_cast<unsigned long long>(prm.L), C = kNotchGrid;
    const unsigned long long r0 = seg0 * L, r1 = r0 + static_cast<unsigned long long>(n_seg) * L, g0 = r0 / C;
    const unsigned long long qb = static_cast<unsigned long long>(blockIdx.x) * blockDim.x + threadIdx.x, g = g0 + qb;
    if (g > (r1 - 1) / C) return;
    const Input<FMT> in = input_of<FMT>(src, src_mask, prm);
    const unsigned long long lo = max(r0, g * C), hi = min(r1, (g + 1) * C);
    double2 A = make_double2(1.0, 0.0), B = make_double2(0.0, 0.0);
    if (lo != g * C)
        {
            A = state->pa;
            B = state->pb;
        }
    for (unsigned long long r = lo; r < hi; r++)
        {
            const int kp = static_cast<int>(r / L - seg0);
            const unsigned char f = flags[kp];
            if (!(f & 1))
                {
                    A = B = make_double2(0.0, 0.0);
                    continue;
                }
            float2 a, b;
            notch_terms<FMT, VAR>(in, prm, r, kp, r - r0, zseg, zs, true, a, b);
            if ((f & 2) && r % L == 0)
                {
                    A = make_double2(0.0, 0.0);
                    B = f2d(b);
                }
            else
                {
                    A = dmul(f2d(a), A);
                    B = dadd(dmul(f2d(a), B), f2d(b));
                }
        }
    block_ab[2 * qb] = A;
    block_ab[2 * qb + 1] = B;
}

// one thread: y from grid point to grid point, y_{g+1} = A_g y_g + B_g in double, writing y entering each block of the push;
// the block left incomplete keeps its partial map.  Notch: z_0_ becomes the last filtered sample's z0.
__global__ void notch_carry_kernel(NotchParams prm, unsigned long long seg0, int n_seg, const double2* __restrict__ block_ab,
    const float2* __restrict__ zs, NotchState* __restrict__ state, double2* __restrict__ y_grid)
{
    const unsigned long long L = static_cast<unsigned long long>(prm.L), C = kNotchGrid;
    const unsigned long long r0 = seg0 * L, r1 = r0 + static_cast<unsigned long long>(n_seg) * L, g0 = r0 / C, nb = (r1 - 1) / C - g0 + 1;
    double2 y = state->y_grid;
    double2 pa = make_double2(1.0, 0.0), pb = make_double2(0.0, 0.0);
    for (unsigned long long q = 0; q < nb; q++)
        {
            y_grid[q] = y;
            const double2 A = block_ab[2 * q], B = block_ab[2 * q + 1];
            if ((g0 + q + 1) * C <= r1)
                y = dadd(dmul(A, y), B);
            else
                {
                    pa = A;
                    pb = B;
                }
        }
    state->y_grid = y;
    state->pa = pa;
    state->pb = pb;
    state->last_in = state->last_out;
    if (prm.variant == B200_NOTCH && state->last_seg >= 0) state->z0 = zs[static_cast<unsigned long long>(state->last_seg + 1) * L - 1];
}

// one thread per grid block of the push: the destination, copied where unfiltered, else the block's float32 recursion
// y = (x - z0 x_prev) + (p z0) last, last = y, started from float(y entering the block) (the block in progress at the push's
// start: from the last output of the previous push), and from 0 at a run start
template <int FMT, int VAR>
__global__ void __launch_bounds__(kGridThreads) notch_apply_kernel(const void* __restrict__ src, unsigned long long src_mask, NotchParams prm,
    unsigned long long seg0, int n_seg, const unsigned char* __restrict__ flags, const float2* __restrict__ zseg, float2* __restrict__ zs,
    const double2* __restrict__ y_grid, NotchState* __restrict__ state, float2* __restrict__ dst, unsigned long long dst_mask)
{
    const unsigned long long L = static_cast<unsigned long long>(prm.L), C = kNotchGrid;
    const unsigned long long r0 = seg0 * L, r1 = r0 + static_cast<unsigned long long>(n_seg) * L, g0 = r0 / C;
    const unsigned long long qb = static_cast<unsigned long long>(blockIdx.x) * blockDim.x + threadIdx.x, g = g0 + qb;
    if (g > (r1 - 1) / C) return;
    const Input<FMT> in = input_of<FMT>(src, src_mask, prm);
    const unsigned long long lo = max(r0, g * C), hi = min(r1, (g + 1) * C);
    const int last_seg = state->last_seg;
    float2 last;
    if (lo != g * C)
        last = state->last_in;
    else
        last = make_float2(__double2float_rn(y_grid[qb].x), __double2float_rn(y_grid[qb].y));
    for (unsigned long long r = lo; r < hi; r++)
        {
            const int kp = static_cast<int>(r / L - seg0);
            const unsigned char f = flags[kp];
            const unsigned long long j = prm.origin + r;
            if (!(f & 1))
                {
                    dst[j & dst_mask] = in(j + (VAR == B200_NOTCH ? 1ULL : 0ULL));
                    continue;
                }
            float2 a, b;
            notch_terms<FMT, VAR>(in, prm, r, kp, r - r0, zseg, zs, false, a, b);
            if ((f & 2) && r % L == 0) last = make_float2(0.f, 0.f);
            const float2 u = cmul(a, last);
            last = make_float2(__fadd_rn(b.x, u.x), __fadd_rn(b.y, u.y));
            dst[j & dst_mask] = last;
            if (kp == last_seg && (r + 1) % L == 0) state->last_out = last;
        }
}
}  // namespace

namespace b200
{
int launch_notch(const void* src, int src_fmt, unsigned long long src_mask, const NotchParams& prm, unsigned long long seg0, int n_seg,
    int fresh, const NotchBufs& b, float2* dst, unsigned long long dst_mask, cudaStream_t st)
{
    if (n_seg <= 0) return B200_OK;
    const unsigned long long L = static_cast<unsigned long long>(prm.L), r0 = seg0 * L, r1 = r0 + static_cast<unsigned long long>(n_seg) * L;
    const unsigned nb = static_cast<unsigned>((r1 - 1) / kNotchGrid - r0 / kNotchGrid + 1);
    const unsigned grid_ctas = (nb + kGridThreads - 1) / kGridThreads;
    const int floor_threads = std::min(B200_IQ_MAX_NOTCH_LENGTH, (prm.L + 31) / 32 * 32);
    const int rc = with_format(src_fmt, [&](auto F) {
        constexpr int FMT = decltype(F)::value;
        notch_energy_kernel<FMT><<<(n_seg + kEnergyThreads - 1) / kEnergyThreads, kEnergyThreads, 0, st>>>(src, src_mask, prm, seg0, n_seg, b.energy);
        notch_floor_kernel<FMT><<<n_seg, floor_threads, 0, st>>>(src, src_mask, prm, seg0, fresh, b.state, b.twiddle, b.sig2lin);
        notch_scan_kernel<FMT><<<1, kScanThreads, 0, st>>>(src, src_mask, prm, seg0, n_seg, fresh, b.energy, b.sig2lin, b.state, b.flags, b.zsrc,
            b.zseg);
        if (prm.variant == B200_NOTCH)
            notch_compose_kernel<FMT, B200_NOTCH><<<grid_ctas, kGridThreads, 0, st>>>(src, src_mask, prm, seg0, n_seg, b.flags, b.zseg, b.zs,
                b.state, b.block_ab);
        else
            notch_compose_kernel<FMT, B200_NOTCH_LITE><<<grid_ctas, kGridThreads, 0, st>>>(src, src_mask, prm, seg0, n_seg, b.flags, b.zseg,
                b.zs, b.state, b.block_ab);
        notch_carry_kernel<<<1, 1, 0, st>>>(prm, seg0, n_seg, b.block_ab, b.zs, b.state, b.y_grid);
        if (prm.variant == B200_NOTCH)
            notch_apply_kernel<FMT, B200_NOTCH><<<grid_ctas, kGridThreads, 0, st>>>(src, src_mask, prm, seg0, n_seg, b.flags, b.zseg, b.zs,
                b.y_grid, b.state, dst, dst_mask);
        else
            notch_apply_kernel<FMT, B200_NOTCH_LITE><<<grid_ctas, kGridThreads, 0, st>>>(src, src_mask, prm, seg0, n_seg, b.flags, b.zseg,
                b.zs, b.y_grid, b.state, dst, dst_mask);
        return B200_OK;
    });
    if (rc) return rc;
    B200_CUDA_TRY(cudaGetLastError());
    return B200_OK;
}
}  // namespace b200
