// Device helpers shared by the tracking kernels (trk_kernels.cu, trk_shared_kernel.cu, trk_variants.cu and, through
// trk_item.cuh, loop_kernels_nofma.cu).  Every contraction is written out, so they compute the same under --fmad=false.
#pragma once

#include "common.cuh"

namespace b200
{
namespace
{
// ---- float32 chip-index arithmetic, bit-compatible with the reference -------------------------
// a_avx/u_avx association (resampler .h:387,393-396): floor(fl(fl(step*n) + fl(shift - rem)))
__device__ __forceinline__ int chip_index_avx(float step, float nf, float aux2)
{
    return __float2int_rd(__fadd_rn(__fmul_rn(step, nf), aux2));
}
// generic association (resampler .h:73 and the AVX kernels' scalar tail :423-433):
// floor(fl(fl(fl(step*n) + shift) - rem))
__device__ __forceinline__ int chip_index_generic(float step, float nf, float shift, float rem)
{
    return __float2int_rd(__fsub_rn(__fadd_rn(__fmul_rn(step, nf), shift), rem));
}
// high-dynamics association (..._high_dynamics_resampler_32f_xn.h:77):
// floor(fl(fl(fl(fl(step*n) + fl(rate*(float)(n*n))) + shift0) - rem)), n*n in uint32 (wraps)
__device__ __forceinline__ int chip_index_hd(float step, float rate, unsigned int n, float shift0, float rem)
{
    const float nf = static_cast<float>(n);
    const float n2 = static_cast<float>(n * n);
    return __float2int_rd(__fsub_rn(__fadd_rn(__fadd_rn(__fmul_rn(step, nf), __fmul_rn(rate, n2)), shift0), rem));
}

// high-dynamics, a_avx/u_avx association (same file :460-466): n*n is a FLOAT product here
// floor(fl(fl(fl(step*n) + fl(rate*fl(n*n))) + fl(shift0 - rem)))
__device__ __forceinline__ int chip_index_hd_avx(float step, float rate, float nf, float aux2)
{
    const float nn = __fmul_rn(nf, nf);
    return __float2int_rd(__fadd_rn(__fadd_rn(__fmul_rn(step, nf), __fmul_rn(rate, nn)), aux2));
}

// chip index of sample n of an epoch: the AVX association below body = 8*(N/8), the generic one in the tail
__device__ __forceinline__ int chip_index_at(float step, int n, int body, float shift, float rem)
{
    const float nf = static_cast<float>(n);
    return (n < body) ? chip_index_avx(step, nf, __fsub_rn(shift, rem)) : chip_index_generic(step, nf, shift, rem);
}

// [lo, hi] of the AVX-association chip indices of every tap over the samples n_first..n_last (monotone in n, so the ends
// suffice); aux(t) = fl(shift_t - rem).
template <int TAPS, class Aux>
__device__ __forceinline__ void chip_range(float step, float n_first, float n_last, const Aux& aux, int& lo, int& hi)
{
    lo = 0x7fffffff;
    hi = -0x7fffffff - 1;
#pragma unroll
    for (int t = 0; t < TAPS; t++)
        {
            const int i0 = chip_index_avx(step, n_first, aux(t));
            const int i1 = chip_index_avx(step, n_last, aux(t));
            lo = min(lo, min(i0, i1));
            hi = max(hi, max(i0, i1));
        }
}

__device__ __forceinline__ int mod_pos(int k, int L)
{
    int r = k % L;
    return r < 0 ? r + L : r;
}

// Stages the code window [base, base + span) (indices modulo L) into a table: entries pos, pos + stride, ... are this
// thread's, store(j, code + i) writes entry j from code value i.
template <class Store>
__device__ __forceinline__ void stage_code_window(const float* code, int L, int base, int span, int pos, int stride, const Store& store)
{
    int r = mod_pos(base + pos, L);
    const int step = stride % L;
    for (int j = pos; j < span; j += stride)
        {
            store(j, code + r);
            r += step;
            if (r >= L) r -= L;
        }
}

// floor() by the 1.5*2^23 trick: fl_rd(x + kFloorMagic) has floor(x) in its low mantissa bits (exact for |x| < 2^22), so a
// table entry's shared-memory address is one LEA, (bits << 2) + table_offset(table, base) for the entry floor(x) - base.
constexpr float kFloorMagic = 12582912.0f;  // bit pattern 0x4B400000
__device__ __forceinline__ unsigned int table_offset(const float* smem_tbl, int base)
{
    // computed inside an asm so the optimiser cannot split the constant back out of the per-lookup LEA
    unsigned int off;
    asm("sub.u32 %0, %1, %2;"
        : "=r"(off)
        : "r"(static_cast<unsigned int>(__cvta_generic_to_shared(smem_tbl))), "r"(4u * (static_cast<unsigned int>(base) + 0x4B400000u)));
    return off;
}

template <class T>
__device__ __forceinline__ T warp_sum(T v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float2 warp_sum(float2 v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1)
        {
            v.x += __shfl_xor_sync(0xffffffffu, v.x, o);
            v.y += __shfl_xor_sync(0xffffffffu, v.y, o);
        }
    return v;
}

// exp(j*2*pi*T/2^64)
__device__ __forceinline__ float2 phasor_from_turns(unsigned long long T)
{
    const int hi = static_cast<int>(T >> 32);
    const float x = static_cast<float>(hi) * 4.656612873077393e-10f;  // half-turns in [-1,1)
    float s, c;
    sincospif(x, &s, &c);
    return make_float2(c, s);
}

// radians -> 64-bit fixed-point turns (two's complement, wraps naturally)
__device__ __forceinline__ unsigned long long turns_from_rad(double rad)
{
    double t = rad * 0.15915494309189535;  // 1/(2*pi)
    t -= rint(t);
    return static_cast<unsigned long long>(__double2ll_rn(t * 18446744073709551616.0));
}

// carrier phase and step of an item in 64-bit turns (phase(n) = -(rem + n*step)), and body = 8*(N/8)
struct ItemPhase
{
    unsigned long long T0, DT;
    int body;
};
__device__ __forceinline__ ItemPhase item_phase(float rem_carrier_phase_rad, float phase_step_rad, int n)
{
    return ItemPhase{turns_from_rad(-static_cast<double>(rem_carrier_phase_rad)), turns_from_rad(-static_cast<double>(phase_step_rad)), (n / 8) * 8};
}

__device__ __forceinline__ float2 cmulf(float2 a, float2 b)
{
    return make_float2(fmaf(a.x, b.x, -a.y * b.y), fmaf(a.x, b.y, a.y * b.x));
}

__device__ __forceinline__ float4 ldg_stream16(const float2* p)
{
    float4 v;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
                 : "l"(p));
    return v;
}

__device__ __forceinline__ float2 ldg_stream8(const float2* p)
{
    float2 v;
    asm volatile("ld.global.nc.L1::no_allocate.v2.f32 {%0,%1}, [%2];" : "=f"(v.x), "=f"(v.y) : "l"(p));
    return v;
}

// Streaming loads of band samples of SampleFormat FMT, widened to float on load (widen_i16 / widen_i8 of common.cuh):
// sample slot k of a band starts at byte 2 * FMT * k of its base.
template <int FMT>
__device__ __forceinline__ const char* sample_ptr(const void* base, unsigned long long k)
{
    return static_cast<const char*>(base) + k * (2ULL * FMT);
}
// samples k and k + 1 (k even) as (re, im, re, im): one 16-, 8- or 4-byte load
template <int FMT>
__device__ __forceinline__ float4 ldg_stream_pair(const char* p)
{
    if constexpr (FMT == kCf32)
        {
            return ldg_stream16(reinterpret_cast<const float2*>(p));
        }
    else if constexpr (FMT == kI16)
        {
            unsigned int w0, w1;
            asm volatile("ld.global.nc.L1::no_allocate.v2.u32 {%0,%1}, [%2];" : "=r"(w0), "=r"(w1) : "l"(p));
            const float2 a = widen_i16(w0), b = widen_i16(w1);
            return make_float4(a.x, a.y, b.x, b.y);
        }
    else
        {
            unsigned int w;
            asm volatile("ld.global.nc.L1::no_allocate.u32 %0, [%1];" : "=r"(w) : "l"(p));
            const float2 a = widen_i8<0>(w), b = widen_i8<1>(w);
            return make_float4(a.x, a.y, b.x, b.y);
        }
}
// one sample: an 8-, 4- or 2-byte load
template <int FMT>
__device__ __forceinline__ float2 ldg_stream_one(const char* p)
{
    if constexpr (FMT == kCf32)
        {
            return ldg_stream8(reinterpret_cast<const float2*>(p));
        }
    else if constexpr (FMT == kI16)
        {
            unsigned int w;
            asm volatile("ld.global.nc.L1::no_allocate.u32 %0, [%1];" : "=r"(w) : "l"(p));
            return widen_i16(w);
        }
    else
        {
            unsigned short h;
            asm volatile("ld.global.nc.L1::no_allocate.u16 %0, [%1];" : "=h"(h) : "l"(p));
            return widen_i8<0>(h);
        }
}


// ---- lane-wise float2 arithmetic on sample pairs (.x = sample n, .y = sample n+1).  Hopper has no
// packed FP32 instructions, so each is two scalar operations with an explicit rounding mode: ptxas
// never contracts a separately rounded mul+add of the chip-index arithmetic into an FMA.
__device__ __forceinline__ float2 add2_rn(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ float2 add2_rd(float2 a, float2 b) { return make_float2(__fadd_rd(a.x, b.x), __fadd_rd(a.y, b.y)); }
__device__ __forceinline__ float2 mul2_rn(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ float2 fma2_rn(float2 a, float2 b, float2 c)
{
    return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}
__device__ __forceinline__ float lds_f32(unsigned int addr)
{
    float v;
    asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr));
    return v;
}

// (zr, zi) *= (Dr2, Di2): the phasors of a sample pair (.x, .y) advance by one step D
__device__ __forceinline__ void advance_pair(float2& zr, float2& zi, float2 Dr2, float2 Di2)
{
    const float2 t1 = mul2_rn(zi, Di2);
    const float2 nzr = fma2_rn(zr, Dr2, make_float2(-t1.x, -t1.y));
    zi = fma2_rn(zr, Di2, mul2_rn(zi, Dr2));
    zr = nzr;
}

// The taps of one sample pair (.x = sample n, .y = n+1) with rotated samples (wr2, wi2) and m2 = fl(step * n): each tap's chip
// is floor(fl(m2 + aux2[t])) by the kFloorMagic trick, looked up in the extended table (tbl_off = table_offset()).
template <int TAPS>
__device__ __forceinline__ void pair_taps(float2 m2, const float2 (&aux2)[TAPS], unsigned int tbl_off, float2 wr2, float2 wi2,
    float2 (&are)[TAPS], float2 (&aim)[TAPS])
{
    const float2 magic2 = make_float2(kFloorMagic, kFloorMagic);
#pragma unroll
    for (int t = 0; t < TAPS; t++)
        {
            const float2 tt = add2_rd(add2_rn(m2, aux2[t]), magic2);
            const float ca = lds_f32((__float_as_uint(tt.x) << 2) + tbl_off);
            const float cb = lds_f32((__float_as_uint(tt.y) << 2) + tbl_off);
            const float2 c2 = make_float2(ca, cb);
            are[t] = fma2_rn(wr2, c2, are[t]);
            aim[t] = fma2_rn(wi2, c2, aim[t]);
        }
}

}  // namespace
}  // namespace b200
