// Device helpers shared by the tracking kernels (trk_kernels.cu, trk_shared_kernel.cu).
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

__device__ __forceinline__ int mod_pos(int k, int L)
{
    int r = k % L;
    return r < 0 ? r + L : r;
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

}  // namespace
}  // namespace b200
