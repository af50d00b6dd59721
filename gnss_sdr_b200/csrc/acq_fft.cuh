// In-shared-memory mixed-radix complex FFT for sm_90a (no cuFFT).
//
// Sizes are whatever the receiver's sampling rate dictates (N = fs * T: 4000, 8000, 16000,
// 25000 = 2^3*5^5 ...), so radices 2,3,4,5,7,8 are supported and the planner factors N into them.
//
// Layout trick that removes every permutation pass: the forward transform is decimation in
// frequency (natural order in, digit-reversed order out), the inverse is decimation in time
// running the same stages backwards (digit-reversed in, natural out).  The local-code spectrum
// is stored in the same digit-reversed order, so the point-wise product between the two
// transforms needs no reordering.  Every butterfly reads r elements and writes them back to the
// same places: one buffer of N complex values (8N bytes, N <= kAcqMaxSmemPoints) and one
// __syncthreads per stage.
//
// Transforms are unnormalised in both directions, like FFTW / gr::fft
// (src/algorithms/libs/gnss_sdr_fft.h:26-62).
#pragma once

#include <cuda_runtime.h>

namespace b200
{
constexpr int kAcqThreads = 1024;
constexpr int kAcqThreads25 = 512;  // plans with radix-25 stages: 25 values per thread need 128 registers
constexpr int kAcqMaxStages = 16;
constexpr int kAcqMaxSmemPoints = 27648;  // 216 KB of float2

struct FftPlan
{
    int n;
    int n_stages;
    int radix[kAcqMaxStages];          // forward DIF order; product = n
    unsigned int mdiv[kAcqMaxStages];  // floor(2^32 / m) + 1 for the stage's m = M / radix (exact i / m for i < 2^16)
    int tw_off[kAcqMaxStages];         // start of the stage's compact twiddle table: exp(-2 pi j k / M), k < m
    // Sizes above kAcqMaxSmemPoints: n_total = n1 * n.  One radix-n1 stage runs through global memory (L2),
    // the remaining stages are the in-shared-memory plan above on each of the n1 blocks of n points.
    int n1;       // 1 = whole transform in shared memory
    int n_total;  // transform size seen by the caller
    int tw_goff;  // twiddles of the global stage: exp(-2 pi j k / n_total), k < n
    // Storage order of spectra in global memory (single-level plans with >= 2 stages): the digit-reversed
    // position p = b * perm_r + q (perm_r = radix of the last forward stage, q < perm_r) lives at
    // q * perm_nb + b.  The last forward stage then stores, and the first inverse stage loads, with
    // consecutive threads on consecutive addresses, so neither needs a pass through shared memory.
    int perm_r;   // 1 = natural digit-reversed order (no fusion)
    int perm_nb;  // n / perm_r
    int threads;  // CTA size the plan was made for: kAcqThreads, or kAcqThreads25 when it has radix-25 stages
};

__device__ __forceinline__ int fast_div(int i, int m, unsigned int magic)
{
    return (m == 1) ? i : static_cast<int>(__umulhi(static_cast<unsigned int>(i), magic));
}

__device__ __forceinline__ float2 cmul(float2 a, float2 b)
{
    return make_float2(fmaf(a.x, b.x, -a.y * b.y), fmaf(a.x, b.y, a.y * b.x));
}
// volk_32fc_x2_multiply_32fc: every product and sum rounded on its own, in the reference's order
__device__ __forceinline__ float2 cmul_rn(float2 a, float2 b)
{
    return make_float2(__fsub_rn(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)), __fadd_rn(__fmul_rn(a.x, b.y), __fmul_rn(a.y, b.x)));
}
__device__ __forceinline__ float2 cmul_conj(float2 a, float2 b)  // a * conj(b)
{
    return make_float2(fmaf(a.x, b.x, a.y * b.y), fmaf(a.y, b.x, -a.x * b.y));
}
__device__ __forceinline__ float2 cadd(float2 a, float2 b) { return make_float2(a.x + b.x, a.y + b.y); }
__device__ __forceinline__ float2 csub(float2 a, float2 b) { return make_float2(a.x - b.x, a.y - b.y); }
// multiply by -j (forward rotation by -90 deg): (x, y) -> (y, -x)
__device__ __forceinline__ float2 mul_mj(float2 a) { return make_float2(a.y, -a.x); }
__device__ __forceinline__ float2 mul_pj(float2 a) { return make_float2(-a.y, a.x); }

// ---- forward butterflies: y_p = sum_q x_q exp(-2 pi j p q / R), in place --------------------------
template <int R>
struct Bfly;

template <>
struct Bfly<2>
{
    static __device__ __forceinline__ void fwd(float2 (&v)[2])
    {
        const float2 a = v[0], b = v[1];
        v[0] = cadd(a, b);
        v[1] = csub(a, b);
    }
};

template <>
struct Bfly<3>
{
    static __device__ __forceinline__ void fwd(float2 (&v)[3])
    {
        const float s = 0.86602540378443865f;
        const float2 t = cadd(v[1], v[2]);
        const float2 d = csub(v[1], v[2]);
        const float2 a = make_float2(fmaf(-0.5f, t.x, v[0].x), fmaf(-0.5f, t.y, v[0].y));
        const float2 b = make_float2(s * d.x, s * d.y);
        v[0] = cadd(v[0], t);
        v[1] = cadd(a, mul_mj(b));
        v[2] = cadd(a, mul_pj(b));
    }
};

template <>
struct Bfly<4>
{
    static __device__ __forceinline__ void fwd(float2 (&v)[4])
    {
        const float2 t0 = cadd(v[0], v[2]), t1 = csub(v[0], v[2]);
        const float2 t2 = cadd(v[1], v[3]), t3 = csub(v[1], v[3]);
        v[0] = cadd(t0, t2);
        v[2] = csub(t0, t2);
        v[1] = cadd(t1, mul_mj(t3));
        v[3] = cadd(t1, mul_pj(t3));
    }
};

template <>
struct Bfly<5>
{
    static __device__ __forceinline__ void fwd(float2 (&v)[5])
    {
        const float c1 = 0.30901699437494742f, c2 = -0.80901699437494742f;
        const float s1 = 0.95105651629515357f, s2 = 0.58778525229247313f;
        const float2 t1 = cadd(v[1], v[4]), t2 = cadd(v[2], v[3]);
        const float2 t3 = csub(v[1], v[4]), t4 = csub(v[2], v[3]);
        const float2 a1 = make_float2(fmaf(c2, t2.x, fmaf(c1, t1.x, v[0].x)), fmaf(c2, t2.y, fmaf(c1, t1.y, v[0].y)));
        const float2 a2 = make_float2(fmaf(c1, t2.x, fmaf(c2, t1.x, v[0].x)), fmaf(c1, t2.y, fmaf(c2, t1.y, v[0].y)));
        const float2 b1 = make_float2(fmaf(s2, t4.x, s1 * t3.x), fmaf(s2, t4.y, s1 * t3.y));
        const float2 b2 = make_float2(fmaf(-s1, t4.x, s2 * t3.x), fmaf(-s1, t4.y, s2 * t3.y));
        v[0] = make_float2(v[0].x + t1.x + t2.x, v[0].y + t1.y + t2.y);
        v[1] = cadd(a1, mul_mj(b1));
        v[4] = cadd(a1, mul_pj(b1));
        v[2] = cadd(a2, mul_mj(b2));
        v[3] = cadd(a2, mul_pj(b2));
    }
};

template <>
struct Bfly<7>
{
    static __device__ __forceinline__ void fwd(float2 (&v)[7])
    {
        const float c1 = 0.62348980185873353f, c2 = -0.22252093395631440f, c3 = -0.90096886790241913f;
        const float s1 = 0.78183148246802981f, s2 = 0.97492791218182361f, s3 = 0.43388373911755812f;
        const float2 p1 = cadd(v[1], v[6]), p2 = cadd(v[2], v[5]), p3 = cadd(v[3], v[4]);
        const float2 m1 = csub(v[1], v[6]), m2 = csub(v[2], v[5]), m3 = csub(v[3], v[4]);
        const float2 x0 = v[0];
        // a_k = x0 + sum_q cos(2 pi k q/7) p_q ; b_k = sum_q sin(2 pi k q/7) m_q ; y_k = a_k - j b_k
        const float2 a1 = make_float2(x0.x + c1 * p1.x + c2 * p2.x + c3 * p3.x, x0.y + c1 * p1.y + c2 * p2.y + c3 * p3.y);
        const float2 a2 = make_float2(x0.x + c2 * p1.x + c3 * p2.x + c1 * p3.x, x0.y + c2 * p1.y + c3 * p2.y + c1 * p3.y);
        const float2 a3 = make_float2(x0.x + c3 * p1.x + c1 * p2.x + c2 * p3.x, x0.y + c3 * p1.y + c1 * p2.y + c2 * p3.y);
        const float2 b1 = make_float2(s1 * m1.x + s2 * m2.x + s3 * m3.x, s1 * m1.y + s2 * m2.y + s3 * m3.y);
        const float2 b2 = make_float2(s2 * m1.x - s3 * m2.x - s1 * m3.x, s2 * m1.y - s3 * m2.y - s1 * m3.y);
        const float2 b3 = make_float2(s3 * m1.x - s1 * m2.x + s2 * m3.x, s3 * m1.y - s1 * m2.y + s2 * m3.y);
        v[0] = make_float2(x0.x + p1.x + p2.x + p3.x, x0.y + p1.y + p2.y + p3.y);
        v[1] = cadd(a1, mul_mj(b1));
        v[6] = cadd(a1, mul_pj(b1));
        v[2] = cadd(a2, mul_mj(b2));
        v[5] = cadd(a2, mul_pj(b2));
        v[3] = cadd(a3, mul_mj(b3));
        v[4] = cadd(a3, mul_pj(b3));
    }
};

template <>
struct Bfly<8>
{
    static __device__ __forceinline__ void fwd(float2 (&v)[8])
    {
        const float h = 0.70710678118654752f;
        // radix-2 step over (q, q+4), then two radix-4s on even/odd outputs
        float2 e[4], o[4];
#pragma unroll
        for (int q = 0; q < 4; q++)
            {
                e[q] = cadd(v[q], v[q + 4]);
                o[q] = csub(v[q], v[q + 4]);
            }
        // odd branch twiddles w8^q, q = 0..3
        o[1] = make_float2(h * (o[1].x + o[1].y), h * (o[1].y - o[1].x));   // * (1 - j)/sqrt2
        o[2] = mul_mj(o[2]);
        o[3] = make_float2(h * (o[3].y - o[3].x), -h * (o[3].x + o[3].y));  // * (-1 - j)/sqrt2
        Bfly<4>::fwd(e);
        Bfly<4>::fwd(o);
#pragma unroll
        for (int q = 0; q < 4; q++)
            {
                v[2 * q] = e[q];
                v[2 * q + 1] = o[q];
            }
    }
};

// 10 = 2 x 5: input n = 5 n1 + n2, output k = k1 + 2 k2 (global stage of 10 ms transforms: 10 blocks of 1 ms)
template <>
struct Bfly<10>
{
    static __device__ __forceinline__ void fwd(float2 (&v)[10])
    {
        // W10^m = cos(2 pi m/10) - j sin(2 pi m/10), m = 1..4
        const float c1 = 0.80901699437494742f, s1 = 0.58778525229247313f;
        const float c2 = 0.30901699437494742f, s2 = 0.95105651629515357f;
        const float c3 = -0.30901699437494742f, s3 = 0.95105651629515357f;
        const float c4 = -0.80901699437494742f, s4 = 0.58778525229247313f;
        float2 a0[5], a1[5];
#pragma unroll
        for (int n2 = 0; n2 < 5; n2++)
            {
                a0[n2] = cadd(v[n2], v[5 + n2]);  // k1 = 0
                a1[n2] = csub(v[n2], v[5 + n2]);  // k1 = 1
            }
        a1[1] = make_float2(fmaf(a1[1].x, c1, a1[1].y * s1), fmaf(a1[1].y, c1, -a1[1].x * s1));
        a1[2] = make_float2(fmaf(a1[2].x, c2, a1[2].y * s2), fmaf(a1[2].y, c2, -a1[2].x * s2));
        a1[3] = make_float2(fmaf(a1[3].x, c3, a1[3].y * s3), fmaf(a1[3].y, c3, -a1[3].x * s3));
        a1[4] = make_float2(fmaf(a1[4].x, c4, a1[4].y * s4), fmaf(a1[4].y, c4, -a1[4].x * s4));
        Bfly<5>::fwd(a0);
        Bfly<5>::fwd(a1);
#pragma unroll
        for (int k2 = 0; k2 < 5; k2++)
            {
                v[2 * k2] = a0[k2];
                v[2 * k2 + 1] = a1[k2];
            }
    }
};

// 25 = 5 x 5 (Cooley-Tukey inside the registers of one thread): input n = 5 n1 + n2, output k = k1 + 5 k2,
// X[k1 + 5 k2] = sum_n2 W5^(n2 k2) W25^(n2 k1) sum_n1 x[5 n1 + n2] W5^(n1 k1).  Two shared-memory passes of a
// radix-5 pair become one.
template <>
struct Bfly<25>
{
    static __device__ __forceinline__ float2 mulw(float2 a, float c, float sn)  // a * (c - j sn)
    {
        return make_float2(fmaf(a.x, c, a.y * sn), fmaf(a.y, c, -a.x * sn));
    }
    static __device__ __forceinline__ void fwd(float2 (&v)[25])
    {
        // W25^m = cos(2 pi m/25) - j sin(2 pi m/25), m = n2 * k1
        const float c1 = 0.96858316112863108f, s1 = 0.24868988716485479f;
        const float c2 = 0.87630668004386358f, s2 = 0.48175367410171532f;
        const float c3 = 0.72896862742141155f, s3 = 0.68454710592868862f;
        const float c4 = 0.53582679497899655f, s4 = 0.84432792550201508f;
        const float c6 = 0.06279051952931353f, s6 = 0.99802672842827156f;
        const float c8 = -0.42577929156507272f, s8 = 0.90482705246601947f;
        const float c9 = -0.63742398974868975f, s9 = 0.77051324277578925f;
        const float c12 = -0.99211470131447783f, s12 = 0.12533323356430454f;
        const float c16 = -0.63742398974868952f, s16 = -0.77051324277578936f;
        float2 t[5];
#pragma unroll
        for (int n2 = 0; n2 < 5; n2++)
            {
#pragma unroll
                for (int n1 = 0; n1 < 5; n1++) t[n1] = v[5 * n1 + n2];
                Bfly<5>::fwd(t);
#pragma unroll
                for (int k1 = 0; k1 < 5; k1++) v[5 * k1 + n2] = t[k1];  // A[k1][n2]
            }
        v[5 * 1 + 1] = mulw(v[5 * 1 + 1], c1, s1);
        v[5 * 1 + 2] = mulw(v[5 * 1 + 2], c2, s2);
        v[5 * 1 + 3] = mulw(v[5 * 1 + 3], c3, s3);
        v[5 * 1 + 4] = mulw(v[5 * 1 + 4], c4, s4);
        v[5 * 2 + 1] = mulw(v[5 * 2 + 1], c2, s2);
        v[5 * 2 + 2] = mulw(v[5 * 2 + 2], c4, s4);
        v[5 * 2 + 3] = mulw(v[5 * 2 + 3], c6, s6);
        v[5 * 2 + 4] = mulw(v[5 * 2 + 4], c8, s8);
        v[5 * 3 + 1] = mulw(v[5 * 3 + 1], c3, s3);
        v[5 * 3 + 2] = mulw(v[5 * 3 + 2], c6, s6);
        v[5 * 3 + 3] = mulw(v[5 * 3 + 3], c9, s9);
        v[5 * 3 + 4] = mulw(v[5 * 3 + 4], c12, s12);
        v[5 * 4 + 1] = mulw(v[5 * 4 + 1], c4, s4);
        v[5 * 4 + 2] = mulw(v[5 * 4 + 2], c8, s8);
        v[5 * 4 + 3] = mulw(v[5 * 4 + 3], c12, s12);
        v[5 * 4 + 4] = mulw(v[5 * 4 + 4], c16, s16);
        float2 o[25];
#pragma unroll
        for (int k1 = 0; k1 < 5; k1++)
            {
#pragma unroll
                for (int n2 = 0; n2 < 5; n2++) t[n2] = v[5 * k1 + n2];
                Bfly<5>::fwd(t);
#pragma unroll
                for (int k2 = 0; k2 < 5; k2++) o[k1 + 5 * k2] = t[k2];
            }
#pragma unroll
        for (int q = 0; q < 25; q++) v[q] = o[q];
    }
};

__device__ __forceinline__ float2 swap_ri(float2 a) { return make_float2(a.y, a.x); }

// w^q for q = 0..R-1 from w^1: a multiply chain for the small radices, a two-level product for radix 25
// (w^(5a+b) = w^(5a) w^b) so that the dependency depth stays short.
template <int R>
__device__ __forceinline__ void twiddle_powers(float2 w1, float2 (&w)[R])
{
    w[0] = make_float2(1.f, 0.f);
    if (R > 1) w[1] = w1;
    if (R == 25)
        {
            w[2] = cmul(w1, w1);
            w[3] = cmul(w[2], w1);
            w[4] = cmul(w[2], w[2]);
            w[5] = cmul(w[4], w1);
            w[10] = cmul(w[5], w[5]);
            w[15] = cmul(w[10], w[5]);
            w[20] = cmul(w[10], w[10]);
#pragma unroll
            for (int a = 1; a < 5; a++)
                {
#pragma unroll
                    for (int b = 1; b < 5; b++) w[5 * a + b] = cmul(w[5 * a], w[b]);
                }
        }
    else
        {
#pragma unroll
            for (int q = 2; q < R; q++) w[q] = cmul(w[q - 1], w1);
        }
}

// Where a stage puts its outputs.  StoreSink writes them back in place (the normal case); the
// acquisition kernels pass a sink that consumes the natural-order outputs of the LAST inverse
// stage directly (|.|^2, max, sum) so the correlation row is never written anywhere.
struct StoreSink
{
    __device__ __forceinline__ void operator()(float2* p, int /*pos*/, float2 v) const { *p = v; }
};

// One DIF (forward) or DIT (inverse) stage over a buffer of n points in shared memory.
// M = current block length, R | M, m = M / R.  tw = this stage's compact table exp(-2 pi j k / M), k < m
// (contiguous, so a warp's twiddle loads are coalesced and the small late-stage tables stay in L1).
// sink(ptr, position, value) receives each output; position = index in the buffer.
template <int R, bool INV, class Sink>
__device__ __forceinline__ void fft_stage(float2* __restrict__ s, int n, int M, unsigned int magic, const float2* __restrict__ tw, Sink& sink)
{
    const int m = M / R;
    const int nb = n / R;
    // Butterfly i works on block b, offset j (pos0 = b M + j, elements pos0 + q m).  Consecutive threads normally take
    // consecutive j: conflict-free while m >= 16.  In the late forward / early inverse stages m is small (5 for the
    // M = 125 stage of 25 000 = 8 . 25 . 25 . 5) and consecutive threads would hop to the next block every m lanes, which
    // put 2-3 lanes on the same bank.  There the block
    // length M is odd (the planner runs the even radices first), so 16 consecutive BLOCKS at the same offset j hit 16
    // different bank pairs (M b mod 16 is a permutation): threads walk over b first.
    const bool by_block = (m < 16) && (M & 1) && (m > 1);
    const int nblk = by_block ? n / M : 1;
#pragma unroll(R >= 16 ? 1 : 2)
    for (int i = threadIdx.x; i < nb; i += blockDim.x)
        {
            int b, j;
            if (by_block)
                {
                    j = i / nblk;
                    b = i - j * nblk;
                }
            else
                {
                    b = fast_div(i, m, magic);
                    j = i - b * m;
                }
            const int pos0 = b * M + j;
            float2* p = s + pos0;
            float2 v[R];
#pragma unroll
            for (int q = 0; q < R; q++) v[q] = p[q * m];
            if (INV)
                {
                    if (m > 1)
                        {
                            const float2 w1 = __ldg(tw + j);
                            if (R == 25)
                                {
                                    float2 wp[R];
                                    twiddle_powers<R>(w1, wp);
#pragma unroll
                                    for (int q = 1; q < R; q++) v[q] = cmul_conj(v[q], wp[q]);
                                }
                            else
                                {
                                    float2 w = w1;
#pragma unroll
                                    for (int q = 1; q < R; q++)
                                        {
                                            v[q] = cmul_conj(v[q], w);
                                            if (q + 1 < R) w = cmul(w, w1);
                                        }
                                }
                        }
#pragma unroll
                    for (int q = 0; q < R; q++) v[q] = swap_ri(v[q]);
                    Bfly<R>::fwd(v);
#pragma unroll
                    for (int q = 0; q < R; q++) v[q] = swap_ri(v[q]);
                }
            else
                {
                    Bfly<R>::fwd(v);
                    if (m > 1)
                        {
                            const float2 w1 = __ldg(tw + j);
                            if (R == 25)
                                {
                                    float2 wp[R];
                                    twiddle_powers<R>(w1, wp);
#pragma unroll
                                    for (int q = 1; q < R; q++) v[q] = cmul(v[q], wp[q]);
                                }
                            else
                                {
                                    float2 w = w1;
#pragma unroll
                                    for (int q = 1; q < R; q++)
                                        {
                                            v[q] = cmul(v[q], w);
                                            if (q + 1 < R) w = cmul(w, w1);
                                        }
                                }
                        }
                }
#pragma unroll
            for (int q = 0; q < R; q++) sink(p + q * m, pos0 + q * m, v[q]);
        }
}

// Last forward (DIF) stage, block length R, no twiddles: shared memory -> global in the permuted storage order
// (see FftPlan::perm_r).  CONJ stores the conjugate (local-code spectrum, volk_32fc_conjugate_32fc).
template <int R, bool CONJ>
__device__ __forceinline__ void fft_last_fwd_stage_to_global(const float2* __restrict__ s, float2* __restrict__ out, int nb)
{
#pragma unroll 2
    for (int i = threadIdx.x; i < nb; i += blockDim.x)
        {
            float2 v[R];
#pragma unroll
            for (int q = 0; q < R; q++) v[q] = s[i * R + q];
            Bfly<R>::fwd(v);
#pragma unroll
            for (int q = 0; q < R; q++) out[q * nb + i] = CONJ ? make_float2(v[q].x, -v[q].y) : v[q];
        }
}

template <bool CONJ>
__device__ __forceinline__ void fft_last_fwd_stage_to_global_dispatch(int radix, const float2* s, float2* out, int nb)
{
    switch (radix)
        {
        case 2: fft_last_fwd_stage_to_global<2, CONJ>(s, out, nb); break;
        case 3: fft_last_fwd_stage_to_global<3, CONJ>(s, out, nb); break;
        case 4: fft_last_fwd_stage_to_global<4, CONJ>(s, out, nb); break;
        case 5: fft_last_fwd_stage_to_global<5, CONJ>(s, out, nb); break;
        case 7: fft_last_fwd_stage_to_global<7, CONJ>(s, out, nb); break;
        default: fft_last_fwd_stage_to_global<8, CONJ>(s, out, nb); break;
        }
}

// First inverse (DIT) stage, block length R, no twiddles: the point-wise product X . C
// (volk_32fc_x2_multiply_32fc, separately rounded like the element-wise kernel) is formed from the two
// permuted-order spectra in global memory and goes through the butterfly into shared memory.
template <int R>
__device__ __forceinline__ void fft_first_inv_stage_from_global(const float2* __restrict__ x, const float2* __restrict__ c,
    float2* __restrict__ s, int nb)
{
#pragma unroll 2
    for (int i = threadIdx.x; i < nb; i += blockDim.x)
        {
            float2 a[R], b[R], v[R];
#pragma unroll
            for (int q = 0; q < R; q++)
                {
                    a[q] = __ldg(x + q * nb + i);
                    b[q] = __ldg(c + q * nb + i);
                }
#pragma unroll
            for (int q = 0; q < R; q++) v[q] = swap_ri(cmul_rn(a[q], b[q]));  // inverse = swap . forward . swap
            Bfly<R>::fwd(v);
#pragma unroll
            for (int q = 0; q < R; q++) s[i * R + q] = swap_ri(v[q]);
        }
}

__device__ __forceinline__ void fft_first_inv_stage_from_global_dispatch(int radix, const float2* x, const float2* c, float2* s, int nb)
{
    switch (radix)
        {
        case 2: fft_first_inv_stage_from_global<2>(x, c, s, nb); break;
        case 3: fft_first_inv_stage_from_global<3>(x, c, s, nb); break;
        case 4: fft_first_inv_stage_from_global<4>(x, c, s, nb); break;
        case 5: fft_first_inv_stage_from_global<5>(x, c, s, nb); break;
        case 7: fft_first_inv_stage_from_global<7>(x, c, s, nb); break;
        default: fft_first_inv_stage_from_global<8>(x, c, s, nb); break;
        }
}

template <bool INV, class Sink, bool A25 = false>
__device__ __forceinline__ void fft_stage_dispatch(int radix, float2* s, int n, int M, unsigned int magic, const float2* tw, Sink& sink)
{
    if (A25)
        {
            if (radix == 25)
                {
                    fft_stage<A25 ? 25 : 5, INV>(s, n, M, magic, tw, sink);
                    return;
                }
        }
    switch (radix)
        {
        case 2: fft_stage<2, INV>(s, n, M, magic, tw, sink); break;
        case 3: fft_stage<3, INV>(s, n, M, magic, tw, sink); break;
        case 4: fft_stage<4, INV>(s, n, M, magic, tw, sink); break;
        case 5: fft_stage<5, INV>(s, n, M, magic, tw, sink); break;
        case 7: fft_stage<7, INV>(s, n, M, magic, tw, sink); break;
        default: fft_stage<8, INV>(s, n, M, magic, tw, sink); break;
        }
}

// forward DIF, spectrum written to global memory in the plan's storage order: all stages in shared memory and
// a copy when perm_r == 1, else the last stage streams straight to global.  CONJ: store the conjugate.
template <bool CONJ, bool A25 = false>
__device__ __forceinline__ void fft_forward_to_global(float2* s, const FftPlan& pl, const float2* tw, float2* __restrict__ out)
{
    StoreSink st_sink;
    int M = pl.n;
    const int n_smem_stages = (pl.perm_r > 1) ? pl.n_stages - 1 : pl.n_stages;
    for (int st = 0; st < n_smem_stages; st++)
        {
            __syncthreads();
            fft_stage_dispatch<false, StoreSink, A25>(pl.radix[st], s, pl.n, M, pl.mdiv[st], tw + pl.tw_off[st], st_sink);
            M /= pl.radix[st];
        }
    __syncthreads();
    if (pl.perm_r > 1)
        {
            fft_last_fwd_stage_to_global_dispatch<CONJ>(pl.perm_r, s, out, pl.perm_nb);
        }
    else
        {
            for (int i = threadIdx.x; i < pl.n; i += blockDim.x) out[i] = CONJ ? make_float2(s[i].x, -s[i].y) : s[i];
        }
}

// forward DIF over all stages: natural order in, digit-reversed out
__device__ __forceinline__ void fft_forward_smem(float2* s, const FftPlan& pl, const float2* tw)
{
    StoreSink st_sink;
    int M = pl.n;
    for (int st = 0; st < pl.n_stages; st++)
        {
            __syncthreads();
            fft_stage_dispatch<false>(pl.radix[st], s, pl.n, M, pl.mdiv[st], tw + pl.tw_off[st], st_sink);
            M /= pl.radix[st];
        }
    __syncthreads();
}

// inverse DIT over stages n_stages-1 .. 1 in place, then stage 0 (block length n, natural-order
// outputs) through `last`: digit-reversed in, natural out.
template <class Sink>
__device__ __forceinline__ void fft_inverse_smem(float2* s, const FftPlan& pl, const float2* tw, Sink& last)
{
    StoreSink st_sink;
    int M = 1;
    for (int st = pl.n_stages - 1; st >= 1; st--)
        {
            M *= pl.radix[st];
            __syncthreads();
            fft_stage_dispatch<true>(pl.radix[st], s, pl.n, M, pl.mdiv[st], tw + pl.tw_off[st], st_sink);
        }
    __syncthreads();
    fft_stage_dispatch<true>(pl.radix[0], s, pl.n, pl.n, pl.mdiv[0], tw + pl.tw_off[0], last);
}


// inverse DIT of the product of two spectra held in global memory in the plan's storage order (perm_r > 1):
// first stage from global, stages n_stages-2 .. 1 in place, stage 0 through `last`.
template <bool A25, class Sink>
__device__ __forceinline__ void fft_inverse_from_global(const float2* x, const float2* c, float2* s, const FftPlan& pl, const float2* tw, Sink& last)
{
    StoreSink st_sink;
    fft_first_inv_stage_from_global_dispatch(pl.perm_r, x, c, s, pl.perm_nb);
    int M = pl.perm_r;
    for (int st = pl.n_stages - 2; st >= 1; st--)
        {
            M *= pl.radix[st];
            __syncthreads();
            fft_stage_dispatch<true, StoreSink, A25>(pl.radix[st], s, pl.n, M, pl.mdiv[st], tw + pl.tw_off[st], st_sink);
        }
    __syncthreads();
    fft_stage_dispatch<true, Sink, A25>(pl.radix[0], s, pl.n, pl.n, pl.mdiv[0], tw + pl.tw_off[0], last);
}

// inverse DIT over all stages in place (two-level path: natural order within the block afterwards)
__device__ __forceinline__ void fft_inverse_smem_inplace(float2* s, const FftPlan& pl, const float2* tw)
{
    StoreSink st_sink;
    int M = 1;
    for (int st = pl.n_stages - 1; st >= 0; st--)
        {
            M *= pl.radix[st];
            __syncthreads();
            fft_stage_dispatch<true>(pl.radix[st], s, pl.n, M, pl.mdiv[st], tw + pl.tw_off[st], st_sink);
        }
    __syncthreads();
}

}  // namespace b200
