// Per-item correlation of the multi-tap tracking correlator (device templates shared by the batch kernel in
// trk_kernels.cu and the persistent free-running kernel in loop_kernels_nofma.cu).  See trk_kernels.cu for the
// mapping to the reference's volk_gnsssdr kernels.  Every floating-point contraction in here is written
// explicitly (fmaf / __fmul_rn / __fadd_rn and the float2 helpers of trk_device.cuh), so the arithmetic does not depend on the
// translation unit's --fmad setting; tests/test_loop_gpu.py checks the two instantiations bit for bit.
#pragma once

#include "common.cuh"
#include "trk_device.cuh"

namespace b200
{
namespace
{
// tiles of the main loop unrolled per thread (one 16-byte load each on a float band): memory-level parallelism vs registers.  With five taps
// (C3, Galileo E1) and one tap (the data correlator of a tracked pilot) the kernel waits on L2, so 16 = a whole re-seed group
// of loads in flight; three taps (C2) take 4.  On an H100 (400 W), ms per step, these values vs 8: five taps C3 5.52 vs 5.94;
// three taps C2 distinct-IQ 1.165 vs 1.178; one tap C3 + pilot 8.93-8.98 vs 8.84 (within the spread of repeated runs of one
// build).
constexpr int kTileUnroll3 = 4;
constexpr int kTileUnroll5 = 16;
constexpr int kTileUnroll1 = 16;   // one tap: the data prompt of a tracked pilot

struct ItemCtx
{
    const void* base;       // the band's samples (sample_ptr)
    unsigned long long mask;
    unsigned long long s0;  // offset of the epoch's first sample in the band
    unsigned long long T0;  // -rem_carrier in turns
    unsigned long long DT;  // -phase_step in turns
    float step, rem;
    int N, body;            // body = 8*(N/8): samples using the AVX association
};

// Code lookup policies -----------------------------------------------------------------------
// FAST: extended table in smem covering [tbl_base, tbl_base+span): no modulo in the loop.
struct LookupExt
{
    const float* tb;  // smem_table - tbl_base
    __device__ __forceinline__ float operator()(int idx) const { return tb[idx]; }
};
// GENERAL: any index range (multi-period epochs, pathological parameters): integer modulo,
// table in smem when it fits, else global.
struct LookupMod
{
    const float* tbl;
    int L;
    __device__ __forceinline__ float operator()(int idx) const { return tbl[mod_pos(idx, L)]; }
};

template <int TAPS, class Lookup>
__device__ __forceinline__ void accumulate_sample(float2 x, float2 z, float m, const float (&aux2)[TAPS],
    const Lookup& lut, float2 (&acc)[TAPS])
{
    const float wr = fmaf(x.x, z.x, -x.y * z.y);
    const float wi = fmaf(x.x, z.y, x.y * z.x);
#pragma unroll
    for (int t = 0; t < TAPS; t++)
        {
            const int idx = __float2int_rd(__fadd_rn(m, aux2[t]));
            const float c = lut(idx);
            acc[t].x = fmaf(wr, c, acc[t].x);
            acc[t].y = fmaf(wi, c, acc[t].y);
        }
}

template <int TAPS, class Lookup, int THREADS = kTrkThreads, int FMT = kCf32>
__device__ __forceinline__ void correlate_range(const ItemCtx& cx, const float (&shifts)[TAPS], const Lookup& lut,
    int tile_begin, int tile_end, int head, bool do_remainder, int n_main_end, float2 (&acc)[TAPS])
{
    constexpr int kTile = 2 * THREADS;  // samples per CTA iteration (one LDG.128 per thread)
    const int tid = threadIdx.x;
    float aux2[TAPS];
#pragma unroll
    for (int t = 0; t < TAPS; t++) aux2[t] = __fsub_rn(shifts[t], cx.rem);

    // ---- main tiles: all samples < body, 16-byte aligned pairs -------------------------------
    const float2 D = phasor_from_turns(cx.DT * static_cast<unsigned long long>(kTile));
    for (int tg = tile_begin; tg < tile_end; tg += kTrkReseed)
        {
            const int tg_end = min(tg + kTrkReseed, tile_end);
            int n0 = head + tg * kTile + 2 * tid;
            float2 za = phasor_from_turns(cx.T0 + cx.DT * static_cast<unsigned long long>(n0));
            float2 zb = phasor_from_turns(cx.T0 + cx.DT * static_cast<unsigned long long>(n0 + 1));
            float nf = static_cast<float>(n0);
#pragma unroll 4
            for (int tile = tg; tile < tg_end; tile++)
                {
                    const float4 v = ldg_stream_pair<FMT>(sample_ptr<FMT>(cx.base, (cx.s0 + static_cast<unsigned long long>(n0)) & cx.mask));
                    accumulate_sample<TAPS>(make_float2(v.x, v.y), za, __fmul_rn(cx.step, nf), aux2, lut, acc);
                    accumulate_sample<TAPS>(make_float2(v.z, v.w), zb, __fmul_rn(cx.step, nf + 1.0f), aux2, lut, acc);
                    za = cmulf(za, D);
                    zb = cmulf(zb, D);
                    n0 += kTile;
                    nf += static_cast<float>(kTile);
                }
        }

    // ---- remainder: optional head sample 0 and everything from n_main_end to N ------------------
    if (do_remainder)
        {
            const int count = head + (cx.N - n_main_end);
            for (int r = tid; r < count; r += THREADS)
                {
                    const int n = (r < head) ? 0 : n_main_end + (r - head);
                    const float2 x = ldg_stream_one<FMT>(sample_ptr<FMT>(cx.base, (cx.s0 + static_cast<unsigned long long>(n)) & cx.mask));
                    const float2 z = phasor_from_turns(cx.T0 + cx.DT * static_cast<unsigned long long>(n));
                    const float wr = fmaf(x.x, z.x, -x.y * z.y);
                    const float wi = fmaf(x.x, z.y, x.y * z.x);
#pragma unroll
                    for (int t = 0; t < TAPS; t++)
                        {
                            const float c = lut(chip_index_at(cx.step, n, cx.body, shifts[t], cx.rem));
                            acc[t].x = fmaf(wr, c, acc[t].x);
                            acc[t].y = fmaf(wi, c, acc[t].y);
                        }
                }
        }
}


// ---- main tiles, FAST path: arithmetic on sample pairs, no modulo, no F2I -----------------------------
// Lane .x of every float2 value belongs to sample n0, lane .y to sample n0+1 (one LDG.128).  The chip lookup is pair_taps'
// floor trick (exact for |index| < 2^22, guaranteed by the caller's range check); tbl_off = table_offset().
template <int TAPS, bool WRAPS, int THREADS = kTrkThreads, int FMT = kCf32>
__device__ __forceinline__ void correlate_tiles_fast(const ItemCtx& cx, const float (&shifts)[TAPS], unsigned int tbl_off,
    int tile_begin, int tile_end, int head, float2 (&acc)[TAPS])
{
    constexpr int kTile = 2 * THREADS;  // samples per CTA iteration (one LDG.128 per thread)
    const int tid = threadIdx.x;
    float2 aux2[TAPS];
#pragma unroll
    for (int t = 0; t < TAPS; t++)
        {
            const float a = __fsub_rn(shifts[t], cx.rem);
            aux2[t] = make_float2(a, a);
        }
    float2 are[TAPS], aim[TAPS];
#pragma unroll
    for (int t = 0; t < TAPS; t++) are[t] = aim[t] = make_float2(0.f, 0.f);

    const float2 D = phasor_from_turns(cx.DT * static_cast<unsigned long long>(kTile));
    const float2 Dr2 = make_float2(D.x, D.x), Di2 = make_float2(D.y, D.y);
    // group-to-group phasor step: kTrkReseed tiles
    const float2 G = phasor_from_turns(cx.DT * static_cast<unsigned long long>(kTile * kTrkReseed));
    const float2 Gr2 = make_float2(G.x, G.x), Gi2 = make_float2(G.y, G.y);

    int n0 = head + tile_begin * kTile + 2 * tid;
    float2 zr2, zi2;   // phasors of the two samples at the start of the current group
    {
        const float2 za = phasor_from_turns(cx.T0 + cx.DT * static_cast<unsigned long long>(n0));
        const float2 zb = phasor_from_turns(cx.T0 + cx.DT * static_cast<unsigned long long>(n0 + 1));
        zr2 = make_float2(za.x, zb.x);
        zi2 = make_float2(za.y, zb.y);
    }
    float nfa = static_cast<float>(n0), nfb = static_cast<float>(n0 + 1);
    const char* ptr = sample_ptr<FMT>(cx.base, (cx.s0 + static_cast<unsigned long long>(n0)) & cx.mask);

    for (int tg = tile_begin; tg < tile_end; tg += kTrkReseed)
        {
            const int tg_end = min(tg + kTrkReseed, tile_end);
            float2 zr = zr2, zi = zi2;   // running phasors inside the group
#pragma unroll (TAPS >= 4 ? kTileUnroll5 : (TAPS == 1 ? kTileUnroll1 : kTileUnroll3))
            for (int tile = tg; tile < tg_end; tile++)
                {
                    float4 v;
                    if (WRAPS)
                        v = ldg_stream_pair<FMT>(sample_ptr<FMT>(cx.base, (cx.s0 + static_cast<unsigned long long>(n0)) & cx.mask));
                    else
                        v = ldg_stream_pair<FMT>(ptr);
                    // w = x * z, scalar: the LDG.128 delivers (re,im,re,im), so packed operands would
                    // need 8 register moves per tile; scalar results land directly in register pairs
                    float2 wr2, wi2;
                    wr2.x = fmaf(v.x, zr.x, -v.y * zi.x);
                    wi2.x = fmaf(v.x, zi.x, v.y * zr.x);
                    wr2.y = fmaf(v.z, zr.y, -v.w * zi.y);
                    wi2.y = fmaf(v.z, zi.y, v.w * zr.y);
                    const float2 m2 = make_float2(__fmul_rn(cx.step, nfa), __fmul_rn(cx.step, nfb));
                    pair_taps<TAPS>(m2, aux2, tbl_off, wr2, wi2, are, aim);
                    advance_pair(zr, zi, Dr2, Di2);
                    nfa += static_cast<float>(kTile);
                    nfb += static_cast<float>(kTile);
                    n0 += kTile;
                    ptr += kTile * 2 * FMT;
                }
            // group seed advances by the rounded G, not re-seeded from the 64-bit phase: its error grows by about 1e-7
            // per group (8192 samples); see the measured bound in trk_kernels.cu
            advance_pair(zr2, zi2, Gr2, Gi2);
        }
#pragma unroll
    for (int t = 0; t < TAPS; t++)
        {
            acc[t].x += are[t].x + are[t].y;
            acc[t].y += aim[t].x + aim[t].y;
        }
}

// High-dynamics variant (a4): quadratic code phase on tap 0, other taps are circular
// integer-sample shifts of tap 0's resampled sequence; carrier has a phase-rate term that lags
// one sample (..._high_dynamic_rotator_dot_prod_32fc_xn.h:92-103).  Not the throughput path:
// one sample per thread per step, exact phasor per sample.
template <int TAPS, class Lookup, int THREADS = kTrkThreads, int FMT = kCf32>
__device__ __forceinline__ void correlate_range_hd(const ItemCtx& cx, float rate, unsigned long long RT,
    const float (&shifts)[TAPS], const Lookup& lut, int n_begin, int n_end, float2 (&acc)[TAPS])
{
    int shift_samples[TAPS];
    shift_samples[0] = 0;
    unsigned int ss = 0;
#pragma unroll
    for (int t = 1; t < TAPS; t++)
        {
            // (int)round((shifts[t]-shifts[t-1])/step) in double like C's round() on a float expr
            ss += static_cast<unsigned int>(static_cast<int>(round(static_cast<double>(__fdiv_rn(__fsub_rn(shifts[t], shifts[t - 1]), cx.step)))));
            shift_samples[t] = static_cast<int>(ss);
        }
    for (int n = n_begin + threadIdx.x; n < n_end; n += THREADS)
        {
            const float2 x = ldg_stream_one<FMT>(sample_ptr<FMT>(cx.base, (cx.s0 + static_cast<unsigned long long>(n)) & cx.mask));
            // rate exponent: (n-1)^2 for n>=1 with the reference's uint32 wrap of k*k, as float
            unsigned long long T = cx.T0 + cx.DT * static_cast<unsigned long long>(n);
            if (n >= 1)
                {
                    const unsigned int k = static_cast<unsigned int>(n - 1);
                    const float e = static_cast<float>(k * k);
                    // RT is the per-unit rate in turns; e is an integer-valued float < 2^32
                    T += RT * static_cast<unsigned long long>(e);
                }
            const float2 z = phasor_from_turns(T);
            const float wr = fmaf(x.x, z.x, -x.y * z.y);
            const float wi = fmaf(x.x, z.y, x.y * z.x);
#pragma unroll
            for (int t = 0; t < TAPS; t++)
                {
                    unsigned int m = static_cast<unsigned int>(n) + static_cast<unsigned int>(shift_samples[t]);
                    if (m >= static_cast<unsigned int>(cx.N)) m -= static_cast<unsigned int>(cx.N);
                    // samples below 8*(N/8) follow the AVX kernel's association, the tail the generic one
                    const int idx = (m < static_cast<unsigned int>(cx.body))
                                        ? chip_index_hd_avx(cx.step, rate, static_cast<float>(m), __fsub_rn(shifts[0], cx.rem))
                                        : chip_index_hd(cx.step, rate, m, shifts[0], cx.rem);
                    const float c = lut(idx);
                    acc[t].x = fmaf(wr, c, acc[t].x);
                    acc[t].y = fmaf(wi, c, acc[t].y);
                }
        }
}

// REUSE (persistent tracker: one CTA keeps serving the same channel): tbl_cache[0..1] = [begin, end) of the chip-index
// window already staged in smem_tbl; an epoch whose window lies inside it skips the staging pass.
// FMT: the SampleFormat of bd (the caller's to check); every path widens each sample to float right after its load and then
// runs the same arithmetic, so a narrow band gives exactly the taps of a float band holding the same integers.
template <int TAPS, bool REUSE = false, int THREADS = kTrkThreads, int FMT = kCf32>
__device__ void process_item(const b200_trk_item& it, const ChanDesc& ch, const BandDesc& bd, float* smem_tbl,
    int tbl_cap, float2* smem_red, int slice, int slices, float2 (&result)[TAPS], int* tbl_cache = nullptr)
{
    constexpr int kTile = 2 * THREADS;  // samples per CTA iteration (one LDG.128 per thread)
    const int tid = threadIdx.x;
    const ItemPhase ph = item_phase(it.rem_carrier_phase_rad, it.phase_step_rad, it.n);
    ItemCtx cx;
    cx.base = bd.base;
    cx.mask = bd.mask;
    cx.s0 = it.sample_index - bd.first_index;
    cx.N = it.n;
    cx.body = ph.body;
    cx.step = it.code_phase_step_chips;
    cx.rem = it.rem_code_phase_chips;
    cx.T0 = ph.T0;
    cx.DT = ph.DT;
    const int L = ch.code_len;

    float shifts[TAPS];
#pragma unroll
    for (int t = 0; t < TAPS; t++) shifts[t] = ch.shifts[t];

    float2 acc[TAPS];
#pragma unroll
    for (int t = 0; t < TAPS; t++) acc[t] = make_float2(0.f, 0.f);

    if (ch.high_dyn)
        {
            // table of exactly L entries (smem if it fits), modulo lookup
            const bool in_smem = L <= tbl_cap;
            if (in_smem)
                {
                    stage_code_window(ch.code, L, 0, L, tid, THREADS, [&](int j, const float* src) { smem_tbl[j] = *src; });
                }
            __syncthreads();
            LookupMod lut{in_smem ? smem_tbl : ch.code, L};
            const unsigned long long RT = turns_from_rad(-static_cast<double>(it.phase_rate_step_rad));
            const int per = (cx.N + slices - 1) / slices;
            const int nb = min(cx.N, slice * per), ne = min(cx.N, nb + per);
            correlate_range_hd<TAPS, LookupMod, THREADS, FMT>(cx, it.code_phase_rate_step_chips, RT, shifts, lut, nb, ne, acc);
        }
    else
        {
            // index range over the epoch (monotone in n within each association): the AVX association's ends, plus the
            // generic association's at body, N-1 and 0 (epochs shorter than 8 samples)
            int lo, hi;
            chip_range<TAPS>(cx.step, 0.f, static_cast<float>(max(cx.body - 1, 0)), [&](int t) { return __fsub_rn(shifts[t], cx.rem); }, lo, hi);
            const float n_last = static_cast<float>(max(cx.N - 1, 0));
            const float n_body = static_cast<float>(cx.body);
#pragma unroll
            for (int t = 0; t < TAPS; t++)
                {
                    const int g0 = chip_index_generic(cx.step, n_body, shifts[t], cx.rem);
                    const int g1 = chip_index_generic(cx.step, n_last, shifts[t], cx.rem);
                    const int g2 = chip_index_generic(cx.step, 0.f, shifts[t], cx.rem);
                    lo = min(lo, min(g0, min(g1, g2)));
                    hi = max(hi, max(g0, max(g1, g2)));
                }
            const long long tbl_base = static_cast<long long>(lo) - 2;
            const long long span = static_cast<long long>(hi) - lo + 5;

            const int head = static_cast<int>(cx.s0 & 1ULL);
            const int ntiles = (cx.body > head) ? (cx.body - head) / kTile : 0;
            const int n_main_end = head + ntiles * kTile;
            const int tb = static_cast<int>((static_cast<long long>(ntiles) * slice) / slices);
            const int te = static_cast<int>((static_cast<long long>(ntiles) * (slice + 1)) / slices);
            const bool rem_here = (slice == slices - 1);

            if (span <= static_cast<long long>(tbl_cap))
                {
                    int base_i = static_cast<int>(tbl_base);
                    int span_st = static_cast<int>(span);
                    bool stage = true;
                    if (REUSE)
                        {
                            const int cb = tbl_cache[0], ce = tbl_cache[1];
                            if (ce > cb && base_i >= cb && base_i + span_st <= ce)
                                {
                                    stage = false;
                                    base_i = cb;
                                }
                            else
                                {
                                    // a little wider than needed: the window drifts by a chip or two per epoch
                                    int margin = (tbl_cap - span_st) / 2;
                                    margin = margin > 8 ? 8 : (margin < 0 ? 0 : margin);
                                    base_i -= margin;
                                    span_st += 2 * margin;
                                }
                        }
                    if (stage) stage_code_window(ch.code, L, base_i, span_st, tid, THREADS, [&](int j, const float* src) { smem_tbl[j] = *src; });
                    __syncthreads();
                    if (REUSE && stage && tid == 0)
                        {
                            tbl_cache[0] = base_i;
                            tbl_cache[1] = base_i + span_st;
                        }
                    LookupExt lut{smem_tbl - base_i};
                    if (lo > -4000000 && hi < 4000000)
                        {
                            const unsigned int tbl_off = table_offset(smem_tbl, base_i);
                            // ring wrap inside the epoch? (uniform per item)
                            const bool wraps = ((cx.s0 & cx.mask) + static_cast<unsigned long long>(cx.N)) > cx.mask;
                            if (wraps)
                                correlate_tiles_fast<TAPS, true, THREADS, FMT>(cx, shifts, tbl_off, tb, te, head, acc);
                            else
                                correlate_tiles_fast<TAPS, false, THREADS, FMT>(cx, shifts, tbl_off, tb, te, head, acc);
                            // remainder samples only (no main tiles) through the scalar path
                            correlate_range<TAPS, LookupExt, THREADS, FMT>(cx, shifts, lut, 0, 0, head, rem_here, n_main_end, acc);
                        }
                    else
                        {
                            correlate_range<TAPS, LookupExt, THREADS, FMT>(cx, shifts, lut, tb, te, head, rem_here, n_main_end, acc);
                        }
                }
            else
                {
                    const bool in_smem = L <= tbl_cap;
                    if (REUSE && tid == 0) tbl_cache[1] = tbl_cache[0];  // smem_tbl no longer holds an extended window
                    if (in_smem)
                        {
                            stage_code_window(ch.code, L, 0, L, tid, THREADS, [&](int j, const float* src) { smem_tbl[j] = *src; });
                        }
                    __syncthreads();
                    LookupMod lut{in_smem ? smem_tbl : ch.code, L};
                    correlate_range<TAPS, LookupMod, THREADS, FMT>(cx, shifts, lut, tb, te, head, rem_here, n_main_end, acc);
                }
        }

    // ---- CTA reduction: shuffles, then 8 warp partials through shared memory -------------------
#pragma unroll
    for (int t = 0; t < TAPS; t++) acc[t] = warp_sum(acc[t]);
    const int warp = tid >> 5, lane = tid & 31;
    if (lane == 0)
        {
#pragma unroll
            for (int t = 0; t < TAPS; t++) smem_red[warp * B200_MAX_TAPS + t] = acc[t];
        }
    __syncthreads();
#pragma unroll
    for (int t = 0; t < TAPS; t++)
        {
            float2 s = make_float2(0.f, 0.f);
#pragma unroll
            for (int w = 0; w < THREADS / 32; w++)
                {
                    const float2 p = smem_red[w * B200_MAX_TAPS + t];
                    s.x += p.x;
                    s.y += p.y;
                }
            result[t] = s;
        }
}

}  // namespace
}  // namespace b200
