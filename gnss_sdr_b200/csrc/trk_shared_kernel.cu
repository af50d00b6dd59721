// Tracking correlator, "shared window" kernel for sm_90a.
//
// Why: the per-item kernel (trk_kernels.cu) re-reads every IQ sample from L2 once per channel.  With
// 32 channels on one band that is 6.4 GB through the L2->SM crossbar per second of signal, and the
// crossbar becomes the bound.  Channels that are
// in lock on the same band correlate the SAME samples, so here one CTA serves a GROUP of up to 8 work
// items (one consumer warp each) from one copy of the samples:
//
//   producer warp   cp.async.bulk (TMA bulk copy, UBLKCP) of 512-sample tiles of the band store into a
//                   4-stage shared-memory ring (8 padded runs per tile), completion signalled on mbarriers
//                   (expect_tx bytes);
//   8 consumer warps each owns one (channel, epoch) item of the group: waits for the tile, reads its
//                   samples with conflict-free LDS.128, correlates them against a warp-private shared-memory
//                   code table, releases the tile.  warp_tile looks every tap's chip up per sample;
//                   warp_tile_chunks (C/A-like steps) splits 16-sample chunks at their one exact chip
//                   boundary per tap and multiplies two chip values into chunk sums kept in registers.
//
// Both use the chip-index float sequence and the 64-bit fixed-point carrier phase of trk_kernels.cu, so
// indices are bit-exact and results follow the same contract.  Items of a group need
// not start at the same sample: the tile range is the hull of the group and a warp only works on
// tiles that intersect its own epoch (masked at the ends).  Group membership is the caller's item
// ORDER (items 8g .. 8g+7); the host API sorts by start sample, bench.py's epoch-major order already
// has that shape.
#include "trk_device.cuh"

namespace b200
{
constexpr int kShK = 8;          // items (consumer warps) per CTA
constexpr int kShTile = 512;     // samples per tile (4 KB)
#ifndef SH_STAGES
#define SH_STAGES 4
#endif
constexpr int kShStages = SH_STAGES;
// Minimum resident CTAs per SM (__launch_bounds__).  sm_90a, 288 threads: 3 caps the kernel at 72 registers and spills
// (<3>: 166 B stores / 248 B loads), 2 gives 96 registers (<3>: 8 B / 8 B), 1 no spills at 127-152.  On an H100 (400 W), ms
// per C2 step: 2 -> 0.969-0.970, 3 -> 1.051-1.058, 1 -> 1.189-1.191, 4 -> 1.179; distinct-IQ through this kernel 1.237 at 2,
// 1.393 at 3.  Since the chunk path keeps its running sums in registers, a CTA takes about 54 KB of shared memory and three
// fit again; at 3 the kernel is capped at 72 registers and <3> spills 134 B / 268 B.  On an H100 80GB HBM3 (700 W, 1980 MHz),
// ms per C2 step, two runs each: 2 -> 0.6946-0.6950, 3 -> 0.6988-0.6989.
constexpr int kShMinBlocks = 2;
// SH_STRESS (test builds only, tests/test_ring_stress_gpu.py): pseudo-random delays in the producer and in every consumer
// warp, before the tile is read and before the slot is released, so that warps drift apart by several tiles and every
// full/empty hand-over of the TMA ring is exercised with 2, 4 and 8 stages.
#ifndef SH_STRESS
#define SH_STRESS 0
#endif
#if SH_STRESS
__device__ __forceinline__ void stress_delay(unsigned int salt)
{
    unsigned int h = salt * 2654435761u;
    h ^= h >> 15;
    h *= 2246822519u;
    h ^= h >> 13;
    if ((h & 3u) == 0u) __nanosleep(100u + ((h >> 4) & 1023u));
}
#endif
constexpr int kShTblCap = 1152;  // floats of warp-private code storage: whole-epoch table when it fits ...
constexpr int kShWin = 256;      // ... else two 256-entry windows (double-buffered, refilled per tile with cp.async)
constexpr int kShThreads = (kShK + 1) * 32;
constexpr int kShReseed = 64;    // 64-sample steps between exact phasor re-seeds (4096 samples)
constexpr int kShReseedTiles = kShReseed / (kShTile / 64);  // ... that is, tiles
static_assert((kShReseedTiles & (kShReseedTiles - 1)) == 0, "the chunk path tests the re-seed tile with a mask");
// Tiles sit in shared memory as 8 runs of 64 samples (4 chunks of 16), each run followed by 16 bytes of padding: 528-byte
// run stride, one bulk copy per run.  On the chunk path lane l owns chunk 4 (l % 8) + l / 8, so the 8 lanes of a quarter
// warp read 8 different runs, whose starts fall on 8 distinct 16-byte bank groups: LDS.128 without conflicts.
constexpr int kShChunk = 16;
constexpr int kShRun = 4 * kShChunk;          // samples per bulk copy
constexpr int kShRunStride = kShRun + 2;      // float2 per run slot
constexpr int kShTileSlot = kShTile / kShRun * kShRunStride;
__device__ __forceinline__ int lane_chunk(int lane) { return 4 * (lane & 7) + (lane >> 3); }

namespace
{
struct __align__(128) ShSmem
{
    float2 tiles[kShStages][kShTileSlot];
    float tbl[kShK][kShTblCap];
    float2 rot[kShK][kShChunk];                // chunk path: D^j, j = 0..15, D = the item's per-sample phasor
    unsigned long long full[kShStages];
    unsigned long long empty[kShStages];
    unsigned long long item_start[kShK];  // offset of the item's first sample in the band (band-relative)
    unsigned long long item_turns[kShK][2];  // the item's T0 and DT (item_phase()), read back after the set-up
    int item_n[kShK];
    int item_band[kShK];
    unsigned long long hull_start;
    int n_tiles;
    int share;
};

__device__ __forceinline__ unsigned int smem_u32(const void* p) { return static_cast<unsigned int>(__cvta_generic_to_shared(p)); }

__device__ __forceinline__ void mbar_init(unsigned long long* bar, unsigned int count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(unsigned long long* bar)
{
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(unsigned long long* bar, unsigned int bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, unsigned int parity)
{
    asm volatile(
        "{\n\t"
        ".reg .pred P1;\n\t"
        "LAB_WAIT:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1, %2;\n\t"
        "@P1 bra DONE;\n\t"
        "bra LAB_WAIT;\n\t"
        "DONE:\n\t"
        "}" ::"r"(smem_u32(bar)),
        "r"(parity), "r"(0x989680u)  // suspend-time hint: the warp sleeps in hardware instead of spinning
        : "memory");
}
// Where tile t sits in the ring: slot t % kShStages, whose barriers are in phase (t / kShStages) & 1.  The chunk path
// carries it from tile to tile (next) instead of recomputing it.
struct RingPos
{
    int s;
    unsigned int par;
    static __device__ __forceinline__ RingPos of(int t) { return {t % kShStages, static_cast<unsigned int>((t / kShStages) & 1)}; }
    __device__ __forceinline__ void next()
    {
        if (++s == kShStages)
            {
                s = 0;
                par ^= 1u;
            }
    }
};
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gmem_src, unsigned int bytes, unsigned long long* bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)),
                 "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

// Correct-for-anything fallback for one warp: direct global loads, exact phasor per sample, integer
// modulo lookup in the global code table.  Used when an item cannot take the table path.
// T0, DT, body: the item's item_phase().
template <int TAPS>
__device__ void warp_correlate_general(const b200_trk_item& it, const ChanDesc& ch, const BandDesc& bd, unsigned long long T0,
    unsigned long long DT, int body, float2 (&acc)[TAPS])
{
    const int lane = threadIdx.x & 31;
    const unsigned long long s0 = it.sample_index - bd.first_index;
    for (int n = lane; n < it.n; n += 32)
        {
            const float2 x = ldg_stream8(static_cast<const float2*>(bd.base) + ((s0 + static_cast<unsigned long long>(n)) & bd.mask));
            const float2 z = phasor_from_turns(T0 + DT * static_cast<unsigned long long>(n));
            const float wr = fmaf(x.x, z.x, -x.y * z.y);
            const float wi = fmaf(x.x, z.y, x.y * z.x);
#pragma unroll
            for (int t = 0; t < TAPS; t++)
                {
                    const int idx = chip_index_at(it.code_phase_step_chips, n, body, ch.shifts[t], it.rem_code_phase_chips);
                    const float c = ch.code[mod_pos(idx, ch.code_len)];
                    acc[t].x = fmaf(wr, c, acc[t].x);
                    acc[t].y = fmaf(wi, c, acc[t].y);
                }
        }
}

// One tile (512 samples in shared memory) for one warp: 8 steps of 64 samples, lane l takes the pair
// (2l, 2l+1) of every step.  fa/fb (sample index within the epoch, as floats) and the running phasors
// are lane state that continues seamlessly from tile to tile (tiles are contiguous).
// MASKED = the tile sticks out of [0, body): samples outside contribute zero and evaluate the chip
// index of the nearest sample inside (always within the code window).
// where a warp gets the tile's samples from: the CTA's shared ring (normal case) ...
struct SmemTileLoader
{
    const float4* p;  // tile + lane: sample pair lane + 32 k is pair `lane` of run k
    __device__ __forceinline__ float4 operator()(int k) const { return p[(kShRunStride / 2) * k]; }
};
// ... or straight from the band store, when the group's items cannot share a window (different bands,
// epochs far apart): same arithmetic, the samples just come through L2 per item as in trk_kernels.cu.
struct GlobalTileLoader
{
    const float2* base;
    unsigned long long mask, off, limit;  // off = band offset of the tile's first sample + 2*lane (even)
    __device__ __forceinline__ float4 operator()(int k) const
    {
        const unsigned long long o = off + 64ULL * static_cast<unsigned long long>(k);
        if (mask == ~0ULL && o + 2ULL > limit) return make_float4(0.f, 0.f, 0.f, 0.f);  // linear band: stay inside
        return ldg_stream16(base + (o & mask));
    }
};

template <int TAPS, bool MASKED, class Loader>
__device__ __forceinline__ void warp_tile(const Loader& load, float vlo, float vhi, float step, const float2 (&aux2)[TAPS],
    unsigned int tbl_off, float2 Dr2, float2 Di2, float& fa, float& fb, float2& zr, float2& zi, float2 (&are)[TAPS], float2 (&aim)[TAPS])
{
#pragma unroll
    for (int k = 0; k < kShTile / 64; k++)
        {
            const float4 v = load(k);
            float ua = fa, ub = fb;
            float2 xa = make_float2(v.x, v.y), xb = make_float2(v.z, v.w);
            if (MASKED)
                {
                    // [vlo, vhi] = the tile's samples that belong to the epoch (indices are exact in float);
                    // the others contribute zero and look the chip of the nearest valid sample up
                    if (fa < vlo || fa > vhi) xa = make_float2(0.f, 0.f);
                    if (fb < vlo || fb > vhi) xb = make_float2(0.f, 0.f);
                    ua = fminf(fmaxf(fa, vlo), vhi);
                    ub = fminf(fmaxf(fb, vlo), vhi);
                }
            float2 wr2, wi2;
            wr2.x = fmaf(xa.x, zr.x, -xa.y * zi.x);
            wi2.x = fmaf(xa.x, zi.x, xa.y * zr.x);
            wr2.y = fmaf(xb.x, zr.y, -xb.y * zi.y);
            wi2.y = fmaf(xb.x, zi.y, xb.y * zr.y);
            const float2 m2 = make_float2(__fmul_rn(step, ua), __fmul_rn(step, ub));
            pair_taps<TAPS>(m2, aux2, tbl_off, wr2, wi2, are, aim);
            advance_pair(zr, zi, Dr2, Di2);
            fa += 64.0f;
            fb += 64.0f;
        }
}

// R[m] for a lane-dependent m in [0, 15] without indexing registers (which would put R in local memory): a 4-level tree
// of selects on the bits of m.
__device__ __forceinline__ float2 select16(const float2 (&R)[kShChunk], int m)
{
    float2 a[8], b[4], c[2];
#pragma unroll
    for (int i = 0; i < 8; i++) a[i] = (m & 1) ? R[2 * i + 1] : R[2 * i];
#pragma unroll
    for (int i = 0; i < 4; i++) b[i] = (m & 2) ? a[2 * i + 1] : a[2 * i];
#pragma unroll
    for (int i = 0; i < 2; i++) c[i] = (m & 4) ? b[2 * i + 1] : b[2 * i];
    return (m & 8) ? c[1] : c[0];
}

// Chunk path: one tile for one warp, lane l owns the 16 contiguous samples of chunk lane_chunk(l) of the tile, n0f is
// the epoch index of the first of them.  The lane rotates its chunk in the chunk frame, u_j = x_j D^j, and forms the
// running sums R_j = u_0 + ... + u_j.  Every tap's chip index rises at most once inside a chunk (the step test at the
// item set-up), so with i0 the index of the first sample and m the last sample that keeps it, the tap gets
//     z0 (c[i0] R_m + c[i0+1] (S - R_m)),   S = R_15,   z0 = the phasor of the chunk's first sample.
// m comes from an estimate that the exact index formula a(n) = fl(fl(step n) + aux), i(n) = floor(a(n)), then decides
// (item set-up: the bound there keeps the estimate within one sample).  From the chunk's first valid sample lo, the
// index rises at b = lo + j, j >= 1 the first with a(b) >= i0 + 1; with e = (i0 + 1) - a(lo) in (0, 1] that is near
// lo + e / step, and c = fl(fl(e) inv_step + 1/2) puts b in {lo + k, lo + k + 1}, k = floor(c).  One evaluation of
// i(lo + k) picks the one: m = b - 1.  c is clamped to 15.5: for b >= lo + 16 that gives k = 15 and i(lo + 15) = i0, so
// m = 15; for b <= lo + 15, c < 16 and k keeps its value.  So k <= 15, and m = k - [i(lo + k) > i0] lies in [0, 15]
// (k = 0 only when b = lo + 1).  The formula is non-decreasing in n for step > 0, and it alone decides, so no sample's
// index is estimated.
// MASKED as in warp_tile: lo is the first sample of the chunk inside the epoch; masked samples add zero to R, so every m
// past the epoch's last sample selects the same sum.  Accumulates into acc_re / acc_im.
// unpaired = 0 (warp-uniform, the item set-up) when the first and the last of three taps are a whole number of chips
// apart, so that in almost every chunk both rise at the same sample; 1 otherwise.  When every lane of the warp finds the
// same m for the two, the last tap takes the first tap's R_m instead of running its own select tree: the same value, so
// nothing in the arithmetic changes.  Each tap still decides its own m and reads its own c[i0], c[i0 + 1] at its own i0
// (fl(y + 1) and fl(y) + 1 may floor differently).
template <int TAPS, bool MASKED>
__device__ __forceinline__ void warp_tile_chunks(const float4* x4, const float4* rot4, float n0f, float vlo, float vhi,
    float step, float inv_step, const float2 (&aux2)[TAPS], unsigned int tbl_off, int unpaired, float2 z0, float2 (&acc_re)[TAPS],
    float2 (&acc_im)[TAPS])
{
    float2 R[kShChunk];
    float2 r = make_float2(0.f, 0.f);
#pragma unroll
    for (int k = 0; k < kShChunk / 2; k++)
        {
            float4 v = x4[k];
            const float4 d = rot4[k];  // D^(2k), D^(2k+1)
            if (MASKED)
                {
                    const float na = n0f + static_cast<float>(2 * k), nb = na + 1.0f;
                    if (na < vlo || na > vhi) v.x = v.y = 0.f;
                    if (nb < vlo || nb > vhi) v.z = v.w = 0.f;
                }
            // two chained FFMA per component: with a zero carrier D^j = (1, 0) and integer data stays exact
            r.x = fmaf(-v.y, d.y, fmaf(v.x, d.x, r.x));
            r.y = fmaf(v.y, d.x, fmaf(v.x, d.y, r.y));
            R[2 * k] = r;
            r.x = fmaf(-v.w, d.w, fmaf(v.z, d.z, r.x));
            r.y = fmaf(v.w, d.z, fmaf(v.z, d.w, r.y));
            R[2 * k + 1] = r;
        }
    const float lo = MASKED ? fminf(fmaxf(n0f, vlo), vhi) : n0f;
    const float lo_m = lo - kFloorMagic;  // exact: lo + k = t_k + lo_m below
    // m relative to the chunk start is (lo - n0f) + (b - lo) - 1
    const int lo_off = MASKED ? __float2int_rn(lo - n0f) : 0;
    float t0[TAPS];
    int m[TAPS];
#pragma unroll
    for (int t = 0; t < TAPS; t++)
        {
            const float a = aux2[t].x;
            const float g = __fadd_rn(__fmul_rn(step, lo), a);
            t0[t] = __fadd_rd(g, kFloorMagic);                                      // kFloorMagic + i0
            const float e = __fsub_rn(__fsub_rn(t0[t], kFloorMagic - 1.0f), g);    // (i0 + 1) - a(lo)
            const float c = fminf(__fmaf_rn(e, inv_step, 0.5f), 15.5f);
            const float tk = __fadd_rd(c, kFloorMagic);                             // kFloorMagic + k
            const float tb = __fadd_rd(__fadd_rn(__fmul_rn(step, __fadd_rn(tk, lo_m)), a), kFloorMagic);
            const int k = __float_as_int(tk) - __float_as_int(kFloorMagic);
            const int mt = lo_off + k - (tb != t0[t] ? 1 : 0);
            m[t] = MASKED ? min(max(mt, 0), kShChunk - 1) : mt;
        }
    // tap t's share of the chunk, P = R_m
    auto add_tap = [&](int t, float2 P) {
        const unsigned int addr = (__float_as_uint(t0[t]) << 2) + tbl_off;
        const float c0 = lds_f32(addr), c1 = lds_f32(addr + 4u);
        const float dc = c0 - c1;
        const float vr = fmaf(dc, P.x, c1 * r.x), vi = fmaf(dc, P.y, c1 * r.y);
        acc_re[t].x = fmaf(z0.x, vr, fmaf(-z0.y, vi, acc_re[t].x));
        acc_im[t].x = fmaf(z0.x, vi, fmaf(z0.y, vr, acc_im[t].x));
    };
    const float2 P0 = select16(R, m[0]);
    add_tap(0, P0);
#pragma unroll
    for (int t = 1; t < (TAPS == 3 ? TAPS - 1 : TAPS); t++) add_tap(t, select16(R, m[t]));
    if (TAPS == 3)
        {
            if (__all_sync(0xffffffffu, ((m[TAPS - 1] ^ m[0]) | unpaired) == 0))
                add_tap(TAPS - 1, P0);
            else
                add_tap(TAPS - 1, select16(R, m[TAPS - 1]));
        }
}

template <int TAPS>
__global__ void __launch_bounds__(kShThreads, kShMinBlocks) trk_shared_kernel(const b200_trk_item* __restrict__ items, int n_items,
    const ChanDesc* __restrict__ chans, const BandDesc* __restrict__ bands, float2* __restrict__ out, int out_stride)
{
    extern __shared__ __align__(128) unsigned char sh_raw[];
    ShSmem& sm = *reinterpret_cast<ShSmem*>(sh_raw);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int group = blockIdx.x;
    const int item_id = group * kShK + warp;
    const bool consumer = warp < kShK;
    const bool have_item = consumer && item_id < n_items;

    b200_trk_item it;
    ChanDesc const* ch = nullptr;
    BandDesc bd;
    if (have_item)
        {
            it = items[item_id];
            ch = &chans[it.channel];
            bd = bands[ch->band];
        }
    if (threadIdx.x == 0)
        {
            for (int s = 0; s < kShStages; s++)
                {
                    mbar_init(&sm.full[s], 1);
                    mbar_init(&sm.empty[s], kShK * 32);  // every consumer lane releases the slot
                }
            asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        }
    if (consumer && lane == 0)
        {
            sm.item_n[warp] = have_item ? it.n : 0;
            sm.item_band[warp] = have_item ? ch->band : -1;
            sm.item_start[warp] = have_item ? (it.sample_index - bd.first_index) : 0ULL;
        }
    __syncthreads();
    if (threadIdx.x == 0)
        {
            // hull of the group's sample ranges (same band only, no ring wrap inside an item's range
            // relative to the hull start, bounded sparsity) -- otherwise the warps load for themselves
            unsigned long long lo = ~0ULL, hi = 0ULL;
            int band = -1, share = 1, nmax = 0;
            for (int w = 0; w < kShK; w++)
                {
                    if (sm.item_n[w] <= 0) continue;
                    if (band < 0) band = sm.item_band[w];
                    if (sm.item_band[w] != band) share = 0;
                    lo = min(lo, sm.item_start[w]);
                    hi = max(hi, sm.item_start[w] + static_cast<unsigned long long>(sm.item_n[w]));
                    nmax = max(nmax, sm.item_n[w]);
                }
            if (band < 0) share = 0;
            lo &= ~1ULL;  // 16-byte aligned tile starts
            if (share && (hi - lo) > 3ULL * static_cast<unsigned long long>(nmax) + 2ULL * kShTile) share = 0;
            sm.hull_start = lo;
            sm.n_tiles = share ? static_cast<int>((hi - lo + kShTile - 1) / kShTile) : 0;
            sm.share = share;
        }
    __syncthreads();
    const int n_tiles = sm.n_tiles;
    const unsigned long long hull_start = sm.hull_start;

    if (!consumer)
        {
            // ---- producer warp: stream the hull through the ring ---------------------------------------
            if (n_tiles > 0)
                {
                    BandDesc pb;
                    {
                        int w0 = 0;
                        while (sm.item_n[w0] <= 0) w0++;
                        pb = bands[sm.item_band[w0]];
                    }
                    const bool ring = (pb.mask != ~0ULL);
                    const unsigned long long cap = ring ? pb.mask + 1ULL : pb.limit;
                    // lane r < 8 copies samples [64r, 64r + 64) of every tile into run slot r (padded layout)
                    const unsigned int c0 = static_cast<unsigned int>(lane) * kShRun;
                    for (int t = 0; t < n_tiles; t++)
                        {
                            const int s = t % kShStages;
                            const unsigned int par = static_cast<unsigned int>((t / kShStages) & 1);
                            mbar_wait(&sm.empty[s], par ^ 1u);
#if SH_STRESS
                            stress_delay(static_cast<unsigned int>(t) * 31u + blockIdx.x * 7u + 3u);
#endif
                            unsigned long long src = hull_start + static_cast<unsigned long long>(t) * kShTile;
                            unsigned int valid = kShTile;
                            if (ring)
                                src &= pb.mask;
                            else if (src >= cap)
                                valid = 0;  // linear band: never read past its end (the clipped samples are outside every item)
                            else if (src + kShTile > cap)
                                valid = static_cast<unsigned int>(cap - src) & ~1u;
                            if (lane == 0) mbar_arrive_expect_tx(&sm.full[s], valid * 8u);
                            __syncwarp();
                            float2* dst = &sm.tiles[s][lane * kShRunStride];
                            if (lane < kShTile / kShRun && ring)
                                {
                                    // a run that straddles the end of the ring is split in two copies
                                    const unsigned long long p = (src + c0) & pb.mask;
                                    const unsigned int n1 = static_cast<unsigned int>(min(static_cast<unsigned long long>(kShRun), cap - p));
                                    bulk_g2s(dst, static_cast<const float2*>(pb.base) + p, n1 * 8u, &sm.full[s]);
                                    if (n1 < kShRun) bulk_g2s(dst + n1, static_cast<const float2*>(pb.base), (kShRun - n1) * 8u, &sm.full[s]);
                                }
                            else if (lane < kShTile / kShRun && valid > c0)
                                {
                                    bulk_g2s(dst, static_cast<const float2*>(pb.base) + src + c0, min(valid - c0, static_cast<unsigned int>(kShRun)) * 8u, &sm.full[s]);
                                }
                        }
                }
            return;
        }

    // ---- consumer warp: one item ---------------------------------------------------------------------
    float2 acc[TAPS];
#pragma unroll
    for (int t = 0; t < TAPS; t++) acc[t] = make_float2(0.f, 0.f);

    bool table_path = false, whole_table = false, chunked = false;
    int unpaired = 1;
    float2 z0 = make_float2(0.f, 0.f), E = z0;  // chunk path: phasor of the lane's chunk start, its advance per tile
    unsigned long long my_hull = 0;
    int body = 0, a_i = 0, t_first = 0, t_last = 0;
    float step = 0.f;
    unsigned int tbl_off = 0;
    float2 aux2[TAPS];
    float2 Dr2, Di2, Gr2, Gi2, zr2, zi2, zr, zi;
    unsigned long long T0 = 0, DT = 0;
    if (have_item && it.n > 0)
        {
            const ItemPhase ph = item_phase(it.rem_carrier_phase_rad, it.phase_step_rad, it.n);
            T0 = ph.T0;
            DT = ph.DT;
            // The chunk path's re-seeds and the epilogue read T0 and DT back from here, so that the two 64-bit words do
            // not hold registers through the tile loops (with them, ptxas spilled a flag word of <3> at 96 registers).
            if (lane == 0)
                {
                    sm.item_turns[warp][0] = T0;
                    sm.item_turns[warp][1] = DT;
                }
            __syncwarp();
            body = ph.body;
            step = it.code_phase_step_chips;
            const float rem = it.rem_code_phase_chips;
            float smin = ch->shifts[0], smax = ch->shifts[0];
#pragma unroll
            for (int t = 0; t < TAPS; t++)
                {
                    const float sh = ch->shifts[t];
                    const float a2 = __fsub_rn(sh, rem);
                    aux2[t] = make_float2(a2, a2);
                    smin = fminf(smin, sh);
                    smax = fmaxf(smax, sh);
                }
            // chunk path, three taps: the first and the last may share their running-sum pick (warp_tile_chunks)
            const float spread = ch->shifts[TAPS - 1] - ch->shifts[0];
            unpaired = (spread != 0.f && spread == rintf(spread)) ? 0 : 1;
            // The code replica is staged per TILE: a tile spans 512*step chips (+ the tap spread), so a
            // 256-entry window per warp serves any code length (1023-chip C/A, 8184-value E1, 10230-chip L5).
            const float span_bound = ceilf(fabsf(step) * static_cast<float>(kShTile)) + ceilf(smax - smin) + 6.0f;
            table_path = !ch->high_dyn && span_bound <= static_cast<float>(kShWin) && fabsf(step) * static_cast<float>(it.n) < 3.0e6f &&
                         fabsf(smax) < 1.0e5f && fabsf(smin) < 1.0e5f && fabsf(rem) < 1.0e6f;
            // (3.0e6 + 1.0e6 + 1.0e5 < 2^22: every chip index of the epoch stays inside the range where the
            //  1.5*2^23 floor trick and the table-offset LEA of warp_tile are exact)
            // Tiles hold whole sample pairs, so the last sample of an attached (linear) band of odd length never reaches
            // one: an epoch whose main part ends there takes the general path.
            if (bd.mask == ~0ULL && (bd.limit & 1ULL) && (it.sample_index - bd.first_index) + static_cast<unsigned long long>(body) == bd.limit)
                table_path = false;
            if (table_path)
                {
                    // whole-epoch table when the epoch's chip range fits the warp's storage (C/A at any rate):
                    // filled once, no per-tile work.  Range from the epoch ends (index monotone in n).
                    {
                        int elo, ehi;
                        const float nl = static_cast<float>(max(body - 1, 0));
                        chip_range<TAPS>(step, 0.f, nl, [&](int q) { return aux2[q].x; }, elo, ehi);
                        whole_table = (static_cast<long long>(ehi) - elo + 3) <= kShTblCap;
                        // Chunk path: the index a(n) = fl(fl(step n) + aux) of every tap may rise at most once over the
                        // 16 samples of a chunk.  warp_tile_chunks evaluates a(n) for 0 <= n <= body - 1 + 16, where
                        // |step n| + |a(n)| <= M = step (body + 15) + max(|elo|, |ehi|) + 3 (16 step < 2).  Both roundings
                        // err by at most half an ulp of their result, so |a(n) - (step n + aux)| <= eps = M 2^-24, and
                        // a(n + 15) - a(n) <= 15 step + 2 eps < 15 step + M 2^-22; below 1, floor(a) rises at most once.
                        // The boundary estimate of warp_tile_chunks: the first j >= 1 with a(lo + j) >= i0 + 1 lies in
                        // [(e - 2 eps) / step, (e + 2 eps) / step + 1), e = (i0 + 1) - a(lo).  fl(e) is within 2^-25 of e
                        // (e <= 1), inv_step = fl(1 / step) within 2^-24 / step, and the FMA rounds c < 17.5 by at most
                        // 2^-20, so |c - (e / step + 1/2)| <= 2^-23 / step + 2^-20.  With
                        // tau = (2 eps + 2^-23) / step + 2^-20 < 1/2, that is (M + 1/2) 2^-22 < step (1 - 2^-19), the first
                        // j lies in (c - 1, c + 1): it is floor(c) or floor(c) + 1.  (C/A at 25 Msps and 1 ms: tau < 0.013;
                        // at 100 Msps and 20 ms: tau < 0.26.)  Only a shared window is laid out in per-lane chunks, so
                        // items that stream their own tiles keep warp_tile.
                        const double M = static_cast<double>(step) * (nl + 16.0) + static_cast<double>(max(abs(elo), abs(ehi))) + 3.0;
                        chunked = whole_table && sm.share && step > 0.f &&
                                  static_cast<double>(kShChunk - 1) * static_cast<double>(step) + M * 0x1p-22 < 1.0 &&
                                  (M + 1.0) * 0x1p-22 < static_cast<double>(step) * (1.0 - 0x1p-18);
                        if (whole_table)
                            {
                                const int wb = elo - 1;
                                const int wspan = ehi - elo + 3;
                                // This copy and stage_window's are written out instead of calling stage_code_window: with it,
                                // ptxas laid the kernel out differently and the C2 step ran 0.8 % slower on an H100 80GB HBM3
                                // at 700 W (1 088 000-1 095 000 against 1 098 000-1 099 000 Msamples/s, three alternating runs).
                                const int L = ch->code_len;
                                int r = mod_pos(wb + lane, L);
                                const int stride = 32 % L;
                                for (int j = lane; j < wspan; j += 32)
                                    {
                                        sm.tbl[warp][j] = __ldg(ch->code + r);
                                        r += stride;
                                        if (r >= L) r -= L;
                                    }
                                tbl_off = table_offset(&sm.tbl[warp][0], wb);
                                __syncwarp();
                            }
                    }
                    // tiles are counted from the group's hull when the window is shared, else from this item's
                    // own (even-aligned) start
                    my_hull = sm.share ? hull_start : (sm.item_start[warp] & ~1ULL);
                    a_i = static_cast<int>(sm.item_start[warp] - my_hull);
                    t_first = a_i / kShTile;
                    t_last = (a_i + body + kShTile - 1) / kShTile;
                    const float2 D = phasor_from_turns(DT * 64ULL);
                    const float2 G = phasor_from_turns(DT * static_cast<unsigned long long>(64 * kShReseed));
                    Dr2 = make_float2(D.x, D.x);
                    Di2 = make_float2(D.y, D.y);
                    Gr2 = make_float2(G.x, G.x);
                    Gi2 = make_float2(G.y, G.y);
                    // phasors of the lane's two samples at the first tile (n may be negative: modular phase)
                    const long long n0 = static_cast<long long>(t_first) * kShTile + 2 * lane - a_i;
                    const float2 za = phasor_from_turns(T0 + DT * static_cast<unsigned long long>(n0));
                    const float2 zb = phasor_from_turns(T0 + DT * static_cast<unsigned long long>(n0 + 1));
                    zr2 = make_float2(za.x, zb.x);
                    zi2 = make_float2(za.y, zb.y);
                    zr = zr2;
                    zi = zi2;
                    if (chunked)
                        {
                            if (lane < kShChunk) sm.rot[warp][lane] = phasor_from_turns(DT * static_cast<unsigned long long>(lane));
                            __syncwarp();
                            E = phasor_from_turns(DT * static_cast<unsigned long long>(kShTile));
                            z0 = phasor_from_turns(T0 + DT * static_cast<unsigned long long>(static_cast<long long>(t_first) * kShTile + kShChunk * lane_chunk(lane) - a_i));
                        }
                }
        }

    float2 are[TAPS], aim[TAPS];
#pragma unroll
    for (int t = 0; t < TAPS; t++) are[t] = aim[t] = make_float2(0.f, 0.f);
    int tiles_in_group = 0;
    int next_wb = 0;
    float fa = static_cast<float>(t_first * kShTile + 2 * lane - a_i), fb = fa + 1.0f;
    // one tile of this warp's epoch; `load` says where the samples come from
    auto process_tile = [&](int t, const auto& load) {
        const int n_tile0 = t * kShTile - a_i;
        const bool interior = (n_tile0 >= 0) && (n_tile0 + kShTile <= body);
        // samples of this tile that belong to the epoch
        const int n_lo = max(n_tile0, 0), n_hi = min(n_tile0 + kShTile, body) - 1;
        const float vlo = static_cast<float>(n_lo), vhi = static_cast<float>(n_hi);
        if (!whole_table)
            {
                // sliding code window: the replica values this tile touches, staged with cp.async
                // (LDGSTS, no registers) one tile AHEAD so the L2 latency hides behind the
                // correlation of the current tile.  window(t) lives in half (t & 1) of tbl[warp].
                auto stage_window = [&](int tt) {
                    const int m0 = tt * kShTile - a_i;
                    const float lo_f = static_cast<float>(max(m0, 0)), hi_f = static_cast<float>(min(m0 + kShTile, body) - 1);
                    int wlo, whi;
                    chip_range<TAPS>(step, lo_f, hi_f, [&](int q) { return aux2[q].x; }, wlo, whi);
                    const int wb = wlo - 1;
                    const int wspan = min(whi - wlo + 3, kShWin);  // <= kShWin by the span_bound test
                    const int L = ch->code_len;
                    int r = mod_pos(wb + lane, L);
                    const int stride = 32 % L;
                    float* dst = &sm.tbl[warp][(tt & 1) * kShWin];
                    for (int j = lane; j < wspan; j += 32)
                        {
                            asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(dst + j)), "l"(ch->code + r) : "memory");
                            r += stride;
                            if (r >= L) r -= L;
                        }
                    return wb;
                };
                if (t == t_first) next_wb = stage_window(t);
                const int wb = next_wb;
                asm volatile("cp.async.wait_all;" ::: "memory");
                __syncwarp();
                if (t + 1 < t_last) next_wb = stage_window(t + 1);
                tbl_off = table_offset(&sm.tbl[warp][(t & 1) * kShWin], wb);
            }
        if (interior)
            warp_tile<TAPS, false>(load, vlo, vhi, step, aux2, tbl_off, Dr2, Di2, fa, fb, zr, zi, are, aim);
        else
            warp_tile<TAPS, true>(load, vlo, vhi, step, aux2, tbl_off, Dr2, Di2, fa, fb, zr, zi, are, aim);
        if (++tiles_in_group == kShReseedTiles)
            {
                // re-seed: the group seed advances by the rounded G = exp(j DT 64*kShReseed) and replaces the
                // running phasor (bounds the drift of the 64 recurrence steps in between; the seed itself is not
                // re-seeded from the 64-bit phase, so its error grows by about 1e-7 per 4096 samples: on 20 ms
                // epochs of 2 000 000 samples, tests/test_trk_paths_gpu.py measured 8.7e-6 |P| on an H100 80GB HBM3, 700 W)
                advance_pair(zr2, zi2, Gr2, Gi2);
                zr = zr2;
                zi = zi2;
                tiles_in_group = 0;
            }
        __syncwarp();
    };

    // Walks the group's tiles through the ring, calling work(t, slot) on the tiles of this warp's epoch.  Every consumer
    // waits for every tile, also the ones it skips: a warp that ran ahead could otherwise arrive twice on empty[s] within
    // one phase and let the producer overwrite a slot that a slower warp is still reading.  Every lane arrives on empty[s]
    // when it is done with the slot, so no lane has to wait for the others before the slot is released.
    auto ring_wait = [&](int t, const RingPos& rp) {
        mbar_wait(&sm.full[rp.s], rp.par);
#if SH_STRESS
        stress_delay(static_cast<unsigned int>(t) * 17u + static_cast<unsigned int>(warp) * 101u + blockIdx.x * 13u);
#endif
    };
    auto ring_release = [&](int t, const RingPos& rp) {
#if SH_STRESS
        stress_delay(static_cast<unsigned int>(t) * 29u + static_cast<unsigned int>(warp) * 53u + blockIdx.x * 5u + 1u);
        __syncwarp();
#endif
        mbar_arrive(&sm.empty[rp.s]);
    };
    auto for_each_ring_tile = [&](const auto& work) {
        for (int t = 0; t < n_tiles; t++)
            {
                const int s = t % kShStages;
                const unsigned int par = static_cast<unsigned int>((t / kShStages) & 1);
                mbar_wait(&sm.full[s], par);
#if SH_STRESS
                stress_delay(static_cast<unsigned int>(t) * 17u + static_cast<unsigned int>(warp) * 101u + blockIdx.x * 13u);
#endif
                if (t >= t_first && t < t_last) work(t, s);
#if SH_STRESS
                stress_delay(static_cast<unsigned int>(t) * 29u + static_cast<unsigned int>(warp) * 53u + blockIdx.x * 5u + 1u);
                __syncwarp();
#endif
                mbar_arrive(&sm.empty[s]);
            }
    };
    // The two paths walk the ring in separate loops, so that none of warp_tile's lane state is live on the chunk path.
    if (chunked)
        {
            const float inv_step = __frcp_rn(step);  // for the boundary estimate (bound at the chunked test)
            const float4* rot4 = reinterpret_cast<const float4*>(&sm.rot[warp][0]);
            // the lane's chunk in ring slot 0; slot s lies s * kShTileSlot samples further
            const float4* x4_0 = reinterpret_cast<const float4*>(&sm.tiles[0][(lane & 7) * kShRunStride + (lane >> 3) * kShChunk]);
            // one tile of the epoch in ring slot s: its first sample is epoch index n_tile0, the lane's chunk n0f; interior =
            // the whole tile lies in the epoch; reseed = z0 is re-seeded after it (every kShReseedTiles-th tile of the epoch)
            auto chunk_tile = [&](const float4* x4, int n_tile0, float n0f, bool interior, bool reseed) {
                if (interior)
                    {
                        warp_tile_chunks<TAPS, false>(x4, rot4, n0f, 0.f, 0.f, step, inv_step, aux2, tbl_off, unpaired, z0, are, aim);
                    }
                else
                    {
                        const float vlo = static_cast<float>(max(n_tile0, 0)), vhi = static_cast<float>(min(n_tile0 + kShTile, body) - 1);
                        warp_tile_chunks<TAPS, true>(x4, rot4, n0f, vlo, vhi, step, inv_step, aux2, tbl_off, unpaired, z0, are, aim);
                    }
                if (reseed)
                    {
                        // exact re-seed from the 64-bit phase of the lane's next chunk start, every 4096 samples
                        const long long n_next = n_tile0 + kShTile + kShChunk * lane_chunk(lane);
                        z0 = phasor_from_turns(sm.item_turns[warp][0] + sm.item_turns[warp][1] * static_cast<unsigned long long>(n_next));
                    }
                else
                    {
                        z0 = cmulf(z0, E);
                    }
            };
            if constexpr (TAPS == 5)
                {
                    // Five taps walk the ring as the other paths do, deriving everything from t: with the carried walk
                    // below, ptxas spilled more in <5>'s set-up and epilogue (38 / 116 B against 22 / 76 B).
                    for_each_ring_tile([&](int t, int s) {
                        const int n_tile0 = t * kShTile - a_i;
                        chunk_tile(x4_0 + s * (kShTileSlot / 2), n_tile0, static_cast<float>(n_tile0 + kShChunk * lane_chunk(lane)), n_tile0 >= 0 && n_tile0 + kShTile <= body,
                            (t - t_first + 1) % kShReseedTiles == 0);
                    });
                }
            else
                {
                    // Tile t of the epoch, t_first <= t < t_last, starts at epoch index n_tile0 = t kShTile - a_i (the last
                    // one holds sample body - 1).  The loop runs on n_tile0 and carries n0f (exact in float: the chunked
                    // test keeps body below 2^22) and the ring position.
                    const int n_first = t_first * kShTile - a_i;
                    float n0f = static_cast<float>(n_first + kShChunk * lane_chunk(lane));
                    // the whole tile lies in the epoch when 0 <= n_tile0 <= body - kShTile
                    const unsigned int n_interior = static_cast<unsigned int>(max(body - kShTile + 1, 0));
                    // n_tile0 - n_first is a multiple of kShTile, so the bits of n_tile0 just above kShTile's say when to
                    // re-seed
                    const int reseed_at = n_first + (kShReseedTiles - 1) * kShTile;
                    // (chunked implies a shared window, so t_last <= n_tiles)
#pragma unroll 1
                    for (int t = 0; t < t_first; t++)
                        {
                            ring_wait(t, RingPos::of(t));
                            ring_release(t, RingPos::of(t));
                        }
                    RingPos ring = RingPos::of(t_first);
                    for (int n_tile0 = n_first; n_tile0 < body; n_tile0 += kShTile)
                        {
                            const int t = (n_tile0 + a_i) / kShTile;  // the stress builds' delays only
                            ring_wait(t, ring);
                            chunk_tile(x4_0 + ring.s * (kShTileSlot / 2), n_tile0, n0f, static_cast<unsigned int>(n_tile0) < n_interior,
                                ((n_tile0 ^ reseed_at) & ((kShReseedTiles - 1) * kShTile)) == 0);
                            ring_release(t, ring);
                            ring.next();
                            n0f += static_cast<float>(kShTile);
                        }
#pragma unroll 1
                    for (int t = t_last; t < n_tiles; t++)
                        {
                            ring_wait(t, RingPos::of(t));
                            ring_release(t, RingPos::of(t));
                        }
                }
        }
    else
        {
            if (table_path)
                for_each_ring_tile([&](int t, int s) {
                    const SmemTileLoader ld{reinterpret_cast<const float4*>(&sm.tiles[s][0]) + lane};
                    process_tile(t, ld);
                });
            else
                for_each_ring_tile([](int, int) {});
            if (!sm.share && table_path)
                {
                    // no shared window for this group: stream this item's own tiles from the band store
                    for (int t = t_first; t < t_last; t++)
                        {
                            const GlobalTileLoader ld{static_cast<const float2*>(bd.base), bd.mask, my_hull + static_cast<unsigned long long>(t) * kShTile + 2ULL * lane, bd.limit};
                            process_tile(t, ld);
                        }
                }
        }
    if (have_item && it.n > 0)
        {
            T0 = sm.item_turns[warp][0];
            DT = sm.item_turns[warp][1];
            if (table_path)
                {
#pragma unroll
                    for (int t = 0; t < TAPS; t++)
                        {
                            acc[t].x = are[t].x + are[t].y;
                            acc[t].y = aim[t].x + aim[t].y;
                        }
                    // tail n in [body, N): generic association, a handful of samples
                    const int n = body + lane;
                    if (n < it.n)
                        {
                            const unsigned long long s0 = it.sample_index - bd.first_index;
                            const float2 x = ldg_stream8(static_cast<const float2*>(bd.base) + ((s0 + static_cast<unsigned long long>(n)) & bd.mask));
                            const float2 z = phasor_from_turns(T0 + DT * static_cast<unsigned long long>(n));
                            const float wr = fmaf(x.x, z.x, -x.y * z.y);
                            const float wi = fmaf(x.x, z.y, x.y * z.x);
#pragma unroll
                            for (int t = 0; t < TAPS; t++)
                                {
                                    const int idx = chip_index_at(step, n, body, ch->shifts[t], it.rem_code_phase_chips);
                                    const float c = __ldg(ch->code + mod_pos(idx, ch->code_len));
                                    acc[t].x = fmaf(wr, c, acc[t].x);
                                    acc[t].y = fmaf(wi, c, acc[t].y);
                                }
                        }
                }
            else
                {
                    warp_correlate_general<TAPS>(it, *ch, bd, T0, DT, body, acc);
                }
#pragma unroll
            for (int t = 0; t < TAPS; t++) acc[t] = warp_sum(acc[t]);
            if (lane < TAPS)
                {
                    float2 r = acc[0];
#pragma unroll
                    for (int t = 1; t < TAPS; t++)
                        if (lane == t) r = acc[t];
                    out[static_cast<size_t>(item_id) * out_stride + lane] = r;
                }
        }
    else if (have_item && lane < ch->taps)
        {
            out[static_cast<size_t>(item_id) * out_stride + lane] = make_float2(0.f, 0.f);
        }
}
template <int TAPS>
int launch_shared(const b200_trk_item* items, int n_items, const ChanDesc* chans, const BandDesc* bands, float2* out, int out_stride,
    cudaStream_t stream)
{
    static DeviceOnce once;  // per device: a second engine on another GPU needs its own opt-in
    const int once_dev = once.begin();
    if (once_dev >= 0)
        {
            B200_CUDA_TRY(cudaFuncSetAttribute(trk_shared_kernel<TAPS>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(sizeof(ShSmem))));
            once.done(once_dev);
        }
    const int groups = (n_items + kShK - 1) / kShK;
    trk_shared_kernel<TAPS><<<groups, kShThreads, sizeof(ShSmem), stream>>>(items, n_items, chans, bands, out, out_stride);
    B200_CUDA_TRY(cudaGetLastError());
    return B200_OK;
}
}  // namespace

int launch_trk_shared(const b200_trk_item* items, int n_items, const ChanDesc* chans, const BandDesc* bands, float2* out,
    int out_stride, int taps, cudaStream_t stream, uint64_t& launched)
{
    if (n_items <= 0) return B200_OK;
    const int rc = with_taps<1, 3, 5>(taps, [&](auto tc) {
        return launch_shared<decltype(tc)::value>(items, n_items, chans, bands, out, out_stride, stream);
    });
    if (rc == B200_OK) launched++;
    return rc;
}

// Longest code table for which every epoch takes the whole-table mode (faster than the per-item kernel on C2).
// Longer tables (E1 8184, L5 10230) work through the sliding window but are slower than the per-item kernel
// (C3), so the engine only picks them when forced.
int trk_shared_max_code_len() { return kShTblCap - 64; }

}  // namespace b200
