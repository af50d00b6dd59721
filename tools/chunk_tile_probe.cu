// A kernel that runs only the chunk path's tile, warp_tile_chunks<TAPS, MASKED>, in a loop over the ring's slots, so that
// its SASS can be counted apart from the rest of trk_shared_kernel (tools/chunk_tile_sass.py).  Compiled for sm_90a with
// the same __launch_bounds__ as the kernel; never launched.
//
// Interior tile, instructions per warp (nvcc 12.9, sm_90a), this probe / the kernel's own chunk-path tile loop with its
// ring walk (DESIGN 4.2):
//   taps   before the shared pick   shared pick   last tap's own pick
//   1      145 / 179                144 / 162     -
//   3      245 / 279                232 / 246     256 / 270
//   5      349 / 383                348 / 380     -   (the kernel's <5> keeps the ring walk of the other paths)
#include "../gnss_sdr_b200/csrc/trk_shared_kernel.cu"

namespace b200
{
namespace
{
template <int TAPS, bool MASKED>
__global__ void __launch_bounds__(kShThreads, kShMinBlocks) chunk_tile_probe(const float* __restrict__ p, float2* __restrict__ out, int tiles)
{
    extern __shared__ __align__(128) unsigned char sh_raw[];
    ShSmem& sm = *reinterpret_cast<ShSmem*>(sh_raw);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const float step = p[0], inv_step = p[1], vlo = p[2], vhi = p[3];
    const float2 E = make_float2(p[4], p[5]);
    float2 z0 = make_float2(p[6], p[7]);
    float2 aux2[TAPS];
#pragma unroll
    for (int t = 0; t < TAPS; t++) aux2[t] = make_float2(p[8 + t], p[8 + t]);
    const unsigned int tbl_off = table_offset(&sm.tbl[warp][0], static_cast<int>(p[16]));
    const int unpaired = p[17] != 0.f;
    float2 are[TAPS], aim[TAPS];
#pragma unroll
    for (int t = 0; t < TAPS; t++) are[t] = aim[t] = make_float2(0.f, 0.f);
    float n0f = static_cast<float>(kShChunk * lane_chunk(lane));
    const float4* rot4 = reinterpret_cast<const float4*>(&sm.rot[warp][0]);
    for (int t = 0; t < tiles; t++)
        {
            const int s = t % kShStages;
            const float4* x4 = reinterpret_cast<const float4*>(&sm.tiles[s][(lane & 7) * kShRunStride + (lane >> 3) * kShChunk]);
            warp_tile_chunks<TAPS, MASKED>(x4, rot4, n0f, vlo, vhi, step, inv_step, aux2, tbl_off, unpaired, z0, are, aim);
            z0 = cmulf(z0, E);
            n0f += static_cast<float>(kShTile);
        }
#pragma unroll
    for (int t = 0; t < TAPS; t++) out[(threadIdx.x * TAPS + t) * 2] = are[t], out[(threadIdx.x * TAPS + t) * 2 + 1] = aim[t];
}

template __global__ void chunk_tile_probe<1, false>(const float*, float2*, int);
template __global__ void chunk_tile_probe<3, false>(const float*, float2*, int);
template __global__ void chunk_tile_probe<5, false>(const float*, float2*, int);
}  // namespace
}  // namespace b200
