// The kernels of the batch field decoder (SURVEY.md 8 row f4); the host orchestration and the C ABI are in
// amb_decode.cu, the per-message arithmetic in amb_decode_core.h. Kept in a header without any <<< >>> launch so that
// tests/simt/ can compile the very same kernel source for the host under a small SIMT emulator (CPU-side check of the
// warp-level logic; the GPU tests remain the parity gate).
#pragma once
#include "amb_decode_core.h"

#define AMB_TABLE_SLOTS (1ull << 26)     // (24-bit ICAO, surface, even/odd)
#define AMB_PAIR_WARPS_PER_CTA 4

struct AmbCprSlot { uint32_t lat, lon; double t; };   // lat == 0xFFFFFFFF: empty

// ---- kernels ------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) amb_fields_kernel(const amb_frame* __restrict__ frames, int n,
                                                         amb_fields* __restrict__ fields, AmbPosRec* __restrict__ pos,
                                                         AmbPair* __restrict__ pair)
{
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    amb_fields r; AmbPosRec p;
    amb_decode_fields(frames[k], &r, &p);
    fields[k] = r;
    pos[k] = p;
    AmbPair z; z.elat = z.elon = z.olat = z.olon = 0; z.have = 0; z.mostrecent = 0;
    pair[k] = z;
}

__device__ __forceinline__ unsigned amb_key_owner(uint32_t key, unsigned n_warps)
{
    return (unsigned)(((uint64_t)(key * 2654435761u) * n_warps) >> 32);     // multiplicative hash -> [0, n_warps)
}

__global__ void __launch_bounds__(32 * AMB_PAIR_WARPS_PER_CTA)
amb_pair_kernel(const AmbPosRec* __restrict__ pos, int n, AmbCprSlot* table, AmbPair* __restrict__ pair)
{
    const unsigned lane = threadIdx.x & 31;
    const unsigned warp = blockIdx.x * AMB_PAIR_WARPS_PER_CTA + (threadIdx.x >> 5);
    const unsigned n_warps = gridDim.x * AMB_PAIR_WARPS_PER_CTA;
    const unsigned lt = (1u << lane) - 1u;
    for (int base = 0; base < n; base += 32) {
        const int k = base + (int)lane;
        AmbPosRec me; me.key = AMB_NO_KEY; me.lat = me.lon = 0; me.fmt = 0; me.t = 0.0;
        if (k < n) me = pos[k];
        const bool mine = me.key != AMB_NO_KEY && amb_key_owner(me.key, n_warps) == warp;
        if (!__any_sync(0xffffffffu, mine)) continue;                      // uniform: all lanes take the same branch
        // same aircraft (same list pair) inside this step; lanes that are not ours get a private value
        const unsigned peers = __match_any_sync(0xffffffffu, mine ? me.key : (0x80000000u | lane));
        const unsigned evens = __ballot_sync(0xffffffffu, mine && me.fmt == 0);
        const unsigned odds = __ballot_sync(0xffffffffu, mine && me.fmt != 0);
        // the latest report of the OTHER format at or before this message: an earlier lane of this step, else the table
        const unsigned other_here = peers & (me.fmt ? evens : odds) & lt;
        const int src = other_here ? (31 - __clz(other_here)) : (int)lane;
        uint32_t o_lat = __shfl_sync(0xffffffffu, me.lat, src);
        uint32_t o_lon = __shfl_sync(0xffffffffu, me.lon, src);
        double o_t = __shfl_sync(0xffffffffu, me.t, src);
        bool o_have = other_here != 0;
        const size_t slot_other = ((size_t)me.key << 1) | (me.fmt ? 0u : 1u);
        const size_t slot_mine = ((size_t)me.key << 1) | (me.fmt ? 1u : 0u);
        if (mine && !o_have) {
            const uint4 v = __ldcg(reinterpret_cast<const uint4*>(&table[slot_other]));     // L2, never a stale L1 line
            if (v.x != 0xFFFFFFFFu) { o_lat = v.x; o_lon = v.y; o_t = __hiloint2double((int)v.w, (int)v.z); o_have = true; }
        }
        if (mine) pair[k] = amb_make_pair(me, o_have ? 1 : 0, o_lat, o_lon, o_t);
        __syncwarp();                                                       // every table read of this step is done
        // cpr.py:214-221: the message's own report replaces the stored one; the last lane per (aircraft, format) wins
        const unsigned same = peers & (me.fmt ? odds : evens);
        if (mine && (int)lane == 31 - __clz(same)) {
            const uint4 v = make_uint4(me.lat, me.lon, (unsigned)__double2loint(me.t), (unsigned)__double2hiint(me.t));
            __stcg(reinterpret_cast<uint4*>(&table[slot_mine]), v);
            __threadfence_block();
        }
        __syncwarp();                                                       // ... and visible to the next step's reads
    }
}

#ifdef AMB_PAIR_V2
// EXPERIMENT (tools/variants.py "pair_v2"; NOT in the product build, not yet run on a GPU). The first pairing kernel is
// L2-bandwidth-bound: each of its warps reads the whole 24-byte report list. Here
// the ownership test reads a 4-byte key array, eight independent steps' keys are in flight per iteration, and only
// the lanes that own a report load the rest of it. The per-step logic is the first kernel's, unchanged.
#define AMB_PAIR_V2_U 8
__global__ void amb_keys_kernel(const AmbPosRec* __restrict__ pos, int n, uint32_t* __restrict__ keys)
{
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k < n) keys[k] = pos[k].key;
}

__device__ __forceinline__ void amb_pair_step_v2(int k, bool mine, unsigned lane, unsigned lt, const AmbPosRec* __restrict__ pos,
                                                 AmbCprSlot* table, AmbPair* __restrict__ pair)
{
    AmbPosRec me; me.key = AMB_NO_KEY; me.lat = me.lon = 0; me.fmt = 0; me.t = 0.0;
    if (mine) me = pos[k];
    const unsigned peers = __match_any_sync(0xffffffffu, mine ? me.key : (0x80000000u | lane));
    const unsigned evens = __ballot_sync(0xffffffffu, mine && me.fmt == 0);
    const unsigned odds = __ballot_sync(0xffffffffu, mine && me.fmt != 0);
    const unsigned other_here = peers & (me.fmt ? evens : odds) & lt;
    const int src = other_here ? (31 - __clz(other_here)) : (int)lane;
    uint32_t o_lat = __shfl_sync(0xffffffffu, me.lat, src);
    uint32_t o_lon = __shfl_sync(0xffffffffu, me.lon, src);
    double o_t = __shfl_sync(0xffffffffu, me.t, src);
    bool o_have = other_here != 0;
    const size_t slot_other = ((size_t)me.key << 1) | (me.fmt ? 0u : 1u);
    const size_t slot_mine = ((size_t)me.key << 1) | (me.fmt ? 1u : 0u);
    if (mine && !o_have) {
        const uint4 v = __ldcg(reinterpret_cast<const uint4*>(&table[slot_other]));
        if (v.x != 0xFFFFFFFFu) { o_lat = v.x; o_lon = v.y; o_t = __hiloint2double((int)v.w, (int)v.z); o_have = true; }
    }
    if (mine) pair[k] = amb_make_pair(me, o_have ? 1 : 0, o_lat, o_lon, o_t);
    __syncwarp();
    const unsigned same = peers & (me.fmt ? odds : evens);
    if (mine && (int)lane == 31 - __clz(same)) {
        const uint4 v = make_uint4(me.lat, me.lon, (unsigned)__double2loint(me.t), (unsigned)__double2hiint(me.t));
        __stcg(reinterpret_cast<uint4*>(&table[slot_mine]), v);
        __threadfence_block();
    }
    __syncwarp();
}

__global__ void __launch_bounds__(32 * AMB_PAIR_WARPS_PER_CTA)
amb_pair_kernel_v2(const uint32_t* __restrict__ keys, const AmbPosRec* __restrict__ pos, int n, AmbCprSlot* table,
                   AmbPair* __restrict__ pair)
{
    const unsigned lane = threadIdx.x & 31;
    const unsigned warp = blockIdx.x * AMB_PAIR_WARPS_PER_CTA + (threadIdx.x >> 5);
    const unsigned n_warps = gridDim.x * AMB_PAIR_WARPS_PER_CTA;
    const unsigned lt = (1u << lane) - 1u;
    for (int base = 0; base < n; base += 32 * AMB_PAIR_V2_U) {
        uint32_t key[AMB_PAIR_V2_U];
#pragma unroll
        for (int u = 0; u < AMB_PAIR_V2_U; u++) {
            const int k = base + 32 * u + (int)lane;
            key[u] = k < n ? __ldg(keys + k) : AMB_NO_KEY;
        }
        bool mine[AMB_PAIR_V2_U], any = false;
#pragma unroll
        for (int u = 0; u < AMB_PAIR_V2_U; u++) {
            mine[u] = key[u] != AMB_NO_KEY && amb_key_owner(key[u], n_warps) == warp;
            any = any || mine[u];
        }
        if (!__any_sync(0xffffffffu, any)) continue;
#pragma unroll
        for (int u = 0; u < AMB_PAIR_V2_U; u++)                     // stream order: step u before step u + 1
            if (__any_sync(0xffffffffu, mine[u]))
                amb_pair_step_v2(base + 32 * u + (int)lane, mine[u], lane, lt, pos, table, pair);
    }
}
#endif

__global__ void __launch_bounds__(128) amb_resolve_kernel(amb_fields* __restrict__ fields, const AmbPosRec* __restrict__ pos,
                                                          const AmbPair* __restrict__ pair, int n, int have_loc,
                                                          double mylat, double mylon, const double* __restrict__ nl_T)
{
    __shared__ double T[AMB_NL_MAX];
    for (int i = threadIdx.x; i < AMB_NL_MAX; i += blockDim.x) T[i] = nl_T[i];
    __syncthreads();
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    if (pos[k].key == AMB_NO_KEY) return;
    amb_fields r = fields[k];
    amb_resolve_position(&r, pair[k], have_loc, mylat, mylon, T);
    fields[k] = r;
}

#ifdef AMB_PAIR_V3
#include "amb_decode_v3.cuh"
#endif
