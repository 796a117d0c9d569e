// Pairing stage of the batch decoder: cpr_decoder's bookkeeping (cpr.py:206-229). For every position message it finds
// the latest even and odd report of its aircraft as of that message; the reference does this one message at a time
// against four dicts. Here the reports are first PARTITIONED by owner: a stable counting sort of the frame indices into
// AMB_V3_B buckets (bucket = hash of the aircraft key), so that each bucket's list keeps stream order. Then one warp per
// bucket walks only its own list, 32 reports per step: same-aircraft reports inside a step are resolved with
// match/ballot, everything older through a direct-mapped table in HBM (AMB_TABLE_SLOTS x 16 B: one slot per (ICAO,
// surface, even/odd), so no probing, no collisions, no locks - a slot has exactly one owner bucket). O(n) memory traffic.
//
//   amb_v3_count    per tile of 8192 frames: histogram of the buckets (shared-memory atomics) -> cnt[bucket][tile]
//   amb_v3_rowscan  one warp per bucket: exclusive scan along the tiles -> off[bucket][tile], tot[bucket]
//   amb_v3_basescan one CTA: exclusive scan of tot -> base[bucket], base[B] = number of position reports
//   amb_v3_scatter  per tile, chunks of 256 frames in order, the 8 warps of a chunk take turns: rank inside the warp
//                   by match_any, running per-bucket cursor in shared memory -> order[] (stable)
//   amb_v3_pair     one warp per bucket over order[base[b] .. base[b+1])
#pragma once

#define AMB_V3_B 1024
#define AMB_V3_TILE 8192

struct AmbV3Bufs {
    uint32_t* cnt = nullptr; uint32_t* off = nullptr; uint32_t* tot = nullptr; uint32_t* base = nullptr; uint32_t* order = nullptr;
    int tiles_cap = 0, order_cap = 0;
};

__device__ __forceinline__ unsigned amb_v3_bucket(uint32_t key)
{
    return (unsigned)(((uint64_t)(key * 2654435761u) * AMB_V3_B) >> 32);
}

__global__ void __launch_bounds__(256) amb_v3_count(const AmbPosRec* __restrict__ pos, int n, int n_tiles, uint32_t* __restrict__ cnt)
{
    __shared__ unsigned h[AMB_V3_B];
    for (int b = threadIdx.x; b < AMB_V3_B; b += 256) h[b] = 0;
    __syncthreads();
    const int start = blockIdx.x * AMB_V3_TILE;
    for (int i = threadIdx.x; i < AMB_V3_TILE; i += 256) {
        const int k = start + i;
        if (k < n) {
            const uint32_t key = pos[k].key;
            if (key != AMB_NO_KEY) atomicAdd(&h[amb_v3_bucket(key)], 1u);
        }
    }
    __syncthreads();
    for (int b = threadIdx.x; b < AMB_V3_B; b += 256) cnt[(size_t)b * n_tiles + blockIdx.x] = h[b];
}

__global__ void __launch_bounds__(256) amb_v3_rowscan(const uint32_t* __restrict__ cnt, int n_tiles, uint32_t* __restrict__ off,
                                                      uint32_t* __restrict__ tot)
{
    const unsigned lane = threadIdx.x & 31;
    const int b = blockIdx.x * 8 + (threadIdx.x >> 5);          // one warp per bucket
    unsigned running = 0;
    for (int t0 = 0; t0 < n_tiles; t0 += 32) {
        const int t = t0 + (int)lane;
        const unsigned v = t < n_tiles ? cnt[(size_t)b * n_tiles + t] : 0u;
        unsigned x = v;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const unsigned y = __shfl_up_sync(0xffffffffu, x, d);
            if ((int)lane >= d) x += y;
        }
        if (t < n_tiles) off[(size_t)b * n_tiles + t] = running + x - v;
        running += __shfl_sync(0xffffffffu, x, 31);
    }
    if (lane == 0) tot[b] = running;
}

__global__ void __launch_bounds__(AMB_V3_B) amb_v3_basescan(const uint32_t* __restrict__ tot, uint32_t* __restrict__ base)
{
    __shared__ unsigned wsum[32];
    const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned v = tot[threadIdx.x];
    unsigned x = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const unsigned y = __shfl_up_sync(0xffffffffu, x, d);
        if ((int)lane >= d) x += y;
    }
    if (lane == 31) wsum[warp] = x;
    __syncthreads();
    if (warp == 0) {
        unsigned s = wsum[lane];
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const unsigned y = __shfl_up_sync(0xffffffffu, s, d);
            if ((int)lane >= d) s += y;
        }
        wsum[lane] = s;                                          // inclusive totals of the 32 warps
    }
    __syncthreads();
    const unsigned before = warp ? wsum[warp - 1] : 0u;
    base[threadIdx.x] = before + x - v;
    if (threadIdx.x == AMB_V3_B - 1) base[AMB_V3_B] = before + x;
}

__global__ void __launch_bounds__(256) amb_v3_scatter(const AmbPosRec* __restrict__ pos, int n, int n_tiles,
                                                      const uint32_t* __restrict__ off, const uint32_t* __restrict__ base,
                                                      uint32_t* __restrict__ order)
{
    __shared__ unsigned run[AMB_V3_B];                           // next free position of every bucket, for this tile
    for (int b = threadIdx.x; b < AMB_V3_B; b += 256) run[b] = base[b] + off[(size_t)b * n_tiles + blockIdx.x];
    __syncthreads();
    const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned lt = (1u << lane) - 1u;
    const int start = blockIdx.x * AMB_V3_TILE;
    for (int c = 0; c < AMB_V3_TILE && start + c < n; c += 256) {          // chunks in stream order (uniform bounds)
        const int k = start + c + (int)threadIdx.x;
        uint32_t key = AMB_NO_KEY;
        if (k < n) key = pos[k].key;
        const bool valid = key != AMB_NO_KEY;
        const unsigned b = valid ? amb_v3_bucket(key) : 0u;
        for (unsigned w = 0; w < 8; w++) {                                 // the chunk's warps in stream order
            if (warp == w) {
                const unsigned peers = __match_any_sync(0xffffffffu, valid ? b : (0x80000000u | lane));
                const int leader = __ffs(peers) - 1;
                unsigned old = 0;
                if (valid && (int)lane == leader) { old = run[b]; run[b] = old + __popc(peers); }
                old = __shfl_sync(0xffffffffu, old, valid ? leader : (int)lane);
                if (valid) order[old + __popc(peers & lt)] = (uint32_t)k;
            }
            __syncthreads();
        }
    }
}

__global__ void __launch_bounds__(128) amb_v3_pair(const AmbPosRec* __restrict__ pos, const uint32_t* __restrict__ order,
                                                   const uint32_t* __restrict__ base, AmbCprSlot* table, AmbPair* __restrict__ pair)
{
    const unsigned lane = threadIdx.x & 31;
    const unsigned b = blockIdx.x * 4 + (threadIdx.x >> 5);     // one warp per bucket; a table slot has one owner bucket
    const unsigned lt = (1u << lane) - 1u;
    const unsigned lo = base[b], hi = base[b + 1];
    for (unsigned i0 = lo; i0 < hi; i0 += 32) {
        const unsigned i = i0 + lane;
        const bool mine = i < hi;
        const int k = mine ? (int)order[i] : 0;
        AmbPosRec me; me.key = AMB_NO_KEY; me.lat = me.lon = 0; me.fmt = 0; me.t = 0.0;
        if (mine) me = pos[k];
        // same aircraft inside this step (lane order = stream order inside the bucket); lanes past the end of the bucket
        // get a private value
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

static cudaError_t amb_v3_ensure(AmbV3Bufs* v, int n)
{
    const int n_tiles = (n + AMB_V3_TILE - 1) / AMB_V3_TILE;
    cudaError_t e = cudaSuccess;
    if (!v->tot) {
        if ((e = cudaMalloc(&v->tot, AMB_V3_B * sizeof(uint32_t))) != cudaSuccess) return e;
        if ((e = cudaMalloc(&v->base, (AMB_V3_B + 1) * sizeof(uint32_t))) != cudaSuccess) return e;
    }
    if (v->tiles_cap < n_tiles) {
        cudaFree(v->cnt); cudaFree(v->off); v->cnt = v->off = nullptr;
        const int cap = n_tiles * 2;
        if ((e = cudaMalloc(&v->cnt, (size_t)AMB_V3_B * cap * sizeof(uint32_t))) != cudaSuccess) return e;
        if ((e = cudaMalloc(&v->off, (size_t)AMB_V3_B * cap * sizeof(uint32_t))) != cudaSuccess) return e;
        v->tiles_cap = cap;
    }
    if (v->order_cap < n) {
        cudaFree(v->order); v->order = nullptr;
        if ((e = cudaMalloc(&v->order, (size_t)n * 2 * sizeof(uint32_t))) != cudaSuccess) return e;
        v->order_cap = n * 2;
    }
    return cudaSuccess;
}

static void amb_v3_free(AmbV3Bufs* v)
{
    cudaFree(v->cnt); cudaFree(v->off); cudaFree(v->tot); cudaFree(v->base); cudaFree(v->order);
    *v = AmbV3Bufs();
}

// Enqueue the five kernels; returns how many were launched (for the launch counter) or -1 with *err set.
static int amb_v3_launch(AmbV3Bufs* v, const AmbPosRec* pos, int n, AmbCprSlot* table, AmbPair* pair, cudaStream_t s, cudaError_t* err)
{
    if ((*err = amb_v3_ensure(v, n)) != cudaSuccess) return -1;
    const int n_tiles = (n + AMB_V3_TILE - 1) / AMB_V3_TILE;
    AMB_LAUNCH((amb_v3_count), n_tiles, 256, 0, s, pos, n, n_tiles, v->cnt);
    AMB_LAUNCH((amb_v3_rowscan), AMB_V3_B / 8, 256, 0, s, v->cnt, n_tiles, v->off, v->tot);
    AMB_LAUNCH((amb_v3_basescan), 1, AMB_V3_B, 0, s, v->tot, v->base);
    AMB_LAUNCH((amb_v3_scatter), n_tiles, 256, 0, s, pos, n, n_tiles, v->off, v->base, v->order);
    AMB_LAUNCH((amb_v3_pair), AMB_V3_B / 4, 128, 0, s, pos, v->order, v->base, table, pair);
    *err = cudaGetLastError();
    return *err == cudaSuccess ? 5 : -1;
}
