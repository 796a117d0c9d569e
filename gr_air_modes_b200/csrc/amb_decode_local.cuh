// Local CPR stage of the batch decoder (decoder option "local_cpr", DESIGN.md §8). Runs after amb_resolve_kernel and
// decodes every position message that has no global fix relative to its aircraft's reference position: the last fix of
// the same 24-bit ICAO, global or local, kept in a direct-mapped table in HBM (AMB_LOCAL_SLOTS x 24 B, one slot per
// ICAO). Each local fix depends on the previous fix of the same aircraft, so the position messages of one aircraft form
// a chain that is walked in stream order:
//
//   amb_local_keys      one thread per frame: the report key reduced to the ICAO (airborne and surface share a chain)
//   amb_v3_count .. amb_v3_scatter   the pairing stage's stable partition (amb_decode_v3.cuh), here on the ICAO keys
//   amb_local_walk      one warp per bucket, 32 messages per step: same-aircraft groups from __match_any_sync; inside a
//                       group the chain is resolved in lane order (= stream order), each member starting from its
//                       predecessor's reference by shuffle, the first one from the table; the last one writes it back.
//                       A slot has exactly one owner bucket: no probing, no atomics.
#pragma once

#define AMB_LOCAL_SLOTS (1ull << 24)

__global__ void __launch_bounds__(128) amb_local_keys(const AmbPosRec* __restrict__ pos, int n, AmbPosRec* __restrict__ lpos)
{
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    const uint32_t key = pos[k].key;
    lpos[k].key = key == AMB_NO_KEY ? AMB_NO_KEY : (key >> 1);
}

__global__ void __launch_bounds__(128) amb_local_walk(const AmbPosRec* __restrict__ pos, const uint32_t* __restrict__ order,
                                                      const uint32_t* __restrict__ base, amb_fields* __restrict__ fields,
                                                      AmbRefPos* table, int max_age, int have_loc, double mylat, double mylon,
                                                      const double* __restrict__ nl_T)
{
    __shared__ double T[AMB_NL_MAX];
    for (int i = threadIdx.x; i < AMB_NL_MAX; i += blockDim.x) T[i] = nl_T[i];
    __syncthreads();
    const unsigned lane = threadIdx.x & 31;
    const unsigned b = blockIdx.x * 4 + (threadIdx.x >> 5);     // one warp per bucket; a table slot has one owner bucket
    const unsigned lt = (1u << lane) - 1u;
    const unsigned lo = base[b], hi = base[b + 1];
    for (unsigned i0 = lo; i0 < hi; i0 += 32) {
        const unsigned i = i0 + lane;
        const bool mine = i < hi;
        const int k = mine ? (int)order[i] : 0;
        const uint32_t icao = mine ? (pos[k].key >> 1) : 0u;
        const double t = mine ? pos[k].t : 0.0;
        // the same aircraft inside this step; lanes past the end of the bucket get a private value (an ICAO has 24 bits)
        const unsigned peers = __match_any_sync(0xffffffffu, mine ? icao : (0x80000000u | lane));
        const unsigned before = peers & lt;
        const int rank = __popc(before);                        // position in the aircraft's chain inside this step
        const int pred = before ? (31 - __clz(before)) : (int)lane;
        AmbRefPos ref; ref.lat = ref.lon = ref.t = NAN;
        if (mine && rank == 0) {
            const double* s = &table[icao].lat;                 // L2, never a stale L1 line
            ref.lat = __ldcg(s); ref.lon = __ldcg(s + 1); ref.t = __ldcg(s + 2);
        }
        // The first member of a group starts from the table, and a message whose global fix stands needs nothing from
        // its predecessors: both are done at once. Every other member waits for its predecessor's final reference, so
        // the rounds are as many as the longest run of members without a global fix.
        int done = !mine;
        if (mine && (rank == 0 || (fields[k].status & AMB_FS_HAS_POS))) {
            amb_local_step(&fields[k], t, &ref, max_age, have_loc, mylat, mylon, T);
            done = 1;
        }
        while (__any_sync(0xffffffffu, !done)) {
            const int pdone = __shfl_sync(0xffffffffu, done, pred);
            const double plat = __shfl_sync(0xffffffffu, ref.lat, pred);
            const double plon = __shfl_sync(0xffffffffu, ref.lon, pred);
            const double pt = __shfl_sync(0xffffffffu, ref.t, pred);
            if (!done && pdone) {
                ref.lat = plat; ref.lon = plon; ref.t = pt;
                amb_local_step(&fields[k], t, &ref, max_age, have_loc, mylat, mylon, T);
                done = 1;
            }
        }
        __syncwarp();                                           // every table read of this step is done
        if (mine && (int)lane == 31 - __clz(peers)) {           // the last member holds the aircraft's reference
            double* s = &table[icao].lat;
            __stcg(s, ref.lat); __stcg(s + 1, ref.lon); __stcg(s + 2, ref.t);
            __threadfence_block();
        }
        __syncwarp();                                           // ... and visible to the next step's reads
    }
}

// Enqueue the stage (six kernels) after amb_resolve_kernel; `v` is the pairing stage's scratch, free again by then.
// Returns how many kernels were launched or -1 with *err set.
static int amb_local_launch(AmbV3Bufs* v, const AmbPosRec* pos, AmbPosRec* lpos, int n, amb_fields* fields, AmbRefPos* table,
                            int max_age, int have_loc, double mylat, double mylon, const double* nl_T, cudaStream_t s,
                            cudaError_t* err)
{
    AMB_LAUNCH((amb_local_keys), (n + 127) / 128, 128, 0, s, pos, n, lpos);
    if (amb_v3_partition(v, lpos, n, s, err) < 0) return -1;
    AMB_LAUNCH((amb_local_walk), AMB_V3_B / 4, 128, 0, s, pos, v->order, v->base, fields, table, max_age, have_loc, mylat,
               mylon, nl_T);
    *err = cudaGetLastError();
    return *err == cudaSuccess ? 6 : -1;
}
