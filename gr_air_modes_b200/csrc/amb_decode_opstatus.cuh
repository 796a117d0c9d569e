// ADS-B operational status, target state and position integrity of the batch decoder (decoder option "opstatus",
// DESIGN.md §8 "Operational status and NIC"). Runs after the Comm-B stage and before the track stage. A queued DF17
// TC 31 (BDS6,5) or TC 29 subtype 1 (BDS6,2) squitter, which the parser does not handle, is decoded into its record;
// every queued DF17 position (BDS0,5 / BDS0,6) gets its NIC and Rc from its address's latest op status, or its NUCp
// (amb_es_* in amb_decode_core.h). That op status is kept in a direct-mapped table in HBM (AMB_OPS_SLOTS x 24 B, one
// slot per address) across calls:
//
//   amb_opstatus_keys   one thread per frame: TC 29 / 31 decoded and written at once; key = icao for op-status writers
//                       and for positions, AMB_NO_KEY otherwise
//   amb_v3_count .. amb_v3_scatter   the pairing stage's stable partition (amb_decode_v3.cuh), here on those keys
//   amb_opstatus_walk   one warp per bucket, 32 records per step: same-address groups from __match_any_sync; a position
//                       takes the last earlier writer of its group (any subtype) and the last earlier surface writer,
//                       or the table's slot where there is none; the group's last writer and last surface writer write
//                       the slot. No chains: one pass per step. A slot has exactly one owner bucket: no atomics.
#pragma once

#define AMB_OPS_SLOTS (1ull << 24)

__global__ void __launch_bounds__(128) amb_opstatus_keys(const amb_frame* __restrict__ frames, amb_fields* __restrict__ fields,
                                                         const AmbPosRec* __restrict__ pos, int n, AmbPosRec* __restrict__ opos)
{
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    AmbPosRec p;
    p.t = pos[k].t;                                         // secs + frac, as the pairing stage has it
    p.fmt = amb_es_classify(frames[k], &fields[k], &p.lat, &p.lon);
    p.key = p.fmt != AMB_ES_KIND_NONE ? fields[k].icao : AMB_NO_KEY;   // DF17: the 24-bit address
    opos[k] = p;
}

__global__ void __launch_bounds__(128) amb_opstatus_walk(const AmbPosRec* __restrict__ opos, const uint32_t* __restrict__ order,
                                                         const uint32_t* __restrict__ base, amb_fields* __restrict__ fields,
                                                         AmbOpsSlot* table, int max_age)
{
    const unsigned lane = threadIdx.x & 31;
    const unsigned b = blockIdx.x * 4 + (threadIdx.x >> 5);     // one warp per bucket; a table slot has one owner bucket
    const unsigned lt = (1u << lane) - 1u;
    const unsigned lo = base[b], hi = base[b + 1];
    for (unsigned i0 = lo; i0 < hi; i0 += 32) {
        const unsigned i = i0 + lane;
        const bool mine = i < hi;
        const int k = mine ? (int)order[i] : 0;
        AmbPosRec p;
        if (mine) p = opos[k];
        else { p.key = 0u; p.t = 0.0; p.fmt = AMB_ES_KIND_NONE; p.lat = p.lon = 0u; }
        const unsigned kind = p.fmt;
        // the same address inside this step; lanes past the end of the bucket get a private value (an address has 24 bits)
        const unsigned peers = __match_any_sync(0xffffffffu, mine ? p.key : (0x80000000u | lane));
        const unsigned writers = __ballot_sync(0xffffffffu, kind == AMB_ES_KIND_AIR || kind == AMB_ES_KIND_SURF) & peers;
        const unsigned surfw = __ballot_sync(0xffffffffu, kind == AMB_ES_KIND_SURF) & peers;
        const unsigned before = writers & lt, sbefore = surfw & lt;
        const int src_a = before ? 31 - __clz(before) : (int)lane;
        const int src_c = sbefore ? 31 - __clz(sbefore) : (int)lane;
        AmbOpsSlot ref;
        ref.t_any = __shfl_sync(0xffffffffu, p.t, src_a);
        ref.any = __shfl_sync(0xffffffffu, p.lat, src_a);
        ref.t_surf = __shfl_sync(0xffffffffu, p.t, src_c);
        ref.surf = __shfl_sync(0xffffffffu, p.lon, src_c);
        if (kind == AMB_ES_KIND_POS) {
            AmbOpsSlot* s = &table[p.key];
            if (!before) { ref.t_any = __ldcg(&s->t_any); ref.any = __ldcg(&s->any); }       // the table, L2 only
            if (!sbefore) { ref.t_surf = __ldcg(&s->t_surf); ref.surf = __ldcg(&s->surf); }
            amb_es_position(&fields[k], (int)p.lat, (int)p.lon, p.t, &ref, max_age);
        }
        __syncwarp();                                           // every table read of this step is done
        if (writers && (int)lane == 31 - __clz(writers)) {       // the group's last writer keeps its version and NIC-A
            __stcg(&table[p.key].t_any, p.t); __stcg(&table[p.key].any, p.lat);
        }
        if (surfw && (int)lane == 31 - __clz(surfw)) {           // ... and its last surface writer its NIC-C
            __stcg(&table[p.key].t_surf, p.t); __stcg(&table[p.key].surf, p.lon);
        }
        __threadfence_block();
        __syncwarp();                                           // ... and visible to the next step's reads
    }
}

// Enqueue the stage (six kernels) after the Comm-B stage; `v` is the pairing stage's scratch, free again by then, `opos`
// the stage's key records. Returns how many kernels were launched or -1 with *err set.
static int amb_opstatus_launch(AmbV3Bufs* v, const amb_frame* frames, amb_fields* fields, const AmbPosRec* pos,
                               AmbPosRec* opos, int n, AmbOpsSlot* table, int max_age, cudaStream_t s, cudaError_t* err)
{
    AMB_LAUNCH((amb_opstatus_keys), (n + 127) / 128, 128, 0, s, frames, fields, pos, n, opos);
    if (amb_v3_partition(v, opos, n, s, err) < 0) return -1;
    AMB_LAUNCH((amb_opstatus_walk), AMB_V3_B / 4, 128, 0, s, opos, v->order, v->base, fields, table, max_age);
    *err = cudaGetLastError();
    return *err == cudaSuccess ? 6 : -1;
}
