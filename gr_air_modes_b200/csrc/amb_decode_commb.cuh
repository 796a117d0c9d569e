// Comm-B register inference of the batch decoder (decoder option "commb", DESIGN.md §8 "Comm-B inference"). Runs after
// the resolve and local CPR stages and before the track stage. A DF20/21 reply whose MB word the parser does not handle
// (AMB_FS_NO_HANDLER) is tested against the layouts of BDS 4,0 / 5,0 / 6,0 (amb_commb_* in amb_decode_core.h); when
// several fit and 5,0 is one of them, the address's latest ADS-B velocity (DF17 BDS0,9 subtype 0/1) decides. That
// reference is kept in a direct-mapped table in HBM (AMB_COMMB_SLOTS x 24 B, one slot per address) across calls:
//
//   amb_commb_keys      one thread per frame: the structural test; every outcome that needs no reference is written at
//                       once; key = icao for velocity records (writers, fmt 1) and for records that need a reference
//                       (fmt 2), AMB_NO_KEY otherwise
//   amb_v3_count .. amb_v3_scatter   the pairing stage's stable partition (amb_decode_v3.cuh), here on those keys
//   amb_commb_walk      one warp per bucket, 32 records per step: same-address groups from __match_any_sync; a record
//                       that needs a reference takes the last earlier writer of its group, or the table when there is
//                       none; the last writer of each group writes the slot. No chains: one pass per step. A slot has
//                       exactly one owner bucket: no probing, no atomics.
#pragma once

#define AMB_COMMB_SLOTS (1ull << 24)
#define AMB_COMMB_WRITER 1u
#define AMB_COMMB_NEEDER 2u

__global__ void __launch_bounds__(128) amb_commb_keys(const amb_frame* __restrict__ frames, amb_fields* __restrict__ fields,
                                                      const AmbPosRec* __restrict__ pos, int n, AmbPosRec* __restrict__ cpos)
{
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    amb_fields* r = &fields[k];
    AmbPosRec p;
    p.key = AMB_NO_KEY; p.lat = p.lon = 0; p.fmt = 0;
    p.t = pos[k].t;                                         // secs + frac, as the pairing stage has it
    const bool in_table = r->icao < AMB_COMMB_SLOTS;       // an address or AP syndrome has 24 bits
    if (amb_commb_is_ref(r)) {
        p.fmt = AMB_COMMB_WRITER;
    } else if (amb_commb_eligible(frames[k], r)) {
        const uint64_t mb = amb_commb_mb(frames[k]);
        if (in_table && amb_commb_needs_ref(mb, amb_commb_candidates(mb))) {
            p.fmt = AMB_COMMB_NEEDER;
        } else {
            const AmbCommbRef none = {NAN, NAN, NAN};
            amb_commb_step(r, mb, p.t, &none, 0);           // final without a reference
        }
    }
    if (p.fmt && in_table) p.key = r->icao;
    cpos[k] = p;
}

__global__ void __launch_bounds__(128) amb_commb_walk(const AmbPosRec* __restrict__ cpos, const uint32_t* __restrict__ order,
                                                      const uint32_t* __restrict__ base, const amb_frame* __restrict__ frames,
                                                      amb_fields* __restrict__ fields, AmbCommbRef* table, int max_age)
{
    const unsigned lane = threadIdx.x & 31;
    const unsigned b = blockIdx.x * 4 + (threadIdx.x >> 5);     // one warp per bucket; a table slot has one owner bucket
    const unsigned lt = (1u << lane) - 1u;
    const unsigned lo = base[b], hi = base[b + 1];
    for (unsigned i0 = lo; i0 < hi; i0 += 32) {
        const unsigned i = i0 + lane;
        const bool mine = i < hi;
        const int k = mine ? (int)order[i] : 0;
        const uint32_t a = mine ? cpos[k].key : 0u;
        const double t = mine ? cpos[k].t : 0.0;
        const unsigned kind = mine ? cpos[k].fmt : 0u;
        // the same address inside this step; lanes past the end of the bucket get a private value (an address has 24 bits)
        const unsigned peers = __match_any_sync(0xffffffffu, mine ? a : (0x80000000u | lane));
        const unsigned writers = __ballot_sync(0xffffffffu, kind == AMB_COMMB_WRITER) & peers;
        AmbCommbRef mine_ref = {t, NAN, NAN};
        if (kind == AMB_COMMB_WRITER) { mine_ref.speed = fields[k].val[0]; mine_ref.track = fields[k].val[1]; }
        const unsigned before = writers & lt;
        const int src = before ? 31 - __clz(before) : (int)lane;
        AmbCommbRef ref;
        ref.t = __shfl_sync(0xffffffffu, mine_ref.t, src);
        ref.speed = __shfl_sync(0xffffffffu, mine_ref.speed, src);
        ref.track = __shfl_sync(0xffffffffu, mine_ref.track, src);
        if (kind == AMB_COMMB_NEEDER) {
            if (!before) {                                      // no earlier writer in this step: the table, L2 only
                const double* s = &table[a].t;
                ref.t = __ldcg(s); ref.speed = __ldcg(s + 1); ref.track = __ldcg(s + 2);
            }
            amb_commb_step(&fields[k], amb_commb_mb(frames[k]), t, &ref, max_age);
        }
        __syncwarp();                                           // every table read of this step is done
        if (kind == AMB_COMMB_WRITER && (int)lane == 31 - __clz(writers)) {   // the group's last writer keeps its velocity
            double* s = &table[a].t;
            __stcg(s, mine_ref.t); __stcg(s + 1, mine_ref.speed); __stcg(s + 2, mine_ref.track);
            __threadfence_block();
        }
        __syncwarp();                                           // ... and visible to the next step's reads
    }
}

// Enqueue the stage (six kernels) after the decode and the local CPR stage; `v` is the pairing stage's scratch, free
// again by then, `cpos` the stage's key records. Returns how many kernels were launched or -1 with *err set.
static int amb_commb_launch(AmbV3Bufs* v, const amb_frame* frames, amb_fields* fields, const AmbPosRec* pos, AmbPosRec* cpos,
                            int n, AmbCommbRef* table, int max_age, cudaStream_t s, cudaError_t* err)
{
    AMB_LAUNCH((amb_commb_keys), (n + 127) / 128, 128, 0, s, frames, fields, pos, n, cpos);
    if (amb_v3_partition(v, cpos, n, s, err) < 0) return -1;
    AMB_LAUNCH((amb_commb_walk), AMB_V3_B / 4, 128, 0, s, cpos, v->order, v->base, frames, fields, table, max_age);
    *err = cudaGetLastError();
    return *err == cudaSuccess ? 6 : -1;
}
