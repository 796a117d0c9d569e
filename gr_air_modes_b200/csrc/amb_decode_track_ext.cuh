// Extension of the per-aircraft table (decoder option "track_ext", DESIGN.md §8 "Aircraft table extension"). Runs
// after the track stage while both options are on. Every queued record that the op-status or the Comm-B stage decoded
// writes one of six groups of its address's extension row (amb_aircraft_ext in include/airmodes_b200.h, where the rules
// are): a copy of its aux / pad_ bytes and its t. Rows are direct-mapped by address (AMB_TRACK_ROWS x 144 B, never
// cleared); an occupancy bitmap says which rows were written since reset, and a row whose bit is clear is never read.
//
//   amb_track_ext_keys  one thread per frame: key = icao for a record that writes a group, AMB_NO_KEY otherwise; fmt =
//                       the group
//   amb_v3_count .. amb_v3_scatter   the pairing stage's stable partition (amb_decode_v3.cuh), here on those keys
//   amb_track_ext_walk  one warp per bucket, 32 records per step: same-address groups from __match_any_sync; for each
//                       group the last lane of the address that writes it copies its record. No chains and no table
//                       reads but the bitmap: one pass per step. A row has exactly one owner bucket: no row atomics.
// The snapshot (amb_decoder_aircraft_ext) is amb_snap_count and amb_snap_scan of the track stage, as they are, and
// amb_snap_gather_ext, which writes the base rows and their extensions.
#pragma once

#define AMB_AXG_NONE 0xFFu

// The helpers below are static: the SIMT host emulator turns __shared__ into function-local statics and threadIdx into
// per-library state, so a helper with external linkage could bind to another library's copy.

// The group a record writes (AMB_AXG_* bit index), or AMB_AXG_NONE.
static __device__ __forceinline__ unsigned amb_track_ext_group(const amb_fields* r)
{
    if (r->status & AMB_FS_NOT_QUEUED) return AMB_AXG_NONE;
    const unsigned es = AMB_FIELDS_ES(r), cb = AMB_FIELDS_COMMB(r), reg = AMB_FIELDS_COMMB_REG(r);
    if (es == AMB_ES_OPSTATUS) return 0;
    if (es == AMB_ES_TARGET_STATE) return 1;
    if ((es == AMB_ES_NIC || es == AMB_ES_NUC) && (r->status & AMB_FS_HAS_POS)) return 2;
    if (cb != AMB_COMMB_DECODED && cb != AMB_COMMB_RESOLVED) return AMB_AXG_NONE;
    return reg == 0x40 ? 3 : reg == 0x50 ? 4 : reg == 0x60 ? 5 : AMB_AXG_NONE;
}

// Group g of row x := the record r of time t.
static __device__ __forceinline__ void amb_track_ext_copy(amb_aircraft_ext* x, unsigned g, const amb_fields* r, double t)
{
    x->t[g] = t;
    switch (g) {
    case 0:
        for (int j = 0; j < 4; j++) x->ops[j] = r->aux[j];
        x->ops_version = AMB_FIELDS_ES_VERSION(r);
        break;
    case 1:
        for (int j = 0; j < 4; j++) x->ts[j] = r->aux[j];
        break;
    case 2:
        for (int j = 0; j < 2; j++) x->integ[j] = r->aux[j];
        x->integ_es = AMB_FIELDS_ES(r);
        x->integ_version = AMB_FIELDS_ES_VERSION(r);
        x->integ_nic = AMB_FIELDS_ES_NIC(r);
        break;
    default: {
        const unsigned c = g - 3;
        for (int i = 0; i < 5; i++) x->commb[c][i] = AMB_FIELDS_COMMB_RAW(r, i);
        x->commb_mask[c] = AMB_FIELDS_COMMB_MASK(r);
        x->commb_outcome[c] = AMB_FIELDS_COMMB(r);
        break;
    }
    }
}

__global__ void __launch_bounds__(128) amb_track_ext_keys(const amb_fields* __restrict__ fields, const AmbPosRec* __restrict__ pos,
                                                          int n, AmbPosRec* __restrict__ xpos)
{
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    amb_fields r = fields[k];
    const unsigned g = amb_track_ext_group(&r);
    AmbPosRec p;
    p.key = g != AMB_AXG_NONE && r.icao < AMB_TRACK_ROWS ? r.icao : AMB_NO_KEY;
    p.fmt = g;
    p.lat = p.lon = 0;
    p.t = pos[k].t;                                         // secs + frac, as the pairing stage has it
    xpos[k] = p;
}

__global__ void __launch_bounds__(128) amb_track_ext_walk(const AmbPosRec* __restrict__ xpos, const uint32_t* __restrict__ order,
                                                          const uint32_t* __restrict__ base, const amb_fields* __restrict__ fields,
                                                          amb_aircraft_ext* rows, unsigned* occ)
{
    const unsigned lane = threadIdx.x & 31;
    const unsigned b = blockIdx.x * 4 + (threadIdx.x >> 5);     // one warp per bucket; a row has one owner bucket
    const unsigned lo = base[b], hi = base[b + 1];
    for (unsigned i0 = lo; i0 < hi; i0 += 32) {
        const unsigned i = i0 + lane;
        const bool mine = i < hi;
        const int k = mine ? (int)order[i] : 0;
        const uint32_t a = mine ? xpos[k].key : 0u;
        const unsigned g = mine ? xpos[k].fmt : AMB_AXG_NONE;
        // the same address inside this step; lanes past the end of the bucket get a private value (an address has 24 bits)
        const unsigned peers = __match_any_sync(0xffffffffu, mine ? a : (0x80000000u | lane));
        unsigned wrote = 0;                                     // the groups this step writes for the address
        bool last = false;                                      // this lane is the last writer of its group
#pragma unroll
        for (unsigned q = 0; q < AMB_AXG_N; q++) {
            const unsigned w = __ballot_sync(0xffffffffu, g == q) & peers;
            if (w) wrote |= 1u << q;
            if (g == q && (int)lane == 31 - __clz(w)) last = true;
        }
        amb_aircraft_ext* row = &rows[a];
        if (mine && (int)lane == __ffs(peers) - 1 && !((__ldcg(&occ[a >> 5]) >> (a & 31)) & 1u)) {
            // first write since reset: the groups this step leaves alone have never been written
            for (unsigned q = 0; q < AMB_AXG_N; q++)
                if (!((wrote >> q) & 1u)) row->t[q] = NAN;
            atomicOr(&occ[a >> 5], 1u << (a & 31));
        }
        if (last) amb_track_ext_copy(row, g, &fields[k], xpos[k].t);
        __threadfence_block();
        __syncwarp();                                           // every write of this step is visible to the next step
    }
}

// Enqueue the stage (six kernels) after the track stage; `v` is the pairing stage's scratch, free again by then, `xpos`
// the stage's key records. Returns how many kernels were launched or -1 with *err set.
static int amb_track_ext_launch(AmbV3Bufs* v, const amb_fields* fields, const AmbPosRec* pos, AmbPosRec* xpos, int n,
                                amb_aircraft_ext* rows, unsigned* occ, cudaStream_t s, cudaError_t* err)
{
    AMB_LAUNCH((amb_track_ext_keys), (n + 127) / 128, 128, 0, s, fields, pos, n, xpos);
    if (amb_v3_partition(v, xpos, n, s, err) < 0) return -1;
    AMB_LAUNCH((amb_track_ext_walk), AMB_V3_B / 4, 128, 0, s, xpos, v->order, v->base, fields, rows, occ);
    *err = cudaGetLastError();
    return *err == cudaSuccess ? 6 : -1;
}

// ---- snapshot ---------------------------------------------------------------------------------------------------------
// The extension of a shown base row (address a, created at `first`) at `now`: a group is shown when its t lies in
// [first, now] and now - t <= max_age; whatever is not shown is NaN (times) or 0.
static __device__ __forceinline__ void amb_track_ext_out(const amb_aircraft_ext* x, bool live, unsigned a, double first,
                                                  double now, int max_age, amb_aircraft_ext* o)
{
    unsigned shown = 0;
#pragma unroll
    for (int q = 0; q < AMB_AXG_N; q++) {
        const double t = live ? x->t[q] : NAN;
        if (t >= first && t <= now && now - t <= (double)max_age) shown |= 1u << q;
    }
    const bool ops = shown & AMB_AXG_OPS, ts = shown & AMB_AXG_TS, integ = shown & AMB_AXG_INTEG;
    o->icao = a;
    o->shown = (uint8_t)shown;
    o->ops_version = ops ? x->ops_version : 0;
    o->integ_es = integ ? x->integ_es : 0;
    o->integ_version = integ ? x->integ_version : 0;
#pragma unroll
    for (int q = 0; q < AMB_AXG_N; q++) o->t[q] = (shown >> q) & 1u ? x->t[q] : NAN;
    for (int j = 0; j < 4; j++) {
        o->ops[j] = ops ? x->ops[j] : 0u;
        o->ts[j] = ts ? x->ts[j] : 0u;
    }
    for (int j = 0; j < 2; j++) o->integ[j] = integ ? x->integ[j] : 0u;
    o->integ_nic = integ ? x->integ_nic : 0;
    for (int c = 0; c < 3; c++) {
        const bool on = (shown >> (3 + c)) & 1u;
        o->commb_mask[c] = on ? x->commb_mask[c] : 0;
        o->commb_outcome[c] = on ? x->commb_outcome[c] : 0;
        for (int i = 0; i < 5; i++) o->commb[c][i] = on ? x->commb[c][i] : (int16_t)0;
    }
    o->pad0_ = 0;
    for (int j = 0; j < 10; j++) o->pad_[j] = 0;
}

// amb_snap_gather, and beside every row its extension (xocc == nullptr: nothing written yet, every group hidden).
__global__ void __launch_bounds__(256) amb_snap_gather_ext(const unsigned* __restrict__ occ, const amb_aircraft* __restrict__ rows,
                                                           const AmbTrackClock* __restrict__ clk, double now, int max_age,
                                                           const uint32_t* __restrict__ off, amb_aircraft* __restrict__ out,
                                                           const unsigned* __restrict__ xocc,
                                                           const amb_aircraft_ext* __restrict__ xrows, int ext_age,
                                                           amb_aircraft_ext* __restrict__ ext)
{
    unsigned before;
    amb_snap_thread(occ, rows, clk, now, max_age, &before);
    const double nw = now == now ? now : clk->last_t;
    unsigned o = off[blockIdx.x] + before;
    const unsigned w0 = (blockIdx.x * 256 + threadIdx.x) * 4;
    for (int q = 0; q < 4; q++) {
        unsigned bits = occ[w0 + q];
        const unsigned xbits = xocc ? xocc[w0 + q] : 0u;
        while (bits) {
            const unsigned j = (unsigned)(__ffs(bits) - 1), a = (w0 + q) * 32 + j;
            bits &= bits - 1;
            if (!amb_track_shown(rows, a, nw, max_age)) continue;
            const uint4* src = reinterpret_cast<const uint4*>(&rows[a]);
            uint4* dst = reinterpret_cast<uint4*>(&out[o]);
            for (int i = 0; i < 8; i++) dst[i] = src[i];
            amb_track_ext_out(&xrows[a], (xbits >> j) & 1u, a, rows[a].first_seen, nw, ext_age, &ext[o]);
            o++;
        }
    }
}

// Copy the counted rows (amb_snap_count_launch) to out[0 .. total) and their extensions to ext[0 .. total), in
// ascending address. One kernel.
static int amb_snap_gather_ext_launch(const unsigned* occ, const amb_aircraft* rows, const AmbTrackClock* clk, double now,
                                      int max_age, unsigned words, const uint32_t* off, amb_aircraft* out,
                                      const unsigned* xocc, const amb_aircraft_ext* xrows, int ext_age,
                                      amb_aircraft_ext* ext, cudaStream_t s, cudaError_t* err)
{
    AMB_LAUNCH((amb_snap_gather_ext), (int)(words / AMB_SNAP_WORDS), 256, 0, s, occ, rows, clk, now, max_age, off, out,
               xocc, xrows, ext_age, ext);
    *err = cudaGetLastError();
    return *err == cudaSuccess ? 1 : -1;
}
