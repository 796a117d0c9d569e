// Per-aircraft state table of the batch decoder (decoder option "track", DESIGN.md §8 "Aircraft table"). Runs after the
// local CPR stage, so that local fixes reach the table, and folds every counting record (status without
// AMB_FS_NOT_QUEUED / AMB_FS_NO_HANDLER) into one row per 24-bit address, in stream order. The rules are in
// include/airmodes_b200.h next to amb_aircraft. Rows are direct-mapped by address (AMB_TRACK_ROWS x 128 B, never
// cleared); an occupancy bitmap says which rows hold data, so that a reset only clears the bitmap.
//
//   amb_track_keys      one thread per frame: the record's address as key (AMB_NO_KEY when it does not count), its t
//                       and its frame's ref_level; one atomic per warp notes the latest queued record of the call
//   amb_v3_count .. amb_v3_scatter   the pairing stage's stable partition (amb_decode_v3.cuh), here on those keys
//   amb_track_walk      one warp per bucket, 32 records per step: same-address groups from __match_any_sync; expiry and
//                       creation resolved in lane order (= stream order); for each column only the last lane that carries
//                       a value writes it (the creator writes the blank when none does). A row has exactly one owner
//                       bucket: no probing, no row atomics.
// The snapshot (amb_decoder_aircraft) is three more kernels: amb_snap_count, amb_snap_scan, amb_snap_gather - count the
// rows to show per 1024 bitmap words, scan the counts, copy the rows out in ascending address.
#pragma once

#define AMB_TRACK_ROWS (1u << 24)
#define AMB_TRACK_WORDS (AMB_TRACK_ROWS / 32)       // occupancy bitmap, 2 MiB
#define AMB_SNAP_WORDS 1024                          // bitmap words per snapshot block (256 threads x 4)

// The latest queued record (for a snapshot at now = NaN): last_k = 1 + its index in the current call, 0 = none yet;
// the walk turns it into last_t.
struct AmbTrackClock { double last_t; unsigned last_k, pad_; };

// What a counting record carries into its row: one bit per column class. Every class has one writer per step.
#define AMB_TC_ALT 0x01      // altitude                       (AMB_AC_HAS_ALT)
#define AMB_TC_GND 0x02      // on ground or not, flag only    (AMB_AC_ON_GROUND)
#define AMB_TC_SQUAWK 0x04   // squawk                         (AMB_AC_HAS_SQUAWK)
#define AMB_TC_IDENT 0x08    // ident, ftc, cat                (AMB_AC_HAS_IDENT)
#define AMB_TC_POS 0x10      // lat, lon, pos_t, range, bearing (AMB_AC_HAS_POS, AMB_AC_HAS_RANGE)
#define AMB_TC_VEL 0x20      // speed, vertical                (AMB_AC_HAS_VELOCITY)
#define AMB_TC_HDG 0x40      // heading                        (AMB_AC_HAS_HEADING)
#define AMB_TC_EPS 0x80      // eps                            (AMB_AC_HAS_EPS)
#define AMB_TC_N 8

__device__ __forceinline__ unsigned amb_track_classes(const amb_fields* r)
{
    const int df = r->df;
    const bool ext = df == 17;
    const bool b05 = ext && r->bds == 0x05, b06 = ext && r->bds == 0x06;
    const bool b09 = ext && r->bds == 0x09 && (r->subtype == 0 || r->subtype == 1);
    unsigned c = 0;
    if (((df == 0 || df == 4 || df == 16 || df == 20 || b05) && r->altitude != AMB_NO_ALTITUDE) || b06) c |= AMB_TC_ALT;
    if (b05 || b06) c |= AMB_TC_GND;
    if (df == 5 || df == 21) c |= AMB_TC_SQUAWK;
    if (ext && r->bds == 0x08) c |= AMB_TC_IDENT;
    if (r->status & AMB_FS_HAS_POS) c |= AMB_TC_POS;
    if (b09) c |= AMB_TC_VEL | AMB_TC_HDG;
    if (b06) c |= AMB_TC_HDG;
    if (ext && r->bds == 0x61) c |= AMB_TC_EPS;
    return c;
}

// The row flags a class owns, and the ones this record sets among them.
__device__ __forceinline__ unsigned amb_track_owned(int q)
{
    switch (1u << q) {
    case AMB_TC_ALT: return AMB_AC_HAS_ALT;
    case AMB_TC_GND: return AMB_AC_ON_GROUND;
    case AMB_TC_SQUAWK: return AMB_AC_HAS_SQUAWK;
    case AMB_TC_IDENT: return AMB_AC_HAS_IDENT;
    case AMB_TC_POS: return AMB_AC_HAS_POS | AMB_AC_HAS_RANGE;
    case AMB_TC_VEL: return AMB_AC_HAS_VELOCITY;
    case AMB_TC_HDG: return AMB_AC_HAS_HEADING;
    default: return AMB_AC_HAS_EPS;
    }
}
__device__ __forceinline__ unsigned amb_track_flags(const amb_fields* r, unsigned classes)
{
    unsigned f = 0;
    if (classes & AMB_TC_ALT) f |= AMB_AC_HAS_ALT;
    if ((classes & AMB_TC_GND) && r->bds == 0x06) f |= AMB_AC_ON_GROUND;
    if (classes & AMB_TC_SQUAWK) f |= AMB_AC_HAS_SQUAWK;
    if (classes & AMB_TC_IDENT) f |= AMB_AC_HAS_IDENT;
    if (classes & AMB_TC_POS) f |= AMB_AC_HAS_POS | ((r->status & AMB_FS_HAS_RANGE) ? AMB_AC_HAS_RANGE : 0u);
    if (classes & AMB_TC_VEL) f |= AMB_AC_HAS_VELOCITY;
    if (classes & AMB_TC_HDG) f |= AMB_AC_HAS_HEADING;
    if (classes & AMB_TC_EPS) f |= AMB_AC_HAS_EPS;
    return f;
}

// The columns of class q: the record's values (r != nullptr) or the blank.
__device__ __forceinline__ void amb_track_write(amb_aircraft* row, int q, const amb_fields* r)
{
    switch (1u << q) {
    case AMB_TC_ALT: row->altitude = r ? (r->bds == 0x06 && r->df == 17 ? 0 : r->altitude) : AMB_NO_ALTITUDE; break;
    case AMB_TC_SQUAWK: row->squawk = r ? r->squawk : -1; break;
    case AMB_TC_IDENT:
        row->ftc = r ? (int8_t)r->ftc : (int8_t)-1;
        row->cat = r ? (int8_t)r->cat : (int8_t)-1;
        for (int j = 0; j < 8; j++) row->ident[j] = r ? r->ident[j] : 0;
        break;
    case AMB_TC_POS: {
        const bool rb = r && (r->status & AMB_FS_HAS_RANGE);
        row->lat = r ? r->lat : NAN; row->lon = r ? r->lon : NAN;
        row->range = rb ? r->range : NAN; row->bearing = rb ? r->bearing : NAN;
        break;                                              // pos_t is written by the caller: it is the lane's t
    }
    case AMB_TC_VEL: row->speed = r ? r->val[0] : NAN; row->vertical = r ? r->val[2] : NAN; break;
    case AMB_TC_HDG: row->heading = r ? (r->bds == 0x06 ? r->val[0] : r->val[1]) : NAN; break;
    case AMB_TC_EPS: row->eps = r ? (int8_t)r->eps : (int8_t)-1; break;
    default: break;                                         // AMB_TC_GND: a flag, written with the header
    }
}

__global__ void __launch_bounds__(128) amb_track_keys(const amb_frame* __restrict__ frames, const amb_fields* __restrict__ fields,
                                                      const AmbPosRec* __restrict__ pos, int n, AmbPosRec* __restrict__ tpos,
                                                      AmbTrackClock* clk)
{
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned st = k < n ? fields[k].status : (unsigned)AMB_FS_NOT_QUEUED;
    const unsigned queued = __ballot_sync(0xffffffffu, !(st & AMB_FS_NOT_QUEUED));
    if (queued && (int)(threadIdx.x & 31) == 31 - __clz(queued)) atomicMax(&clk->last_k, (unsigned)k + 1u);
    if (k >= n) return;
    const uint32_t a = fields[k].icao;
    AmbPosRec p;
    p.key = (st & (AMB_FS_NOT_QUEUED | AMB_FS_NO_HANDLER)) || a >= AMB_TRACK_ROWS ? AMB_NO_KEY : a;
    p.lat = __float_as_uint(frames[k].ref_level);          // the partition's record type; lat carries ref_level's bits
    p.lon = 0; p.fmt = 0;
    p.t = pos[k].t;                                         // secs + frac, as the pairing stage has it
    tpos[k] = p;
}

__global__ void __launch_bounds__(128) amb_track_walk(const AmbPosRec* __restrict__ tpos, const uint32_t* __restrict__ order,
                                                      const uint32_t* __restrict__ base, const amb_fields* __restrict__ fields,
                                                      amb_aircraft* rows, unsigned* occ, AmbTrackClock* clk, int max_age)
{
    if (blockIdx.x == 0 && threadIdx.x == 0 && clk->last_k) {   // amb_track_keys is complete: every atomic has landed
        clk->last_t = tpos[clk->last_k - 1].t;
        clk->last_k = 0;
    }
    const unsigned lane = threadIdx.x & 31;
    const unsigned b = blockIdx.x * 4 + (threadIdx.x >> 5);     // one warp per bucket; a row has one owner bucket
    const unsigned lo = base[b], hi = base[b + 1];
    for (unsigned i0 = lo; i0 < hi; i0 += 32) {
        const unsigned i = i0 + lane;
        const bool mine = i < hi;
        const int m = hi - i0 < 32 ? (int)(hi - i0) : 32;
        const int k = mine ? (int)order[i] : 0;
        const uint32_t a = mine ? tpos[k].key : 0u;
        const double t = mine ? tpos[k].t : 0.0;
        // the same aircraft inside this step; lanes past the end of the bucket get a private value (an address has 24 bits)
        const unsigned peers = __match_any_sync(0xffffffffu, mine ? a : (0x80000000u | lane));
        amb_aircraft* row = &rows[a];
        bool live = false;
        double seen = 0.0;
        if (mine) {
            live = (__ldcg(&occ[a >> 5]) >> (a & 31)) & 1u;   // L2, never a stale L1 line
            if (live) seen = __ldcg(&row->seen);
        }
        const int df = mine ? fields[k].df : 0;
        // Expiry and creation in lane order: lane j decides against the row its group's earlier lanes left, then every
        // member of its group takes the outcome over.
        bool applied = false, created = false;
        for (int j = 0; j < m; j++) {
            if ((int)lane == j && mine) {
                const bool alive = live && !(t - seen > (double)max_age);
                created = !alive && df == 17;
                applied = alive || created;
            }
            const int aj = __shfl_sync(0xffffffffu, (int)applied, j);
            const double tj = __shfl_sync(0xffffffffu, t, j);
            if (((peers >> j) & 1u) && aj) { live = true; seen = tj; }
        }
        const unsigned app = __ballot_sync(0xffffffffu, applied) & peers;
        const unsigned cre = __ballot_sync(0xffffffffu, created) & peers;
        const int c = cre ? 31 - __clz(cre) : -1;             // the last creator: what came before it is blanked
        const unsigned eff = c >= 0 ? (app & ~((1u << c) - 1u)) : app;   // the lanes whose values stay in the row
        const bool on = ((eff >> lane) & 1u) != 0;
        const amb_fields* r = &fields[k];
        const unsigned cls = on ? amb_track_classes(r) : 0u;
        const unsigned fl = on ? amb_track_flags(r, cls) : 0u;
        const double t_first = __shfl_sync(0xffffffffu, t, c >= 0 ? c : (int)lane);
        const int last = eff ? 31 - __clz(eff) : -1;
        unsigned flags = 0;
        if ((int)lane == last && c < 0) flags = __ldcg(&row->flags);   // no creation: the row's flags are the base
#pragma unroll
        for (int q = 0; q < AMB_TC_N; q++) {
            const unsigned carriers = __ballot_sync(0xffffffffu, (cls >> q) & 1u) & peers;
            const int w = carriers ? 31 - __clz(carriers) : c;
            const unsigned wf = __shfl_sync(0xffffffffu, fl, w >= 0 ? w : (int)lane);
            if (carriers) flags = (flags & ~amb_track_owned(q)) | (wf & amb_track_owned(q));
            if ((int)lane == w && eff) {
                amb_track_write(row, q, carriers ? r : nullptr);
                if ((1u << q) == AMB_TC_POS) row->pos_t = carriers ? t : NAN;
            }
        }
        if ((int)lane == c) {                                   // a new row: the rest of it, and its bit
            for (int j = 0; j < 15; j++) row->pad_[j] = 0;
            atomicOr(&occ[a >> 5], 1u << (a & 31));
        }
        if ((int)lane == last) {
            const unsigned msgs = (c >= 0 ? 0u : __ldcg(&row->messages)) + (unsigned)__popc(eff);
            if (c >= 0) row->first_seen = t_first;
            row->icao = a;
            row->messages = msgs;
            row->seen = t;
            *reinterpret_cast<uint32_t*>(&row->ref_level) = tpos[k].lat;
            row->flags = (uint16_t)flags;
        }
        __threadfence_block();
        __syncwarp();                                           // every write of this step is visible to the next step
    }
}

// Enqueue the stage (six kernels) after the decode (and the local CPR stage); `v` is the pairing stage's scratch, free
// again by then, `tpos` the stage's key records. Returns how many kernels were launched or -1 with *err set.
static int amb_track_launch(AmbV3Bufs* v, const amb_frame* frames, const amb_fields* fields, const AmbPosRec* pos,
                            AmbPosRec* tpos, int n, amb_aircraft* rows, unsigned* occ, AmbTrackClock* clk, int max_age,
                            cudaStream_t s, cudaError_t* err)
{
    AMB_LAUNCH((amb_track_keys), (n + 127) / 128, 128, 0, s, frames, fields, pos, n, tpos, clk);
    if (amb_v3_partition(v, tpos, n, s, err) < 0) return -1;
    AMB_LAUNCH((amb_track_walk), AMB_V3_B / 4, 128, 0, s, tpos, v->order, v->base, fields, rows, occ, clk, max_age);
    *err = cudaGetLastError();
    return *err == cudaSuccess ? 6 : -1;
}

// ---- snapshot ---------------------------------------------------------------------------------------------------------
__device__ __forceinline__ bool amb_track_shown(const amb_aircraft* rows, unsigned a, double now, int max_age)
{
    const double s = rows[a].seen;
    return s <= now && now - s <= (double)max_age;
}

// Rows to show among this thread's four bitmap words, and their exclusive prefix over the 256 threads of the block.
// Static, so that each library compiled from this header - and each host-emulated one, where the __shared__ array
// becomes a function-local static - calls its own copy.
static __device__ __forceinline__ unsigned amb_snap_thread(const unsigned* occ, const amb_aircraft* rows, const AmbTrackClock* clk,
                                                    double now, int max_age, unsigned* before)
{
    __shared__ unsigned ws[8];
    const double nw = now == now ? now : clk->last_t;      // NaN: the latest queued record decoded since reset
    const unsigned w0 = (blockIdx.x * 256 + threadIdx.x) * 4;
    unsigned cnt = 0;
    for (int q = 0; q < 4; q++) {
        unsigned bits = occ[w0 + q];
        while (bits) {
            const unsigned a = (w0 + q) * 32 + (unsigned)(__ffs(bits) - 1);
            bits &= bits - 1;
            cnt += amb_track_shown(rows, a, nw, max_age) ? 1u : 0u;
        }
    }
    const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned x = cnt;
    for (int d = 1; d < 32; d <<= 1) {
        const unsigned y = __shfl_up_sync(0xffffffffu, x, d);
        if ((int)lane >= d) x += y;
    }
    if (lane == 31) ws[warp] = x;
    __syncthreads();
    unsigned pre = 0;
    for (unsigned w = 0; w < warp; w++) pre += ws[w];
    *before = pre + x - cnt;
    const unsigned total = ws[0] + ws[1] + ws[2] + ws[3] + ws[4] + ws[5] + ws[6] + ws[7];
    __syncthreads();
    return total;
}

__global__ void __launch_bounds__(256) amb_snap_count(const unsigned* __restrict__ occ, const amb_aircraft* __restrict__ rows,
                                                      const AmbTrackClock* __restrict__ clk, double now, int max_age,
                                                      uint32_t* __restrict__ cnt)
{
    unsigned before;
    const unsigned total = amb_snap_thread(occ, rows, clk, now, max_age, &before);
    if (threadIdx.x == 0) cnt[blockIdx.x] = total;
}

// one CTA of 1024 threads: exclusive scan of nb <= 1024 block counts -> off[0 .. nb), off[nb] = the total
__global__ void __launch_bounds__(1024) amb_snap_scan(const uint32_t* __restrict__ cnt, int nb, uint32_t* __restrict__ off)
{
    __shared__ unsigned wsum[32];
    const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned v = (int)threadIdx.x < nb ? cnt[threadIdx.x] : 0u;
    unsigned x = v;
    for (int d = 1; d < 32; d <<= 1) {
        const unsigned y = __shfl_up_sync(0xffffffffu, x, d);
        if ((int)lane >= d) x += y;
    }
    if (lane == 31) wsum[warp] = x;
    __syncthreads();
    unsigned pre = 0;
    for (unsigned w = 0; w < warp; w++) pre += wsum[w];
    if ((int)threadIdx.x < nb) off[threadIdx.x] = pre + x - v;
    if (threadIdx.x == 1023) off[nb] = pre + x;
}

__global__ void __launch_bounds__(256) amb_snap_gather(const unsigned* __restrict__ occ, const amb_aircraft* __restrict__ rows,
                                                       const AmbTrackClock* __restrict__ clk, double now, int max_age,
                                                       const uint32_t* __restrict__ off, amb_aircraft* __restrict__ out)
{
    unsigned before;
    amb_snap_thread(occ, rows, clk, now, max_age, &before);
    const double nw = now == now ? now : clk->last_t;
    unsigned o = off[blockIdx.x] + before;
    const unsigned w0 = (blockIdx.x * 256 + threadIdx.x) * 4;
    for (int q = 0; q < 4; q++) {
        unsigned bits = occ[w0 + q];
        while (bits) {
            const unsigned a = (w0 + q) * 32 + (unsigned)(__ffs(bits) - 1);
            bits &= bits - 1;
            if (!amb_track_shown(rows, a, nw, max_age)) continue;
            const uint4* src = reinterpret_cast<const uint4*>(&rows[a]);
            uint4* dst = reinterpret_cast<uint4*>(&out[o++]);
            for (int j = 0; j < 8; j++) dst[j] = src[j];
        }
    }
}

// Count the rows a snapshot at `now` shows, over `words` bitmap words (a multiple of AMB_SNAP_WORDS, at most 1024 of
// them): cnt[] gets the per-block counts, off[] their scan, off[words / AMB_SNAP_WORDS] the total. Two kernels.
static int amb_snap_count_launch(const unsigned* occ, const amb_aircraft* rows, const AmbTrackClock* clk, double now,
                                 int max_age, unsigned words, uint32_t* cnt, uint32_t* off, cudaStream_t s, cudaError_t* err)
{
    const int nb = (int)(words / AMB_SNAP_WORDS);
    AMB_LAUNCH((amb_snap_count), nb, 256, 0, s, occ, rows, clk, now, max_age, cnt);
    AMB_LAUNCH((amb_snap_scan), 1, 1024, 0, s, cnt, nb, off);
    *err = cudaGetLastError();
    return *err == cudaSuccess ? 2 : -1;
}

// Copy the counted rows to out[0 .. total) in ascending address. One kernel.
static int amb_snap_gather_launch(const unsigned* occ, const amb_aircraft* rows, const AmbTrackClock* clk, double now,
                                  int max_age, unsigned words, const uint32_t* off, amb_aircraft* out, cudaStream_t s,
                                  cudaError_t* err)
{
    AMB_LAUNCH((amb_snap_gather), (int)(words / AMB_SNAP_WORDS), 256, 0, s, occ, rows, clk, now, max_age, off, out);
    *err = cudaGetLastError();
    return *err == cudaSuccess ? 1 : -1;
}
