// SBS-1 (BaseStation) feed (decoder option "sbs1", DESIGN.md §8 "SBS-1 feed"). Runs last, after every other stage, so
// that local CPR fixes reach the lines; it reads the records and writes nothing into them. Every published record
// (amb_sbs1_published) takes an aircraft id in stream order, as output_sbs1.get_aircraft_id does (sbs1.py:73-90), and
// writes its line (amb_sbs1_line, amb_sbs1_format.h); the lines of one call are packed into one buffer in record order.
//
// Ids: G counts every id handed out since the decoder was made and is never reset; amb_decoder_reset records base = G.
// A record whose address holds id g (a global value) before it reuses g when g > base and g + 10000 > G (the window
// of sbs1.py:83-88, G the counter before the record), and otherwise takes G + 1. The latest g of each address lives in
// a direct-mapped table (2^24 x 8 B, 0 = none) carried from call to call.
//
//   amb_sbs1_keys    one thread per frame: key = icao of a published record, AMB_NO_KEY otherwise; clears the call's
//                    look-back flags and ticket
//   amb_v3_count .. amb_v3_scatter   the pairing stage's stable partition (amb_decode_v3.cuh), on those keys
//   amb_sbs1_walk    one warp per bucket, 32 records per step: each record learns where its address's previous id comes
//                    from - the latest earlier lane of its address (__match_any_sync), else the table slot, which holds
//                    either the id of an earlier call or MARK | the index of this call's latest record of the address
//                    (the walk leaves that mark; amb_sbs1_format puts the id back). A slot has one owner bucket.
//   amb_sbs1_ids     a single-pass chained scan over 1024-record chunks of stream order (atomic ticket for the chunk
//                    order, look-back on the previous chunk's flag). Whether a record needs a new id depends on G at its
//                    position, so a chunk's total depends on its carry: a chunk first tests whether any of its first
//                    occurrences lies near the window edge; if none does, every record is settled at once (block scan
//                    and pointer jumping), otherwise its warps settle their lanes one after another. Each record's id
//                    is written before the chunk publishes its G, so a later record of the same address reads it.
//   amb_sbs1_format  one thread per frame: the line into a fixed-stride slot, its length, the block's byte count
//   amb_sbs1_scan    one block: the byte offset of every block of lines, and the total
//   amb_sbs1_gather  one thread per frame: its line at its byte offset
#pragma once
#include "amb_sbs1_format.h"

#define AMB_SBS1_MARK (1ull << 63)
#define AMB_SBS1_CHUNK 1024
#define AMB_SBS1_SLOTS (1u << 24)                // one id slot per 24-bit address

#ifdef AMB_SIMT_EMUL
static inline void __threadfence() {}                // the emulator's fibers share one OS thread: every store is visible
#endif

// Device-resident counter of the stage, kept across calls.
struct AmbSbs1Ctr {
    unsigned long long G;        // ids handed out since the decoder was made
    unsigned long long base;     // G at the last amb_decoder_reset
    unsigned ticket, pad_;       // next chunk of the running call
};

// The stage's per-call scratch (n frames).
struct AmbSbs1Bufs {
    unsigned long long* src = nullptr;   // per record: MARK | index of the address's previous record, or its table g
    unsigned long long* gid = nullptr;   // per record: its global id
    unsigned long long* flag = nullptr;  // per chunk: (G after the chunk << 1) | 1 once it is settled, 0 before
    char* slots = nullptr;               // per record: AMB_SBS1_STRIDE bytes
    uint32_t* len = nullptr;             // per record: bytes of its line
    uint32_t* bsum = nullptr;            // per block of 128 records: bytes of its lines
    unsigned long long* boff = nullptr;  // per block: byte offset of its lines; [blocks] = the total
    char* text = nullptr;                // the packed lines
};

static __device__ __forceinline__ bool amb_sbs1_live(unsigned long long g, unsigned long long G, unsigned long long base)
{
    return g > base && g + AMB_SBS1_WINDOW > G;
}

__global__ void __launch_bounds__(128) amb_sbs1_keys(const amb_fields* __restrict__ fields, int n, AmbPosRec* __restrict__ keys,
                                                     unsigned long long* __restrict__ flag, int chunks, AmbSbs1Ctr* ctr)
{
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    amb_fields r = fields[k];
    AmbPosRec p;
    p.key = amb_sbs1_published(&r) ? r.icao : AMB_NO_KEY;
    p.lat = p.lon = p.fmt = 0;
    p.t = 0.0;
    keys[k] = p;
    if (k < chunks) flag[k] = 0ull;
    if (k == 0) ctr->ticket = 0u;
}

__global__ void __launch_bounds__(128) amb_sbs1_walk(const AmbPosRec* __restrict__ keys, const uint32_t* __restrict__ order,
                                                     const uint32_t* __restrict__ base, unsigned long long* table,
                                                     unsigned long long* __restrict__ src)
{
    const unsigned lane = threadIdx.x & 31;
    const unsigned b = blockIdx.x * 4 + (threadIdx.x >> 5);     // one warp per bucket; a slot has one owner bucket
    const unsigned lo = base[b], hi = base[b + 1];
    for (unsigned i0 = lo; i0 < hi; i0 += 32) {
        const unsigned i = i0 + lane;
        const bool mine = i < hi;
        const unsigned k = mine ? order[i] : 0u;
        const uint32_t a = mine ? keys[k].key : 0u;
        const unsigned long long slot = mine ? __ldcg(&table[a]) : 0ull;
        // the same address inside this step; lanes past the end of the bucket get a private value (an address has 24 bits)
        const unsigned peers = __match_any_sync(0xffffffffu, mine ? a : (0x80000000u | lane));
        const unsigned before = peers & ((1u << lane) - 1u), later = peers & ~((2u << lane) - 1u);
        const int prev = before ? 31 - __clz(before) : (int)lane;
        const unsigned pk = __shfl_sync(0xffffffffu, k, prev);
        __syncwarp();                                           // every lane has read its slot before the marks below
        if (mine) {
            src[k] = before ? (AMB_SBS1_MARK | pk) : slot;
            if (!later) table[a] = AMB_SBS1_MARK | k;
        }
        __threadfence_block();
        __syncwarp();                                           // this step's marks are visible to the next step
    }
}

__global__ void __launch_bounds__(AMB_SBS1_CHUNK) amb_sbs1_ids(const AmbPosRec* __restrict__ keys,
                                                               const unsigned long long* __restrict__ src, int n,
                                                               unsigned long long* gid, AmbSbs1Ctr* ctr,
                                                               unsigned long long* flag)
{
    __shared__ unsigned s_chunk, s_amb, s_wnew[32];
    __shared__ unsigned long long s_G;
    __shared__ unsigned long long s_id[AMB_SBS1_CHUNK];
    __shared__ unsigned short s_root[AMB_SBS1_CHUNK];
    const unsigned t = threadIdx.x, lane = t & 31, warp = t >> 5;
    if (t == 0) { s_chunk = atomicAdd(&ctr->ticket, 1u); s_amb = 0u; }
    __syncthreads();
    const unsigned c = s_chunk;
    const int k = (int)(c * AMB_SBS1_CHUNK + t);
    const bool pub = k < n && keys[k].key != AMB_NO_KEY;
    const uint32_t a = pub ? keys[k].key : (0x80000000u | lane);
    const unsigned long long s = pub ? src[k] : 0ull;
    const unsigned first = c * AMB_SBS1_CHUNK;
    const bool marked = pub && (s & AMB_SBS1_MARK);
    const unsigned p = (unsigned)s;                             // the previous record, when marked
    const int q = marked && p >= first ? (int)(p - first) : -1; // ... when it is in this chunk: its thread
    if (t == 0) {                                               // G before the chunk
        unsigned long long G;
        if (c == 0) G = ctr->G;
        else {
            const volatile unsigned long long* f = &flag[c - 1];
            while ((G = *f) == 0ull) {}
            G >>= 1;
        }
        __threadfence();
        s_G = G;
    }
    __syncthreads();
    const unsigned long long G0 = s_G, base = ctr->base;
    unsigned long long g = 0ull;                                // the address's id before this record (0: none)
    if (pub && q < 0) g = marked ? __ldcg(&gid[p]) : s;         // an earlier chunk wrote it before its flag
    // A first occurrence in the chunk is settled now unless the window edge can pass it inside the chunk.
    if (pub && q < 0 && amb_sbs1_live(g, G0, base) != amb_sbs1_live(g, G0 + AMB_SBS1_CHUNK, base)) s_amb = 1u;
    __syncthreads();
    unsigned long long id = 0ull;
    if (!s_amb) {
        // Nothing expires inside the chunk: first occurrences are new iff their id is dead at G0, and every later
        // occurrence reuses the id of its address's first occurrence (live for at least 10000 - 1024 more ids).
        const bool nw = pub && q < 0 && !amb_sbs1_live(g, G0, base);
        const unsigned bal = __ballot_sync(0xffffffffu, nw);
        if (lane == 0) s_wnew[warp] = __popc(bal);
        unsigned r = q < 0 ? t : (unsigned)q;
        s_root[t] = (unsigned short)r;
        __syncthreads();
        unsigned rank = __popc(bal & ((1u << lane) - 1u));
        for (unsigned w = 0; w < warp; w++) rank += s_wnew[w];
        for (int j = 0; j < 10; j++) {                          // pointer jumping: root of the chain of predecessors
            r = s_root[r];
            __syncthreads();
            s_root[t] = (unsigned short)r;
            __syncthreads();
        }
        if (q < 0) s_id[t] = nw ? G0 + rank + 1 : g;
        __syncthreads();
        id = s_id[r];
        if (t == AMB_SBS1_CHUNK - 1) {
            unsigned tot = 0;
            for (unsigned w = 0; w < 32; w++) tot += s_wnew[w];
            s_G = G0 + tot;
        }
    } else {
        for (unsigned w = 0; w < 32; w++) {                     // warp by warp, in stream order
            if (warp == w) {
                const unsigned long long Gw = s_G;
                const bool inwarp = q >= 0 && (unsigned)q >> 5 == w;
                if (q >= 0 && !inwarp) g = s_id[q];             // an earlier warp settled it
                // lanes whose previous id comes from outside the warp (leaders), near the window edge within 32 ids?
                const unsigned amb = __ballot_sync(0xffffffffu, pub && !inwarp &&
                                                   amb_sbs1_live(g, Gw, base) != amb_sbs1_live(g, Gw + 32, base));
                unsigned long long Gn;
                if (!amb) {
                    const bool nw = pub && !inwarp && !amb_sbs1_live(g, Gw, base);
                    const unsigned bal = __ballot_sync(0xffffffffu, nw);
                    const unsigned peers = __match_any_sync(0xffffffffu, a);
                    const unsigned long long mine = nw ? Gw + __popc(bal & ((1u << lane) - 1u)) + 1 : g;
                    id = __shfl_sync(0xffffffffu, mine, __ffs(peers) - 1);
                    Gn = Gw + __popc(bal);
                } else {                                        // one lane after another
                    unsigned long long G = Gw;
                    for (int j = 0; j < 32; j++) {
                        const int pj = __shfl_sync(0xffffffffu, (int)pub, j);
                        const int ij = __shfl_sync(0xffffffffu, (int)inwarp, j);
                        const int qj = __shfl_sync(0xffffffffu, q & 31, j);
                        const unsigned long long from_lane = __shfl_sync(0xffffffffu, id, qj);
                        const unsigned long long gl = __shfl_sync(0xffffffffu, g, j);
                        if (!pj) continue;
                        const unsigned long long gj = ij ? from_lane : gl;
                        const bool nj = !amb_sbs1_live(gj, G, base);
                        if ((int)lane == j) id = nj ? G + 1 : gj;
                        G += nj ? 1ull : 0ull;
                    }
                    Gn = G;
                }
                s_id[t] = id;
                if (lane == 0) s_G = Gn;
            }
            __syncthreads();
        }
    }
    if (pub) gid[k] = id;
    __threadfence();
    __syncthreads();
    if (t == 0) {
        const unsigned long long G = s_G;
        *(volatile unsigned long long*)&flag[c] = (G << 1) | 1ull;
        if (c == gridDim.x - 1) ctr->G = G;
    }
}

__global__ void __launch_bounds__(128) amb_sbs1_format(const amb_frame* __restrict__ frames, const amb_fields* __restrict__ fields,
                                                       const AmbPosRec* __restrict__ keys,
                                                       const unsigned long long* __restrict__ gid, int n,
                                                       const AmbSbs1Ctr* __restrict__ ctr, int tz_min,
                                                       unsigned long long* table, char* __restrict__ slots,
                                                       uint32_t* __restrict__ len, uint32_t* __restrict__ bsum)
{
    __shared__ unsigned s_w[4];
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    unsigned L = 0;
    if (k < n && keys[k].key != AMB_NO_KEY) {
        const unsigned long long g = gid[k];
        const uint32_t a = keys[k].key;
        if (table[a] == (AMB_SBS1_MARK | (unsigned)k)) table[a] = g;   // the call's last record of the address
        amb_fields r = fields[k];
        L = (unsigned)amb_sbs1_line(&r, g - ctr->base, frames[k].secs, frames[k].frac, tz_min,
                                    slots + (size_t)k * AMB_SBS1_STRIDE);
    }
    if (k < n) len[k] = L;
    unsigned v = L;
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x == 0) bsum[blockIdx.x] = s_w[0] + s_w[1] + s_w[2] + s_w[3];
}

// Exclusive byte offsets of the nb blocks of lines, and the total in boff[nb]. One block of 1024 threads.
__global__ void __launch_bounds__(1024) amb_sbs1_scan(const uint32_t* __restrict__ bsum, int nb, unsigned long long* boff)
{
    __shared__ unsigned long long s_w[32], s_carry;
    const unsigned t = threadIdx.x, lane = t & 31, warp = t >> 5;
    if (t == 0) s_carry = 0ull;
    __syncthreads();
    for (int i0 = 0; i0 < nb; i0 += 1024) {
        const int i = i0 + (int)t;
        const unsigned long long x = i < nb ? bsum[i] : 0ull;
        unsigned long long v = x;
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned long long y = __shfl_up_sync(0xffffffffu, v, o);
            if (lane >= (unsigned)o) v += y;
        }
        if (lane == 31) s_w[warp] = v;
        __syncthreads();
        unsigned long long before = s_carry;
        for (unsigned w = 0; w < warp; w++) before += s_w[w];
        if (i < nb) boff[i] = before + v - x;
        __syncthreads();
        if (t == 1023) s_carry = before + v;
        __syncthreads();
    }
    if (t == 0) boff[nb] = s_carry;
}

__global__ void __launch_bounds__(128) amb_sbs1_gather(const char* __restrict__ slots, const uint32_t* __restrict__ len, int n,
                                                       const unsigned long long* __restrict__ boff, char* __restrict__ text)
{
    __shared__ unsigned s_w[4];
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned L = k < n ? len[k] : 0u;
    unsigned v = L;
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned y = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= (unsigned)o) v += y;
    }
    if (lane == 31) s_w[warp] = v;
    __syncthreads();
    unsigned long long off = boff[blockIdx.x] + v - L;
    for (unsigned w = 0; w < warp; w++) off += s_w[w];
    const char* from = slots + (size_t)k * AMB_SBS1_STRIDE;
    for (unsigned i = 0; i < L; i++) text[off + i] = from[i];
}

// Enqueue the stage (ten kernels) after every other stage; `v` is the pairing stage's scratch, free again by then,
// `keys` the stage's key records. Returns how many kernels were launched or -1 with *err set.
static int amb_sbs1_launch(AmbV3Bufs* v, const amb_frame* frames, const amb_fields* fields, AmbPosRec* keys, int n,
                           unsigned long long* table, AmbSbs1Ctr* ctr, const AmbSbs1Bufs* b, int tz_min, cudaStream_t s,
                           cudaError_t* err)
{
    const int nb = (n + 127) / 128, chunks = (n + AMB_SBS1_CHUNK - 1) / AMB_SBS1_CHUNK;
    AMB_LAUNCH((amb_sbs1_keys), nb, 128, 0, s, fields, n, keys, b->flag, chunks, ctr);
    if (amb_v3_partition(v, keys, n, s, err) < 0) return -1;
    AMB_LAUNCH((amb_sbs1_walk), AMB_V3_B / 4, 128, 0, s, keys, v->order, v->base, table, b->src);
    AMB_LAUNCH((amb_sbs1_ids), chunks, AMB_SBS1_CHUNK, 0, s, keys, b->src, n, b->gid, ctr, b->flag);
    AMB_LAUNCH((amb_sbs1_format), nb, 128, 0, s, frames, fields, keys, b->gid, n, ctr, tz_min, table, b->slots, b->len,
               b->bsum);
    AMB_LAUNCH((amb_sbs1_scan), 1, 1024, 0, s, b->bsum, nb, b->boff);
    AMB_LAUNCH((amb_sbs1_gather), nb, 128, 0, s, b->slots, b->len, n, b->boff, b->text);
    *err = cudaGetLastError();
    return *err == cudaSuccess ? 10 : -1;
}
