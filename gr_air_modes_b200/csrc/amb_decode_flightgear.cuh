// FlightGear multiplayer feed (decoder option "flightgear", DESIGN.md §8 "FlightGear multiplayer feed"). Runs last,
// after every other stage, so that local CPR fixes reach it; it reads the records and writes nothing into them. Every
// position record (amb_fg_kind) of an address that has had a callsign and a velocity since the last reset writes one
// position packet (amb_fg_packet, amb_fg_format.h); the packets of one call are packed into one buffer in record order.
//
// State: per address, the latest callsign (ident, model) and velocity (heading, vel_ms, turn) since the reset, in a
// direct-mapped table (2^24 x 32 B) carried from call to call. amb_decoder_reset clears it with a memset.
//
//   amb_fg_keys    one thread per frame: key = icao of a record that sets or reads the state, AMB_NO_KEY otherwise
//   amb_v3_count .. amb_v3_scatter   the pairing stage's stable partition (amb_decode_v3.cuh), on those keys
//   amb_fg_walk    one warp per bucket, 32 records per step: each record's state after it - its own callsign or
//                  velocity, else the latest earlier lane's of its address (__match_any_sync), else the table slot;
//                  a position record keeps its state in the call's scratch, the address's last lane of the step
//                  writes the slot. A slot has one owner bucket.
//   amb_fg_count   one thread per frame: 232 bytes for a position record that writes a packet, else 0; the block's sum
//   amb_sbs1_scan  one block: the byte offset of every block of packets, and the total (amb_decode_sbs1.cuh)
//   amb_fg_write   one thread per frame: its packet at its byte offset
#pragma once
#include "amb_fg_format.h"

#define AMB_FG_SLOTS (1u << 24)                  // one state slot per 24-bit address
#define AMB_FG_HAS_CALLSIGN 0x01
#define AMB_FG_HAS_VELOCITY 0x02

// An address's state, and a position record's state as the walk leaves it (32 bytes).
struct AmbFgSlot {
    char ident[8];               // callsign of the latest BDS0,8
    double hdg;                  // heading, degrees, of the latest BDS0,9 subtype 0 / 1
    float vel_ms, turn;          // (float)(velocity * 0.514444444), (float)(turn rate * (pi / 180.))
    uint8_t model, flags, pad_[6];   // model of the callsign's category; AMB_FG_HAS_*
};
static_assert(sizeof(AmbFgSlot) == 32, "FlightGear slot layout");

__global__ void __launch_bounds__(128) amb_fg_keys(const amb_fields* __restrict__ fields, int n, AmbPosRec* __restrict__ keys)
{
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    amb_fields r = fields[k];
    AmbPosRec p;
    p.key = amb_fg_kind(&r) != AMB_FG_NONE ? r.icao : AMB_NO_KEY;
    p.lat = p.lon = p.fmt = 0;
    p.t = 0.0;
    keys[k] = p;
}

__global__ void __launch_bounds__(128) amb_fg_walk(const amb_fields* __restrict__ fields, const AmbPosRec* __restrict__ keys,
                                                   const uint32_t* __restrict__ order, const uint32_t* __restrict__ base,
                                                   AmbFgSlot* table, AmbFgSlot* __restrict__ st)
{
    const unsigned lane = threadIdx.x & 31;
    const unsigned b = blockIdx.x * 4 + (threadIdx.x >> 5);     // one warp per bucket; a slot has one owner bucket
    const unsigned lo = base[b], hi = base[b + 1];
    for (unsigned i0 = lo; i0 < hi; i0 += 32) {
        const unsigned i = i0 + lane;
        const bool mine = i < hi;
        const unsigned k = mine ? order[i] : 0u;
        const uint32_t a = mine ? keys[k].key : 0u;
        int kind = AMB_FG_NONE;
        unsigned long long ident = 0ull;
        int model = 0;
        double hdg = 0.0;
        float vel = 0.f, turn = 0.f;
        AmbFgSlot slot;
        memset(&slot, 0, sizeof slot);
        if (mine) {
            const amb_fields* r = &fields[k];
            kind = amb_fg_kind(r);
            if (kind == AMB_FG_CALLSIGN) {
                memcpy(&ident, r->ident, 8);
                model = amb_fg_model(r->ftc, r->cat);
            } else if (kind == AMB_FG_VELOCITY) {               // rule 3: subtype 1 has no turn rate
                hdg = r->val[1];
                vel = (float)(r->val[0] * AMB_FG_KTS_MS);
                turn = (float)((r->subtype == 0 ? r->val[3] : 0.0) * (M_PI / 180.));
            }
            const uint4* p = reinterpret_cast<const uint4*>(&table[a]);
            const uint4 w0 = __ldcg(p), w1 = __ldcg(p + 1);
            memcpy(&slot, &w0, 16);
            memcpy(reinterpret_cast<char*>(&slot) + 16, &w1, 16);
        }
        // the same address inside this step; lanes past the end of the bucket get a private value (an address has 24 bits)
        const unsigned peers = __match_any_sync(0xffffffffu, mine ? a : (0x80000000u | lane));
        const unsigned upto = peers & ((2u << lane) - 1u), later = peers & ~((2u << lane) - 1u);
        const unsigned cs = __ballot_sync(0xffffffffu, kind == AMB_FG_CALLSIGN) & upto;
        const unsigned vs = __ballot_sync(0xffffffffu, kind == AMB_FG_VELOCITY) & upto;
        const int pc = cs ? 31 - __clz(cs) : (int)lane, pv = vs ? 31 - __clz(vs) : (int)lane;
        const unsigned long long c_ident = __shfl_sync(0xffffffffu, ident, pc);
        const int c_model = __shfl_sync(0xffffffffu, model, pc);
        const double v_hdg = __shfl_sync(0xffffffffu, hdg, pv);
        const float v_vel = __shfl_sync(0xffffffffu, vel, pv), v_turn = __shfl_sync(0xffffffffu, turn, pv);
        if (cs) {                                               // the state after this record
            memcpy(slot.ident, &c_ident, 8);
            slot.model = (uint8_t)c_model;
            slot.flags |= AMB_FG_HAS_CALLSIGN;
        }
        if (vs) {
            slot.hdg = v_hdg; slot.vel_ms = v_vel; slot.turn = v_turn;
            slot.flags |= AMB_FG_HAS_VELOCITY;
        }
        __syncwarp();                                           // every lane has read its slot before the writes below
        if (mine) {
            if (kind == AMB_FG_POSITION) st[k] = slot;
            if (!later) {
                uint4 w0, w1;
                memcpy(&w0, &slot, 16);
                memcpy(&w1, reinterpret_cast<const char*>(&slot) + 16, 16);
                uint4* p = reinterpret_cast<uint4*>(&table[a]);
                p[0] = w0; p[1] = w1;
            }
        }
        __threadfence_block();
        __syncwarp();                                           // this step's writes are visible to the next step
    }
}

// The packet of record k into out (or only its length when out is NULL): rule 4.
static __device__ __forceinline__ unsigned amb_fg_record_packet(const amb_frame* frames, const amb_fields* fields,
                                                                const AmbPosRec* keys, const AmbFgSlot* st, int k, char* out)
{
    if (keys[k].key == AMB_NO_KEY) return 0u;
    const amb_fields* r = &fields[k];
    if (amb_fg_kind(r) != AMB_FG_POSITION) return 0u;
    const AmbFgSlot s = st[k];
    if ((s.flags & (AMB_FG_HAS_CALLSIGN | AMB_FG_HAS_VELOCITY)) != (AMB_FG_HAS_CALLSIGN | AMB_FG_HAS_VELOCITY)) return 0u;
    const double alt = r->bds == 0x05 ? (double)r->altitude : 0.0;
    const double t = (double)frames[k].secs + frames[k].frac;
    if (!out) {
        float o[3];
        return amb_fg_orientation(r->lat, r->lon, s.hdg, o) ? (unsigned)AMB_FG_PACKET : 0u;
    }
    return amb_fg_packet(s.ident, s.model, r->lat, r->lon, alt, t, s.hdg, s.vel_ms, s.turn, out);
}

__global__ void __launch_bounds__(128) amb_fg_count(const amb_frame* __restrict__ frames, const amb_fields* __restrict__ fields,
                                                    const AmbPosRec* __restrict__ keys, const AmbFgSlot* __restrict__ st,
                                                    int n, uint32_t* __restrict__ len, uint32_t* __restrict__ bsum)
{
    __shared__ unsigned s_w[4];
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned L = k < n ? amb_fg_record_packet(frames, fields, keys, st, k, nullptr) : 0u;
    if (k < n) len[k] = L;
    unsigned v = L;
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x == 0) bsum[blockIdx.x] = s_w[0] + s_w[1] + s_w[2] + s_w[3];
}

__global__ void __launch_bounds__(128) amb_fg_write(const amb_frame* __restrict__ frames, const amb_fields* __restrict__ fields,
                                                    const AmbPosRec* __restrict__ keys, const AmbFgSlot* __restrict__ st,
                                                    int n, const uint32_t* __restrict__ len,
                                                    const unsigned long long* __restrict__ boff, char* __restrict__ out)
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
    if (L) amb_fg_record_packet(frames, fields, keys, st, k, out + off);
}

// Enqueue the stage (nine kernels) after every other stage; `v` is the pairing stage's scratch, free again by then,
// `keys` the stage's key records, `st` the per-frame state the walk leaves, b the packets. Returns how many kernels
// were launched or -1 with *err set.
static int amb_fg_launch(AmbV3Bufs* v, const amb_frame* frames, const amb_fields* fields, AmbPosRec* keys, int n,
                         AmbFgSlot* table, AmbFgSlot* st, const AmbReportBufs* b, cudaStream_t s, cudaError_t* err)
{
    const int nb = (n + 127) / 128;
    AMB_LAUNCH((amb_fg_keys), nb, 128, 0, s, fields, n, keys);
    if (amb_v3_partition(v, keys, n, s, err) < 0) return -1;
    AMB_LAUNCH((amb_fg_walk), AMB_V3_B / 4, 128, 0, s, fields, keys, v->order, v->base, table, st);
    AMB_LAUNCH((amb_fg_count), nb, 128, 0, s, frames, fields, keys, st, n, b->len, b->bsum);
    AMB_LAUNCH((amb_sbs1_scan), 1, 1024, 0, s, b->bsum, nb, b->boff);
    AMB_LAUNCH((amb_fg_write), nb, 128, 0, s, frames, fields, keys, st, n, b->len, b->boff, b->text);
    *err = cudaGetLastError();
    return *err == cudaSuccess ? 9 : -1;
}
