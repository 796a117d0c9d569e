// The kernels of the batch field decoder (SURVEY.md 8 row f4): amb_fields_kernel and amb_resolve_kernel here, the CPR
// pairing stage between them in amb_decode_v3.cuh. The host orchestration and the C ABI are in amb_decode.cu, the
// per-message arithmetic in amb_decode_core.h. Kept in headers without any <<< >>> launch so that tests/simt/ can
// compile the very same kernel source for the host under a small SIMT emulator (CPU-side check of the warp-level logic;
// the GPU tests remain the parity gate).
#pragma once
#include "amb_decode_core.h"

#define AMB_TABLE_SLOTS (1ull << 26)     // (24-bit ICAO, surface, even/odd)

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

#include "amb_decode_v3.cuh"
#include "amb_decode_local.cuh"
#include "amb_decode_commb.cuh"
#include "amb_decode_opstatus.cuh"
#include "amb_decode_track.cuh"
#include "amb_decode_track_ext.cuh"
#include "amb_decode_sbs1.cuh"

// ---- launch sequence ----------------------------------------------------------------------------------------------
// What the stages of one decode read and write besides the frames and the records: amb_decoder keeps one in device
// memory, tests/simt/decode_emul.cc one in host memory. A stage's tables are only touched while its S is > 0.
struct AmbDecodeState {
    AmbCprSlot* table = nullptr;         // pairing: latest even / odd report per (ICAO, surface), AMB_TABLE_SLOTS
    double* nl_T = nullptr;              // NL transition table, AMB_NL_MAX
    AmbV3Bufs v3;                        // pairing scratch, reused by the partitions of the stages after it
    AmbPosRec* pos = nullptr; AmbPair* pair = nullptr;   // one per frame
    AmbPosRec* keys = nullptr;           // one per frame: address-keyed records of the local, Comm-B, op-status and track stage
    int local_cpr = 0;                   // option "local_cpr" = S seconds, 0 = off
    AmbRefPos* ltable = nullptr;         // reference position per ICAO, AMB_LOCAL_SLOTS
    int commb = 0;                       // option "commb" = S seconds, 0 = off
    AmbCommbRef* ctable = nullptr;       // ADS-B velocity per address, AMB_COMMB_SLOTS
    int opstatus = 0;                    // option "opstatus" = S seconds, 0 = off
    AmbOpsSlot* otable = nullptr;        // latest op status per address, AMB_OPS_SLOTS
    int track = 0;                       // option "track" = S seconds, 0 = off
    amb_aircraft* trows = nullptr;       // one row per address, AMB_TRACK_ROWS
    unsigned* tocc = nullptr;            // which rows hold data, AMB_TRACK_WORDS
    AmbTrackClock* tclk = nullptr;       // t of the latest queued record since reset
    int track_ext = 0;                   // option "track_ext" = S2 seconds, 0 = off; runs only while track is on too
    amb_aircraft_ext* xrows = nullptr;   // one extension row per address, AMB_TRACK_ROWS
    unsigned* xocc = nullptr;            // which extension rows were written since reset, AMB_TRACK_WORDS
    int sbs1 = 0;                        // option "sbs1": 1 = on, 0 = off
    int sbs1_tz = 0;                     // option "sbs1_tz": minutes added to UTC in the lines' date and time
    unsigned long long* stable = nullptr;   // latest aircraft id per address (a global value, 0 = none), AMB_SBS1_SLOTS
    AmbSbs1Ctr* sctr = nullptr;          // the id counter and the base recorded at reset
    AmbSbs1Bufs sb;                      // the stage's per-call scratch and the packed lines, one entry per frame
    int have_loc = 0; double lat = 0.0, lon = 0.0;      // receiver location
};

// What amb_decode_launch returns when a stage fails to launch.
enum { AMB_STAGE_FIELDS = -1, AMB_STAGE_PAIRING = -2, AMB_STAGE_RESOLVE = -3, AMB_STAGE_LOCAL = -4,
       AMB_STAGE_COMMB = -5, AMB_STAGE_TRACK = -6, AMB_STAGE_OPSTATUS = -7, AMB_STAGE_TRACK_EXT = -8,
       AMB_STAGE_SBS1 = -9 };

// Enqueue one decode of the n frames into the n records on stream s, in this order: fields, pairing, resolve, then the
// local CPR, Comm-B, op-status and track stages whose S is > 0, and the track extension when track and track_ext are
// both > 0, then the SBS-1 feed when sbs1 is on. Returns how many kernels were launched (7, plus 6 per stage that is
// on, plus 10 for the SBS-1 feed), or an AMB_STAGE_* code with *err set.
static int amb_decode_launch(AmbDecodeState* st, const amb_frame* frames, int n, amb_fields* fields, cudaStream_t s,
                             cudaError_t* err)
{
    const int nb = (n + 127) / 128;
    AMB_LAUNCH((amb_fields_kernel), nb, 128, 0, s, frames, n, fields, st->pos, st->pair);
    if ((*err = cudaGetLastError()) != cudaSuccess) return AMB_STAGE_FIELDS;
    const int kp = amb_v3_launch(&st->v3, st->pos, n, st->table, st->pair, s, err);
    if (kp < 0) return AMB_STAGE_PAIRING;
    AMB_LAUNCH((amb_resolve_kernel), nb, 128, 0, s, fields, st->pos, st->pair, n, st->have_loc, st->lat, st->lon,
               st->nl_T);
    if ((*err = cudaGetLastError()) != cudaSuccess) return AMB_STAGE_RESOLVE;
    int k = 2 + kp;
    if (st->local_cpr > 0) {
        const int kl = amb_local_launch(&st->v3, st->pos, st->keys, n, fields, st->ltable, st->local_cpr, st->have_loc,
                                        st->lat, st->lon, st->nl_T, s, err);
        if (kl < 0) return AMB_STAGE_LOCAL;
        k += kl;
    }
    if (st->commb > 0) {
        const int kc = amb_commb_launch(&st->v3, frames, fields, st->pos, st->keys, n, st->ctable, st->commb, s, err);
        if (kc < 0) return AMB_STAGE_COMMB;
        k += kc;
    }
    if (st->opstatus > 0) {
        const int ko = amb_opstatus_launch(&st->v3, frames, fields, st->pos, st->keys, n, st->otable, st->opstatus, s, err);
        if (ko < 0) return AMB_STAGE_OPSTATUS;
        k += ko;
    }
    if (st->track > 0) {
        const int kt = amb_track_launch(&st->v3, frames, fields, st->pos, st->keys, n, st->trows, st->tocc, st->tclk,
                                        st->track, s, err);
        if (kt < 0) return AMB_STAGE_TRACK;
        k += kt;
        if (st->track_ext > 0) {
            const int kx = amb_track_ext_launch(&st->v3, fields, st->pos, st->keys, n, st->xrows, st->xocc, s, err);
            if (kx < 0) return AMB_STAGE_TRACK_EXT;
            k += kx;
        }
    }
    if (st->sbs1 > 0) {
        const int ks = amb_sbs1_launch(&st->v3, frames, fields, st->keys, n, st->stable, st->sctr, &st->sb, st->sbs1_tz,
                                       s, err);
        if (ks < 0) return AMB_STAGE_SBS1;
        k += ks;
    }
    return k;
}
