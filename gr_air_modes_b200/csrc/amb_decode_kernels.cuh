// The kernels of the batch field decoder (SURVEY.md 8 row f4): amb_fields_kernel and amb_resolve_kernel here, the CPR
// pairing stage between them in amb_decode_v3.cuh, the optional stages in the headers included below; then the state
// every stage reads and writes, its lifecycle (amb_decode_prepare, amb_decode_reset, amb_decode_free) and the one launch
// sequence of a decode (amb_decode_launch). The staging of frames and records and the C ABI are in amb_decode.cu, the
// per-message arithmetic in amb_decode_core.h. Beside the state: its option table (amb_decode_set_option); last, the
// read-outs of the stages' results (amb_decode_text, amb_decode_snapshot_*, amb_decode_coverage). Kept in headers
// without any <<< >>> launch, and with the state's memory handled through cudaMalloc / cudaMemsetAsync /
// cudaMemcpyAsync / cudaFree only, so that tests/simt/ can compile the very same kernel source and state handling for
// the host under a small SIMT emulator (CPU-side check of the warp-level logic; the GPU tests remain the parity gate).
#pragma once
#include "amb_decode_core.h"

#include <string.h>

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
#include "amb_decode_coverage.cuh"
#include "amb_decode_reports.cuh"

// ---- state and launch sequence ------------------------------------------------------------------------------------
// What the stages of one decode read and write besides the frames and the records, and the one owner of that memory:
// amb_decoder keeps one in device memory, tests/simt/decode_emul.cc one in host memory, and both allocate, clear and
// free it with amb_decode_prepare, amb_decode_reset and amb_decode_free below. A stage's tables are only allocated and
// touched while its S is > 0.
struct AmbDecodeState {
    AmbCprSlot* table = nullptr;         // pairing: latest even / odd report per (ICAO, surface), table_slots
    size_t table_slots = AMB_TABLE_SLOTS, local_slots = AMB_LOCAL_SLOTS;   // smaller only in the emulator's tests
    double* nl_T = nullptr;              // NL transition table, AMB_NL_MAX
    AmbV3Bufs v3;                        // pairing scratch, reused by the partitions of the stages after it
    AmbPosRec* pos = nullptr; AmbPair* pair = nullptr;   // one per frame
    int cap = 0;                         // frames pos and pair hold
    AmbPosRec* keys = nullptr;           // one per frame: address-keyed records of the local, Comm-B, op-status and track stage
    int kcap = 0;                        // frames keys holds
    int local_cpr = 0;                   // option "local_cpr" = S seconds, 0 = off
    AmbRefPos* ltable = nullptr;         // reference position per ICAO, local_slots
    int commb = 0;                       // option "commb" = S seconds, 0 = off
    AmbCommbRef* ctable = nullptr;       // ADS-B velocity per address, AMB_COMMB_SLOTS
    int opstatus = 0;                    // option "opstatus" = S seconds, 0 = off
    AmbOpsSlot* otable = nullptr;        // latest op status per address, AMB_OPS_SLOTS
    int track = 0;                       // option "track" = S seconds, 0 = off
    amb_aircraft* trows = nullptr;       // one row per address, AMB_TRACK_ROWS
    unsigned* tocc = nullptr;            // which rows hold data, AMB_TRACK_WORDS
    AmbTrackClock* tclk = nullptr;       // t of the latest queued record since reset
    uint32_t* snap_cnt = nullptr;        // snapshot: per-block counts, then their scan and the total
    int track_ext = 0;                   // option "track_ext" = S2 seconds, 0 = off; runs only while track is on too
    amb_aircraft_ext* xrows = nullptr;   // one extension row per address, AMB_TRACK_ROWS
    unsigned* xocc = nullptr;            // which extension rows were written since reset, AMB_TRACK_WORDS
    int sbs1 = 0;                        // option "sbs1": 1 = on, 0 = off
    int sbs1_tz = 0;                     // option "sbs1_tz": minutes added to UTC in the lines' date and time
    unsigned long long* stable = nullptr;   // latest aircraft id per address (a global value, 0 = none), AMB_SBS1_SLOTS
    AmbSbs1Ctr* sctr = nullptr;          // the id counter and the base recorded at reset
    AmbSbs1Bufs sb;                      // the stage's per-call scratch and the packed lines, one entry per frame
    int scap = 0;                        // frames sb holds
    int coverage = 0;                    // option "coverage": 1 = on, 0 = off
    unsigned long long* cgrid = nullptr; // the coverage grid: the bits of AMB_COVERAGE_CELLS doubles, all >= +0.0
    int reports = 0;                     // option "reports": 1 = on, 0 = off
    unsigned* rfirst = nullptr;          // 1 until the first queued frame since creation or reset has been formatted
    AmbReportBufs rb;                    // the stage's per-call scratch and the packed lines
    int rcap = 0;                        // frames rb holds
    int sbs1_nb = -1;                    // blocks of lines of the last decode (its byte total is sb.boff[sbs1_nb]);
                                         // -1: the last decode wrote no lines
    int reports_nb = -1;                 // the same for the text reports (rb.boff[reports_nb])
    int have_loc = 0; double lat = 0.0, lon = 0.0;      // receiver location
};

// The options of amb_decoder_set_option: the member each one sets, the values it takes and what any other value reports.
static const struct {
    const char* name; int AmbDecodeState::*member; int lo, hi; const char* range;
} amb_decode_options[] = {
    {"local_cpr", &AmbDecodeState::local_cpr, 0, AMB_LOCAL_CPR_MAX, "local_cpr: 0 (off) .. 600 seconds"},
    {"commb", &AmbDecodeState::commb, 0, AMB_COMMB_MAX, "commb: 0 (off) .. 600 seconds"},
    {"track", &AmbDecodeState::track, 0, AMB_TRACK_MAX, "track: 0 (off) .. 3600 seconds"},
    {"opstatus", &AmbDecodeState::opstatus, 0, AMB_OPSTATUS_MAX, "opstatus: 0 (off) .. 600 seconds"},
    {"track_ext", &AmbDecodeState::track_ext, 0, AMB_TRACK_EXT_MAX, "track_ext: 0 (off) .. 3600 seconds"},
    {"sbs1", &AmbDecodeState::sbs1, 0, 1, "sbs1: 0 (off) or 1 (on)"},
    {"sbs1_tz", &AmbDecodeState::sbs1_tz, AMB_SBS1_TZ_MIN, AMB_SBS1_TZ_MAX, "sbs1_tz: -720 .. 840 minutes"},
    {"coverage", &AmbDecodeState::coverage, 0, 1, "coverage: 0 (off) or 1 (on)"},
    {"reports", &AmbDecodeState::reports, 0, 1, "reports: 0 (off) or 1 (on)"},
};

// Set option `name` of st to `value`, from the next decode on. Returns NULL, or why the setting is refused.
static const char* amb_decode_set_option(AmbDecodeState* st, const char* name, int value)
{
    for (const auto& o : amb_decode_options) {
        if (strcmp(name, o.name) != 0) continue;
        if (value < o.lo || value > o.hi) return o.range;
        st->*o.member = value;
        return nullptr;
    }
    return "amb_decoder_set_option: unknown option";
}

static void amb_decode_set_location(AmbDecodeState* st, int have_location, double lat, double lon)
{
    st->have_loc = have_location ? 1 : 0; st->lat = lat; st->lon = lon;
}

// What amb_decode_prepare, amb_decode_reset and amb_decode_launch return when a stage's memory or launch fails.
enum { AMB_STAGE_FIELDS = -1, AMB_STAGE_PAIRING = -2, AMB_STAGE_RESOLVE = -3, AMB_STAGE_LOCAL = -4,
       AMB_STAGE_COMMB = -5, AMB_STAGE_TRACK = -6, AMB_STAGE_OPSTATUS = -7, AMB_STAGE_TRACK_EXT = -8,
       AMB_STAGE_SBS1 = -9, AMB_STAGE_COVERAGE = -10,
       AMB_STAGE_REPORTS = -11 };

// By -AMB_STAGE_* - 1: what a failed launch of the stage reports, and what a failure of its memory reports.
static const struct { const char* launch; const char* memory; } amb_stage_names[] = {
    {"cudaGetLastError()", "per-frame records"},
    {"pairing", "report table (1 GiB)"},
    {"cudaGetLastError()", "NL transition table"},
    {"local CPR", "reference position table (384 MiB)"},
    {"Comm-B inference", "Comm-B velocity table (384 MiB)"},
    {"aircraft table", "aircraft table (2 GiB)"},
    {"op status", "op status table (384 MiB)"},
    {"aircraft table extension", "aircraft table extension (2.25 GiB)"},
    {"SBS-1 feed", "SBS-1 id table (128 MiB)"},
    {"coverage map", "coverage grid (5184 B)"},
    {"text reports", "text report buffers (478 B per frame)"},
};

// cudaMalloc, then every byte set to `fill` unless it is < 0; *p is NULL after a failed cudaMalloc
template <typename T> static cudaError_t amb_decode_alloc(T** p, size_t bytes, int fill, cudaStream_t s)
{
    const cudaError_t e = cudaMalloc(p, bytes);
    if (e != cudaSuccess) { *p = nullptr; return e; }
    return fill < 0 ? cudaSuccess : cudaMemsetAsync(*p, fill, bytes, s);
}

static void amb_sbs1_bufs_free(AmbSbs1Bufs* b)
{
    void* const all[] = {b->src, b->gid, b->flag, b->slots, b->len, b->bsum, b->boff, b->text};
    for (void* p : all) cudaFree(p);
    *b = AmbSbs1Bufs();
}

static void amb_report_bufs_free(AmbReportBufs* b)
{
    void* const all[] = {b->len, b->bsum, b->boff, b->text};
    for (void* p : all) cudaFree(p);
    *b = AmbReportBufs();
}

#define AMB_STAGE_TRY(stage, call) do { if ((*err = (call)) != cudaSuccess) return (stage); } while (0)

// Allocate on stream s what the stages that are on need for a decode of n frames (n = 0: only the pairing and NL
// tables, which every decode needs): the per-frame records, from 4096 frames up, doubling; the address-keyed records
// once a stage that partitions them is on; each stage's table, bitmap, clock and counter at its first decode with the
// option on, filled as an empty one (the track extension only while track is on too); the SBS-1 scratch as the frame
// capacity grows; the coverage grid at the first decode with the option on; the text reports' first-message flag (set)
// at the first decode with the option on, and their buffers as the frame capacity grows. Returns 0, or the AMB_STAGE_* code of the
// stage whose memory could not be had, with *err set.
static int amb_decode_prepare(AmbDecodeState* st, int n, cudaStream_t s, cudaError_t* err)
{
    if (!st->table) AMB_STAGE_TRY(AMB_STAGE_PAIRING, amb_decode_alloc(&st->table, st->table_slots * sizeof(AmbCprSlot), 0xFF, s));
    if (!st->nl_T) {
        double T[AMB_NL_MAX];
        amb_build_nl_table(T);                          // cpr.py:46-51 through the host libm, once
        AMB_STAGE_TRY(AMB_STAGE_RESOLVE, amb_decode_alloc(&st->nl_T, sizeof T, -1, s));
        AMB_STAGE_TRY(AMB_STAGE_RESOLVE, cudaMemcpyAsync(st->nl_T, T, sizeof T, cudaMemcpyHostToDevice, s));
    }
    if (n > st->cap) {
        int cap = st->cap ? st->cap : 4096;
        while (cap < n) cap *= 2;
        cudaFree(st->pos); cudaFree(st->pair);
        st->pos = nullptr; st->pair = nullptr; st->cap = 0;
        AMB_STAGE_TRY(AMB_STAGE_FIELDS, amb_decode_alloc(&st->pos, (size_t)cap * sizeof(AmbPosRec), -1, s));
        AMB_STAGE_TRY(AMB_STAGE_FIELDS, amb_decode_alloc(&st->pair, (size_t)cap * sizeof(AmbPair), -1, s));
        st->cap = cap;
    }
    if ((st->local_cpr > 0 || st->commb > 0 || st->opstatus > 0 || st->track > 0 || st->sbs1 > 0) && st->kcap < st->cap) {
        cudaFree(st->keys);
        st->keys = nullptr; st->kcap = 0;
        AMB_STAGE_TRY(AMB_STAGE_FIELDS, amb_decode_alloc(&st->keys, (size_t)st->cap * sizeof(AmbPosRec), -1, s));
        st->kcap = st->cap;
    }
    if (st->local_cpr > 0 && !st->ltable)               // the tables start empty: all NaN
        AMB_STAGE_TRY(AMB_STAGE_LOCAL, amb_decode_alloc(&st->ltable, st->local_slots * sizeof(AmbRefPos), 0xFF, s));
    if (st->commb > 0 && !st->ctable)
        AMB_STAGE_TRY(AMB_STAGE_COMMB, amb_decode_alloc(&st->ctable, AMB_COMMB_SLOTS * sizeof(AmbCommbRef), 0xFF, s));
    if (st->opstatus > 0 && !st->otable)
        AMB_STAGE_TRY(AMB_STAGE_OPSTATUS, amb_decode_alloc(&st->otable, AMB_OPS_SLOTS * sizeof(AmbOpsSlot), 0xFF, s));
    if (st->track > 0) {                                // rows are not initialised: the bitmaps start empty
        static const AmbTrackClock none = {NAN, 0u, 0u};   // "nothing decoded"
        if (!st->trows)
            AMB_STAGE_TRY(AMB_STAGE_TRACK, amb_decode_alloc(&st->trows, (size_t)AMB_TRACK_ROWS * sizeof(amb_aircraft), -1, s));
        if (!st->tclk) {
            AMB_STAGE_TRY(AMB_STAGE_TRACK, amb_decode_alloc(&st->tclk, sizeof none, -1, s));
            AMB_STAGE_TRY(AMB_STAGE_TRACK, cudaMemcpyAsync(st->tclk, &none, sizeof none, cudaMemcpyHostToDevice, s));
        }
        if (!st->snap_cnt)
            AMB_STAGE_TRY(AMB_STAGE_TRACK, amb_decode_alloc(&st->snap_cnt, (2 * AMB_TRACK_WORDS / AMB_SNAP_WORDS + 1) *
                                                                               sizeof(uint32_t), -1, s));
        if (!st->tocc)                                  // last: a snapshot and a reset take a bitmap as "everything is there"
            AMB_STAGE_TRY(AMB_STAGE_TRACK, amb_decode_alloc(&st->tocc, AMB_TRACK_WORDS * sizeof(unsigned), 0, s));
        if (st->track_ext > 0 && !st->xrows)
            AMB_STAGE_TRY(AMB_STAGE_TRACK_EXT, amb_decode_alloc(&st->xrows, (size_t)AMB_TRACK_ROWS * sizeof(amb_aircraft_ext),
                                                                -1, s));
        if (st->track_ext > 0 && !st->xocc)             // last, likewise
            AMB_STAGE_TRY(AMB_STAGE_TRACK_EXT, amb_decode_alloc(&st->xocc, AMB_TRACK_WORDS * sizeof(unsigned), 0, s));
    }
    if (st->sbs1 > 0) {                                 // no id yet, the counter at 0
        if (!st->stable)
            AMB_STAGE_TRY(AMB_STAGE_SBS1, amb_decode_alloc(&st->stable, (size_t)AMB_SBS1_SLOTS * sizeof(unsigned long long),
                                                           0, s));
        if (!st->sctr) AMB_STAGE_TRY(AMB_STAGE_SBS1, amb_decode_alloc(&st->sctr, sizeof(AmbSbs1Ctr), 0, s));
        if (st->scap < st->cap) {
            amb_sbs1_bufs_free(&st->sb);
            st->scap = 0;
            const size_t c = (size_t)st->cap, nb = (c + 127) / 128, chunks = (c + AMB_SBS1_CHUNK - 1) / AMB_SBS1_CHUNK;
            AmbSbs1Bufs& b = st->sb;
            AMB_STAGE_TRY(AMB_STAGE_SBS1, amb_decode_alloc(&b.src, c * sizeof(unsigned long long), -1, s));
            AMB_STAGE_TRY(AMB_STAGE_SBS1, amb_decode_alloc(&b.gid, c * sizeof(unsigned long long), -1, s));
            AMB_STAGE_TRY(AMB_STAGE_SBS1, amb_decode_alloc(&b.flag, chunks * sizeof(unsigned long long), -1, s));
            AMB_STAGE_TRY(AMB_STAGE_SBS1, amb_decode_alloc(&b.slots, c * AMB_SBS1_STRIDE, -1, s));
            AMB_STAGE_TRY(AMB_STAGE_SBS1, amb_decode_alloc(&b.len, c * sizeof(uint32_t), -1, s));
            AMB_STAGE_TRY(AMB_STAGE_SBS1, amb_decode_alloc(&b.bsum, nb * sizeof(uint32_t), -1, s));
            AMB_STAGE_TRY(AMB_STAGE_SBS1, amb_decode_alloc(&b.boff, (nb + 1) * sizeof(unsigned long long), -1, s));
            AMB_STAGE_TRY(AMB_STAGE_SBS1, amb_decode_alloc(&b.text, c * AMB_SBS1_STRIDE, -1, s));
            st->scap = st->cap;
        }
    }
    if (st->coverage > 0 && !st->cgrid)                 // every cell +0.0
        AMB_STAGE_TRY(AMB_STAGE_COVERAGE, amb_decode_alloc(&st->cgrid, AMB_COVERAGE_CELLS * sizeof(unsigned long long), 0, s));
    if (st->reports > 0) {
        if (!st->rfirst) {
            static const unsigned one = 1u;
            AMB_STAGE_TRY(AMB_STAGE_REPORTS, amb_decode_alloc(&st->rfirst, sizeof one, -1, s));
            AMB_STAGE_TRY(AMB_STAGE_REPORTS, cudaMemcpyAsync(st->rfirst, &one, sizeof one, cudaMemcpyHostToDevice, s));
        }
        if (st->rcap < st->cap) {
            amb_report_bufs_free(&st->rb);
            st->rcap = 0;
            const size_t c = (size_t)st->cap, nb = (c + 127) / 128;
            AmbReportBufs& b = st->rb;
            AMB_STAGE_TRY(AMB_STAGE_REPORTS, amb_decode_alloc(&b.len, c * sizeof(uint32_t), -1, s));
            AMB_STAGE_TRY(AMB_STAGE_REPORTS, amb_decode_alloc(&b.bsum, nb * sizeof(uint32_t), -1, s));
            AMB_STAGE_TRY(AMB_STAGE_REPORTS, amb_decode_alloc(&b.boff, (nb + 1) * sizeof(unsigned long long), -1, s));
            AMB_STAGE_TRY(AMB_STAGE_REPORTS, amb_decode_alloc(&b.text, c * AMB_REP_MAX_LINE, -1, s));
            st->rcap = st->cap;
        }
    }
    return 0;
}

// amb_decoder_reset on stream s, for whatever is allocated: every table empty again. The rows of the aircraft table
// and its extension stay (a row whose bit is clear is never read), and so does the SBS-1 id table (ids up to G are
// dead once base = G); the coverage grid is cleared; the text reports' first-message flag is set again. Returns 0, or
// the AMB_STAGE_* code of the stage whose memory could not be cleared, with *err set.
static int amb_decode_reset(AmbDecodeState* st, cudaStream_t s, cudaError_t* err)
{
    static const AmbTrackClock none = {NAN, 0u, 0u};
    if (st->table) AMB_STAGE_TRY(AMB_STAGE_PAIRING, cudaMemsetAsync(st->table, 0xFF, st->table_slots * sizeof(AmbCprSlot), s));
    if (st->ltable) AMB_STAGE_TRY(AMB_STAGE_LOCAL, cudaMemsetAsync(st->ltable, 0xFF, st->local_slots * sizeof(AmbRefPos), s));
    if (st->ctable) AMB_STAGE_TRY(AMB_STAGE_COMMB, cudaMemsetAsync(st->ctable, 0xFF, AMB_COMMB_SLOTS * sizeof(AmbCommbRef), s));
    if (st->otable) AMB_STAGE_TRY(AMB_STAGE_OPSTATUS, cudaMemsetAsync(st->otable, 0xFF, AMB_OPS_SLOTS * sizeof(AmbOpsSlot), s));
    if (st->tocc) {
        AMB_STAGE_TRY(AMB_STAGE_TRACK, cudaMemsetAsync(st->tocc, 0, AMB_TRACK_WORDS * sizeof(unsigned), s));
        AMB_STAGE_TRY(AMB_STAGE_TRACK, cudaMemcpyAsync(st->tclk, &none, sizeof none, cudaMemcpyHostToDevice, s));
    }
    if (st->xocc) AMB_STAGE_TRY(AMB_STAGE_TRACK_EXT, cudaMemsetAsync(st->xocc, 0, AMB_TRACK_WORDS * sizeof(unsigned), s));
    if (st->sctr)
        AMB_STAGE_TRY(AMB_STAGE_SBS1, cudaMemcpyAsync(&st->sctr->base, &st->sctr->G, sizeof(unsigned long long),
                                                      cudaMemcpyDeviceToDevice, s));
    if (st->cgrid)
        AMB_STAGE_TRY(AMB_STAGE_COVERAGE, cudaMemsetAsync(st->cgrid, 0, AMB_COVERAGE_CELLS * sizeof(unsigned long long), s));
    if (st->rfirst) {
        static const unsigned one = 1u;
        AMB_STAGE_TRY(AMB_STAGE_REPORTS, cudaMemcpyAsync(st->rfirst, &one, sizeof one, cudaMemcpyHostToDevice, s));
    }
    return 0;
}
#undef AMB_STAGE_TRY

// Free everything the state owns and leave it as a new one (the caller has synchronised with its last use).
static void amb_decode_free(AmbDecodeState* st)
{
    void* const all[] = {st->table, st->nl_T, st->pos, st->pair, st->keys, st->ltable, st->ctable, st->otable, st->trows,
                         st->tocc, st->tclk, st->snap_cnt, st->xrows, st->xocc, st->stable, st->sctr, st->cgrid,
                         st->rfirst};
    for (void* p : all) cudaFree(p);
    amb_v3_free(&st->v3);
    amb_sbs1_bufs_free(&st->sb);
    amb_report_bufs_free(&st->rb);
    *st = AmbDecodeState();
}

// Enqueue one decode of the n frames into the n records on stream s, in this order: fields, pairing, resolve, then the
// local CPR stage when its S is > 0, the coverage map when coverage is on (after the local stage, so that local fixes
// reach it), the Comm-B, op-status and track stages whose S is > 0, and the track extension when track and track_ext
// are both > 0, then the SBS-1 feed when sbs1 is on, then the text reports when reports is on. Returns how many kernels
// were launched (7, plus 6 per stage that is on, plus 1 for the coverage map, 10 for the SBS-1 feed and 3 for the text
// reports), or an AMB_STAGE_* code with *err set. Only a decode that launches every stage leaves lines of the SBS-1
// feed and the text reports, whichever is on, for amb_decode_text: sbs1_nb and reports_nb are -1 otherwise, and a
// caller that ends a decode before this call (n = 0, a failure) sets them to -1 itself.
static int amb_decode_launch(AmbDecodeState* st, const amb_frame* frames, int n, amb_fields* fields, cudaStream_t s,
                             cudaError_t* err)
{
    const int nb = (n + 127) / 128;
    st->sbs1_nb = st->reports_nb = -1;
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
    if (st->coverage > 0) {
        if (amb_coverage_launch(fields, n, st->cgrid, s, err) < 0) return AMB_STAGE_COVERAGE;
        k += 1;
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
    if (st->reports > 0) {
        const int kr = amb_reports_launch(frames, fields, n, st->rfirst, &st->rb, s, err);
        if (kr < 0) return AMB_STAGE_REPORTS;
        k += kr;
    }
    if (st->sbs1 > 0) st->sbs1_nb = nb;
    if (st->reports > 0) st->reports_nb = nb;
    return k;
}

// ---- read-outs ----------------------------------------------------------------------------------------------------
// The lines of the last decode, the text reports' (reports) or the SBS-1 feed's, on stream s: *text their packed bytes
// in the state's memory and *bytes their count, or NULL and 0 when the last decode wrote none.
static cudaError_t amb_decode_text(const AmbDecodeState* st, bool reports, cudaStream_t s, const char** text,
                                   unsigned long long* bytes)
{
    const int nb = reports ? st->reports_nb : st->sbs1_nb;
    *text = nullptr; *bytes = 0;
    if (nb < 0) return cudaSuccess;
    *text = reports ? st->rb.text : st->sb.text;
    const cudaError_t e = cudaMemcpyAsync(bytes, (reports ? st->rb.boff : st->sb.boff) + nb, sizeof *bytes,
                                          cudaMemcpyDeviceToHost, s);
    return e != cudaSuccess ? e : cudaStreamSynchronize(s);
}

// The aircraft table at `now` over the first `words` words of its bitmap (a multiple of AMB_SNAP_WORDS; the decoder
// scans all AMB_TRACK_WORDS), on stream s, once the track stage has allocated it. amb_decode_snapshot_count counts the
// rows shown and returns their total (2 launches); amb_decode_snapshot_gather then writes them to out, and their
// extensions to ext unless it is NULL (1 launch). Both return -1 with *err set when a launch or a copy fails.
static int amb_decode_snapshot_count(const AmbDecodeState* st, double now, unsigned words, cudaStream_t s, cudaError_t* err)
{
    const unsigned nb = words / AMB_SNAP_WORDS;
    uint32_t* const off = st->snap_cnt + nb;
    uint32_t total = 0;
    if (amb_snap_count_launch(st->tocc, st->trows, st->tclk, now, st->track, words, st->snap_cnt, off, s, err) < 0 ||
        (*err = cudaMemcpyAsync(&total, off + nb, sizeof total, cudaMemcpyDeviceToHost, s)) != cudaSuccess ||
        (*err = cudaStreamSynchronize(s)) != cudaSuccess)
        return -1;
    return (int)total;
}

static int amb_decode_snapshot_gather(const AmbDecodeState* st, double now, unsigned words, amb_aircraft* out,
                                      amb_aircraft_ext* ext, cudaStream_t s, cudaError_t* err)
{
    const uint32_t* off = st->snap_cnt + words / AMB_SNAP_WORDS;
    const int k = ext ? amb_snap_gather_ext_launch(st->tocc, st->trows, st->tclk, now, st->track, words, off, out, st->xocc,
                                                   st->xrows, st->track_ext, ext, s, err)
                      : amb_snap_gather_launch(st->tocc, st->trows, st->tclk, now, st->track, words, off, out, s, err);
    return k < 0 ? -1 : k;
}

// The coverage grid into out (AMB_COVERAGE_CELLS doubles, in device memory when out_on_device, else in host memory) on
// stream s: all zeros while the grid is not allocated yet.
static cudaError_t amb_decode_coverage(const AmbDecodeState* st, double* out, bool out_on_device, cudaStream_t s)
{
    static_assert(sizeof(double) == sizeof(unsigned long long), "coverage cell layout");
    const size_t bytes = AMB_COVERAGE_CELLS * sizeof(double);
    if (!st->cgrid && !out_on_device) { memset(out, 0, bytes); return cudaSuccess; }
    const cudaError_t e = st->cgrid ? cudaMemcpyAsync(out, st->cgrid, bytes, out_on_device ? cudaMemcpyDeviceToDevice
                                                                                            : cudaMemcpyDeviceToHost, s)
                                    : cudaMemsetAsync(out, 0, bytes, s);
    return e != cudaSuccess ? e : cudaStreamSynchronize(s);
}
