// The per-call rules of the receive chain, shared by the library (amb_api.cu) and the kernel harness
// (tests/simt/kernels_emul.cc): the geometry of a call (carry and guard, segments, scan rows and spans, candidate and
// frame bounds), the one owner of the per-call buffers (AmbChainBufs with amb_chain_prepare / _reset / _free) and the
// one sparse launch sequence, compact -> exact -> [walk -> slice -> ec -> ap], which returns how many kernels it
// launched, and beside it the Mode A/C sequence of option "modeac" (amb_chain_modeac). Host code only, with memory
// handled through cudaMalloc / cudaMemsetAsync / cudaMemcpy / cudaFree, so that tests/simt/simt_cudart.h can stand in
// for the runtime.
#pragma once
#include "amb_internal.h"

#include <math.h>

#include <algorithm>

#define AMB_TAIL_CAP (4 * AMB_STAGE)   // samples of a tail buffer: the call's last partial tile and >= 512 zeros

// ---- geometry -----------------------------------------------------------------------------------------------------
// Reported positions before the end of the input that a call may not decide yet (the streaming guard), and the carry
// that keeps them for the next call together with the noise-floor and PMF windows in front of them, in whole tiles.
static inline int amb_chain_guard(const AmbParams& P) { return P.maxlate + (int)ceilf(P.skip_f) + 4; }
static inline int amb_chain_carry(const AmbParams& P)
{
    const int need = amb_chain_guard(P) + P.L + 2 * P.spc_i + 64;
    return (need + AMB_STAGE - 1) / AMB_STAGE * AMB_STAGE;
}

// carry ++ main ++ tail of a call over n_new fresh samples at src: main holds their whole tiles, the tail the rest
// followed by at least 512 zeros (<= 3 tiles).
static inline AmbSegs amb_chain_segs(const float2* carry, int kc, const float2* src, int n_new, const float2* tail)
{
    AmbSegs S;
    S.carry = carry; S.main_ = src; S.tail = tail;
    S.n_carry = kc; S.n_main = n_new & ~(AMB_STAGE - 1);
    S.n_tail = (n_new - S.n_main + 512 + AMB_STAGE - 1) / AMB_STAGE * AMB_STAGE;
    S.n_valid = kc + n_new;
    return S;
}

// Rows and spans of a scan over j in [j_lo, j_hi). Rows run from row_lo to the row of j_hi - 1. row_lo is 0 for the
// split form, whose candidate kernel writes the bitmap from row 0; otherwise it is j_lo's row rounded down to a coarse
// word. Spans are whole coarse words, about one per warp of a scan grid of `ctas` CTAs of 4 warps (ctas = 0: 4 per
// SM), and there is at least one.
static inline void amb_chain_geometry(AmbScanArgs* a, long long j_lo, long long j_hi, bool from_row0, int sm_count, int ctas)
{
    a->j_lo = (int)j_lo; a->j_hi = (int)j_hi;
    a->row_lo = from_row0 ? 0 : (int)(j_lo / AMB_ROW) & ~(AMB_SPAN_ROWS_ALIGN - 1);
    a->row_hi = (int)((j_hi + AMB_ROW - 1) / AMB_ROW);
    const int rows = a->row_hi - a->row_lo;
    const int target = (ctas > 0 ? ctas : sm_count * 4) * 4;
    int rps = (rows + target - 1) / target;
    rps = (rps + AMB_SPAN_ROWS_ALIGN - 1) / AMB_SPAN_ROWS_ALIGN * AMB_SPAN_ROWS_ALIGN;
    if (rps < AMB_SPAN_ROWS_ALIGN) rps = AMB_SPAN_ROWS_ALIGN;
    a->rows_per_span = rps;
    a->n_spans = std::max(1, (rows + rps - 1) / rps);
}

// Candidate capacity for a call that evaluates `len` start positions. Up to 2^25 positions (24 bytes per candidate
// over the five arrays = 800 MB) the list can hold every position, so not even a flood of candidates (all-pass
// filter on denormal-power input, DESIGN.md) can overflow it; longer calls get len / 8, at least 2^25.
static inline unsigned amb_chain_cand_capacity(long long len)
{
    const long long big = 1ll << 25;
    const long long cap = len <= big ? len : std::max<long long>(len / 8, big);
    return (unsigned)std::max<long long>(1 << 16, cap + 1024);
}

// A detection consumes >= skip0 samples (preamble_impl.cc:237): that bounds the frames of a call over len positions.
static inline unsigned amb_chain_frame_bound(const AmbParams& P, long long len)
{
    return (unsigned)(len / std::max(P.skip0, 1) + 2);
}

// ---- buffers ------------------------------------------------------------------------------------------------------
// The per-call buffers of a context: two sets of scan bitmaps and span counts (a call uses set call_idx & 1, so that
// the next call's scan does not overwrite what this call's sparse kernels read), the candidate arrays with the
// resolver's work list and scratch, the frame buffer (with the chips when they are kept), and the ap_filter state.
struct AmbChainBufs {
    uint32_t* coarse[2] = {nullptr, nullptr}; uint32_t* fine[2] = {nullptr, nullptr};
    uint32_t* span_count[2] = {nullptr, nullptr};
    size_t rows_cap = 0; int spans_cap = 0;
    int* cand_j = nullptr; uint32_t* cand_info = nullptr; float* cand_avg = nullptr; unsigned cand_cap = 0;
    int* det_list = nullptr;
    void* walk_scratch = nullptr;
    amb_frame* frames = nullptr; unsigned frame_cap = 0;
    unsigned frames_ub = 0;              // bound on the frames queued since they were last read out
    float* chips = nullptr;
    AmbApState ap{};                     // allocated at the first call with option "ap_filter" on
    // option "modeac": per-call tile slots and counts, the queue of replies not read out yet, and the state
    // {last_prev, last_cur, candidates, replies, overlap drops, with altitude, queue count} (amb_modeac.cuh)
    amb_modeac* mac_rec = nullptr; unsigned* mac_tile_count = nullptr; size_t mac_rec_cap = 0; int mac_tiles_cap = 0;
    amb_modeac* mac_queue = nullptr; unsigned mac_queue_cap = 0;
    unsigned mac_ub = 0;                 // bound on the replies queued since they were last read out
    unsigned long long* mac_state = nullptr;
};

// What failed: the call's text and its error.
struct AmbChainErr { cudaError_t e; const char* what; };
#define AMB_CHAIN_TRY(call) do { const cudaError_t e_ = (call); if (e_ != cudaSuccess) { err->e = e_; err->what = #call; return -1; } } while (0)

// Grow the buffers for a call whose scan is *a and which may queue fr_ub more frames, then point a's bitmaps and counts
// at set `set`. sync() runs once before the first growth: the context's streams may still use what is replaced, and
// queued frames (and chips) are copied over. In steady state nothing happens here. Returns 0, or -1 with *err set.
template <class Sync>
static int amb_chain_prepare(AmbChainBufs* b, AmbScanArgs* a, int set, unsigned cap_need, unsigned fr_ub, bool keep_chips,
                             Sync sync, AmbChainErr* err)
{
    bool synced = false;
    auto grow = [&]() -> cudaError_t { if (synced) return cudaSuccess; synced = true; return sync(); };
    const size_t rows_need = (size_t)a->row_hi + 64;
    if (b->rows_cap < rows_need) {
        AMB_CHAIN_TRY(grow());
        const size_t rc = rows_need + rows_need / 8;
        for (int k = 0; k < 2; k++) {
            cudaFree(b->fine[k]); cudaFree(b->coarse[k]); b->fine[k] = b->coarse[k] = nullptr;
            AMB_CHAIN_TRY(cudaMalloc(&b->fine[k], rc * 8 * sizeof(uint32_t)));
            AMB_CHAIN_TRY(cudaMalloc(&b->coarse[k], (rc / 32 + 2) * sizeof(uint32_t)));
        }
        b->rows_cap = rc;
    }
    if (b->spans_cap < a->n_spans) {
        AMB_CHAIN_TRY(grow());
        for (int k = 0; k < 2; k++) {          // 128 group counts behind the span counts
            cudaFree(b->span_count[k]); b->span_count[k] = nullptr;
            AMB_CHAIN_TRY(cudaMalloc(&b->span_count[k], (size_t)(a->n_spans + 64 + 128) * sizeof(uint32_t)));
        }
        b->spans_cap = a->n_spans + 64;
    }
    if (b->cand_cap < cap_need) {
        AMB_CHAIN_TRY(grow());
        cudaFree(b->cand_j); cudaFree(b->cand_info); cudaFree(b->cand_avg); cudaFree(b->walk_scratch); cudaFree(b->det_list);
        b->cand_j = nullptr; b->cand_info = nullptr; b->cand_avg = nullptr; b->walk_scratch = nullptr; b->det_list = nullptr;
        AMB_CHAIN_TRY(cudaMalloc(&b->det_list, (size_t)cap_need * sizeof(int)));
        AMB_CHAIN_TRY(cudaMalloc(&b->walk_scratch, amb_walk_scratch_bytes(cap_need, (long long)cap_need * 8 + 4096)));
        AMB_CHAIN_TRY(cudaMalloc(&b->cand_j, (size_t)cap_need * sizeof(int)));
        AMB_CHAIN_TRY(cudaMalloc(&b->cand_info, (size_t)cap_need * sizeof(uint32_t)));
        AMB_CHAIN_TRY(cudaMalloc(&b->cand_avg, (size_t)cap_need * sizeof(float)));
        b->cand_cap = cap_need;
    }
    if (b->frame_cap < b->frames_ub + fr_ub) {
        AMB_CHAIN_TRY(grow());
        const unsigned ncap = (b->frames_ub + fr_ub) * 2 + 1024;
        const size_t queued = std::min(b->frames_ub, b->frame_cap);
        amb_frame* nf = nullptr; float* nc = nullptr;
        AMB_CHAIN_TRY(cudaMalloc(&nf, (size_t)ncap * sizeof(amb_frame)));
        if (b->frames && b->frames_ub) AMB_CHAIN_TRY(cudaMemcpy(nf, b->frames, queued * sizeof(amb_frame), cudaMemcpyDeviceToDevice));
        if (keep_chips) {
            AMB_CHAIN_TRY(cudaMalloc(&nc, (size_t)ncap * 240 * sizeof(float)));
            if (b->chips && b->frames_ub) AMB_CHAIN_TRY(cudaMemcpy(nc, b->chips, queued * 240 * sizeof(float), cudaMemcpyDeviceToDevice));
        }
        cudaFree(b->frames); cudaFree(b->chips);
        b->frames = nf; b->chips = nc; b->frame_cap = ncap;
    }
    if (keep_chips && !b->chips) AMB_CHAIN_TRY(cudaMalloc(&b->chips, (size_t)b->frame_cap * 240 * sizeof(float)));
    a->coarse = b->coarse[set]; a->fine = b->fine[set]; a->span_count = b->span_count[set];
    a->group_count = b->span_count[set] + b->spans_cap;
    return 0;
}

// A call that scans nothing still runs the walk when it closes the stream: candidate arrays of 64 entries when no call
// has made any yet.
static int amb_chain_prepare_empty(AmbChainBufs* b, AmbChainErr* err)
{
    if (b->cand_j) return 0;
    AMB_CHAIN_TRY(cudaMalloc(&b->cand_j, 64 * sizeof(int)));
    AMB_CHAIN_TRY(cudaMalloc(&b->cand_info, 64 * sizeof(uint32_t)));
    AMB_CHAIN_TRY(cudaMalloc(&b->cand_avg, 64 * sizeof(float)));
    AMB_CHAIN_TRY(cudaMalloc(&b->det_list, 64 * sizeof(int)));
    b->cand_cap = 64;
    return 0;
}

// The ap_filter state for frame_cap frames: at the first call with the option on, the 128 MiB table of 2^24 addresses
// and the bucket counts, zeroed in order on s (all or nothing: the next call tries again); the entries grow with the
// frame buffer, which synchronised when it grew.
static cudaError_t amb_chain_prepare_ap(AmbApState& ap, unsigned frame_cap, cudaStream_t s)
{
    cudaError_t e = cudaSuccess;
    if (!ap.last) {
        unsigned long long* last = nullptr;
        e = cudaMalloc(&last, sizeof(unsigned long long) << 24);
        if (e == cudaSuccess) e = cudaMalloc(&ap.count, AMB_AP_BUCKETS * sizeof(unsigned));
        if (e == cudaSuccess) e = cudaMalloc(&ap.off, AMB_AP_BUCKETS * sizeof(unsigned));
        if (e == cudaSuccess) e = cudaMalloc(&ap.cursor, AMB_AP_BUCKETS * sizeof(unsigned));
        if (e == cudaSuccess) e = cudaMemsetAsync(last, 0, sizeof(unsigned long long) << 24, s);
        if (e == cudaSuccess) e = cudaMemsetAsync(ap.count, 0, AMB_AP_BUCKETS * sizeof(unsigned), s);
        if (e != cudaSuccess) {
            cudaFree(last); cudaFree(ap.count); cudaFree(ap.off); cudaFree(ap.cursor);
            ap.count = ap.off = ap.cursor = nullptr;
            return e;
        }
        ap.last = last;
    }
    if (ap.ent_cap < frame_cap) {
        if ((e = cudaStreamSynchronize(s)) != cudaSuccess) return e;
        cudaFree(ap.ent); ap.ent = nullptr; ap.ent_cap = 0;
        if ((e = cudaMalloc(&ap.ent, (size_t)frame_cap * sizeof(AmbApEntry))) != cudaSuccess) return e;
        ap.ent_cap = frame_cap;
    }
    return cudaSuccess;
}

// A new stream, on s: nothing queued, no confirmed address. The ap_filter table stays allocated: the option is the
// context's, not the stream's. Returns 0, or -1 with *err set.
static int amb_chain_reset(AmbChainBufs* b, cudaStream_t s, AmbChainErr* err)
{
    b->frames_ub = 0;
    if (b->ap.last) {
        AMB_CHAIN_TRY(cudaMemsetAsync(b->ap.last, 0, sizeof(unsigned long long) << 24, s));
        AMB_CHAIN_TRY(cudaMemsetAsync(b->ap.count, 0, AMB_AP_BUCKETS * sizeof(unsigned), s));
    }
    return 0;
}

// ---- Mode A/C replies (option "modeac") ---------------------------------------------------------------------------
#define AMB_MODEAC_STATE_WORDS 7
static inline int amb_modeac_off(double t_us, int rate_int) { return (int)floor(t_us * (double)rate_int / 1e6 + 0.5); }
static inline AmbModeacGeom amb_chain_modeac_geom(int rate_int)
{
    AmbModeacGeom G;
    for (int k = 0; k < 15; k++) G.slot[k] = amb_modeac_off(1.45 * k, rate_int);
    for (int g = 0; g < 14; g++) G.gap[g] = amb_modeac_off(1.45 * g + 0.725, rate_int);
    G.spi = amb_modeac_off(24.65, rate_int);
    G.back = amb_modeac_off(25.1, rate_int);
    return G;
}

// The state on s for a new stream (allocated at the first use), and nothing queued.
static int amb_chain_modeac_reset(AmbChainBufs* b, cudaStream_t s, AmbChainErr* err)
{
    if (!b->mac_state) AMB_CHAIN_TRY(cudaMalloc(&b->mac_state, AMB_MODEAC_STATE_WORDS * sizeof(unsigned long long)));
    AMB_CHAIN_TRY(cudaMemsetAsync(b->mac_state, 0, AMB_MODEAC_STATE_WORDS * sizeof(unsigned long long), s));
    b->mac_ub = 0;
    return 0;
}

// A call's Mode A/C pass on s over the starts [a.j_lo, a.j_hi) of the scan a (org: reported index of j = 0): buffers
// grown (sync() once before the first growth; queued replies are copied over), then the tile and emit kernels. Returns
// the kernels launched, or -1 with *err set.
template <class Sync>
static int amb_chain_modeac(const AmbScanArgs& a, long long org, AmbChainBufs* b, cudaStream_t s, Sync sync, AmbChainErr* err)
{
    AmbModeacArgs m{};
    m.P = a.P; m.S = a.S; m.G = amb_chain_modeac_geom(a.P.rate_int);
    m.j_lo = a.j_lo; m.j_hi = a.j_hi; m.org = org;
    m.na_cap = AMB_MODEAC_TILE + m.G.back + a.P.L;
    m.nb_cap = m.na_cap + m.G.spi + 2;
    m.cap_tile = AMB_MODEAC_TILE / (m.G.back + 1) + 1;
    const int n_tiles = (a.j_hi - a.j_lo + AMB_MODEAC_TILE - 1) / AMB_MODEAC_TILE;
    const size_t rec_need = (size_t)n_tiles * m.cap_tile;
    const unsigned ub = (unsigned)std::min<size_t>(rec_need, (size_t)(a.j_hi - a.j_lo) / (m.G.back + 1) + 1);
    bool synced = false;
    auto grow = [&]() -> cudaError_t { if (synced) return cudaSuccess; synced = true; return sync(); };
    if (b->mac_rec_cap < rec_need || b->mac_tiles_cap < n_tiles) {
        AMB_CHAIN_TRY(grow());
        cudaFree(b->mac_rec); cudaFree(b->mac_tile_count); b->mac_rec = nullptr; b->mac_tile_count = nullptr;
        AMB_CHAIN_TRY(cudaMalloc(&b->mac_rec, (rec_need + rec_need / 8) * sizeof(amb_modeac)));
        AMB_CHAIN_TRY(cudaMalloc(&b->mac_tile_count, (size_t)(n_tiles + n_tiles / 8 + 1) * sizeof(unsigned)));
        b->mac_rec_cap = rec_need + rec_need / 8; b->mac_tiles_cap = n_tiles + n_tiles / 8 + 1;
    }
    if (b->mac_queue_cap < b->mac_ub + ub) {
        AMB_CHAIN_TRY(grow());
        const unsigned ncap = (b->mac_ub + ub) * 2 + 1024;
        amb_modeac* nq = nullptr;
        AMB_CHAIN_TRY(cudaMalloc(&nq, (size_t)ncap * sizeof(amb_modeac)));
        if (b->mac_queue && b->mac_ub)
            AMB_CHAIN_TRY(cudaMemcpy(nq, b->mac_queue, (size_t)std::min(b->mac_ub, b->mac_queue_cap) * sizeof(amb_modeac), cudaMemcpyDeviceToDevice));
        cudaFree(b->mac_queue);
        b->mac_queue = nq; b->mac_queue_cap = ncap;
    }
    b->mac_ub += ub;
    m.rec = b->mac_rec; m.tile_count = b->mac_tile_count;
    m.last_prev = b->mac_state; m.last_cur = b->mac_state + 1; m.stats = b->mac_state + 2;
    m.queue = b->mac_queue; m.q_count = reinterpret_cast<unsigned*>(b->mac_state + 6);
    cudaError_t e = cudaSuccess;
    const int k = amb_launch_modeac(m, s, &e);
    AMB_CHAIN_TRY(e);
    return k;
}

// Free everything and leave the buffers as new ones (the caller has synchronised with their last use).
static void amb_chain_free(AmbChainBufs* b)
{
    void* const all[] = {b->coarse[0], b->coarse[1], b->fine[0], b->fine[1], b->span_count[0], b->span_count[1],
                         b->cand_j, b->cand_info, b->cand_avg, b->det_list, b->walk_scratch, b->frames, b->chips,
                         b->ap.last, b->ap.count, b->ap.off, b->ap.cursor, b->ap.ent,
                         b->mac_rec, b->mac_tile_count, b->mac_queue, b->mac_state};
    for (void* p : all) cudaFree(p);
    *b = AmbChainBufs();
}

// ---- sparse sequence ----------------------------------------------------------------------------------------------
// The options a call's sparse kernels run with (amb_set_option).
struct AmbChainOpts {
    int sm_count;
    bool par;                  // the parallel resolver (option "resolver" != 1), else the sequential walk
    unsigned exact_dense;      // option "exact_dense"
    bool keep_chips;
    int ec, ec_any, ap_filter; // options "ec", "ec_any", "ap_filter" (0 = off)
    int rate_int;              // ap_filter's window is ap_filter * rate_int samples
};

// One call: its input - IQ segments S, or the split form's two float streams (in0 != NULL) - where it sits in the
// stream, what its walk may decide, and the counters and resolver state it updates.
struct AmbChainCall {
    AmbParams P; AmbSegs S;
    const float* in0; const float* in1; long long n_streams;
    long long org, ntot, r_safe; int flush;
    AmbCounters* ctr; AmbWalkState* st;
    long long n_samples;       // samples the parallel resolver's time buckets cover
};

// A call whose candidates are decided: what its walk and slice stages read. Kept across a deferred call (amb_resolve).
struct AmbChainSpan {
    AmbWalkArgs wa; AmbSliceArgs sl;
    bool par;
    bool walk_only;            // a call that scanned nothing: the walk closes the stream, there is nothing to slice
    long long n_samples;
};

static AmbWalkArgs amb_chain_walk_args(const AmbChainCall& c, const AmbChainBufs& b, int sm_count)
{
    AmbWalkArgs wa{};
    wa.P = c.P; wa.org = c.org; wa.ntot = c.ntot; wa.r_safe = c.r_safe; wa.flush = c.flush;
    wa.ctr = c.ctr; wa.st = c.st; wa.sm_count = sm_count;
    wa.cand_j = b.cand_j; wa.cand_info = b.cand_info; wa.det_list = b.det_list;
    return wa;
}

// The split form's bitmap in set 0 from two float streams of n items: bitmap and counts zeroed, which the candidate
// kernel needs, the call's counters too, and the resolver state when st != NULL (the stream's first call). One launch.
static int amb_chain_split_scan(const AmbScanArgs& a, const AmbChainBufs& b, const float* in0, const float* in1, long long n,
                                AmbCounters* ctr, AmbWalkState* st, int sm_count, cudaStream_t s, AmbChainErr* err)
{
    AMB_CHAIN_TRY(cudaMemsetAsync(b.coarse[0], 0, ((size_t)a.row_hi / 32 + 2) * sizeof(uint32_t), s));
    AMB_CHAIN_TRY(cudaMemsetAsync(b.span_count[0], 0, (size_t)(b.spans_cap + 128) * sizeof(uint32_t), s));
    AMB_CHAIN_TRY(cudaMemsetAsync(ctr, 0, sizeof(AmbCounters), s));
    if (st) AMB_CHAIN_TRY(cudaMemsetAsync(st, 0, sizeof(AmbWalkState), s));
    AMB_CHAIN_TRY(amb_launch_stream_candidates(a, in0, in1, n, sm_count, s));
    return 1;
}

// With option "ec" or "ec_any" on, correct the frames a slice kernel dropped for their CRC, in place: one launch for
// both passes. ctr != NULL: the call's slots; ctr == NULL: frames [0, n).
static int amb_chain_ec(amb_frame* frames, unsigned frame_cap, AmbCounters* ctr, int n, const AmbChainOpts& o, cudaStream_t s,
                        AmbChainErr* err)
{
    if (!o.ec && !o.ec_any) return 0;
    AMB_CHAIN_TRY(amb_launch_ec(frames, frame_cap, ctr, n, o.ec, o.ec_any, o.sm_count, s));
    return 1;
}

// [walk -> slice -> ec -> ap] of a decided call on s: the walk (sequential, or the parallel resolver's three kernels),
// then, unless the span is walk-only, the slicer, the error correction and - with "ap_filter" on - the address/parity
// check (four launches). Everything that reads frames or the call's counters is enqueued after this on the same
// stream. Returns the kernels launched, or -1 with *err set.
static int amb_chain_resolve(const AmbChainSpan& sp, AmbChainBufs* b, const AmbChainOpts& o, cudaStream_t s, AmbChainErr* err)
{
    int k;
    if (!sp.par) { AMB_CHAIN_TRY(amb_launch_walk_seq(sp.wa, s)); k = 1; }
    else { AMB_CHAIN_TRY(amb_launch_walk_par(sp.wa, b->walk_scratch, b->cand_cap, sp.n_samples, s)); k = 3; }
    if (sp.walk_only) return k;
    AMB_CHAIN_TRY(amb_launch_slice(sp.sl, o.sm_count, s));
    k++;
    const int ke = amb_chain_ec(sp.sl.frames, sp.sl.frame_cap, sp.sl.ctr, 0, o, s, err);
    if (ke < 0) return -1;
    k += ke;
    if (o.ap_filter) {
        AMB_CHAIN_TRY(amb_chain_prepare_ap(b->ap, sp.sl.frame_cap, s));
        const unsigned long long window = (unsigned long long)o.ap_filter * (unsigned long long)o.rate_int;
        cudaError_t e = cudaSuccess;
        k += amb_launch_ap(sp.sl.frames, sp.sl.frame_cap, sp.sl.ctr, b->ap, window, o.sm_count, s, &e);
        AMB_CHAIN_TRY(e);
    }
    return k;
}

// One call's sparse chain on s, once its bitmap *a is written: compact -> exact, then - unless the call is deferred -
// amb_chain_resolve. *sp receives the decided span either way. Returns the kernels launched, or -1 with *err set.
static int amb_chain_launch(const AmbScanArgs& a, const AmbChainCall& c, AmbChainBufs* b, const AmbChainOpts& o, bool defer,
                            cudaStream_t s, AmbChainSpan* sp, AmbChainErr* err)
{
    AMB_CHAIN_TRY(amb_launch_compact(a, b->cand_j, b->cand_cap, c.ctr, o.par ? b->walk_scratch : nullptr, c.n_samples, s));
    AmbExactArgs ea{};
    ea.P = c.P; ea.S = c.S; ea.cand_j = b->cand_j; ea.cand_info = b->cand_info; ea.cand_avg = b->cand_avg; ea.ctr = c.ctr;
    ea.dense_threshold = o.exact_dense;
    ea.in0 = c.in0; ea.in1 = c.in1; ea.n_streams = c.n_streams;
    AMB_CHAIN_TRY(amb_launch_exact(ea, o.sm_count, s));
    const int k = c.in0 ? 2 : 3;             // the exact stage: one kernel on float streams, two on IQ (both regimes)
    sp->wa = amb_chain_walk_args(c, *b, o.sm_count);
    AmbSliceArgs& sl = sp->sl;
    sl = AmbSliceArgs{};
    sl.P = c.P; sl.S = c.S; sl.cand_j = b->cand_j; sl.cand_info = b->cand_info; sl.cand_avg = b->cand_avg;
    sl.det_list = b->det_list; sl.ctr = c.ctr; sl.frames = b->frames; sl.frame_cap = b->frame_cap;
    sl.chips_out = o.keep_chips ? b->chips : nullptr; sl.org = c.org;
    sl.in0 = c.in0; sl.in1 = c.in1; sl.n_streams = c.n_streams;
    sp->par = o.par; sp->walk_only = false; sp->n_samples = c.n_samples;
    if (defer) return k;
    const int kr = amb_chain_resolve(*sp, b, o, s, err);
    return kr < 0 ? -1 : k + kr;
}
#undef AMB_CHAIN_TRY
