// Host side of libairmodes_b200.so: stream context, per-call orchestration and the C ABI declared in
// include/airmodes_b200.h. No CPU implementation of the hot path lives here: every compute entry point
// launches the kernels in amb_kernels.cu or fails. Citations are file:line under gr-air-modes.
#include "amb_chain.h"
#include "amb_params.h"
#include "amb_order_kernels.cuh"

#include <math.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <condition_variable>
#include <deque>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#define AMB_VERSION "gr-air-modes_b200 0.1 (sm_90a)"

typedef CUresult (*amb_encode_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

#define AMB_ING_SLOTS 4
#define AMB_SNAPS 8
struct AmbIngestSlot {
    float2* dev = nullptr;        // chunk of float32 I/Q the chain reads
    void* dev_raw = nullptr;      // 16-bit chunk before widening (allocated on first use)
    void* pin = nullptr;          // pinned host chunk (pageable / small input is gathered here)
    cudaEvent_t e_h2d = nullptr;  // copy (+ widening) of this slot's chunk done
    cudaEvent_t e_free_b = nullptr, e_free_c = nullptr;   // last readers of dev (sparse kernels, carry) done
    bool used = false, h2d_pending = false;
};
struct amb_time_tag { uint64_t offset; uint64_t secs; double frac; };

struct amb_ctx {
    int device = 0, sm_count = 0;
    amb_encode_fn encode = nullptr;
    CUtensorMap tm_carry[3], tm_tail[2];
    cudaStream_t stream = nullptr;       // stream A: prologue, scan, carry (the caller-visible stream)
    cudaStream_t stream_b = nullptr;     // stream B: compact, exact, resolve, slice - overlaps the next call's scan
    cudaStream_t stream_c = nullptr;     // stream C: prologue + carry, so that stream A is scans back to back
    cudaEvent_t e_aux[2] = {nullptr, nullptr}, e_in = nullptr;
    bool aux_valid[2] = {false, false};
    bool own_stream = false;
    int overlap = 1;
    cudaEvent_t e_scan[2] = {nullptr, nullptr}, e_done[2] = {nullptr, nullptr};
    bool done_valid[2] = {false, false};
    unsigned long long call_idx = 0;
    int carry_in = 2;                    // index of the carry buffer the next call reads (2 = the all-zero one)
    float rate_arg = 0.f, thr_db = 0.f;
    int use_pmf = 0;
    AmbParams P{};
    int chip_off[240];
    int kc = 0, guard = 0;
    float2* carry[3] = {nullptr, nullptr, nullptr};   // [2] stays all zero (sample history before the stream)
    float2* tail[2] = {nullptr, nullptr};   // AMB_TAIL_CAP samples each
    float2* staging = nullptr; size_t staging_cap = 0;
    // host ingest pipeline (amb_process with host memory): ring of pinned + device chunk buffers, copy stream
    cudaStream_t stream_h = nullptr;
    size_t ing_chunk = (size_t)1 << 22;  // samples per chunk (32 MiB of float32 I/Q)
    size_t coalesce = (size_t)1 << 18;   // small host calls are gathered until this many samples are pending
    AmbIngestSlot ing[AMB_ING_SLOTS];
    unsigned ing_next = 0;               // slot the next chunk uses
    size_t pend_n = 0; int pend_kind = 0;  // samples gathered in ing[ing_next].pin, not dispatched yet
    int copy_threads = 0;                // 0 = default
    int scan_ctas = 0;                   // CTAs of the scan kernel (0 = 4 per SM: one full wave)
    unsigned exact_dense = 65536;        // candidates per call beyond which the row-based exact kernel takes over
    // non-blocking poll: counter snapshots of the calls in flight (pinned), frames already handed out
    AmbCounters* ctr_snap = nullptr; cudaEvent_t snap_ev[AMB_SNAPS] = {}; unsigned long long snap_head = 0, snap_tail = 0;
    unsigned polled = 0;                 // frames [0, polled) of the device frame buffer were returned by amb_poll_ready
    std::vector<amb_time_tag> time_tags; // rx_time tags (absolute item offset -> time), ascending
    // device-side drain (amb_drain_device): sort scratch, device copy of the tags
    unsigned long long* ord_key = nullptr; unsigned* ord_val = nullptr; unsigned ord_cap = 0; unsigned order_tile = 2048;
    AmbTagDev* tags_dev = nullptr; int tags_dev_cap = 0;
    // optional DC blocker (rx_path.py:39-41)
    int use_dcblock = 0, dc_D = 0, dc_nc = 0, dc_cur = 0;
    float2* dc_carry[2] = {nullptr, nullptr}; float2* dc_out = nullptr; float2* dc_ma0 = nullptr; size_t dc_cap = 0;
    AmbChainBufs bufs;                   // bitmaps, candidates, frames, chips, ap_filter state (amb_chain.h)
    bool keep_chips = false;
    AmbCounters* ctr = nullptr; AmbWalkState* st = nullptr;
    // stream state
    uint64_t n_in = 0; long long r_done = 0; bool flushed = false;
    uint64_t t0_secs = 0; double t0_frac = 0.0;
    // split-form preamble stream state: undecided tail of the two float streams + counters
    std::vector<float> sf0, sf1; uint64_t sf_total = 0; long long sf_rdone = 0;          // rx_time tag at item 0 (preamble_impl.cc:104-116)
    long long last_org = 0; bool have_last = false;
    std::vector<amb_frame> pending;
    // stats / timing
    amb_stats stats{};
    bool timing = false;
    cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
    bool ev_valid = false;
    cudaEvent_t ring[128] = {};          // 64 (start, stop) pairs around the scan kernel of the last calls
    cudaEvent_t ring_done[64] = {};      // ... and the end of the same calls' sparse stages (stream B)
    unsigned ring_n = 0;
    int resolver = 0;
    int ec = 0;                          // option "ec": error correction over up to K low-confidence bits (0 = off)
    int ec_any = 0;                      // option "ec_any": DF17 correction over up to M (1, 2) bits anywhere (0 = off)
    int ap_filter = 0;                   // option "ap_filter": address/parity check against the last S seconds (0 = off)
    bool seeked = false;                 // positioned by amb_seek since the last reset (no "ap_filter" there)
    // time-sharded operation (amb_seek / amb_resolve): a call whose walk + slice stages are still to run
    int defer = 0;                       // option "defer_resolve"
    int def_kind = 0;                    // 0 nothing pending, 1 full (walk + slice), 2 sequential walk only, 3 state only
    int def_set = 0;
    bool def_resolved = false;           // resolved once already: amb_resolve again = re-resolution with another entry
    AmbChainSpan def{};                  // what its walk + slice stages read
    std::string err;
};

extern "C" {
static void ingest_free(amb_ctx* c);
static int ingest_dispatch_pending(amb_ctx* ctx, int flush);
}

static cudaError_t sync_all(amb_ctx* c)
{
    cudaError_t e = cudaStreamSynchronize(c->stream);
    if (e == cudaSuccess && c->stream_c) e = cudaStreamSynchronize(c->stream_c);
    if (e == cudaSuccess && c->stream_b) e = cudaStreamSynchronize(c->stream_b);
    return e;
}

// IQ as a 2-D tensor of 128-byte lines (16 complex samples each); tiles of 32 lines = 512 samples land in
// shared memory with the 128B swizzle the scan kernel reads through.
static int make_tmap(amb_ctx* ctx, CUtensorMap* m, const void* base, size_t n_samples)
{
    const cuuint64_t dims[2] = {32, (cuuint64_t)(n_samples / 16)};
    const cuuint64_t strides[1] = {128};
    const cuuint32_t box[2] = {32, 32};
    const cuuint32_t estr[2] = {1, 1};
    CUresult r = ctx->encode(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<void*>(base), dims, strides, box, estr,
                             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        char buf[96]; snprintf(buf, sizeof buf, "cuTensorMapEncodeTiled failed (%d)", (int)r);
        ctx->err = buf; return AMB_ERR_CUDA;
    }
    return AMB_OK;
}

static int chain_fail(amb_ctx* c, const AmbChainErr& er) { return fail(c, AMB_ERR_CUDA, er.what, er.e); }

// The options the call's sparse kernels run with
static AmbChainOpts chain_opts(const amb_ctx* c)
{
    return AmbChainOpts{c->sm_count, c->resolver != 1, c->exact_dense, c->keep_chips, c->ec, c->ec_any, c->ap_filter,
                        c->P.rate_int};
}

static int setup_rate(amb_ctx* ctx)
{
    AmbParams P; int off[240];
    int rc = compute_params(ctx->rate_arg, ctx->thr_db, ctx->use_pmf, &P, off);
    if (rc != AMB_OK) return fail(ctx, rc, "unsupported rate (need 2e6 <= rate <= 20e6 and int(rate/2e6) consistent)");
    ctx->P = P;
    memcpy(ctx->chip_off, off, sizeof off);
    CK(ctx, amb_upload_tables(off));
    ctx->guard = amb_chain_guard(P);
    ctx->kc = amb_chain_carry(P);
    if (ctx->use_dcblock) {                              // filter.dc_blocker_cc(100*self._spc, False)  rx_path.py:40
        ctx->dc_D = 100 * P.spc_i;
        ctx->dc_nc = 2 * ctx->dc_D - 2;
        for (int k = 0; k < 2; k++) {
            cudaFree(ctx->dc_carry[k]); ctx->dc_carry[k] = nullptr;
            CK(ctx, cudaMalloc(&ctx->dc_carry[k], (size_t)ctx->dc_nc * sizeof(float2)));
        }
    }
    for (int k = 0; k < 3; k++) {
        cudaFree(ctx->carry[k]); ctx->carry[k] = nullptr;
        CK(ctx, cudaMalloc(&ctx->carry[k], (size_t)ctx->kc * sizeof(float2)));
        CK(ctx, cudaMemset(ctx->carry[k], 0, (size_t)ctx->kc * sizeof(float2)));
        int rc2 = make_tmap(ctx, &ctx->tm_carry[k], ctx->carry[k], (size_t)ctx->kc); if (rc2) return rc2;
    }
    for (int k = 0; k < 2; k++) {
        cudaFree(ctx->tail[k]); ctx->tail[k] = nullptr;
        CK(ctx, cudaMalloc(&ctx->tail[k], (size_t)AMB_TAIL_CAP * sizeof(float2)));
        int rc2 = make_tmap(ctx, &ctx->tm_tail[k], ctx->tail[k], (size_t)AMB_TAIL_CAP); if (rc2) return rc2;
    }
    return AMB_OK;
}

static int reset_stream(amb_ctx* ctx)
{
    // counters and resolver state belong to stream B (in order after the previous call's tail kernels);
    // the sample history restarts from the all-zero carry buffer, so nothing has to be cleared on stream A
    CK(ctx, cudaMemsetAsync(ctx->ctr, 0, sizeof(AmbCounters), ctx->stream_b));
    CK(ctx, cudaMemsetAsync(ctx->st, 0, sizeof(AmbWalkState), ctx->stream_b));
    if (ctx->use_dcblock) {   // raw-sample history of the DC blocker restarts from zeros (only stream A touches it)
        CK(ctx, cudaMemsetAsync(ctx->dc_carry[0], 0, (size_t)ctx->dc_nc * sizeof(float2), ctx->stream));
        CK(ctx, cudaMemsetAsync(ctx->dc_carry[1], 0, (size_t)ctx->dc_nc * sizeof(float2), ctx->stream));
        ctx->dc_cur = 0;
    }
    ctx->sf0.clear(); ctx->sf1.clear(); ctx->sf_total = 0; ctx->sf_rdone = 0;
    ctx->carry_in = 2; ctx->n_in = 0; ctx->r_done = 0; ctx->flushed = false; ctx->have_last = false;
    ctx->pending.clear();
    ctx->def_kind = 0; ctx->def_resolved = false;
    ctx->pend_n = 0;                                   // samples gathered but not dispatched belong to the old stream
    ctx->snap_tail = ctx->snap_head; ctx->polled = 0;
    ctx->time_tags.clear();
    ctx->seeked = false;
    AmbChainErr er;
    if (amb_chain_reset(&ctx->bufs, ctx->stream_b, &er) < 0) return chain_fail(ctx, er);
    return AMB_OK;
}

extern "C" {

const char* amb_version(void) { return AMB_VERSION; }

const char* amb_strerror(int code)
{
    switch (code) {
        case AMB_OK: return "ok";
        case AMB_ERR_INVALID: return "invalid argument";
        case AMB_ERR_NO_DEVICE: return "no usable sm_90 CUDA device (there is no CPU path)";
        case AMB_ERR_CUDA: return "CUDA runtime error";
        case AMB_ERR_RATE: return "unsupported sample rate";
        case AMB_ERR_OVERFLOW: return "internal buffer overflow";
        case AMB_ERR_UNSUPPORTED: return "feature not supported";
        case AMB_ERR_ALIGN: return "device pointer not 16-byte aligned";
        case AMB_ERR_STATE: return "invalid state for this call";
    }
    return "unknown error";
}

const char* amb_last_error(const amb_ctx* ctx) { return ctx ? ctx->err.c_str() : ""; }

int amb_create(int device, float rate, float threshold_db, int use_pmf, int use_dcblock, amb_ctx** out)
{
    if (!out) return AMB_ERR_INVALID;
    *out = nullptr;
    cudaDeviceProp prop;
    if (amb_check_device(device, &prop) != AMB_OK) return AMB_ERR_NO_DEVICE;
    amb_ctx* ctx = new amb_ctx();
    ctx->device = device; ctx->sm_count = prop.multiProcessorCount;
    ctx->rate_arg = rate; ctx->thr_db = threshold_db; ctx->use_pmf = use_pmf ? 1 : 0;
    ctx->use_dcblock = use_dcblock ? 1 : 0;
    int rc = AMB_OK;
    do {
        if (cudaSetDevice(device) != cudaSuccess) { rc = AMB_ERR_NO_DEVICE; break; }
        if (cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking) != cudaSuccess) { rc = AMB_ERR_CUDA; break; }
        ctx->own_stream = true;
        if (cudaStreamCreateWithFlags(&ctx->stream_b, cudaStreamNonBlocking) != cudaSuccess) { rc = AMB_ERR_CUDA; break; }
        if (cudaStreamCreateWithFlags(&ctx->stream_c, cudaStreamNonBlocking) != cudaSuccess) { rc = AMB_ERR_CUDA; break; }
        if (cudaEventCreateWithFlags(&ctx->e_in, cudaEventDisableTiming) != cudaSuccess) { rc = AMB_ERR_CUDA; break; }
        for (int k = 0; k < 2 && rc == AMB_OK; k++)
            if (cudaEventCreateWithFlags(&ctx->e_scan[k], cudaEventDisableTiming) != cudaSuccess ||
                cudaEventCreateWithFlags(&ctx->e_aux[k], cudaEventDisableTiming) != cudaSuccess ||
                cudaEventCreateWithFlags(&ctx->e_done[k], cudaEventDisableTiming) != cudaSuccess) rc = AMB_ERR_CUDA;
        if (rc != AMB_OK) break;
        if (cudaMalloc(&ctx->ctr, sizeof(AmbCounters)) != cudaSuccess || cudaMalloc(&ctx->st, sizeof(AmbWalkState)) != cudaSuccess) { rc = AMB_ERR_CUDA; break; }
        if (cudaMallocHost(&ctx->ctr_snap, AMB_SNAPS * sizeof(AmbCounters)) != cudaSuccess) { rc = AMB_ERR_CUDA; break; }
        for (int k = 0; k < AMB_SNAPS && rc == AMB_OK; k++)
            if (cudaEventCreateWithFlags(&ctx->snap_ev[k], cudaEventDisableTiming) != cudaSuccess) rc = AMB_ERR_CUDA;
        if (rc != AMB_OK) break;
        for (int k = 0; k < 4; k++) if (cudaEventCreate(&ctx->ev[k]) != cudaSuccess) { rc = AMB_ERR_CUDA; break; }
        for (int k = 0; k < 128 && rc == AMB_OK; k++) if (cudaEventCreate(&ctx->ring[k]) != cudaSuccess) rc = AMB_ERR_CUDA;
        for (int k = 0; k < 64 && rc == AMB_OK; k++) if (cudaEventCreate(&ctx->ring_done[k]) != cudaSuccess) rc = AMB_ERR_CUDA;
        if (rc != AMB_OK) break;
        {   // driver entry point for tensor-map encoding (no link-time dependency on libcuda)
            void* fn = nullptr; cudaDriverEntryPointQueryResult qr;
            if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qr) != cudaSuccess || !fn) { rc = AMB_ERR_CUDA; break; }
            ctx->encode = (amb_encode_fn)fn;
        }
        if (amb_prefer_max_shared() != cudaSuccess) { rc = AMB_ERR_CUDA; break; }
        rc = setup_rate(ctx);
        if (rc != AMB_OK) break;
        rc = reset_stream(ctx);
    } while (0);
    if (rc != AMB_OK) { amb_destroy(ctx); return rc; }
    *out = ctx;
    return AMB_OK;
}

void amb_destroy(amb_ctx* ctx)
{
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    if (ctx->stream) sync_all(ctx);
    if (ctx->stream_h) { cudaStreamSynchronize(ctx->stream_h); }
    for (int k = 0; k < 3; k++) cudaFree(ctx->carry[k]);
    cudaFree(ctx->tail[0]); cudaFree(ctx->tail[1]); cudaFree(ctx->staging);
    cudaFree(ctx->dc_carry[0]); cudaFree(ctx->dc_carry[1]); cudaFree(ctx->dc_out); cudaFree(ctx->dc_ma0);
    cudaFree(ctx->ctr); cudaFree(ctx->st);
    amb_chain_free(&ctx->bufs);
    ingest_free(ctx);
    cudaFree(ctx->ord_key); cudaFree(ctx->ord_val); cudaFree(ctx->tags_dev);
    if (ctx->stream_h) cudaStreamDestroy(ctx->stream_h);
    if (ctx->ctr_snap) cudaFreeHost(ctx->ctr_snap);
    for (int k = 0; k < AMB_SNAPS; k++) if (ctx->snap_ev[k]) cudaEventDestroy(ctx->snap_ev[k]);
    for (int k = 0; k < 2; k++) {
        if (ctx->e_scan[k]) cudaEventDestroy(ctx->e_scan[k]);
        if (ctx->e_done[k]) cudaEventDestroy(ctx->e_done[k]);
        if (ctx->e_aux[k]) cudaEventDestroy(ctx->e_aux[k]);
    }
    if (ctx->e_in) cudaEventDestroy(ctx->e_in);
    if (ctx->stream_b) cudaStreamDestroy(ctx->stream_b);
    if (ctx->stream_c) cudaStreamDestroy(ctx->stream_c);
    for (int k = 0; k < 4; k++) if (ctx->ev[k]) cudaEventDestroy(ctx->ev[k]);
    for (int k = 0; k < 128; k++) if (ctx->ring[k]) cudaEventDestroy(ctx->ring[k]);
    for (int k = 0; k < 64; k++) if (ctx->ring_done[k]) cudaEventDestroy(ctx->ring_done[k]);
    if (ctx->own_stream && ctx->stream) cudaStreamDestroy(ctx->stream);
    delete ctx;
}

int amb_reset(amb_ctx* ctx)
{
    if (!ctx) return AMB_ERR_INVALID;
    CK(ctx, cudaSetDevice(ctx->device));
    return reset_stream(ctx);
}

int amb_set_rate(amb_ctx* ctx, float channel_rate)
{
    if (!ctx) return AMB_ERR_INVALID;
    CK(ctx, cudaSetDevice(ctx->device));
    CK(ctx, sync_all(ctx));
    const float old = ctx->rate_arg;
    ctx->rate_arg = channel_rate;
    int rc = setup_rate(ctx);
    if (rc != AMB_OK) { ctx->rate_arg = old; setup_rate(ctx); reset_stream(ctx); return rc; }
    return reset_stream(ctx);
}

int amb_set_threshold(amb_ctx* ctx, float threshold_db)
{
    if (!ctx) return AMB_ERR_INVALID;
    ctx->thr_db = threshold_db;                          // preamble_impl.cc:65-68
    AmbParams P; int off[240];
    int rc = compute_params(ctx->rate_arg, threshold_db, ctx->use_pmf, &P, off);
    if (rc != AMB_OK) return rc;
    ctx->P = P;
    return AMB_OK;
}

float amb_get_rate(const amb_ctx* ctx) { return ctx ? (float)ctx->P.rate_int : 0.f; }   // preamble_impl.cc:74-76
float amb_get_threshold(const amb_ctx* ctx) { return ctx ? ctx->thr_db : 0.f; }         // :70-72
int amb_get_pmf(const amb_ctx* ctx) { return ctx ? ctx->use_pmf : 0; }

int amb_set_start_time(amb_ctx* ctx, uint64_t secs, double frac)
{
    if (!ctx) return AMB_ERR_INVALID;
    ctx->t0_secs = secs; ctx->t0_frac = frac;
    return AMB_OK;
}

int amb_query_geometry(float rate, float threshold_db, int use_pmf, amb_geometry* out)
{
    if (!out) return AMB_ERR_INVALID;
    AmbParams P; int off[240];
    int rc = compute_params(rate, threshold_db, use_pmf, &P, off);
    if (rc != AMB_OK) return rc;
    out->samples_per_chip = P.spc_f; out->samples_per_symbol = P.sps_f; out->threshold = P.thr;
    out->rate_int = P.rate_int; out->history = P.H + 1; out->check_width = (int)(120 * P.sps_f);   // preamble_impl.cc:59
    out->pulse_offset[0] = 0; out->pulse_offset[1] = P.po1; out->pulse_offset[2] = P.po2; out->pulse_offset[3] = P.po3;
    out->quiet_a[0] = P.qa0; out->quiet_a[1] = P.qa1; out->quiet_b[0] = P.qb0; out->quiet_b[1] = P.qb1;
    out->max_late = P.maxlate; out->packet_skip = P.skip0;
    out->pmf_len = use_pmf ? P.spc_i : 1; out->floor_len = P.L;
    out->chip_offset_239 = off[239];
    out->shard_back = P.H + P.L + P.spc_i;                         // block history + floor window + PMF window
    out->shard_fwd = amb_chain_guard(P) - P.H;                    // the streaming guard, in sample coordinates
    return AMB_OK;
}

int amb_set_stream(amb_ctx* ctx, void* cuda_stream)
{
    if (!ctx) return AMB_ERR_INVALID;
    CK(ctx, sync_all(ctx));
    if (ctx->own_stream) { cudaStreamDestroy(ctx->stream); ctx->own_stream = false; }
    ctx->stream = (cudaStream_t)cuda_stream;
    return AMB_OK;
}

int amb_enable_timing(amb_ctx* ctx, int on) { if (!ctx) return AMB_ERR_INVALID; ctx->timing = on != 0; return AMB_OK; }

int amb_set_option(amb_ctx* ctx, const char* name, int value)
{
    if (!ctx || !name) return AMB_ERR_INVALID;
    if (!strcmp(name, "resolver")) { ctx->resolver = value; return AMB_OK; }
    if (!strcmp(name, "ec")) { if (value < 0 || value > 23) return AMB_ERR_INVALID; ctx->ec = value; return AMB_OK; }
    if (!strcmp(name, "ec_any")) { if (value < 0 || value > 2) return AMB_ERR_INVALID; ctx->ec_any = value; return AMB_OK; }
    if (!strcmp(name, "ap_filter")) {
        if (value < 0 || value > 3600) return AMB_ERR_INVALID;
        if (value && (ctx->defer || ctx->seeked))
            return fail(ctx, AMB_ERR_STATE, "ap_filter needs the whole stream: not available in time-sharded operation");
        ctx->ap_filter = value; return AMB_OK;
    }
    if (!strcmp(name, "keep_chips")) { ctx->keep_chips = value != 0; return AMB_OK; }
    if (!strcmp(name, "overlap")) { ctx->overlap = value != 0; return AMB_OK; }
    if (!strcmp(name, "coalesce")) {                       // samples of small host calls gathered before a dispatch
        if (value < 1) return AMB_ERR_INVALID;
        ctx->coalesce = std::min((size_t)value, ctx->ing_chunk); return AMB_OK;
    }
    if (!strcmp(name, "exact_dense")) { if (value < 0) return AMB_ERR_INVALID; ctx->exact_dense = (unsigned)value; return AMB_OK; }
    if (!strcmp(name, "scan_ctas")) { if (value < 0 || value > 65536) return AMB_ERR_INVALID; ctx->scan_ctas = value; return AMB_OK; }
    if (!strcmp(name, "order_tile")) {                     // elements per CTA of the device-side drain's sorting network
        if (value < 2 || value > 2048 || (value & (value - 1))) return AMB_ERR_INVALID;
        ctx->order_tile = (unsigned)value; return AMB_OK;
    }
    if (!strcmp(name, "copy_threads")) { if (value < 0 || value > 64) return AMB_ERR_INVALID; ctx->copy_threads = value; return AMB_OK; }
    if (!strcmp(name, "ingest_chunk")) {                   // samples per chunk of the host ingest ring (multiple of 512)
        if (value < 4096 || (value & 511)) return AMB_ERR_INVALID;
        CK(ctx, cudaSetDevice(ctx->device));
        if (ctx->pend_n) { int rc = ingest_dispatch_pending(ctx, 0); if (rc) return rc; }
        CK(ctx, sync_all(ctx));
        if (ctx->stream_h) CK(ctx, cudaStreamSynchronize(ctx->stream_h));
        ingest_free(ctx);
        ctx->ing_chunk = (size_t)value;
        if (ctx->coalesce > ctx->ing_chunk) ctx->coalesce = ctx->ing_chunk;
        return AMB_OK;
    }
    if (!strcmp(name, "defer_resolve")) {
        if (ctx->def_kind && !ctx->def_resolved) return fail(ctx, AMB_ERR_STATE, "amb_resolve pending");
        if (value && ctx->ap_filter) return fail(ctx, AMB_ERR_STATE, "defer_resolve is not available with ap_filter on");
        ctx->def_kind = 0; ctx->def_resolved = false;
        ctx->defer = value != 0; return AMB_OK;
    }
    return AMB_ERR_INVALID;
}

int amb_synchronize(amb_ctx* ctx)
{
    if (!ctx) return AMB_ERR_INVALID;
    CK(ctx, cudaSetDevice(ctx->device));
    if (ctx->pend_n) { int rc = ingest_dispatch_pending(ctx, 0); if (rc) return rc; }
    CK(ctx, sync_all(ctx));
    return AMB_OK;
}

// One call of the chain over n_complex samples that are in DEVICE memory (or, mem_kind == AMB_MEM_HOST, in host
// memory that goes through the one-piece staging buffer: the deferred / time-sharded mode only).
static int process_core(amb_ctx* ctx, const float* iq, size_t n_complex, int mem_kind, int flush)
{
    if (n_complex > 0x40000000ull) return fail(ctx, AMB_ERR_INVALID, "internal: at most 2^30 samples per pass");
    ctx->def_kind = 0; ctx->def_resolved = false;
    cudaStream_t sa = ctx->stream, sb = ctx->stream_b, sc = ctx->stream_c;
    const AmbParams& P = ctx->P;
    const int kc = ctx->kc;
    const int set = (int)(ctx->call_idx & 1u);             // double-buffered per-call scratch
    if (ctx->timing) CK(ctx, cudaEventRecord(ctx->ev[2], sa));
    // stream C stages the tail and the next carry. It starts where the caller's stream is now (the input is
    // ready there) and after call k-2's sparse kernels, the last users of this set's buffers.
    CK(ctx, cudaEventRecord(ctx->e_in, sa));
    CK(ctx, cudaStreamWaitEvent(sc, ctx->e_in, 0));
    if (ctx->done_valid[set]) { CK(ctx, cudaStreamWaitEvent(sc, ctx->e_done[set], 0)); CK(ctx, cudaStreamWaitEvent(sa, ctx->e_done[set], 0)); }

    // ---- input placement: device pointers are used in place, host data goes through a staging buffer
    const float2* src = reinterpret_cast<const float2*>(iq);
    if (mem_kind == AMB_MEM_HOST || ((uintptr_t)iq & 15u)) {
        if (ctx->staging_cap < n_complex) {
            CK(ctx, sync_all(ctx));
            cudaFree(ctx->staging); ctx->staging = nullptr;
            size_t ncap = n_complex + 1024;
            CK(ctx, cudaMalloc(&ctx->staging, ncap * sizeof(float2)));
            ctx->staging_cap = ncap;
        }
        // the previous call's exact/slice kernels and its carry kernel may still read the staging buffer
        if (ctx->done_valid[set ^ 1]) CK(ctx, cudaStreamWaitEvent(sa, ctx->e_done[set ^ 1], 0));
        if (ctx->aux_valid[set ^ 1]) CK(ctx, cudaStreamWaitEvent(sa, ctx->e_aux[set ^ 1], 0));
        if (n_complex)
            CK(ctx, cudaMemcpyAsync(ctx->staging, iq, n_complex * sizeof(float2),
                               mem_kind == AMB_MEM_HOST ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice, sa));
        src = ctx->staging;
        CK(ctx, cudaEventRecord(ctx->e_in, sa));
        CK(ctx, cudaStreamWaitEvent(sc, ctx->e_in, 0));
    }
    if (ctx->use_dcblock) {
        // ---- DC blocker: x -> out[n] = x[n-D+1] - MA(MA(x))[n] into a ctx-owned buffer that then plays the input
        if (ctx->dc_cap < n_complex + (size_t)ctx->dc_D) {
            CK(ctx, sync_all(ctx));
            cudaFree(ctx->dc_out); ctx->dc_out = nullptr;
            const size_t ncap = n_complex + (size_t)ctx->dc_D + 1024;
            CK(ctx, cudaMalloc(&ctx->dc_out, ncap * sizeof(float2)));
            ctx->dc_cap = ncap;
        }
        // the previous call's exact/slice kernels and its carry kernel still read dc_out
        if (ctx->done_valid[set ^ 1]) CK(ctx, cudaStreamWaitEvent(sa, ctx->e_done[set ^ 1], 0));
        if (ctx->aux_valid[set ^ 1]) CK(ctx, cudaStreamWaitEvent(sa, ctx->e_aux[set ^ 1], 0));
        CK(ctx, amb_launch_dcblock(ctx->dc_carry[ctx->dc_cur], ctx->dc_nc, src, (long long)n_complex, ctx->dc_D,
                              ctx->dc_ma0, ctx->dc_out, ctx->dc_carry[ctx->dc_cur ^ 1], sa));
        ctx->dc_cur ^= 1;
        ctx->stats.kernel_launches += n_complex ? 2 : 1;
        src = ctx->dc_out;
        CK(ctx, cudaEventRecord(ctx->e_in, sa));
        CK(ctx, cudaStreamWaitEvent(sc, ctx->e_in, 0));
    }
    const AmbSegs S = amb_chain_segs(ctx->carry[ctx->carry_in], kc, src, (int)n_complex, ctx->tail[set]);
    const int n_tv = (int)n_complex - S.n_main;
    const int cin = ctx->carry_in;                         // carry this call reads
    const int cout = (cin == 0) ? 1 : 0;                   // carry this call writes (never the zero buffer [2])

    const long long org = (long long)ctx->n_in - kc + P.H;        // reported index of j = 0
    const long long n_after = (long long)ctx->n_in + (long long)n_complex;
    long long j_lo = ctx->r_done - org;
    long long j_hi, r_safe = 0, ntot = 0;
    if (flush) { ntot = n_after + P.H; j_hi = S.n_valid; }
    else { r_safe = n_after + P.H - ctx->guard; if (r_safe < ctx->r_done) r_safe = ctx->r_done; j_hi = r_safe - org; }
    ctx->last_org = org; ctx->have_last = true;

    AmbChainCall call{};
    call.P = P; call.S = S; call.org = org; call.ntot = ntot; call.r_safe = r_safe; call.flush = flush ? 1 : 0;
    call.ctr = ctx->ctr; call.st = ctx->st; call.n_samples = (long long)S.n_carry + S.n_main + S.n_tail;
    const AmbChainOpts opts = chain_opts(ctx);
    AmbChainErr er;

    if (j_hi > j_lo) {
        AmbScanArgs a{};
        a.P = P; a.S = S;
        amb_chain_geometry(&a, j_lo, j_hi, false, ctx->sm_count, ctx->scan_ctas);
        // ---- buffers (growth synchronises every stream; steady state does not)
        const unsigned fr_ub = amb_chain_frame_bound(P, j_hi - j_lo);
        if (amb_chain_prepare(&ctx->bufs, &a, set, amb_chain_cand_capacity(j_hi - j_lo), fr_ub, ctx->keep_chips,
                              [ctx] { return sync_all(ctx); }, &er) < 0) return chain_fail(ctx, er);
        ctx->bufs.frames_ub += fr_ub;
        a.tm_carry = ctx->tm_carry[cin]; a.tm_tail = ctx->tm_tail[set];
        if (S.n_main) { int rc2 = make_tmap(ctx, &a.tm_main, src, (size_t)S.n_main); if (rc2) return rc2; }
        else a.tm_main = ctx->tm_tail[set];

        // ---- stream A: stage the tail + reset the group counts (in front of the scan: a hop over to stream C and
        // back would leave the scan stream idle), then stream over the IQ. Stream C's carry kernel reads the tail.
        CK(ctx, amb_launch_prologue(ctx->tail[set], AMB_TAIL_CAP, src + S.n_main, n_tv, a.group_count, 128, sa));
        ctx->stats.kernel_launches += 1;
        CK(ctx, cudaEventRecord(ctx->e_in, sa));
        CK(ctx, cudaStreamWaitEvent(sc, ctx->e_in, 0));
        if (ctx->aux_valid[set ^ 1]) CK(ctx, cudaStreamWaitEvent(sa, ctx->e_aux[set ^ 1], 0));   // carry written by the previous call
        const unsigned slot = (ctx->ring_n & 63u) * 2;
        if (ctx->timing) { CK(ctx, cudaEventRecord(ctx->ev[0], sa)); CK(ctx, cudaEventRecord(ctx->ring[slot], sa)); }
        CK(ctx, amb_launch_scan(a, ctx->sm_count, sa));
        ctx->stats.kernel_launches += 1;
        if (ctx->timing) { CK(ctx, cudaEventRecord(ctx->ev[1], sa)); CK(ctx, cudaEventRecord(ctx->ring[slot + 1], sa)); ctx->ring_n++; }
        CK(ctx, cudaEventRecord(ctx->e_scan[set], sa));

        // ---- stream B: everything sparse; runs under the NEXT call's scan. A time-sharded span stops before the
        // walk: its loop state arrives later (amb_resolve).
        CK(ctx, cudaStreamWaitEvent(sb, ctx->e_scan[set], 0));
        const int k = amb_chain_launch(a, call, &ctx->bufs, opts, ctx->defer != 0, sb, &ctx->def, &er);
        if (k < 0) return chain_fail(ctx, er);
        ctx->stats.kernel_launches += (uint64_t)k;
        if (ctx->defer) { ctx->def_kind = 1; ctx->def_resolved = false; ctx->def_set = set; }
        ctx->ev_valid = ctx->timing;
    } else {
        // nothing can be decided yet (tiny call): keep it simple and serial
        if (ctx->done_valid[set ^ 1]) CK(ctx, cudaStreamWaitEvent(sa, ctx->e_done[set ^ 1], 0));
        CK(ctx, amb_launch_prologue(ctx->tail[set], AMB_TAIL_CAP, src + S.n_main, n_tv, nullptr, 0, sa));
        ctx->stats.kernel_launches += 1;
        CK(ctx, cudaEventRecord(ctx->e_in, sa));
        CK(ctx, cudaStreamWaitEvent(sc, ctx->e_in, 0));
        if (ctx->aux_valid[set ^ 1]) CK(ctx, cudaStreamWaitEvent(sa, ctx->e_aux[set ^ 1], 0));
        CK(ctx, cudaEventRecord(ctx->e_scan[set], sa));
        CK(ctx, cudaStreamWaitEvent(sb, ctx->e_scan[set], 0));
        if (ctx->defer) { ctx->def_kind = flush ? 2 : 3; ctx->def_resolved = false; ctx->def_set = set; }
        if (flush) {   // the resolver still has to close the stream
            if (amb_chain_prepare_empty(&ctx->bufs, &er) < 0) return chain_fail(ctx, er);
            AmbChainSpan& sp = ctx->def;
            sp.wa = amb_chain_walk_args(call, ctx->bufs, ctx->sm_count);
            sp.par = false; sp.walk_only = true;
            CK(ctx, cudaMemsetAsync(&ctx->ctr->ncand, 0, sizeof(unsigned), sb));
            if (!ctx->defer) {
                const int k = amb_chain_resolve(sp, &ctx->bufs, opts, sb, &er);
                if (k < 0) return chain_fail(ctx, er);
                ctx->stats.kernel_launches += (uint64_t)k;
            }
        }
        ctx->ev_valid = false;
    }
    if (!ctx->defer && ctx->ctr_snap && ctx->snap_head - ctx->snap_tail < AMB_SNAPS) {
        // where the frame counter stands once this call is through: read without blocking by amb_poll_ready
        const unsigned k = (unsigned)(ctx->snap_head % AMB_SNAPS);
        CK(ctx, cudaMemcpyAsync(&ctx->ctr_snap[k], ctx->ctr, sizeof(AmbCounters), cudaMemcpyDeviceToHost, sb));
        CK(ctx, cudaEventRecord(ctx->snap_ev[k], sb));
        ctx->snap_head++;
    }
    CK(ctx, cudaEventRecord(ctx->e_done[set], sb));
    ctx->done_valid[set] = true;
    if (ctx->timing) {
        CK(ctx, cudaEventRecord(ctx->ev[3], sb));
        if (ctx->ev_valid) CK(ctx, cudaEventRecord(ctx->ring_done[(ctx->ring_n - 1) & 63u], sb));
    }
    // ---- carry the tail of the stream into the next call (stream C, concurrently with this call's scan).
    // The buffer written here is the one the PREVIOUS call's scan and sparse kernels read as their carry.
    if (ctx->done_valid[set ^ 1]) CK(ctx, cudaStreamWaitEvent(sc, ctx->e_done[set ^ 1], 0));
    CK(ctx, amb_launch_carry(S, ctx->carry[cout], kc, sc));
    CK(ctx, cudaEventRecord(ctx->e_aux[set], sc));
    ctx->aux_valid[set] = true;
    ctx->stats.kernel_launches += 1;
    ctx->carry_in = cout;
    ctx->n_in = (uint64_t)n_after;
    if (flush) ctx->flushed = true;
    else if (j_hi > j_lo) ctx->r_done = r_safe;
    ctx->call_idx++;
    if (!ctx->overlap) {                                                    // strict stream-ordered behaviour on stream A
        CK(ctx, cudaStreamWaitEvent(sa, ctx->e_done[set], 0));
        CK(ctx, cudaStreamWaitEvent(sa, ctx->e_aux[set], 0));
    }
    return AMB_OK;
}

/* ---- host ingest pipeline ------------------------------------------------------------------------------------
 * Host memory never reaches the chain as one monolithic copy. The stream is cut into chunks of ing_chunk samples
 * that travel through a ring of AMB_ING_SLOTS device buffers on a copy stream of their own: the H2D copy (and, for
 * 16-bit input, the widening kernel) of chunk k+1 runs under the scan of chunk k, the streaming carry makes the cut
 * invisible in the results. Pinned caller memory is DMA'd from where it lies; pageable memory and small calls (what a
 * GNU Radio scheduler hands over: <= 32 k items per work()) are first gathered in the ring's pinned host buffers by a
 * few copy threads, and a partly filled chunk is only dispatched once `coalesce` samples are pending or somebody asks
 * for results (poll / flush / synchronize). */
namespace {
struct CopyPool {
    std::vector<std::thread> th;
    std::mutex m;
    std::condition_variable cv, done_cv;
    struct Task { char* d; const char* s; size_t n; int* left; };   // left: the submitting call's count of unfinished pieces
    std::deque<Task> q;
    bool stop = false;
    explicit CopyPool(int n)
    {
        for (int k = 0; k < n; k++) th.emplace_back([this] {
            for (;;) {
                Task t;
                {
                    std::unique_lock<std::mutex> lk(m);
                    cv.wait(lk, [this] { return stop || !q.empty(); });
                    if (stop && q.empty()) return;
                    t = q.front(); q.pop_front();
                }
                memcpy(t.d, t.s, t.n);
                { std::lock_guard<std::mutex> lk(m); if (--*t.left == 0) done_cv.notify_all(); }
            }
        });
    }
    ~CopyPool()
    {
        { std::lock_guard<std::mutex> lk(m); stop = true; }
        cv.notify_all();
        for (auto& t : th) t.join();
    }
    void copy(char* d, const char* s, size_t n)
    {
        const size_t piece = (size_t)1 << 20;
        if (th.empty() || n < 2 * piece) { memcpy(d, s, n); return; }
        size_t per = (n / (th.size() + 1) + 4095) & ~(size_t)4095;
        if (per < piece) per = piece;
        size_t off = per;                                   // the caller copies the first piece itself
        int left = 0;                                       // several contexts / threads may share the pool: each call counts its own pieces
        {
            std::lock_guard<std::mutex> lk(m);
            for (; off < n; off += per) { q.push_back({d + off, s + off, std::min(per, n - off), &left}); left++; }
        }
        cv.notify_all();
        memcpy(d, s, std::min(per, n));
        std::unique_lock<std::mutex> lk(m);
        done_cv.wait(lk, [&left] { return left == 0; });
    }
};
std::mutex g_pool_mutex;
CopyPool* g_pools[65] = {};                                 // one pool per thread count, created on first use, never torn down:
CopyPool* copy_pool(int want)                               // a context of another thread may be inside copy() of any of them
{
    std::lock_guard<std::mutex> lk(g_pool_mutex);
    if (want <= 0) {
        static const int dflt = (int)std::min(24u, std::max(1u, std::thread::hardware_concurrency() / 6));
        want = dflt;                                        // enough to outrun a PCIe Gen5 x16 link, never the whole box
    }
    if (want > 64) want = 64;
    if (!g_pools[want]) g_pools[want] = new CopyPool(want - 1);
    return g_pools[want];
}
}  // namespace

// also used by the decoder's staging (amb_decode.cu)
void amb_parallel_memcpy(void* dst, const void* src, size_t n) { copy_pool(0)->copy(static_cast<char*>(dst), static_cast<const char*>(src), n); }

static int ingest_setup(amb_ctx* ctx, bool need_raw)
{
    if (!ctx->stream_h) CK(ctx, cudaStreamCreateWithFlags(&ctx->stream_h, cudaStreamNonBlocking));
    for (int k = 0; k < AMB_ING_SLOTS; k++) {
        AmbIngestSlot& sl = ctx->ing[k];
        if (!sl.dev) {
            CK(ctx, cudaMalloc(&sl.dev, ctx->ing_chunk * sizeof(float2)));
            CK(ctx, cudaMallocHost(&sl.pin, ctx->ing_chunk * sizeof(float2)));
            CK(ctx, cudaEventCreateWithFlags(&sl.e_h2d, cudaEventDisableTiming));
            CK(ctx, cudaEventCreateWithFlags(&sl.e_free_b, cudaEventDisableTiming));
            CK(ctx, cudaEventCreateWithFlags(&sl.e_free_c, cudaEventDisableTiming));
        }
        if (need_raw && !sl.dev_raw) CK(ctx, cudaMalloc(&sl.dev_raw, ctx->ing_chunk * 4));
    }
    return AMB_OK;
}

static void ingest_free(amb_ctx* c)
{
    for (int k = 0; k < AMB_ING_SLOTS; k++) {
        AmbIngestSlot& sl = c->ing[k];
        cudaFree(sl.dev); cudaFree(sl.dev_raw);
        if (sl.pin) cudaFreeHost(sl.pin);
        if (sl.e_h2d) cudaEventDestroy(sl.e_h2d);
        if (sl.e_free_b) cudaEventDestroy(sl.e_free_b);
        if (sl.e_free_c) cudaEventDestroy(sl.e_free_c);
        sl = AmbIngestSlot();
    }
    c->pend_n = 0; c->ing_next = 0;
}

// One chunk: `src` (host or device memory, float32 I/Q or 16-bit I/Q) -> ring slot -> the chain.
static int ingest_dispatch(amb_ctx* ctx, const void* src, size_t m, bool sc16, bool src_on_device, int flush)
{
    const unsigned s_idx = ctx->ing_next % AMB_ING_SLOTS;
    AmbIngestSlot& sl = ctx->ing[s_idx];
    cudaStream_t sh = ctx->stream_h;
    if (sl.used) {        // the chunk that lived here before: its sparse kernels and its carry kernel must be through
        CK(ctx, cudaStreamWaitEvent(sh, sl.e_free_b, 0));
        CK(ctx, cudaStreamWaitEvent(sh, sl.e_free_c, 0));
    }
    if (m) {
        const cudaMemcpyKind kind = src_on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
        if (sc16) {
            CK(ctx, cudaMemcpyAsync(sl.dev_raw, src, m * 4, kind, sh));
            CK(ctx, amb_launch_widen_sc16(sl.dev_raw, sl.dev, (long long)m, ctx->sm_count, sh));
            ctx->stats.kernel_launches += 1;
        } else {
            CK(ctx, cudaMemcpyAsync(sl.dev, src, m * sizeof(float2), kind, sh));
        }
    }
    CK(ctx, cudaEventRecord(sl.e_h2d, sh));
    sl.h2d_pending = true;
    CK(ctx, cudaStreamWaitEvent(ctx->stream, sl.e_h2d, 0));
    int rc = process_core(ctx, reinterpret_cast<const float*>(sl.dev), m, AMB_MEM_DEVICE, flush);
    if (rc != AMB_OK) return rc;
    CK(ctx, cudaEventRecord(sl.e_free_b, ctx->stream_b));
    CK(ctx, cudaEventRecord(sl.e_free_c, ctx->stream_c));
    sl.used = true;
    ctx->ing_next++;
    return AMB_OK;
}

// The pinned buffer of the slot the next chunk will use, safe to write into (its last H2D has completed).
static int ingest_pinned_slot(amb_ctx* ctx, char** out)
{
    AmbIngestSlot& sl = ctx->ing[ctx->ing_next % AMB_ING_SLOTS];
    if (sl.h2d_pending) { CK(ctx, cudaEventSynchronize(sl.e_h2d)); sl.h2d_pending = false; }
    *out = static_cast<char*>(sl.pin);
    return AMB_OK;
}

static int ingest_dispatch_pending(amb_ctx* ctx, int flush)
{
    if (!ctx->pend_n && !flush) return AMB_OK;
    const size_t m = ctx->pend_n;
    ctx->pend_n = 0;
    return ingest_dispatch(ctx, ctx->ing[ctx->ing_next % AMB_ING_SLOTS].pin, m, ctx->pend_kind == AMB_MEM_HOST_SC16, false, flush);
}

static bool is_pinned_host(const void* p)
{
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, p) != cudaSuccess) { cudaGetLastError(); return false; }
    return at.type == cudaMemoryTypeHost;
}

static int ingest(amb_ctx* ctx, const void* data, size_t n, int mem_kind, int flush)
{
    const bool sc16 = mem_kind == AMB_MEM_HOST_SC16 || mem_kind == AMB_MEM_DEVICE_SC16;
    const bool on_dev = mem_kind == AMB_MEM_DEVICE_SC16 || mem_kind == AMB_MEM_DEVICE;
    const size_t esz = sc16 ? 4 : sizeof(float2);
    { int rc = ingest_setup(ctx, sc16); if (rc) return rc; }
    const size_t CH = ctx->ing_chunk;
    if (ctx->pend_n && (on_dev || ctx->pend_kind != mem_kind)) { int rc = ingest_dispatch_pending(ctx, 0); if (rc) return rc; }
    const char* p = static_cast<const char*>(data);
    size_t left = n;
    bool flushed = false;
    const bool direct_ok = on_dev || is_pinned_host(p);
    cudaEvent_t last_direct = nullptr;                         // last DMA out of the caller's own (pinned) host memory
    while (left) {
        if (!ctx->pend_n && direct_ok && (on_dev || left >= ctx->coalesce)) {
            const size_t m = std::min(left, CH);               // straight from the caller's memory
            const int fl = flush && m == left;
            if (!on_dev) last_direct = ctx->ing[ctx->ing_next % AMB_ING_SLOTS].e_h2d;
            int rc = ingest_dispatch(ctx, p, m, sc16, on_dev, fl); if (rc) return rc;
            flushed = fl != 0;
            p += m * esz; left -= m;
            continue;
        }
        char* pin = nullptr;
        { int rc = ingest_pinned_slot(ctx, &pin); if (rc) return rc; }
        const size_t m = std::min(left, CH - ctx->pend_n);
        copy_pool(ctx->copy_threads)->copy(pin + ctx->pend_n * esz, p, m * esz);
        ctx->pend_n += m; ctx->pend_kind = mem_kind;
        p += m * esz; left -= m;
        if (ctx->pend_n == CH || (!left && (flush || ctx->pend_n >= ctx->coalesce))) {
            const int fl = flush && !left;
            int rc = ingest_dispatch_pending(ctx, fl); if (rc) return rc;
            flushed = fl != 0;
        }
    }
    if (flush && !flushed) { int rc = ingest_dispatch_pending(ctx, 1); if (rc) return rc; }   // also closes an empty stream
    // host memory is consumed when the call returns: the copies out of a pinned caller buffer are asynchronous, so wait
    // for the last of them (the kernels behind it stay asynchronous)
    if (last_direct) CK(ctx, cudaEventSynchronize(last_direct));
    return AMB_OK;
}

int amb_process(amb_ctx* ctx, const float* iq, size_t n_complex, int mem_kind, int flush)
{
    if (!ctx || (!iq && n_complex)) return AMB_ERR_INVALID;
    if (mem_kind < AMB_MEM_HOST || mem_kind > AMB_MEM_DEVICE_SC16) return AMB_ERR_INVALID;
    if (ctx->flushed) return fail(ctx, AMB_ERR_STATE, "stream already flushed; amb_reset first");
    if (ctx->def_kind && !ctx->def_resolved)
        return fail(ctx, AMB_ERR_STATE, "amb_resolve pending (deferred mode allows one call per span)");
    CK(ctx, cudaSetDevice(ctx->device));
    if (ctx->defer) {     // time-sharded span: one pass, input stays where it is (or goes through the one-piece staging buffer)
        if (mem_kind != AMB_MEM_HOST && mem_kind != AMB_MEM_DEVICE)
            return fail(ctx, AMB_ERR_UNSUPPORTED, "16-bit input is not available in deferred (time-sharded) mode");
        if (n_complex > 0x40000000ull) return fail(ctx, AMB_ERR_INVALID, "a time-sharded span holds at most 2^30 samples");
        return process_core(ctx, iq, n_complex, mem_kind, flush);
    }
    if (mem_kind == AMB_MEM_DEVICE && !((uintptr_t)iq & 15u)) {
        // device-resident float32 input is read in place; only very long buffers are cut (int indexing inside a pass)
        if (ctx->pend_n) { int rc = ingest_dispatch_pending(ctx, 0); if (rc) return rc; }
        const size_t piece = (size_t)1 << 30;
        size_t done = 0;
        do {
            const size_t m = std::min(piece, n_complex - done);
            int rc = process_core(ctx, iq + 2 * done, m, AMB_MEM_DEVICE, flush && done + m == n_complex);
            if (rc) return rc;
            done += m;
        } while (done < n_complex);
        return AMB_OK;
    }
    return ingest(ctx, iq, n_complex, mem_kind, flush);
}

/* ---- time-sharding: see the header ---------------------------------------------------------------------- */
int amb_seek(amb_ctx* ctx, uint64_t first_sample, uint64_t first_decision, const amb_walk_state* entry)
{
    if (!ctx) return AMB_ERR_INVALID;
    CK(ctx, cudaSetDevice(ctx->device));
    const AmbParams& P = ctx->P;
    if (first_sample) {
        if (ctx->use_dcblock) return fail(ctx, AMB_ERR_UNSUPPORTED, "amb_seek into a stream is not available with the DC blocker");
        if (first_decision < first_sample + (uint64_t)(P.H + P.L + P.spc_i))
            return fail(ctx, AMB_ERR_INVALID, "first_decision must be at least first_sample + shard_back");
    }
    if (first_sample > (1ull << 62) || first_decision > (1ull << 62)) return fail(ctx, AMB_ERR_INVALID, "index out of range");
    if (ctx->ap_filter) return fail(ctx, AMB_ERR_STATE, "amb_seek is not available with ap_filter on (it needs the whole stream)");
    int rc = reset_stream(ctx);
    if (rc != AMB_OK) return rc;
    ctx->n_in = first_sample;
    ctx->r_done = (long long)first_decision;
    const long long pos = entry ? (long long)entry->pos : (long long)first_decision;
    const long long p = entry ? (long long)entry->p : (long long)first_decision;
    CK(ctx, amb_launch_set_state(ctx->st, pos, p, ctx->stream_b));          // after reset_stream's memset on stream B
    ctx->stats.kernel_launches += 1;
    ctx->seeked = true;
    return AMB_OK;
}

// The deferred call's walk + slice stages on stream B (amb_resolve, amb_resolve_device), from the entry state in
// entry_dev (device memory, read when the kernel runs) or entry (NULL: where the previous span left the resolver).
static int resolve_deferred(amb_ctx* ctx, const amb_walk_state* entry, const int64_t* entry_dev)
{
    cudaStream_t sb = ctx->stream_b;
    if (ctx->def_resolved && ctx->def_kind == 1) {     // forget the earlier (speculative) resolution of this span
        CK(ctx, amb_launch_walk_reset(ctx->def.wa, ctx->def.par ? ctx->bufs.walk_scratch : nullptr, ctx->def.n_samples, sb));
        ctx->stats.kernel_launches += 1;
    }
    if (entry_dev) CK(ctx, amb_launch_set_state_dev(ctx->st, reinterpret_cast<const long long*>(entry_dev), sb));
    else if (entry) CK(ctx, amb_launch_set_state(ctx->st, (long long)entry->pos, (long long)entry->p, sb));
    if (entry_dev || entry) ctx->stats.kernel_launches += 1;
    if (ctx->def_kind != 3) {
        AmbChainErr er;
        const int k = amb_chain_resolve(ctx->def, &ctx->bufs, chain_opts(ctx), sb, &er);
        if (k < 0) return chain_fail(ctx, er);
        ctx->stats.kernel_launches += (uint64_t)k;
    }
    CK(ctx, cudaEventRecord(ctx->e_done[ctx->def_set], sb));
    if (ctx->timing) CK(ctx, cudaEventRecord(ctx->ev[3], sb));
    if (!ctx->overlap) CK(ctx, cudaStreamWaitEvent(ctx->stream, ctx->e_done[ctx->def_set], 0));
    ctx->def_resolved = true;
    return AMB_OK;
}

int amb_resolve(amb_ctx* ctx, const amb_walk_state* entry)
{
    if (!ctx) return AMB_ERR_INVALID;
    if (!ctx->def_kind) return fail(ctx, AMB_ERR_STATE, "no deferred call to resolve");
    if (ctx->def_resolved && !entry) return fail(ctx, AMB_ERR_INVALID, "re-resolution needs an entry state");
    CK(ctx, cudaSetDevice(ctx->device));
    return resolve_deferred(ctx, entry, nullptr);
}

int amb_get_walk_state(amb_ctx* ctx, amb_walk_state* out)
{
    if (!ctx || !out) return AMB_ERR_INVALID;
    if (ctx->def_kind && !ctx->def_resolved) return fail(ctx, AMB_ERR_STATE, "amb_resolve pending");
    CK(ctx, cudaSetDevice(ctx->device));
    CK(ctx, cudaStreamSynchronize(ctx->stream_b));
    AmbWalkState st;
    CK(ctx, cudaMemcpy(&st, ctx->st, sizeof st, cudaMemcpyDeviceToHost));
    out->pos = st.pos; out->p = st.p;
    return AMB_OK;
}

int amb_get_walk_summary(amb_ctx* ctx, amb_walk_summary* out)
{
    if (!ctx || !out) return AMB_ERR_INVALID;
    if (!ctx->def_kind || !ctx->def_resolved) return fail(ctx, AMB_ERR_STATE, "no resolved deferred span");
    CK(ctx, cudaSetDevice(ctx->device));
    const bool have = ctx->def_kind == 1;
    if (have) { CK(ctx, amb_launch_walk_summary(ctx->def.wa, ctx->stream_b)); ctx->stats.kernel_launches += 1; }
    CK(ctx, cudaStreamSynchronize(ctx->stream_b));
    AmbWalkState st; AmbCounters h;
    CK(ctx, cudaMemcpy(&st, ctx->st, sizeof st, cudaMemcpyDeviceToHost));
    CK(ctx, cudaMemcpy(&h, ctx->ctr, sizeof h, cudaMemcpyDeviceToHost));
    out->pos = st.pos; out->p = st.p;
    out->first_real = (have && st.first_real != ~0ull) ? (int64_t)st.first_real : -1;
    out->first_packet = (have && st.first_packet != ~0ull) ? (int64_t)st.first_packet : -1;
    out->exact_span = ctx->P.i_exact;
    out->frames_passed = have ? (int64_t)h.npassed_call : 0;
    return AMB_OK;
}

/* The same summary, written as six int64 to DEVICE memory by a kernel on the context's second stream: no host
 * synchronisation (amb_join then orders the caller's stream, e.g. an NCCL all-gather, after it). */
int amb_walk_summary_async(amb_ctx* ctx, int64_t* dev_out6)
{
    if (!ctx || !dev_out6) return AMB_ERR_INVALID;
    if (!ctx->def_kind || !ctx->def_resolved) return fail(ctx, AMB_ERR_STATE, "no resolved deferred span");
    CK(ctx, cudaSetDevice(ctx->device));
    const bool have = ctx->def_kind == 1;
    if (have) { CK(ctx, amb_launch_walk_summary(ctx->def.wa, ctx->stream_b)); ctx->stats.kernel_launches += 1; }
    AmbWalkArgs wa = ctx->def.wa; wa.st = ctx->st; wa.ctr = ctx->ctr;
    CK(ctx, amb_launch_pack_summary(wa, ctx->P.i_exact, have ? 1 : 0, reinterpret_cast<long long*>(dev_out6), ctx->stream_b));
    CK(ctx, cudaEventRecord(ctx->e_done[ctx->def_set], ctx->stream_b));
    ctx->stats.kernel_launches += 1;
    return AMB_OK;
}

/* gathered_dev: n_spans x 6 int64 (every span's summary, device memory, ready on the caller-visible stream);
 * out_dev: 1 + 3 n_spans int64: [0] first span whose speculation fails (n_spans - 1: none), [1 + 2k .. 2 + 2k] the true
 * entry (pos, p) of span k, [1 + 2 n_spans + k] messages queued before span k. One tiny kernel on the caller-visible
 * stream; shard.compose_entries is the same computation on the host. */
int amb_compose_entries_async(amb_ctx* ctx, const int64_t* gathered_dev, int n_spans, int64_t* out_dev, void* cuda_stream)
{
    if (!ctx || !gathered_dev || !out_dev || n_spans < 1 || n_spans > 4096) return AMB_ERR_INVALID;
    CK(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : ctx->stream;
    CK(ctx, amb_launch_compose(reinterpret_cast<const long long*>(gathered_dev), n_spans, reinterpret_cast<long long*>(out_dev), st));
    ctx->stats.kernel_launches += 1;
    return AMB_OK;
}

/* amb_resolve with the entry state (pos, p) read from device memory at execution time (e.g. a row of
 * amb_compose_entries_async's output): the walk + slice of the deferred span are enqueued behind whatever produced
 * entry_dev on the caller-visible stream; nothing waits on the host. */
int amb_resolve_device(amb_ctx* ctx, const int64_t* entry_dev, void* after_stream)
{
    if (!ctx || !entry_dev) return AMB_ERR_INVALID;
    if (!ctx->def_kind) return fail(ctx, AMB_ERR_STATE, "no deferred call to resolve");
    CK(ctx, cudaSetDevice(ctx->device));
    CK(ctx, cudaEventRecord(ctx->e_in, after_stream ? (cudaStream_t)after_stream : ctx->stream));
    CK(ctx, cudaStreamWaitEvent(ctx->stream_b, ctx->e_in, 0));
    return resolve_deferred(ctx, nullptr, entry_dev);
}

/* Make a stream wait for everything enqueued so far (no host synchronisation): amb_join = the caller-visible stream,
 * amb_join_stream = any other stream of the caller's (e.g. the one a collective runs on, so that the scan stream is
 * not held up by it). */
int amb_join_stream(amb_ctx* ctx, void* cuda_stream)
{
    if (!ctx) return AMB_ERR_INVALID;
    CK(ctx, cudaSetDevice(ctx->device));
    if (ctx->pend_n) { int rc = ingest_dispatch_pending(ctx, 0); if (rc) return rc; }
    cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : ctx->stream;
    for (int k = 0; k < 2; k++) {
        if (ctx->done_valid[k]) CK(ctx, cudaStreamWaitEvent(st, ctx->e_done[k], 0));
        if (ctx->aux_valid[k]) CK(ctx, cudaStreamWaitEvent(st, ctx->e_aux[k], 0));
    }
    return AMB_OK;
}

int amb_join(amb_ctx* ctx) { return amb_join_stream(ctx, nullptr); }

// tag_to_timestamp with no rx_time tag (preamble_impl.cc:100-137)
// tag_to_timestamp (preamble_impl.cc:100-137) against the rx_time tag in force at the frame: the most recent tag at or
// before it (amb_add_time_tag), else the stream's start time (amb_set_start_time; (0, 0.0) = "no rx_time tag")
static void stamp(const amb_ctx* ctx, amb_frame* f)
{
    const uint64_t rate = (uint64_t)ctx->P.rate_int;
    uint64_t off = 0, t_secs = ctx->t0_secs; double t_frac = ctx->t0_frac;
    for (size_t k = ctx->time_tags.size(); k-- > 0;)
        if (ctx->time_tags[k].offset <= f->sample_index) { off = ctx->time_tags[k].offset; t_secs = ctx->time_tags[k].secs; t_frac = ctx->time_tags[k].frac; break; }
    const uint64_t cnt = f->sample_index - off;                                    // abs_sample_cnt - tstamp.offset
    f->secs = t_secs + cnt / rate;                                                 // :122,:125
    f->frac = t_frac + (double)(cnt % rate) / (double)rate;                        // :123,:126
    if (f->frac > 1.0f) { f->frac -= 1.0f; f->secs += 1; }                         // :127-130
}

// Frames [polled, upto) of the device frame buffer (complete by now) -> pending list, in stream order, stamped.
static int fetch_frames(amb_ctx* ctx, unsigned upto)
{
    if (upto <= ctx->polled) return AMB_OK;
    const size_t base = ctx->pending.size();
    const unsigned cnt = upto - ctx->polled;
    ctx->pending.resize(base + cnt);
    CK(ctx, cudaMemcpy(ctx->pending.data() + base, ctx->bufs.frames + ctx->polled, (size_t)cnt * sizeof(amb_frame), cudaMemcpyDeviceToHost));
    std::sort(ctx->pending.begin() + base, ctx->pending.end(),
              [](const amb_frame& x, const amb_frame& y) { return x.sample_index < y.sample_index; });
    for (size_t k = base; k < ctx->pending.size(); k++) stamp(ctx, &ctx->pending[k]);
    ctx->polled = upto;
    return AMB_OK;
}

// Everything enqueued so far is through; counters of the last call read back.
static int collect_sync(amb_ctx* ctx, AmbCounters* h)
{
    CK(ctx, cudaSetDevice(ctx->device));
    if (ctx->pend_n) { int rc = ingest_dispatch_pending(ctx, 0); if (rc) return rc; }
    CK(ctx, sync_all(ctx));
    CK(ctx, cudaMemcpy(h, ctx->ctr, sizeof *h, cudaMemcpyDeviceToHost));
    ctx->stats.candidates = h->ncand;
    ctx->stats.candidates_real = h->nreal_call;
    ctx->stats.detections = h->ndet_call;
    ctx->stats.frames_passed = h->npassed_call;
    ctx->stats.ec_fixed = (int)h->nec_fixed;
    if (h->overflow) return fail(ctx, AMB_ERR_OVERFLOW, "candidate buffer overflow");
    if (h->frame_overflow) return fail(ctx, AMB_ERR_OVERFLOW, "frame buffer overflow");
    return AMB_OK;
}

static int collect(amb_ctx* ctx)
{
    AmbCounters h;
    { int rc = collect_sync(ctx, &h); if (rc) return rc; }
    { int rc = fetch_frames(ctx, h.nframes); if (rc) return rc; }
    if (h.nframes) CK(ctx, cudaMemset(&ctx->ctr->nframes, 0, sizeof(unsigned)));
    ctx->polled = 0;
    ctx->snap_tail = ctx->snap_head;
    ctx->bufs.frames_ub = 0;
    if (ctx->def_kind && ctx->def_resolved) { ctx->def_kind = 0; ctx->def_resolved = false; }   // frames read: span is final
    return AMB_OK;
}

int amb_pending_frames(amb_ctx* ctx)
{
    if (!ctx) return AMB_ERR_INVALID;
    int rc = collect(ctx);
    if (rc != AMB_OK) return rc;
    return (int)ctx->pending.size();
}

int amb_poll_frames(amb_ctx* ctx, amb_frame* out, int max)
{
    if (!ctx || (!out && max > 0)) return AMB_ERR_INVALID;
    int rc = collect(ctx);
    if (rc != AMB_OK) return rc;
    const int n = (int)std::min<size_t>(ctx->pending.size(), (size_t)std::max(max, 0));
    if (n) memcpy(out, ctx->pending.data(), (size_t)n * sizeof(amb_frame));
    ctx->pending.erase(ctx->pending.begin(), ctx->pending.begin() + n);
    return n;
}

/* Non-blocking: frames of the calls that have already completed on the device; work in flight stays in flight. */
int amb_poll_ready(amb_ctx* ctx, amb_frame* out, int max)
{
    if (!ctx || (!out && max > 0)) return AMB_ERR_INVALID;
    CK(ctx, cudaSetDevice(ctx->device));
    bool have = false; AmbCounters last{};
    while (ctx->snap_tail < ctx->snap_head) {
        const unsigned k = (unsigned)(ctx->snap_tail % AMB_SNAPS);
        const cudaError_t q = cudaEventQuery(ctx->snap_ev[k]);
        if (q == cudaErrorNotReady) { cudaGetLastError(); break; }
        if (q != cudaSuccess) return fail(ctx, AMB_ERR_CUDA, "cudaEventQuery", q);
        last = ctx->ctr_snap[k]; have = true; ctx->snap_tail++;
    }
    if (have) {
        if (last.overflow) return fail(ctx, AMB_ERR_OVERFLOW, "candidate buffer overflow");
        if (last.frame_overflow) return fail(ctx, AMB_ERR_OVERFLOW, "frame buffer overflow");
        int rc = fetch_frames(ctx, last.nframes); if (rc) return rc;
    }
    const int n = (int)std::min<size_t>(ctx->pending.size(), (size_t)std::max(max, 0));
    if (n) memcpy(out, ctx->pending.data(), (size_t)n * sizeof(amb_frame));
    ctx->pending.erase(ctx->pending.begin(), ctx->pending.begin() + n);
    return n;
}

/* The device-side amb_poll_frames: every frame not handed out yet, in stream order and stamped, written to DEVICE memory.
 * out_dev == NULL: only report how many there are. Frames that an earlier amb_poll_ready already moved to the host's
 * pending list are not included (they come out of amb_poll_frames / amb_poll_ready). */
int amb_drain_device(amb_ctx* ctx, amb_frame* out_dev, int cap)
{
    if (!ctx || cap < 0) return AMB_ERR_INVALID;
    AmbCounters h;
    { int rc = collect_sync(ctx, &h); if (rc) return rc; }
    const unsigned n = h.nframes > ctx->polled ? h.nframes - ctx->polled : 0u;
    if (!out_dev) return (int)n;
    if ((unsigned)cap < n) return fail(ctx, AMB_ERR_OVERFLOW, "amb_drain_device: output buffer too small");
    if (n) {
        unsigned npad = 1; while (npad < n) npad <<= 1;
        if (ctx->ord_cap < npad) {
            cudaFree(ctx->ord_key); cudaFree(ctx->ord_val); ctx->ord_key = nullptr; ctx->ord_val = nullptr; ctx->ord_cap = 0;
            CK(ctx, cudaMalloc(&ctx->ord_key, (size_t)npad * sizeof(unsigned long long)));
            CK(ctx, cudaMalloc(&ctx->ord_val, (size_t)npad * sizeof(unsigned)));
            ctx->ord_cap = npad;
        }
        const int ntags = (int)ctx->time_tags.size();
        if (ntags) {
            if (ctx->tags_dev_cap < ntags) {
                cudaFree(ctx->tags_dev); ctx->tags_dev = nullptr; ctx->tags_dev_cap = 0;
                CK(ctx, cudaMalloc(&ctx->tags_dev, (size_t)ntags * 2 * sizeof(AmbTagDev)));
                ctx->tags_dev_cap = ntags * 2;
            }
            std::vector<AmbTagDev> t((size_t)ntags);
            for (int k = 0; k < ntags; k++) t[(size_t)k] = {ctx->time_tags[(size_t)k].offset, ctx->time_tags[(size_t)k].secs, ctx->time_tags[(size_t)k].frac};
            CK(ctx, cudaMemcpy(ctx->tags_dev, t.data(), (size_t)ntags * sizeof(AmbTagDev), cudaMemcpyHostToDevice));
        }
        cudaError_t e = cudaSuccess;
        const int launched = amb_launch_order(ctx->bufs.frames + ctx->polled, n, npad, ctx->order_tile, ctx->ord_key, ctx->ord_val, out_dev,
                                              (unsigned long long)ctx->P.rate_int, ctx->t0_secs, ctx->t0_frac, ctx->tags_dev, ntags,
                                              ctx->stream_b, &e);
        if (e != cudaSuccess) return fail(ctx, AMB_ERR_CUDA, "amb_drain_device launch", e);
        ctx->stats.kernel_launches += (uint64_t)launched;
        CK(ctx, cudaStreamSynchronize(ctx->stream_b));
    }
    if (h.nframes) CK(ctx, cudaMemset(&ctx->ctr->nframes, 0, sizeof(unsigned)));
    ctx->polled = 0;
    ctx->snap_tail = ctx->snap_head;
    ctx->bufs.frames_ub = 0;
    if (ctx->def_kind && ctx->def_resolved) { ctx->def_kind = 0; ctx->def_resolved = false; }
    return (int)n;
}

int amb_add_time_tag(amb_ctx* ctx, uint64_t offset, uint64_t secs, double frac)
{
    if (!ctx) return AMB_ERR_INVALID;
    if (!ctx->time_tags.empty() && ctx->time_tags.back().offset >= offset)
        return fail(ctx, AMB_ERR_INVALID, "rx_time tags must be added in ascending offset order");
    ctx->time_tags.push_back({offset, secs, frac});
    return AMB_OK;
}

/* Order the context's work after whatever has been enqueued so far on another CUDA stream (e.g. the stream that
 * produces a device-resident input buffer). No host synchronisation. */
int amb_wait_stream(amb_ctx* ctx, void* cuda_stream)
{
    if (!ctx) return AMB_ERR_INVALID;
    CK(ctx, cudaSetDevice(ctx->device));
    if ((cudaStream_t)cuda_stream == ctx->stream) return AMB_OK;
    CK(ctx, cudaEventRecord(ctx->e_in, (cudaStream_t)cuda_stream));
    CK(ctx, cudaStreamWaitEvent(ctx->stream, ctx->e_in, 0));
    return AMB_OK;
}

int amb_get_stats(amb_ctx* ctx, amb_stats* out)
{
    if (!ctx || !out) return AMB_ERR_INVALID;
    CK(ctx, cudaSetDevice(ctx->device));
    if (ctx->pend_n) { int rc = ingest_dispatch_pending(ctx, 0); if (rc) return rc; }
    CK(ctx, sync_all(ctx));
    AmbCounters h; AmbWalkState st;
    CK(ctx, cudaMemcpy(&h, ctx->ctr, sizeof h, cudaMemcpyDeviceToHost));
    CK(ctx, cudaMemcpy(&st, ctx->st, sizeof st, cudaMemcpyDeviceToHost));
    ctx->stats.samples_in = ctx->n_in;
    ctx->stats.candidates = h.ncand;
    ctx->stats.candidates_real = h.nreal_call;
    ctx->stats.detections = h.ndet_call;
    ctx->stats.frames_passed = h.npassed_call;
    ctx->stats.ec_fixed = (int)h.nec_fixed;
    ctx->stats.resolver_fallback = st.fallback;
    if (ctx->timing) {
        float ms = 0.f;
        if (ctx->ev_valid && cudaEventElapsedTime(&ms, ctx->ev[0], ctx->ev[1]) == cudaSuccess) ctx->stats.ms_scan = ms;
        if (cudaEventElapsedTime(&ms, ctx->ev[2], ctx->ev[3]) == cudaSuccess) ctx->stats.ms_total = ms;
    }
    *out = ctx->stats;
    return AMB_OK;
}

int amb_get_scan_times(amb_ctx* ctx, float* ms_out, int max)
{
    if (!ctx || (!ms_out && max > 0)) return AMB_ERR_INVALID;
    CK(ctx, cudaSetDevice(ctx->device));
    if (ctx->pend_n) { int rc = ingest_dispatch_pending(ctx, 0); if (rc) return rc; }
    CK(ctx, sync_all(ctx));
    const unsigned have = ctx->ring_n < 64u ? ctx->ring_n : 64u;
    const unsigned n = have < (unsigned)(max > 0 ? max : 0) ? have : (unsigned)(max > 0 ? max : 0);
    for (unsigned k = 0; k < n; k++) {
        const unsigned call = ctx->ring_n - n + k;
        float ms = 0.f;
        CK(ctx, cudaEventElapsedTime(&ms, ctx->ring[(call & 63u) * 2], ctx->ring[(call & 63u) * 2 + 1]));
        ms_out[k] = ms;
    }
    return (int)n;
}

/* Per call, oldest first: [0] idle time of the scan stream in front of this call's scan (previous scan end -> this
 * scan start), [1] the scan kernel, [2] scan end -> end of the call's sparse stages. Timing must be on. */
int amb_get_timeline(amb_ctx* ctx, float* ms_out, int max_calls)
{
    if (!ctx || (!ms_out && max_calls > 0)) return AMB_ERR_INVALID;
    CK(ctx, cudaSetDevice(ctx->device));
    if (ctx->pend_n) { int rc = ingest_dispatch_pending(ctx, 0); if (rc) return rc; }
    CK(ctx, sync_all(ctx));
    const unsigned have = ctx->ring_n < 63u ? ctx->ring_n : 63u;
    const unsigned n = have < (unsigned)(max_calls > 0 ? max_calls : 0) ? have : (unsigned)(max_calls > 0 ? max_calls : 0);
    for (unsigned k = 0; k < n; k++) {
        const unsigned call = ctx->ring_n - n + k;
        float gap = 0.f, sc = 0.f, tail = 0.f;
        if (call > 0 && ctx->ring_n - (call - 1) <= 64u)
            if (cudaEventElapsedTime(&gap, ctx->ring[((call - 1) & 63u) * 2 + 1], ctx->ring[(call & 63u) * 2]) != cudaSuccess) { gap = 0.f; cudaGetLastError(); }
        CK(ctx, cudaEventElapsedTime(&sc, ctx->ring[(call & 63u) * 2], ctx->ring[(call & 63u) * 2 + 1]));
        if (cudaEventElapsedTime(&tail, ctx->ring[(call & 63u) * 2 + 1], ctx->ring_done[call & 63u]) != cudaSuccess) { tail = 0.f; cudaGetLastError(); }
        ms_out[3 * k] = gap; ms_out[3 * k + 1] = sc; ms_out[3 * k + 2] = tail;
    }
    return (int)n;
}

int amb_debug_candidates(amb_ctx* ctx, uint64_t* index, uint32_t* info, int max)
{
    if (!ctx) return AMB_ERR_INVALID;
    CK(ctx, cudaSetDevice(ctx->device));
    CK(ctx, sync_all(ctx));
    if (!ctx->have_last || !ctx->bufs.cand_j) return 0;
    AmbCounters h;
    CK(ctx, cudaMemcpy(&h, ctx->ctr, sizeof h, cudaMemcpyDeviceToHost));
    const int n = (int)std::min<unsigned>(h.ncand, (unsigned)std::max(max, 0));
    if (n <= 0) return 0;
    std::vector<int> j(n);
    CK(ctx, cudaMemcpy(j.data(), ctx->bufs.cand_j, (size_t)n * sizeof(int), cudaMemcpyDeviceToHost));
    if (info) CK(ctx, cudaMemcpy(info, ctx->bufs.cand_info, (size_t)n * sizeof(uint32_t), cudaMemcpyDeviceToHost));
    if (index) for (int k = 0; k < n; k++) index[k] = (uint64_t)(ctx->last_org + j[k]);
    return n;
}

// slicer_impl.cc:186-192
int amb_format_message(const amb_frame* f, int first, char* buf, size_t buflen)
{
    if (!f || !buf) return AMB_ERR_INVALID;
    char tmp[192];
    int o = 0;
    static const char hexd[] = "0123456789abcdef";
    for (int m = 0; m < f->nbits / 8 && m < 14; m++) { tmp[o++] = hexd[f->data[m] >> 4]; tmp[o++] = hexd[f->data[m] & 15]; }
    o += snprintf(tmp + o, sizeof tmp - o, " %06lx %.*g %llu %.10g", (unsigned long)f->crc, first ? 6 : 10,
                  (double)f->ref_level, (unsigned long long)f->secs, f->frac);
    if ((size_t)o + 1 > buflen) return AMB_ERR_INVALID;
    memcpy(buf, tmp, (size_t)o + 1);
    return o;
}

// The same for a whole batch: one line per frame with passed != 0, in order, separated by '\n'. The stream's first
// message has precision 6, every later one 10 (the sticky setprecision of slicer_impl.cc:192).
int amb_format_messages(const amb_frame* frames, int n, int first, char* buf, size_t buflen)
{
    if (n < 0 || (n > 0 && !frames) || !buf || buflen == 0) return AMB_ERR_INVALID;
    size_t o = 0;
    int count = 0;
    buf[0] = 0;
    for (int k = 0; k < n; k++) {
        if (!frames[k].passed) continue;
        char tmp[192];
        const int len = amb_format_message(&frames[k], first && count == 0, tmp, sizeof tmp);
        if (len < 0) return len;
        if (o + (size_t)len + 2 > buflen) return AMB_ERR_INVALID;
        if (count) buf[o++] = '\n';
        memcpy(buf + o, tmp, (size_t)len + 1);
        o += (size_t)len;
        count++;
    }
    return count;
}

// modes_crc.cc:33-63
uint32_t amb_modes_check_crc(const uint8_t* data, int length)
{
    static uint32_t table[256];
    static bool ready = false;
    if (!ready) {
        for (int n = 0; n < 256; n++) {
            uint32_t crc = (uint32_t)n << 16;
            for (int k = 0; k < 8; k++) crc = (crc & 0x800000u) ? (((crc << 1) ^ 0xFFF409u) & 0xFFFFFFu) : ((crc << 1) & 0xFFFFFFu);
            table[n] = crc;
        }
        ready = true;
    }
    uint32_t crc = 0;
    for (int i = 0; i < length; i++) crc = table[((crc >> 16) ^ data[i]) & 0xff] ^ (crc << 8);
    return crc & 0xFFFFFFu;
}

int amb_device_crc(amb_ctx* ctx, const uint8_t* data, int n, int length, uint32_t* out)
{
    if (!ctx || !data || !out || n < 0 || length < 1 || length > 11) return AMB_ERR_INVALID;
    if (n == 0) return AMB_OK;
    CK(ctx, cudaSetDevice(ctx->device));
    uint8_t* d = nullptr; uint32_t* o = nullptr;
    CK(ctx, cudaMalloc(&d, (size_t)n * length));
    CK(ctx, cudaMalloc(&o, (size_t)n * sizeof(uint32_t)));
    cudaError_t e = cudaMemcpyAsync(d, data, (size_t)n * length, cudaMemcpyHostToDevice, ctx->stream);
    if (e == cudaSuccess) e = amb_launch_crc(d, n, length, o, ctx->stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(out, o, (size_t)n * sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    cudaFree(d); cudaFree(o);
    ctx->stats.kernel_launches += 1;
    if (e != cudaSuccess) return fail(ctx, AMB_ERR_CUDA, "amb_device_crc", e);
    return AMB_OK;
}

int amb_dump_stage(amb_ctx* ctx, int stage, const float* iq, size_t n_complex, float* out)
{
    if (!ctx || stage < AMB_STAGE_M2 || stage > AMB_STAGE_DC || (n_complex && (!iq || !out))) return AMB_ERR_INVALID;
    if (n_complex > (1u << 26)) return fail(ctx, AMB_ERR_INVALID, "amb_dump_stage is a parity tool: at most 2^26 samples");
    if (ctx->use_dcblock && stage != AMB_STAGE_DC)
        return fail(ctx, AMB_ERR_UNSUPPORTED, "m2/bb/avg dumps take the demodulator's input; dump AMB_STAGE_DC and feed it to a context without the DC blocker");
    if (n_complex == 0) return AMB_OK;
    CK(ctx, cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->stream;
    if (stage == AMB_STAGE_DC) {     // the whole buffer as one stream: zero history (GNU Radio's delay lines start at zero)
        const int D = 100 * ctx->P.spc_i, nc = 2 * D - 2;                       // rx_path.py:40
        float2 *d = nullptr, *t = nullptr, *o = nullptr, *c0 = nullptr, *c1 = nullptr;
        cudaError_t e = cudaMalloc(&d, n_complex * sizeof(float2));
        if (e == cudaSuccess) e = cudaMalloc(&o, n_complex * sizeof(float2));
        if (e == cudaSuccess) e = cudaMalloc(&c0, (size_t)nc * sizeof(float2));
        if (e == cudaSuccess) e = cudaMalloc(&c1, (size_t)nc * sizeof(float2));
        if (e == cudaSuccess) e = cudaMemsetAsync(c0, 0, (size_t)nc * sizeof(float2), s);
        if (e == cudaSuccess) e = cudaMemcpyAsync(d, iq, n_complex * sizeof(float2), cudaMemcpyHostToDevice, s);
        if (e == cudaSuccess) e = amb_launch_dcblock(c0, nc, d, (long long)n_complex, D, t, o, c1, s);
        if (e == cudaSuccess) e = cudaMemcpyAsync(out, o, n_complex * sizeof(float2), cudaMemcpyDeviceToHost, s);
        if (e == cudaSuccess) e = cudaStreamSynchronize(s);
        cudaFree(d); cudaFree(t); cudaFree(o); cudaFree(c0); cudaFree(c1);
        ctx->stats.kernel_launches += 2;
        if (e != cudaSuccess) return fail(ctx, AMB_ERR_CUDA, "amb_dump_stage", e);
        return AMB_OK;
    }
    float2* d = nullptr; float* t = nullptr; float* o = nullptr;
    CK(ctx, cudaMalloc(&d, n_complex * sizeof(float2)));
    cudaError_t e = cudaMalloc(&t, n_complex * sizeof(float));
    if (e == cudaSuccess) e = cudaMalloc(&o, n_complex * sizeof(float));
    if (e == cudaSuccess) e = cudaMemcpyAsync(d, iq, n_complex * sizeof(float2), cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) e = amb_launch_dump(d, (long long)n_complex, ctx->P, stage, t, o, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(out, o, n_complex * sizeof(float), cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    cudaFree(d); cudaFree(t); cudaFree(o);
    ctx->stats.kernel_launches += stage == AMB_STAGE_AVG ? 2 : 1;
    if (e != cudaSuccess) return fail(ctx, AMB_ERR_CUDA, "amb_dump_stage", e);
    return AMB_OK;
}

int amb_slicer_process(amb_ctx* ctx, const float* chips, int ndet, const uint64_t* secs, const double* frac, amb_frame* out)
{
    if (!ctx || ndet < 0 || (ndet && (!chips || !out))) return AMB_ERR_INVALID;
    if (ndet == 0) return 0;
    CK(ctx, cudaSetDevice(ctx->device));
    float* d = nullptr; amb_frame* f = nullptr;
    CK(ctx, cudaMalloc(&d, (size_t)ndet * 240 * sizeof(float)));
    CK(ctx, cudaMalloc(&f, (size_t)ndet * sizeof(amb_frame)));
    cudaError_t e = cudaMemsetAsync(f, 0, (size_t)ndet * sizeof(amb_frame), ctx->stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d, chips, (size_t)ndet * 240 * sizeof(float), cudaMemcpyHostToDevice, ctx->stream);
    if (e == cudaSuccess) e = amb_launch_slice_chips(d, ndet, f, ctx->stream);
    if (e == cudaSuccess) {
        AmbChainErr er;
        const int k = amb_chain_ec(f, (unsigned)ndet, nullptr, ndet, chain_opts(ctx), ctx->stream, &er);
        if (k < 0) e = er.e; else ctx->stats.kernel_launches += (uint64_t)k;
    }
    if (e == cudaSuccess) e = cudaMemcpyAsync(out, f, (size_t)ndet * sizeof(amb_frame), cudaMemcpyDeviceToHost, ctx->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    cudaFree(d); cudaFree(f);
    ctx->stats.kernel_launches += 1;
    if (e != cudaSuccess) return fail(ctx, AMB_ERR_CUDA, "amb_slicer_process", e);
    for (int k = 0; k < ndet; k++) {
        out[k].secs = secs ? secs[k] : 0;
        out[k].frac = frac ? frac[k] : 0.0;
        out[k].sample_index = secs ? (uint64_t)(secs[k] * (uint64_t)ctx->P.rate_int + (uint64_t)llround((frac ? frac[k] : 0.0) * ctx->P.rate_int)) : 0;
    }
    return ndet;
}

int amb_preamble_process(amb_ctx* ctx, const float* in0, const float* in1, size_t n, int flush,
                         float* chips_out, uint64_t* index_out, int max_det)
{
    if (!ctx || (n && (!in0 || !in1)) || max_det < 0 || (max_det && (!chips_out || !index_out))) return AMB_ERR_INVALID;
    if (n > 0x40000000ull) return fail(ctx, AMB_ERR_INVALID, "at most 2^30 items per call");
    CK(ctx, cudaSetDevice(ctx->device));
    CK(ctx, sync_all(ctx));
    const AmbParams& P = ctx->P;
    cudaStream_t s = ctx->stream;
    // combined = undecided tail of the previous calls ++ new items; item index of combined[0] is b0
    const long long b0 = (long long)ctx->sf_total - (long long)ctx->sf0.size();
    const size_t m = ctx->sf0.size() + n;
    const bool first = (ctx->sf_total == 0);
    const long long total = (long long)ctx->sf_total + (long long)n;
    const long long ntot = total + P.H;                              // items incl. history (reported coordinates)
    const long long r_safe = std::max<long long>(ctx->sf_rdone, total + P.H - ctx->guard);
    float* d0 = nullptr; float* d1 = nullptr;
    CK(ctx, cudaMalloc(&d0, (m + 1) * sizeof(float)));
    CK(ctx, cudaMalloc(&d1, (m + 1) * sizeof(float)));
    int rc = AMB_OK;
    do {
        cudaError_t e = cudaSuccess;
        const size_t nt = ctx->sf0.size();
        if (nt) {
            e = cudaMemcpyAsync(d0, ctx->sf0.data(), nt * sizeof(float), cudaMemcpyHostToDevice, s);
            if (e == cudaSuccess) e = cudaMemcpyAsync(d1, ctx->sf1.data(), nt * sizeof(float), cudaMemcpyHostToDevice, s);
        }
        if (e == cudaSuccess && n) e = cudaMemcpyAsync(d0 + nt, in0, n * sizeof(float), cudaMemcpyHostToDevice, s);
        if (e == cudaSuccess && n) e = cudaMemcpyAsync(d1 + nt, in1, n * sizeof(float), cudaMemcpyHostToDevice, s);
        if (e != cudaSuccess) { rc = fail(ctx, AMB_ERR_CUDA, "H2D", e); break; }
        // local reported coordinate j = r - b0; evaluate starts in [r_done, flush ? ntot : r_safe)
        const long long j_lo = ctx->sf_rdone - b0, j_hi = (flush ? ntot : r_safe) - b0;
        AmbScanArgs a{};
        a.P = P;
        amb_chain_geometry(&a, j_lo, std::max(j_hi, j_lo), true, ctx->sm_count, 0);
        ctx->bufs.frames_ub = 0;
        AmbChainErr er;
        if (amb_chain_prepare(&ctx->bufs, &a, 0, amb_chain_cand_capacity((long long)m + P.H), amb_chain_frame_bound(P, (long long)m),
                              true, [ctx] { return sync_all(ctx); }, &er) < 0) { rc = chain_fail(ctx, er); break; }
        AmbChainCall call{};
        call.P = P; call.in0 = d0; call.in1 = d1; call.n_streams = (long long)m;
        call.org = b0; call.ntot = ntot; call.r_safe = r_safe; call.flush = flush ? 1 : 0;
        call.ctr = ctx->ctr; call.st = ctx->st; call.n_samples = (long long)m + P.H + 4096;
        AmbChainOpts opts = chain_opts(ctx);
        opts.keep_chips = true;
        AmbChainSpan sp;
        int k = amb_chain_split_scan(a, ctx->bufs, d0, d1, (long long)m, ctx->ctr, first ? ctx->st : nullptr, ctx->sm_count, s, &er);
        if (k >= 0) { const int k2 = amb_chain_launch(a, call, &ctx->bufs, opts, false, s, &sp, &er); k = k2 < 0 ? -1 : k + k2; }
        e = k < 0 ? er.e : cudaStreamSynchronize(s);
        if (k > 0) ctx->stats.kernel_launches += (uint64_t)k;
        if (e != cudaSuccess) { rc = fail(ctx, AMB_ERR_CUDA, "amb_preamble_process", e); break; }
        AmbCounters h;
        e = cudaMemcpy(&h, ctx->ctr, sizeof h, cudaMemcpyDeviceToHost);
        if (e != cudaSuccess) { rc = fail(ctx, AMB_ERR_CUDA, "counters", e); break; }
        if (h.overflow || h.frame_overflow) { rc = fail(ctx, AMB_ERR_OVERFLOW, "buffer overflow"); break; }
        const unsigned nd = h.nframes;
        std::vector<amb_frame> fr(nd);
        std::vector<float> ch((size_t)nd * 240);
        if (nd) {
            e = cudaMemcpy(fr.data(), ctx->bufs.frames, (size_t)nd * sizeof(amb_frame), cudaMemcpyDeviceToHost);
            if (e == cudaSuccess) e = cudaMemcpy(ch.data(), ctx->bufs.chips, (size_t)nd * 240 * sizeof(float), cudaMemcpyDeviceToHost);
            if (e != cudaSuccess) { rc = fail(ctx, AMB_ERR_CUDA, "D2H", e); break; }
        }
        std::vector<unsigned> order(nd);
        for (unsigned k = 0; k < nd; k++) order[k] = k;
        std::sort(order.begin(), order.end(), [&](unsigned x, unsigned y) { return fr[x].sample_index < fr[y].sample_index; });
        const int nout = (int)std::min<unsigned>(nd, (unsigned)max_det);
        for (int k = 0; k < nout; k++) {
            index_out[k] = fr[order[k]].sample_index;
            memcpy(chips_out + (size_t)k * 240, ch.data() + (size_t)order[k] * 240, 240 * sizeof(float));
        }
        cudaMemset(&ctx->ctr->nframes, 0, sizeof(unsigned));
        ctx->bufs.frames_ub = 0;
        // keep what a later call still has to look at: items from (r_safe - H) on
        if (flush) { ctx->sf0.clear(); ctx->sf1.clear(); ctx->sf_total = 0; ctx->sf_rdone = 0; }
        else {
            const long long keep_from = std::max<long long>(r_safe - P.H, b0);       // item index
            std::vector<float> t0, t1;
            for (long long it = keep_from; it < total; it++) {
                const long long k = it - b0;
                t0.push_back((size_t)k < nt ? ctx->sf0[(size_t)k] : in0[(size_t)k - nt]);
                t1.push_back((size_t)k < nt ? ctx->sf1[(size_t)k] : in1[(size_t)k - nt]);
            }
            ctx->sf0.swap(t0); ctx->sf1.swap(t1);
            ctx->sf_total = (uint64_t)total; ctx->sf_rdone = r_safe;
        }
        rc = nd > (unsigned)max_det ? fail(ctx, AMB_ERR_OVERFLOW, "max_det too small") : nout;
    } while (0);
    cudaFree(d0); cudaFree(d1);
    return rc;
}

}  // extern "C"
