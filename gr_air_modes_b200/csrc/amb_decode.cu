// Batch field decode (SURVEY.md 8 row f4): kernels + C ABI of amb_decoder (include/airmodes_b200.h).
// The per-message arithmetic is in amb_decode_core.h, the kernels and amb_decode_launch - the one launch sequence of a
// decode - in amb_decode_kernels.cuh and the stage headers it includes (launch-free headers, so that tests/simt can run
// the same kernel source and sequence under a host emulator); this file allocates the tables and buffers the stages
// need, copies the frames in and the records out. Compiled with -fmad=false: latitude/longitude follow cpr.py
// operation by operation in IEEE double, nothing may be contracted. Citations are file:line under gr-air-modes/python.
//
// Seven launches per decode, in stream order:
//   amb_fields_kernel   one thread per frame: bit fields, altitude, squawk, ident, velocity; emits the CPR report
//   amb_v3_*            five kernels, cpr_decoder's bookkeeping (cpr.py:206-229): for every position message, the latest
//                       even and odd report of its aircraft as of that message, from the reports partitioned by owner
//                       bucket and a direct-mapped table in HBM (2^26 x 16 B) that carries them from batch to batch
//   amb_resolve_kernel  one thread per frame: global CPR decode, range/bearing.
// With option "local_cpr" on, six more (amb_decode_local.cuh): amb_local_keys, the four partition kernels of the pairing
// stage on ICAO keys, amb_local_walk - the local decode of the position messages the global decode left without a fix,
// with a direct-mapped table of reference positions in HBM (2^24 x 24 B) carried from batch to batch.
// With option "commb" on, six more after those (amb_decode_commb.cuh): amb_commb_keys, the four partition kernels on
// address keys, amb_commb_walk - Comm-B register inference of the DF20/21 replies the parser does not handle, with a
// direct-mapped table of ADS-B velocities in HBM (2^24 x 24 B) carried from batch to batch.
// With option "track" on, six more after those (amb_decode_track.cuh): amb_track_keys, the four partition kernels on
// address keys, amb_track_walk - the per-aircraft table, direct-mapped in HBM (2^24 x 128 B) with an occupancy bitmap;
// amb_decoder_aircraft reads it out with three kernels of its own.
#include "amb_launch.h"
#include "amb_decode_core.h"
#include "amb_decode_kernels.cuh"

#include <stdio.h>
#include <string.h>

#include <new>
#include <string>

struct amb_decoder {
    int device = 0;
    cudaStream_t stream = nullptr;
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    AmbDecodeState st;                   // the stages' tables, scratch and options (amb_decode_kernels.cuh)
    amb_frame* d_frames = nullptr; amb_fields* d_fields = nullptr;
    int cap = 0;                         // frames d_frames, d_fields, st.pos and st.pair hold
    int kcap = 0;                        // frames st.keys holds
    // host <-> device staging: pageable caller arrays go through two pinned bounce buffers per direction so that the
    // copies run at PCIe speed and overlap the memcpy of the next piece
    void* pin[2] = {nullptr, nullptr}; cudaEvent_t pin_ev[2] = {nullptr, nullptr}; size_t pin_bytes = 0;
    uint32_t* snap_cnt = nullptr;        // snapshot: per-block counts, then their scan and the total
    amb_aircraft* d_snap = nullptr; int snap_cap = 0;   // snapshot rows on their way to host memory
    uint64_t launches = 0; float ms_last = 0.f;
    std::string err;
};

static thread_local std::string g_create_err;          // why the last amb_decoder_create on this thread failed

static int dfail(amb_decoder* d, int code, const char* what, cudaError_t e = cudaSuccess)
{
    if (d) {
        char buf[256];
        if (e != cudaSuccess) snprintf(buf, sizeof buf, "%s: %s", what, cudaGetErrorString(e));
        else snprintf(buf, sizeof buf, "%s", what);
        d->err = buf;
    }
    return code;
}
#define DCK(call)                                                                  \
    do { cudaError_t e_ = (call); if (e_ != cudaSuccess) return dfail(d, AMB_ERR_CUDA, #call, e_); } while (0)

// ---- host ---------------------------------------------------------------------------------------------------------
extern "C" void amb_parallel_memcpy(void* dst, const void* src, size_t n);      // amb_api.cu (the ingest copy threads)
#define AMB_DEC_PIECE ((size_t)8 << 20)

static int ensure_pinned(amb_decoder* d)
{
    if (d->pin[0]) return AMB_OK;
    for (int k = 0; k < 2; k++) {
        DCK(cudaMallocHost(&d->pin[k], AMB_DEC_PIECE));
        DCK(cudaEventCreateWithFlags(&d->pin_ev[k], cudaEventDisableTiming));
    }
    d->pin_bytes = AMB_DEC_PIECE;
    return AMB_OK;
}

// pageable host -> device through the pinned pieces (memcpy of piece k+1 overlaps the DMA of piece k)
static int staged_h2d(amb_decoder* d, void* dst, const void* src, size_t bytes, cudaStream_t s)
{
    int rc = ensure_pinned(d); if (rc) return rc;
    size_t off = 0; int k = 0;
    while (off < bytes) {
        const size_t m = bytes - off < AMB_DEC_PIECE ? bytes - off : AMB_DEC_PIECE;
        DCK(cudaEventSynchronize(d->pin_ev[k]));
        amb_parallel_memcpy(d->pin[k], static_cast<const char*>(src) + off, m);
        DCK(cudaMemcpyAsync(static_cast<char*>(dst) + off, d->pin[k], m, cudaMemcpyHostToDevice, s));
        DCK(cudaEventRecord(d->pin_ev[k], s));
        off += m; k ^= 1;
    }
    return AMB_OK;
}

// device -> pageable host: the DMA of piece i overlaps the memcpy of piece i-1 out of its pinned buffer
static int staged_d2h(amb_decoder* d, void* dst, const void* src, size_t bytes, cudaStream_t s)
{
    int rc = ensure_pinned(d); if (rc) return rc;
    const size_t np = (bytes + AMB_DEC_PIECE - 1) / AMB_DEC_PIECE;
    for (size_t i = 0; i <= np; i++) {
        if (i < np) {
            const size_t off = i * AMB_DEC_PIECE, m = bytes - off < AMB_DEC_PIECE ? bytes - off : AMB_DEC_PIECE;
            DCK(cudaMemcpyAsync(d->pin[i & 1], static_cast<const char*>(src) + off, m, cudaMemcpyDeviceToHost, s));
            DCK(cudaEventRecord(d->pin_ev[i & 1], s));
        }
        if (i >= 1) {
            const size_t off = (i - 1) * AMB_DEC_PIECE, m = bytes - off < AMB_DEC_PIECE ? bytes - off : AMB_DEC_PIECE;
            DCK(cudaEventSynchronize(d->pin_ev[(i - 1) & 1]));
            amb_parallel_memcpy(static_cast<char*>(dst) + off, d->pin[(i - 1) & 1], m);
        }
    }
    return AMB_OK;
}

static void free_bufs(amb_decoder* d)
{
    if (d->d_frames) cudaFree(d->d_frames);
    if (d->d_fields) cudaFree(d->d_fields);
    if (d->st.pos) cudaFree(d->st.pos);
    if (d->st.pair) cudaFree(d->st.pair);
    d->d_frames = nullptr; d->d_fields = nullptr; d->st.pos = nullptr; d->st.pair = nullptr; d->cap = 0;
}

static int ensure_cap(amb_decoder* d, int n)
{
    if (n <= d->cap) return AMB_OK;
    int cap = d->cap ? d->cap : 4096;
    while (cap < n) cap *= 2;
    free_bufs(d);
    DCK(cudaMalloc(&d->d_frames, (size_t)cap * sizeof(amb_frame)));
    DCK(cudaMalloc(&d->d_fields, (size_t)cap * sizeof(amb_fields)));
    DCK(cudaMalloc(&d->st.pos, (size_t)cap * sizeof(AmbPosRec)));
    DCK(cudaMalloc(&d->st.pair, (size_t)cap * sizeof(AmbPair)));
    d->cap = cap;
    return AMB_OK;
}

extern "C" {

int amb_decoder_create(int device, int have_location, double lat, double lon, amb_decoder** out)
{
    static_assert(sizeof(amb_fields) == 144, "amb_fields layout");
    static_assert(sizeof(AmbCprSlot) == 16, "table slot layout");
    static_assert(sizeof(AmbRefPos) == 24, "reference position slot layout");
    static_assert(sizeof(AmbCommbRef) == 24, "velocity reference slot layout");
    static_assert(sizeof(amb_aircraft) == 128, "amb_aircraft layout");
    if (!out) return AMB_ERR_INVALID;
    *out = nullptr;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0 || device < 0 || device >= ndev) return AMB_ERR_NO_DEVICE;
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) return AMB_ERR_NO_DEVICE;
    if (prop.major != 9 || prop.minor != 0) return AMB_ERR_NO_DEVICE;   // sm_90a cubin only; there is no CPU path
    amb_decoder* d = new (std::nothrow) amb_decoder();
    if (!d) return AMB_ERR_INVALID;
    d->device = device;
    d->st.have_loc = have_location ? 1 : 0; d->st.lat = lat; d->st.lon = lon;
    int rc = AMB_OK;
    do {
        if (cudaSetDevice(device) != cudaSuccess) { rc = AMB_ERR_NO_DEVICE; break; }
        if (cudaStreamCreateWithFlags(&d->stream, cudaStreamNonBlocking) != cudaSuccess ||
            cudaEventCreate(&d->e0) != cudaSuccess || cudaEventCreate(&d->e1) != cudaSuccess) { rc = AMB_ERR_CUDA; break; }
        cudaError_t e = cudaMalloc(&d->st.table, AMB_TABLE_SLOTS * sizeof(AmbCprSlot));
        if (e != cudaSuccess) { rc = dfail(d, AMB_ERR_CUDA, "report table (1 GiB)", e); break; }
        if (cudaMalloc(&d->st.nl_T, AMB_NL_MAX * sizeof(double)) != cudaSuccess) { rc = AMB_ERR_CUDA; break; }
        double T[AMB_NL_MAX];
        amb_build_nl_table(T);                          // cpr.py:46-51 through the host libm, once
        if (cudaMemcpyAsync(d->st.nl_T, T, sizeof T, cudaMemcpyHostToDevice, d->stream) != cudaSuccess ||
            cudaMemsetAsync(d->st.table, 0xFF, AMB_TABLE_SLOTS * sizeof(AmbCprSlot), d->stream) != cudaSuccess ||
            cudaStreamSynchronize(d->stream) != cudaSuccess) { rc = AMB_ERR_CUDA; break; }
    } while (0);
    if (rc != AMB_OK) { g_create_err = d->err.empty() ? "CUDA resource creation failed" : d->err; amb_decoder_destroy(d); return rc; }
    g_create_err.clear();
    *out = d;
    return AMB_OK;
}

void amb_decoder_destroy(amb_decoder* d)
{
    if (!d) return;
    cudaSetDevice(d->device);
    if (d->stream) cudaStreamSynchronize(d->stream);
    free_bufs(d);
    amb_v3_free(&d->st.v3);
    if (d->st.ltable) cudaFree(d->st.ltable);
    if (d->st.keys) cudaFree(d->st.keys);
    if (d->st.ctable) cudaFree(d->st.ctable);
    if (d->st.trows) cudaFree(d->st.trows);
    if (d->st.tocc) cudaFree(d->st.tocc);
    if (d->st.tclk) cudaFree(d->st.tclk);
    if (d->snap_cnt) cudaFree(d->snap_cnt);
    if (d->d_snap) cudaFree(d->d_snap);
    for (int k = 0; k < 2; k++) { if (d->pin[k]) cudaFreeHost(d->pin[k]); if (d->pin_ev[k]) cudaEventDestroy(d->pin_ev[k]); }
    if (d->st.table) cudaFree(d->st.table);
    if (d->st.nl_T) cudaFree(d->st.nl_T);
    if (d->e0) cudaEventDestroy(d->e0);
    if (d->e1) cudaEventDestroy(d->e1);
    if (d->stream) cudaStreamDestroy(d->stream);
    delete d;
}

int amb_decoder_set_location(amb_decoder* d, int have_location, double lat, double lon)
{
    if (!d) return AMB_ERR_INVALID;
    d->st.have_loc = have_location ? 1 : 0; d->st.lat = lat; d->st.lon = lon;
    return AMB_OK;
}

int amb_decoder_reset(amb_decoder* d)
{
    if (!d) return AMB_ERR_INVALID;
    DCK(cudaSetDevice(d->device));
    DCK(cudaMemsetAsync(d->st.table, 0xFF, AMB_TABLE_SLOTS * sizeof(AmbCprSlot), d->stream));
    if (d->st.ltable) DCK(cudaMemsetAsync(d->st.ltable, 0xFF, AMB_LOCAL_SLOTS * sizeof(AmbRefPos), d->stream));
    if (d->st.ctable) DCK(cudaMemsetAsync(d->st.ctable, 0xFF, AMB_COMMB_SLOTS * sizeof(AmbCommbRef), d->stream));
    if (d->st.tocc) {                    // the rows themselves stay: a row whose bit is clear is never read
        static const AmbTrackClock none = {NAN, 0u, 0u};
        DCK(cudaMemsetAsync(d->st.tocc, 0, AMB_TRACK_WORDS * sizeof(unsigned), d->stream));
        DCK(cudaMemcpyAsync(d->st.tclk, &none, sizeof none, cudaMemcpyHostToDevice, d->stream));
    }
    DCK(cudaStreamSynchronize(d->stream));
    return AMB_OK;
}

int amb_decoder_set_option(amb_decoder* d, const char* name, int value)
{
    static const struct { const char* name; int max; int AmbDecodeState::*seconds; } options[] = {
        {"local_cpr", AMB_LOCAL_CPR_MAX, &AmbDecodeState::local_cpr},
        {"commb", AMB_COMMB_MAX, &AmbDecodeState::commb},
        {"track", AMB_TRACK_MAX, &AmbDecodeState::track},
    };
    if (!d || !name) return AMB_ERR_INVALID;
    for (const auto& o : options) {
        if (strcmp(name, o.name) != 0) continue;
        if (value < 0 || value > o.max) {
            char what[64];
            snprintf(what, sizeof what, "%s: 0 (off) .. %d seconds", o.name, o.max);
            return dfail(d, AMB_ERR_INVALID, what);
        }
        d->st.*o.seconds = value;
        return AMB_OK;
    }
    return dfail(d, AMB_ERR_INVALID, "amb_decoder_set_option: unknown option");
}

// the key records of the local, the Comm-B and the track stage, one per frame
static int ensure_keys(amb_decoder* d)
{
    if (d->kcap < d->cap) {
        if (d->st.keys) cudaFree(d->st.keys);
        d->st.keys = nullptr; d->kcap = 0;
        DCK(cudaMalloc(&d->st.keys, (size_t)d->cap * sizeof(AmbPosRec)));
        d->kcap = d->cap;
    }
    return AMB_OK;
}

// the local stage's device memory, at the first decode with the option on (the table starts empty: all NaN)
static int ensure_local(amb_decoder* d)
{
    if (!d->st.ltable) {
        DCK(cudaMalloc(&d->st.ltable, AMB_LOCAL_SLOTS * sizeof(AmbRefPos)));
        DCK(cudaMemsetAsync(d->st.ltable, 0xFF, AMB_LOCAL_SLOTS * sizeof(AmbRefPos), d->stream));
    }
    return ensure_keys(d);
}

// the Comm-B stage's device memory, at the first decode with the option on (the table starts empty: all NaN)
static int ensure_commb(amb_decoder* d)
{
    if (!d->st.ctable) {
        cudaError_t e = cudaMalloc(&d->st.ctable, AMB_COMMB_SLOTS * sizeof(AmbCommbRef));
        if (e != cudaSuccess) { d->st.ctable = nullptr; return dfail(d, AMB_ERR_CUDA, "Comm-B velocity table (384 MiB)", e); }
        DCK(cudaMemsetAsync(d->st.ctable, 0xFF, AMB_COMMB_SLOTS * sizeof(AmbCommbRef), d->stream));
    }
    return ensure_keys(d);
}

// the track stage's device memory, at the first decode with the option on: the rows are not initialised (the bitmap
// starts empty), the clock starts at "nothing decoded"
static int ensure_track(amb_decoder* d)
{
    if (!d->st.trows) {
        cudaError_t e = cudaMalloc(&d->st.trows, (size_t)AMB_TRACK_ROWS * sizeof(amb_aircraft));
        if (e != cudaSuccess) { d->st.trows = nullptr; return dfail(d, AMB_ERR_CUDA, "aircraft table (2 GiB)", e); }
    }
    if (!d->st.tclk) {
        static const AmbTrackClock none = {NAN, 0u, 0u};
        DCK(cudaMalloc(&d->st.tclk, sizeof(AmbTrackClock)));
        DCK(cudaMemcpyAsync(d->st.tclk, &none, sizeof none, cudaMemcpyHostToDevice, d->stream));
    }
    if (!d->snap_cnt) DCK(cudaMalloc(&d->snap_cnt, (2 * AMB_TRACK_WORDS / AMB_SNAP_WORDS + 1) * sizeof(uint32_t)));
    if (!d->st.tocc) {                   // last: snapshot_impl and reset take a bitmap as "everything is there"
        DCK(cudaMalloc(&d->st.tocc, AMB_TRACK_WORDS * sizeof(unsigned)));
        DCK(cudaMemsetAsync(d->st.tocc, 0, AMB_TRACK_WORDS * sizeof(unsigned), d->stream));
    }
    return ensure_keys(d);
}

static int decode_impl(amb_decoder* d, const amb_frame* frames, int n, int mem_kind, amb_fields* out, bool out_on_device);

int amb_decode_frames(amb_decoder* d, const amb_frame* frames, int n, int mem_kind, amb_fields* out)
{
    return decode_impl(d, frames, n, mem_kind, out, false);
}

/* Frames AND records in device memory (e.g. the frames of a poll copied to the device once, or produced there): no
 * host copy at all; the records stay on the device for whatever consumes them next. Synchronises the decoder's stream. */
int amb_decode_frames_device(amb_decoder* d, const amb_frame* frames_dev, int n, amb_fields* out_dev)
{
    return decode_impl(d, frames_dev, n, AMB_MEM_DEVICE, out_dev, true);
}

static int decode_impl(amb_decoder* d, const amb_frame* frames, int n, int mem_kind, amb_fields* out, bool out_on_device)
{
    if (!d || n < 0 || (n > 0 && (!frames || !out)) || (mem_kind != AMB_MEM_HOST && mem_kind != AMB_MEM_DEVICE))
        return dfail(d, AMB_ERR_INVALID, "amb_decode_frames: bad argument");
    if (n == 0) return AMB_OK;
    DCK(cudaSetDevice(d->device));
    int rc = ensure_cap(d, n);
    if (rc == AMB_OK && d->st.local_cpr > 0) rc = ensure_local(d);
    if (rc == AMB_OK && d->st.commb > 0) rc = ensure_commb(d);
    if (rc == AMB_OK && d->st.track > 0) rc = ensure_track(d);
    if (rc != AMB_OK) return rc;
    cudaStream_t s = d->stream;
    amb_fields* const fields = out_on_device ? out : d->d_fields;
    DCK(cudaEventRecord(d->e0, s));
    const amb_frame* src = frames;
    if (mem_kind == AMB_MEM_HOST) {
        rc = staged_h2d(d, d->d_frames, frames, (size_t)n * sizeof(amb_frame), s);
        if (rc != AMB_OK) return rc;
        src = d->d_frames;
    }
    cudaError_t e = cudaSuccess;
    const int k = amb_decode_launch(&d->st, src, n, fields, s, &e);
    if (k < 0) {
        static const char* const stage[] = {"cudaGetLastError()", "pairing", "cudaGetLastError()", "local CPR",
                                            "Comm-B inference", "aircraft table"};   // by -AMB_STAGE_* - 1
        return dfail(d, AMB_ERR_CUDA, stage[-k - 1], e);
    }
    d->launches += (uint64_t)k;
    if (!out_on_device) {
        rc = staged_d2h(d, out, d->d_fields, (size_t)n * sizeof(amb_fields), s);
        if (rc != AMB_OK) return rc;
    }
    DCK(cudaEventRecord(d->e1, s));
    DCK(cudaStreamSynchronize(s));
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, d->e0, d->e1) == cudaSuccess) d->ms_last = ms;
    return AMB_OK;
}

static int snapshot_impl(amb_decoder* d, double now, amb_aircraft* out, int max, bool out_on_device)
{
    if (!d || max < 0) return dfail(d, AMB_ERR_INVALID, "amb_decoder_aircraft: bad argument");
    if (d->st.track <= 0) return dfail(d, AMB_ERR_STATE, "amb_decoder_aircraft: option track is off");
    if (!d->st.tocc) return 0;                           // nothing decoded with the option on yet
    DCK(cudaSetDevice(d->device));
    cudaStream_t s = d->stream;
    const unsigned nb = AMB_TRACK_WORDS / AMB_SNAP_WORDS;
    uint32_t* off = d->snap_cnt + nb;
    cudaError_t e = cudaSuccess;
    if (amb_snap_count_launch(d->st.tocc, d->st.trows, d->st.tclk, now, d->st.track, AMB_TRACK_WORDS, d->snap_cnt, off,
                              s, &e) < 0)
        return dfail(d, AMB_ERR_CUDA, "aircraft snapshot", e);
    d->launches += 2;
    uint32_t total = 0;
    DCK(cudaMemcpyAsync(&total, off + nb, sizeof total, cudaMemcpyDeviceToHost, s));
    DCK(cudaStreamSynchronize(s));
    if (!out) return (int)total;
    if (total > (uint32_t)max) return dfail(d, AMB_ERR_OVERFLOW, "amb_decoder_aircraft: output buffer too small");
    if (total == 0) return 0;
    amb_aircraft* dst = out;
    if (!out_on_device) {
        if (d->snap_cap < (int)total) {
            if (d->d_snap) cudaFree(d->d_snap);
            d->d_snap = nullptr; d->snap_cap = 0;
            DCK(cudaMalloc(&d->d_snap, (size_t)total * sizeof(amb_aircraft)));
            d->snap_cap = (int)total;
        }
        dst = d->d_snap;
    }
    if (amb_snap_gather_launch(d->st.tocc, d->st.trows, d->st.tclk, now, d->st.track, AMB_TRACK_WORDS, off, dst, s, &e) < 0)
        return dfail(d, AMB_ERR_CUDA, "aircraft snapshot", e);
    d->launches += 1;
    if (!out_on_device) {
        const int rc = staged_d2h(d, out, d->d_snap, (size_t)total * sizeof(amb_aircraft), s);
        if (rc != AMB_OK) return rc;
    }
    DCK(cudaStreamSynchronize(s));
    return (int)total;
}

int amb_decoder_aircraft(amb_decoder* d, double now, amb_aircraft* out, int max)
{
    return snapshot_impl(d, now, out, max, false);
}

int amb_decoder_aircraft_device(amb_decoder* d, double now, amb_aircraft* out_dev, int cap)
{
    return snapshot_impl(d, now, out_dev, cap, true);
}

int amb_decoder_stats(amb_decoder* d, uint64_t* kernel_launches, float* ms_last)
{
    if (!d) return AMB_ERR_INVALID;
    if (kernel_launches) *kernel_launches = d->launches;
    if (ms_last) *ms_last = d->ms_last;
    return AMB_OK;
}

const char* amb_decoder_last_error(const amb_decoder* d) { return d ? d->err.c_str() : g_create_err.c_str(); }

uint64_t amb_frame_bits(const amb_frame* f, int start, int num)
{
    if (!f || start < 1 || num < 1 || num > 64) return 0;
    return amb_bits(amb_msg_from_frame(*f), start, num);
}

}  // extern "C"
