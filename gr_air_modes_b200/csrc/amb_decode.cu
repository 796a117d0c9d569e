// Batch field decode (SURVEY.md 8 row f4): kernels + C ABI of amb_decoder (include/airmodes_b200.h).
// The per-message arithmetic is in amb_decode_core.h, the kernels, amb_decode_launch - the one launch sequence of a
// decode - and the stages' memory (amb_decode_prepare / amb_decode_reset / amb_decode_free) in amb_decode_kernels.cuh
// and the stage headers it includes (launch-free headers, so that tests/simt can run the same kernel source, sequence
// and memory rules under a host emulator); this file keeps the frames, records and snapshot rows on their way between
// the caller and the stages, copies the frames in and the records out. Compiled with -fmad=false: latitude/longitude follow cpr.py
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
// With option "opstatus" on, six more between the Comm-B and the track stage (amb_decode_opstatus.cuh):
// amb_opstatus_keys, the four partition kernels on address keys, amb_opstatus_walk - DF17 TC 29 / 31 decoded, and NIC / Rc
// or NUCp for every position, with a direct-mapped table of op status in HBM (2^24 x 24 B) carried from batch to batch.
// With options "track" and "track_ext" both on, six more after the track stage (amb_decode_track_ext.cuh):
// amb_track_ext_keys, the four partition kernels on address keys, amb_track_ext_walk - the op-status and Comm-B groups
// of every address, direct-mapped in HBM (2^24 x 144 B) with an occupancy bitmap; amb_decoder_aircraft_ext reads them
// out beside the aircraft rows with amb_snap_count, amb_snap_scan and amb_snap_gather_ext.
// With option "sbs1" on, ten more after every other stage (amb_decode_sbs1.cuh): amb_sbs1_keys, the four partition
// kernels on address keys, amb_sbs1_walk, amb_sbs1_ids - the aircraft ids of sbs1.py, with a direct-mapped table of the
// latest id per address in HBM (2^24 x 8 B) carried from batch to batch - and amb_sbs1_format, amb_sbs1_scan,
// amb_sbs1_gather, which write the call's SBS-1 lines and pack them on the device; amb_decoder_sbs1 copies them out.
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
    AmbDecodeState st;                   // the stages' memory and options (amb_decode_kernels.cuh)
    amb_frame* d_frames = nullptr; amb_fields* d_fields = nullptr;
    int cap = 0;                         // frames d_frames and d_fields hold
    // host <-> device staging: pageable caller arrays go through two pinned bounce buffers per direction so that the
    // copies run at PCIe speed and overlap the memcpy of the next piece
    void* pin[2] = {nullptr, nullptr}; cudaEvent_t pin_ev[2] = {nullptr, nullptr}; size_t pin_bytes = 0;
    amb_aircraft* d_snap = nullptr; int snap_cap = 0;   // snapshot rows on their way to host memory
    amb_aircraft_ext* d_xsnap = nullptr; int xsnap_cap = 0;   // ... and their extensions
    int sbs1_nb = -1;                    // blocks of lines of the last decode (its byte total is st.sb.boff[sbs1_nb]);
                                         // -1: the last decode wrote no lines
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

static int alloc_pinned(amb_decoder* d)
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
    int rc = alloc_pinned(d); if (rc) return rc;
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
    int rc = alloc_pinned(d); if (rc) return rc;
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
    d->d_frames = nullptr; d->d_fields = nullptr; d->cap = 0;
}

// the stages' memory for n frames (amb_decode_prepare), and the frames and records as many as the stages hold
static int prepare(amb_decoder* d, int n)
{
    cudaError_t e = cudaSuccess;
    const int k = amb_decode_prepare(&d->st, n, d->stream, &e);
    if (k < 0) return dfail(d, AMB_ERR_CUDA, amb_stage_names[-k - 1].memory, e);
    if (d->cap < d->st.cap) {
        free_bufs(d);
        DCK(cudaMalloc(&d->d_frames, (size_t)d->st.cap * sizeof(amb_frame)));
        DCK(cudaMalloc(&d->d_fields, (size_t)d->st.cap * sizeof(amb_fields)));
        d->cap = d->st.cap;
    }
    return AMB_OK;
}

extern "C" {

int amb_decoder_create(int device, int have_location, double lat, double lon, amb_decoder** out)
{
    static_assert(sizeof(amb_fields) == 144, "amb_fields layout");
    static_assert(sizeof(AmbCprSlot) == 16, "table slot layout");
    static_assert(sizeof(AmbRefPos) == 24, "reference position slot layout");
    static_assert(sizeof(AmbCommbRef) == 24, "velocity reference slot layout");
    static_assert(sizeof(AmbOpsSlot) == 24, "op status slot layout");
    static_assert(sizeof(amb_aircraft) == 128, "amb_aircraft layout");
    static_assert(sizeof(amb_aircraft_ext) == 144 && sizeof(amb_aircraft_ext) % 16 == 0, "amb_aircraft_ext layout");
    static_assert(offsetof(amb_aircraft_ext, t) == 8 && offsetof(amb_aircraft_ext, ops) == 56 &&
                  offsetof(amb_aircraft_ext, integ_nic) == 96 && offsetof(amb_aircraft_ext, commb) == 104,
                  "amb_aircraft_ext layout");
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
        if ((rc = prepare(d, 0)) != AMB_OK) break;      // the report and NL tables now, so that a lack of memory shows here
        if (cudaStreamSynchronize(d->stream) != cudaSuccess) { rc = AMB_ERR_CUDA; break; }
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
    amb_decode_free(&d->st);
    if (d->d_xsnap) cudaFree(d->d_xsnap);
    if (d->d_snap) cudaFree(d->d_snap);
    for (int k = 0; k < 2; k++) { if (d->pin[k]) cudaFreeHost(d->pin[k]); if (d->pin_ev[k]) cudaEventDestroy(d->pin_ev[k]); }
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
    cudaError_t e = cudaSuccess;
    const int k = amb_decode_reset(&d->st, d->stream, &e);
    if (k < 0) return dfail(d, AMB_ERR_CUDA, amb_stage_names[-k - 1].memory, e);
    DCK(cudaStreamSynchronize(d->stream));
    return AMB_OK;
}

int amb_decoder_set_option(amb_decoder* d, const char* name, int value)
{
    static const struct { const char* name; int max; int AmbDecodeState::*seconds; } options[] = {
        {"local_cpr", AMB_LOCAL_CPR_MAX, &AmbDecodeState::local_cpr},
        {"commb", AMB_COMMB_MAX, &AmbDecodeState::commb},
        {"track", AMB_TRACK_MAX, &AmbDecodeState::track},
        {"opstatus", AMB_OPSTATUS_MAX, &AmbDecodeState::opstatus},
        {"track_ext", AMB_TRACK_EXT_MAX, &AmbDecodeState::track_ext},
    };
    if (!d || !name) return AMB_ERR_INVALID;
    if (strcmp(name, "sbs1") == 0) {
        if (value != 0 && value != 1) return dfail(d, AMB_ERR_INVALID, "sbs1: 0 (off) or 1 (on)");
        d->st.sbs1 = value;
        return AMB_OK;
    }
    if (strcmp(name, "sbs1_tz") == 0) {
        if (value < AMB_SBS1_TZ_MIN || value > AMB_SBS1_TZ_MAX)
            return dfail(d, AMB_ERR_INVALID, "sbs1_tz: -720 .. 840 minutes");
        d->st.sbs1_tz = value;
        return AMB_OK;
    }
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
    if (n == 0) { d->sbs1_nb = -1; return AMB_OK; }
    DCK(cudaSetDevice(d->device));
    d->sbs1_nb = -1;
    int rc = prepare(d, n);
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
    if (k < 0) return dfail(d, AMB_ERR_CUDA, amb_stage_names[-k - 1].launch, e);
    d->launches += (uint64_t)k;
    if (d->st.sbs1 > 0) d->sbs1_nb = (n + 127) / 128;
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

// with_ext: amb_decoder_aircraft_ext(_device), ext[] beside out[]; else amb_decoder_aircraft(_device)
static int snapshot_impl(amb_decoder* d, double now, amb_aircraft* out, amb_aircraft_ext* ext, int max, bool out_on_device,
                         bool with_ext)
{
    const char* fn = with_ext ? "amb_decoder_aircraft_ext" : "amb_decoder_aircraft";
    char what[96];
    if (!d || max < 0 || (with_ext && out && !ext)) {
        snprintf(what, sizeof what, "%s: bad argument", fn);
        return dfail(d, AMB_ERR_INVALID, what);
    }
    if (d->st.track <= 0) { snprintf(what, sizeof what, "%s: option track is off", fn); return dfail(d, AMB_ERR_STATE, what); }
    if (with_ext && d->st.track_ext <= 0) return dfail(d, AMB_ERR_STATE, "amb_decoder_aircraft_ext: option track_ext is off");
    if (!d->st.tocc) return 0;                           // nothing decoded with the option on yet
    DCK(cudaSetDevice(d->device));
    cudaStream_t s = d->stream;
    const unsigned nb = AMB_TRACK_WORDS / AMB_SNAP_WORDS;
    uint32_t* off = d->st.snap_cnt + nb;
    cudaError_t e = cudaSuccess;
    if (amb_snap_count_launch(d->st.tocc, d->st.trows, d->st.tclk, now, d->st.track, AMB_TRACK_WORDS, d->st.snap_cnt, off,
                              s, &e) < 0)
        return dfail(d, AMB_ERR_CUDA, "aircraft snapshot", e);
    d->launches += 2;
    uint32_t total = 0;
    DCK(cudaMemcpyAsync(&total, off + nb, sizeof total, cudaMemcpyDeviceToHost, s));
    DCK(cudaStreamSynchronize(s));
    if (!out) return (int)total;
    if (total > (uint32_t)max) { snprintf(what, sizeof what, "%s: output buffer too small", fn); return dfail(d, AMB_ERR_OVERFLOW, what); }
    if (total == 0) return 0;
    amb_aircraft* dst = out;
    amb_aircraft_ext* xdst = ext;
    if (!out_on_device) {
        if (d->snap_cap < (int)total) {
            if (d->d_snap) cudaFree(d->d_snap);
            d->d_snap = nullptr; d->snap_cap = 0;
            DCK(cudaMalloc(&d->d_snap, (size_t)total * sizeof(amb_aircraft)));
            d->snap_cap = (int)total;
        }
        if (with_ext && d->xsnap_cap < (int)total) {
            if (d->d_xsnap) cudaFree(d->d_xsnap);
            d->d_xsnap = nullptr; d->xsnap_cap = 0;
            DCK(cudaMalloc(&d->d_xsnap, (size_t)total * sizeof(amb_aircraft_ext)));
            d->xsnap_cap = (int)total;
        }
        dst = d->d_snap;
        xdst = d->d_xsnap;
    }
    const int k = with_ext ? amb_snap_gather_ext_launch(d->st.tocc, d->st.trows, d->st.tclk, now, d->st.track, AMB_TRACK_WORDS,
                                                   off, dst, d->st.xocc, d->st.xrows, d->st.track_ext, xdst, s, &e)
                      : amb_snap_gather_launch(d->st.tocc, d->st.trows, d->st.tclk, now, d->st.track, AMB_TRACK_WORDS, off,
                                               dst, s, &e);
    if (k < 0) return dfail(d, AMB_ERR_CUDA, "aircraft snapshot", e);
    d->launches += 1;
    if (!out_on_device) {
        int rc = staged_d2h(d, out, d->d_snap, (size_t)total * sizeof(amb_aircraft), s);
        if (rc == AMB_OK && with_ext) rc = staged_d2h(d, ext, d->d_xsnap, (size_t)total * sizeof(amb_aircraft_ext), s);
        if (rc != AMB_OK) return rc;
    }
    DCK(cudaStreamSynchronize(s));
    return (int)total;
}

int amb_decoder_aircraft(amb_decoder* d, double now, amb_aircraft* out, int max)
{
    return snapshot_impl(d, now, out, nullptr, max, false, false);
}

int amb_decoder_aircraft_device(amb_decoder* d, double now, amb_aircraft* out_dev, int cap)
{
    return snapshot_impl(d, now, out_dev, nullptr, cap, true, false);
}

int amb_decoder_aircraft_ext(amb_decoder* d, double now, amb_aircraft* out, amb_aircraft_ext* ext, int max)
{
    return snapshot_impl(d, now, out, ext, max, false, true);
}

int amb_decoder_aircraft_ext_device(amb_decoder* d, double now, amb_aircraft* out_dev, amb_aircraft_ext* ext_dev, int cap)
{
    return snapshot_impl(d, now, out_dev, ext_dev, cap, true, true);
}

// the last decode's lines into out (host or device memory)
static int sbs1_impl(amb_decoder* d, char* out, size_t cap, size_t* n_bytes, bool out_on_device)
{
    if (!d || !n_bytes || (cap > 0 && !out)) return dfail(d, AMB_ERR_INVALID, "amb_decoder_sbs1: bad argument");
    *n_bytes = 0;
    if (d->st.sbs1 <= 0) return dfail(d, AMB_ERR_STATE, "amb_decoder_sbs1: option sbs1 is off");
    if (d->sbs1_nb < 0) return AMB_OK;                   // no decode with the option on since it was set
    DCK(cudaSetDevice(d->device));
    cudaStream_t s = d->stream;
    unsigned long long total = 0;
    DCK(cudaMemcpyAsync(&total, d->st.sb.boff + d->sbs1_nb, sizeof total, cudaMemcpyDeviceToHost, s));
    DCK(cudaStreamSynchronize(s));
    *n_bytes = (size_t)total;
    if (total > cap) return dfail(d, AMB_ERR_OVERFLOW, "amb_decoder_sbs1: output buffer too small");
    if (total == 0) return AMB_OK;
    if (out_on_device) DCK(cudaMemcpyAsync(out, d->st.sb.text, (size_t)total, cudaMemcpyDeviceToDevice, s));
    else {
        int rc = staged_d2h(d, out, d->st.sb.text, (size_t)total, s);
        if (rc != AMB_OK) return rc;
    }
    DCK(cudaStreamSynchronize(s));
    return AMB_OK;
}

int amb_decoder_sbs1(amb_decoder* d, char* out, size_t cap, size_t* n_bytes)
{
    return sbs1_impl(d, out, cap, n_bytes, false);
}

int amb_decoder_sbs1_device(amb_decoder* d, char* out_dev, size_t cap, size_t* n_bytes)
{
    return sbs1_impl(d, out_dev, cap, n_bytes, true);
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
