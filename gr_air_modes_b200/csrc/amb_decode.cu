// Batch field decode (SURVEY.md 8 row f4): kernels + C ABI of amb_decoder (include/airmodes_b200.h).
// The per-message arithmetic is in amb_decode_core.h, the kernels, amb_decode_launch - the one launch sequence of a
// decode - the stages' memory (amb_decode_prepare / amb_decode_reset / amb_decode_free), the option table and the
// read-outs of the results in amb_decode_kernels.cuh and the stage headers it includes (launch-free headers, so that
// tests/simt can run the same kernel source, sequence, memory, option and read-out rules under a host emulator); this
// file keeps the frames, records and snapshot rows on their way between the caller and the stages, copies the frames
// in and the records out. Compiled with -fmad=false: latitude/longitude follow cpr.py operation by operation in IEEE
// double, nothing may be contracted. Citations are file:line under gr-air-modes/python.
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
// With option "coverage" on, one more right after those (amb_decode_coverage.cuh): amb_coverage_kernel - the greatest
// range per 5-degree bearing sector and altitude band of az_map_model, folded into a 72 x 9 grid in HBM (5184 B) by
// shared and global atomicMax on the bits of the ranges, carried from batch to batch; amb_decoder_coverage copies it out.
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
// With option "reports" on, three more after those (amb_decode_reports.cuh): amb_reports_len, amb_sbs1_scan,
// amb_reports_write - the call's text reports, the lines of report.py, packed on the device; amb_decoder_reports copies
// them out.
// The multilateration object amb_mlat (amb_mlat.cuh) lives here too: its C ABI is at the end of this file.
#include "amb_launch.h"
#include "amb_decode_core.h"
#include "amb_decode_kernels.cuh"
#include "amb_mlat.cuh"

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
    uint64_t launches = 0; float ms_last = 0.f;
    std::string err;
};

static thread_local std::string g_create_err;          // why the last amb_decoder_create on this thread failed

// ---- host ---------------------------------------------------------------------------------------------------------
extern "C" void amb_parallel_memcpy(void* dst, const void* src, size_t n);      // amb_api.cu (the ingest copy threads)
#define AMB_DEC_PIECE ((size_t)8 << 20)

static int alloc_pinned(amb_decoder* d)
{
    if (d->pin[0]) return AMB_OK;
    for (int k = 0; k < 2; k++) {
        CK(d, cudaMallocHost(&d->pin[k], AMB_DEC_PIECE));
        CK(d, cudaEventCreateWithFlags(&d->pin_ev[k], cudaEventDisableTiming));
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
        CK(d, cudaEventSynchronize(d->pin_ev[k]));
        amb_parallel_memcpy(d->pin[k], static_cast<const char*>(src) + off, m);
        CK(d, cudaMemcpyAsync(static_cast<char*>(dst) + off, d->pin[k], m, cudaMemcpyHostToDevice, s));
        CK(d, cudaEventRecord(d->pin_ev[k], s));
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
            CK(d, cudaMemcpyAsync(d->pin[i & 1], static_cast<const char*>(src) + off, m, cudaMemcpyDeviceToHost, s));
            CK(d, cudaEventRecord(d->pin_ev[i & 1], s));
        }
        if (i >= 1) {
            const size_t off = (i - 1) * AMB_DEC_PIECE, m = bytes - off < AMB_DEC_PIECE ? bytes - off : AMB_DEC_PIECE;
            CK(d, cudaEventSynchronize(d->pin_ev[(i - 1) & 1]));
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
    if (k < 0) return fail(d, AMB_ERR_CUDA, amb_stage_names[-k - 1].memory, e);
    if (d->cap < d->st.cap) {
        free_bufs(d);
        CK(d, cudaMalloc(&d->d_frames, (size_t)d->st.cap * sizeof(amb_frame)));
        CK(d, cudaMalloc(&d->d_fields, (size_t)d->st.cap * sizeof(amb_fields)));
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
    cudaDeviceProp prop;
    if (amb_check_device(device, &prop) != AMB_OK) return AMB_ERR_NO_DEVICE;
    amb_decoder* d = new (std::nothrow) amb_decoder();
    if (!d) return AMB_ERR_INVALID;
    d->device = device;
    amb_decode_set_location(&d->st, have_location, lat, lon);
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
    amb_decode_set_location(&d->st, have_location, lat, lon);
    return AMB_OK;
}

int amb_decoder_reset(amb_decoder* d)
{
    if (!d) return AMB_ERR_INVALID;
    CK(d, cudaSetDevice(d->device));
    cudaError_t e = cudaSuccess;
    const int k = amb_decode_reset(&d->st, d->stream, &e);
    if (k < 0) return fail(d, AMB_ERR_CUDA, amb_stage_names[-k - 1].memory, e);
    CK(d, cudaStreamSynchronize(d->stream));
    return AMB_OK;
}

int amb_decoder_set_option(amb_decoder* d, const char* name, int value)
{
    if (!d || !name) return AMB_ERR_INVALID;
    const char* refused = amb_decode_set_option(&d->st, name, value);
    return refused ? fail(d, AMB_ERR_INVALID, refused) : AMB_OK;
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
        return fail(d, AMB_ERR_INVALID, "amb_decode_frames: bad argument");
    d->st.sbs1_nb = d->st.reports_nb = -1;              // until amb_decode_launch has launched every stage
    if (n == 0) return AMB_OK;
    CK(d, cudaSetDevice(d->device));
    int rc = prepare(d, n);
    if (rc != AMB_OK) return rc;
    cudaStream_t s = d->stream;
    amb_fields* const fields = out_on_device ? out : d->d_fields;
    CK(d, cudaEventRecord(d->e0, s));
    const amb_frame* src = frames;
    if (mem_kind == AMB_MEM_HOST) {
        rc = staged_h2d(d, d->d_frames, frames, (size_t)n * sizeof(amb_frame), s);
        if (rc != AMB_OK) return rc;
        src = d->d_frames;
    }
    cudaError_t e = cudaSuccess;
    const int k = amb_decode_launch(&d->st, src, n, fields, s, &e);
    if (k < 0) return fail(d, AMB_ERR_CUDA, amb_stage_names[-k - 1].launch, e);
    d->launches += (uint64_t)k;
    if (!out_on_device) {
        rc = staged_d2h(d, out, d->d_fields, (size_t)n * sizeof(amb_fields), s);
        if (rc != AMB_OK) return rc;
    }
    CK(d, cudaEventRecord(d->e1, s));
    CK(d, cudaStreamSynchronize(s));
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
        return fail(d, AMB_ERR_INVALID, what);
    }
    if (d->st.track <= 0) { snprintf(what, sizeof what, "%s: option track is off", fn); return fail(d, AMB_ERR_STATE, what); }
    if (with_ext && d->st.track_ext <= 0) return fail(d, AMB_ERR_STATE, "amb_decoder_aircraft_ext: option track_ext is off");
    if (!d->st.tocc) return 0;                           // nothing decoded with the option on yet
    CK(d, cudaSetDevice(d->device));
    cudaStream_t s = d->stream;
    cudaError_t e = cudaSuccess;
    const int total = amb_decode_snapshot_count(&d->st, now, AMB_TRACK_WORDS, s, &e);
    if (total < 0) return fail(d, AMB_ERR_CUDA, "aircraft snapshot", e);
    d->launches += 2;
    if (!out) return total;
    if (total > max) { snprintf(what, sizeof what, "%s: output buffer too small", fn); return fail(d, AMB_ERR_OVERFLOW, what); }
    if (total == 0) return 0;
    amb_aircraft* dst = out;
    amb_aircraft_ext* xdst = ext;
    if (!out_on_device) {
        if (d->snap_cap < total) {
            if (d->d_snap) cudaFree(d->d_snap);
            d->d_snap = nullptr; d->snap_cap = 0;
            CK(d, cudaMalloc(&d->d_snap, (size_t)total * sizeof(amb_aircraft)));
            d->snap_cap = total;
        }
        if (with_ext && d->xsnap_cap < total) {
            if (d->d_xsnap) cudaFree(d->d_xsnap);
            d->d_xsnap = nullptr; d->xsnap_cap = 0;
            CK(d, cudaMalloc(&d->d_xsnap, (size_t)total * sizeof(amb_aircraft_ext)));
            d->xsnap_cap = total;
        }
        dst = d->d_snap;
        xdst = d->d_xsnap;
    }
    if (amb_decode_snapshot_gather(&d->st, now, AMB_TRACK_WORDS, dst, with_ext ? xdst : nullptr, s, &e) < 0)
        return fail(d, AMB_ERR_CUDA, "aircraft snapshot", e);
    d->launches += 1;
    if (!out_on_device) {
        int rc = staged_d2h(d, out, d->d_snap, (size_t)total * sizeof(amb_aircraft), s);
        if (rc == AMB_OK && with_ext) rc = staged_d2h(d, ext, d->d_xsnap, (size_t)total * sizeof(amb_aircraft_ext), s);
        if (rc != AMB_OK) return rc;
    }
    CK(d, cudaStreamSynchronize(s));
    return total;
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

// amb_decoder_sbs1(_device), and amb_decoder_reports(_device) when `reports`: the last decode's lines into out (host or
// device memory)
static int text_impl(amb_decoder* d, bool reports, char* out, size_t cap, size_t* n_bytes, bool out_on_device)
{
    const char* fn = !reports ? "amb_decoder_sbs1" : out_on_device ? "amb_decoder_reports_device" : "amb_decoder_reports";
    char what[96];
    if (!d || !n_bytes || (cap > 0 && !out)) { snprintf(what, sizeof what, "%s: bad argument", fn); return fail(d, AMB_ERR_INVALID, what); }
    *n_bytes = 0;
    if ((reports ? d->st.reports : d->st.sbs1) <= 0) {
        snprintf(what, sizeof what, "%s: option %s is off", fn, reports ? "reports" : "sbs1");
        return fail(d, AMB_ERR_STATE, what);
    }
    CK(d, cudaSetDevice(d->device));
    cudaStream_t s = d->stream;
    const char* text = nullptr;
    unsigned long long total = 0;
    CK(d, amb_decode_text(&d->st, reports, s, &text, &total));
    *n_bytes = (size_t)total;
    if (total > cap) { snprintf(what, sizeof what, "%s: output buffer too small", fn); return fail(d, AMB_ERR_OVERFLOW, what); }
    if (total == 0) return AMB_OK;
    if (out_on_device) CK(d, cudaMemcpyAsync(out, text, (size_t)total, cudaMemcpyDeviceToDevice, s));
    else {
        int rc = staged_d2h(d, out, text, (size_t)total, s);
        if (rc != AMB_OK) return rc;
    }
    CK(d, cudaStreamSynchronize(s));
    return AMB_OK;
}

int amb_decoder_sbs1(amb_decoder* d, char* out, size_t cap, size_t* n_bytes)
{
    return text_impl(d, false, out, cap, n_bytes, false);
}

int amb_decoder_sbs1_device(amb_decoder* d, char* out_dev, size_t cap, size_t* n_bytes)
{
    return text_impl(d, false, out_dev, cap, n_bytes, true);
}

int amb_decoder_reports(amb_decoder* d, char* out, size_t cap, size_t* n_bytes)
{
    return text_impl(d, true, out, cap, n_bytes, false);
}

int amb_decoder_reports_device(amb_decoder* d, char* out_dev, size_t cap, size_t* n_bytes)
{
    return text_impl(d, true, out_dev, cap, n_bytes, true);
}

// the coverage grid into out (host or device memory)
static int coverage_impl(amb_decoder* d, double* out, bool out_on_device)
{
    const char* fn = out_on_device ? "amb_decoder_coverage_device" : "amb_decoder_coverage";
    char what[96];
    if (!d || !out) { snprintf(what, sizeof what, "%s: bad argument", fn); return fail(d, AMB_ERR_INVALID, what); }
    if (d->st.coverage <= 0) { snprintf(what, sizeof what, "%s: option coverage is off", fn); return fail(d, AMB_ERR_STATE, what); }
    CK(d, cudaSetDevice(d->device));
    CK(d, amb_decode_coverage(&d->st, out, out_on_device, d->stream));
    return AMB_OK;
}

int amb_decoder_coverage(amb_decoder* d, double* out)
{
    return coverage_impl(d, out, false);
}

int amb_decoder_coverage_device(amb_decoder* d, double* out_dev)
{
    return coverage_impl(d, out_dev, true);
}

int amb_decoder_coverage_reset(amb_decoder* d)
{
    if (!d) return AMB_ERR_INVALID;
    if (d->st.coverage <= 0) return fail(d, AMB_ERR_STATE, "amb_decoder_coverage_reset: option coverage is off");
    if (!d->st.cgrid) return AMB_OK;
    CK(d, cudaSetDevice(d->device));
    CK(d, cudaMemsetAsync(d->st.cgrid, 0, AMB_COVERAGE_CELLS * sizeof(unsigned long long), d->stream));
    CK(d, cudaStreamSynchronize(d->stream));
    return AMB_OK;
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

// ---- multilateration (amb_mlat.cuh) ---------------------------------------------------------------------------------
struct amb_mlat {
    int device = 0;
    cudaStream_t stream = nullptr;
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    AmbMlatState st;
    amb_mlat_counts totals = {};
    std::string err;
};

static thread_local std::string g_mlat_create_err;

// llh2ecef (mlat.py:77-86) of a station, and the terms of the start point overhead it
static AmbMlatStation mlat_station(double lat_deg, double lon_deg, double height)
{
    AmbMlatStation o;
    const double lat = lat_deg * (M_PI / 180.0), lon = lon_deg * (M_PI / 180.0);
    o.sl = sin(lat); o.cl = cos(lat); o.so = sin(lon); o.co = cos(lon);
    o.n = AMB_MLAT_WGS_A / sqrt(1 - AMB_MLAT_WGS_E2 * (o.sl * o.sl));
    o.s[0] = (o.n + height) * o.cl * o.co; o.s[1] = (o.n + height) * o.cl * o.so;
    o.s[2] = (o.n * (1 - AMB_MLAT_WGS_E2) + height) * o.sl;
    return o;
}

extern "C" {

int amb_mlat_create(int device, int K, const double* lat, const double* lon, const double* height, amb_mlat** out)
{
    static_assert(sizeof(amb_mlat_fix) == 112, "amb_mlat_fix layout");
    static_assert(sizeof(amb_mlat_counts) == 80, "amb_mlat_counts layout");
    static_assert(sizeof(AmbMlatItem) == 48, "item layout");
    if (!out) return AMB_ERR_INVALID;
    *out = nullptr;
    if (K < AMB_MLAT_MIN_STATIONS || K > AMB_MLAT_MAX_STATIONS || !lat || !lon || !height) {
        g_mlat_create_err = "amb_mlat_create: K must be 3 .. 32, with lat, lon and height for each station";
        return AMB_ERR_INVALID;
    }
    for (int k = 0; k < K; k++)
        if (!(fabs(lat[k]) <= 90.0) || !(fabs(lon[k]) <= 360.0) || !(fabs(height[k]) < 1e6)) {
            g_mlat_create_err = "amb_mlat_create: a station position is out of range";
            return AMB_ERR_INVALID;
        }
    cudaDeviceProp prop;
    if (amb_check_device(device, &prop) != AMB_OK) return AMB_ERR_NO_DEVICE;
    amb_mlat* m = new (std::nothrow) amb_mlat();
    if (!m) return AMB_ERR_INVALID;
    m->device = device;
    m->st.K = K;
    AmbMlatStation sta[AMB_MLAT_MAX_STATIONS];
    double dmax = 0.0;
    for (int k = 0; k < K; k++) sta[k] = mlat_station(lat[k], lon[k], height[k]);
    for (int i = 0; i < K; i++)
        for (int j = i + 1; j < K; j++) {
            const double d = amb_mlat_norm3(sta[i].s[0] - sta[j].s[0], sta[i].s[1] - sta[j].s[1], sta[i].s[2] - sta[j].s[2]);
            dmax = d > dmax ? d : dmax;
        }
    m->st.W = dmax / AMB_MLAT_C + 2e-6;
    int rc = AMB_OK;
    do {
        if (cudaSetDevice(device) != cudaSuccess) { rc = AMB_ERR_NO_DEVICE; break; }
        if (cudaStreamCreateWithFlags(&m->stream, cudaStreamNonBlocking) != cudaSuccess ||
            cudaEventCreate(&m->e0) != cudaSuccess || cudaEventCreate(&m->e1) != cudaSuccess) { rc = AMB_ERR_CUDA; break; }
        if (cudaMalloc(&m->st.sta, (size_t)K * sizeof(AmbMlatStation)) != cudaSuccess ||
            cudaMemcpy(m->st.sta, sta, (size_t)K * sizeof(AmbMlatStation), cudaMemcpyHostToDevice) != cudaSuccess) {
            rc = AMB_ERR_CUDA; break;
        }
    } while (0);
    if (rc != AMB_OK) { g_mlat_create_err = "CUDA resource creation failed"; amb_mlat_destroy(m); return rc; }
    g_mlat_create_err.clear();
    *out = m;
    return AMB_OK;
}

void amb_mlat_destroy(amb_mlat* m)
{
    if (!m) return;
    cudaSetDevice(m->device);
    if (m->stream) cudaStreamSynchronize(m->stream);
    amb_mlat_free(&m->st);
    if (m->e0) cudaEventDestroy(m->e0);
    if (m->e1) cudaEventDestroy(m->e1);
    if (m->stream) cudaStreamDestroy(m->stream);
    delete m;
}

int amb_mlat_set_option(amb_mlat* m, const char* name, double value)
{
    if (!m || !name) return AMB_ERR_INVALID;
    if (strcmp(name, "window_us") == 0) {
        if (!(value > 0.0) || !(value <= 1e6)) return fail(m, AMB_ERR_INVALID, "window_us: > 0 .. 1e6 microseconds");
        m->st.W = value / 1e6;
        return AMB_OK;
    }
    return fail(m, AMB_ERR_INVALID, "amb_mlat_set_option: unknown option");
}

int amb_mlat_get_option(amb_mlat* m, const char* name, double* value)
{
    if (!m || !name || !value) return AMB_ERR_INVALID;
    if (strcmp(name, "window_us") == 0) { *value = m->st.W * 1e6; return AMB_OK; }
    return fail(m, AMB_ERR_INVALID, "amb_mlat_get_option: unknown option");
}

int amb_mlat_set_offset(amb_mlat* m, int k, double seconds)
{
    if (!m) return AMB_ERR_INVALID;
    if (k < 0 || k >= m->st.K) return fail(m, AMB_ERR_INVALID, "amb_mlat_set_offset: no such station");
    if (!(fabs(seconds) <= 1.0)) return fail(m, AMB_ERR_INVALID, "amb_mlat_set_offset: |seconds| <= 1");
    m->st.off[k] = seconds;
    return AMB_OK;
}

int amb_mlat_reset(amb_mlat* m)
{
    if (!m) return AMB_ERR_INVALID;
    m->st.C = 0;
    m->totals.carried = 0;
    return AMB_OK;
}

static int mlat_impl(amb_mlat* m, const amb_frame* const* frames, const int* counts, uint64_t end_secs, double end_frac,
                     int flush, amb_mlat_fix* out, int cap, int* n_out, bool on_device)
{
    const char* fn = on_device ? "amb_mlat_process_device" : "amb_mlat_process";
    char what[128];
    if (!m || !frames || !counts || !n_out || cap < 0 || (cap > 0 && !out) || (!flush && !(end_frac - end_frac == 0.0))) {
        snprintf(what, sizeof what, "%s: bad argument", fn);
        return fail(m, AMB_ERR_INVALID, what);
    }
    *n_out = 0;
    AmbMlatState* s = &m->st;
    AmbMlatCall c;
    memset(&c, 0, sizeof c);
    c.K = s->K;
    long long P = 0, total = 0;
    for (int k = 0; k < s->K; k++) {
        if (counts[k] < 0 || (counts[k] > 0 && !frames[k])) { snprintf(what, sizeof what, "%s: bad frames of station %d", fn, k); return fail(m, AMB_ERR_INVALID, what); }
        c.count[k] = counts[k]; c.base[k] = (int)P; c.off[k] = s->off[k];
        P += (counts[k] + AMB_MLAT_BLOCK - 1) / AMB_MLAT_BLOCK * AMB_MLAT_BLOCK;
        total += counts[k];
    }
    if (P + s->C > (1ll << 30)) { snprintf(what, sizeof what, "%s: more than 2^30 frames in one call", fn); return fail(m, AMB_ERR_INVALID, what); }
    c.base[s->K] = (int)P;
    const int nb = (int)(P / AMB_MLAT_BLOCK);
    CK(m, cudaSetDevice(m->device));
    cudaStream_t st = m->stream;
    cudaError_t e = cudaSuccess;
    // the scan buffers serve the raw blocks and, after the count, the N <= C + total items: sized for both now, because
    // the count's offsets in boff[0] are read again after it
    const long long nbn_max = (s->C + total + AMB_MLAT_BLOCK - 1) / AMB_MLAT_BLOCK;
    if (amb_mlat_prepare_raw(s, nbn_max > nb ? (int)nbn_max : nb, &e) < 0)
        return fail(m, AMB_ERR_CUDA, "amb_mlat: scratch memory", e);
    CK(m, cudaEventRecord(m->e0, st));
    if (on_device) {
        for (int k = 0; k < s->K; k++) c.f[k] = frames[k];
    } else if (total) {
        if (s->raw_cap < (size_t)total) {
            if (s->raw) cudaFree(s->raw);
            s->raw = nullptr; s->raw_cap = 0;
            CK(m, cudaMalloc(&s->raw, (size_t)total * sizeof(amb_frame)));
            s->raw_cap = (size_t)total;
        }
        size_t at = 0;
        for (int k = 0; k < s->K; k++) {
            if (counts[k]) CK(m, cudaMemcpyAsync(s->raw + at, frames[k], (size_t)counts[k] * sizeof(amb_frame), cudaMemcpyHostToDevice, st));
            c.f[k] = s->raw + at;
            at += (size_t)counts[k];
        }
    }
    uint64_t launches = 0;
    unsigned long long E = 0;
    if (nb) {
        launches += (uint64_t)amb_mlat_launch_count(c, nb, s, st, &e);
        if (e != cudaSuccess) return fail(m, AMB_ERR_CUDA, "amb_mlat: count", e);
        CK(m, cudaMemcpyAsync(&E, s->boff[0] + nb, sizeof E, cudaMemcpyDeviceToHost, st));
        CK(m, cudaStreamSynchronize(st));
    }
    const int N = s->C + (int)E;
    int G = 0, Cn = 0;
    unsigned long long ctr[AMB_MC_N] = {};
    if (N > 0) {
        int npad = 1;
        while (npad < N) npad <<= 1;
        if (amb_mlat_prepare_items(s, N, npad, &e) < 0) return fail(m, AMB_ERR_CUDA, "amb_mlat: scratch memory", e);
        launches += (uint64_t)amb_mlat_launch_group(c, nb, N, npad, 2048u, end_secs, end_frac, flush, s, st, &e);
        if (e != cudaSuccess) return fail(m, AMB_ERR_CUDA, "amb_mlat: grouping", e);
        const int nbn = (N + AMB_MLAT_BLOCK - 1) / AMB_MLAT_BLOCK;
        unsigned long long g = 0, cn = 0;
        CK(m, cudaMemcpyAsync(&g, s->boff[0] + nbn, sizeof g, cudaMemcpyDeviceToHost, st));
        CK(m, cudaMemcpyAsync(&cn, s->boff[1] + nbn, sizeof cn, cudaMemcpyDeviceToHost, st));
        CK(m, cudaMemcpyAsync(ctr, s->ctr, sizeof ctr, cudaMemcpyDeviceToHost, st));
        CK(m, cudaStreamSynchronize(st));
        if (ctr[AMB_MC_UNORDERED]) {
            snprintf(what, sizeof what, "%s: a station's frames are not in time order", fn);
            return fail(m, AMB_ERR_INVALID, what);
        }
        G = (int)g; Cn = (int)cn;
        if (G > cap) {
            *n_out = G;
            snprintf(what, sizeof what, "%s: output buffer too small", fn);
            return fail(m, AMB_ERR_OVERFLOW, what);
        }
        if (!on_device && s->fix_cap < G) {
            if (s->fix) cudaFree(s->fix);
            s->fix = nullptr; s->fix_cap = 0;
            CK(m, cudaMalloc(&s->fix, (size_t)G * sizeof(amb_mlat_fix)));
            s->fix_cap = G;
        }
        launches += (uint64_t)amb_mlat_launch_solve(N, G, on_device ? out : s->fix, s, st, &e);
        if (e != cudaSuccess) return fail(m, AMB_ERR_CUDA, "amb_mlat: solve", e);
        if (!on_device && G) CK(m, cudaMemcpyAsync(out, s->fix, (size_t)G * sizeof(amb_mlat_fix), cudaMemcpyDeviceToHost, st));
        CK(m, cudaMemcpyAsync(ctr, s->ctr, sizeof ctr, cudaMemcpyDeviceToHost, st));
    }
    CK(m, cudaEventRecord(m->e1, st));
    CK(m, cudaStreamSynchronize(st));
    // commit
    s->C = Cn;
    *n_out = G;
    amb_mlat_counts& t = m->totals;
    t.eligible += E; t.carried = (uint64_t)Cn;
    t.solved += ctr[AMB_MC_SOLVED]; t.no_convergence += ctr[AMB_MC_NO_CONV]; t.degenerate += ctr[AMB_MC_DEGENERATE];
    t.too_few += ctr[AMB_MC_TOO_FEW]; t.duplicate += ctr[AMB_MC_DUPLICATE]; t.span += ctr[AMB_MC_SPAN];
    t.kernel_launches += launches;
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, m->e0, m->e1) == cudaSuccess) t.ms_last = ms;
    return AMB_OK;
}

int amb_mlat_process(amb_mlat* m, const amb_frame* const* frames, const int* counts, uint64_t end_secs, double end_frac,
                     int flush, amb_mlat_fix* out, int cap, int* n_out)
{
    return mlat_impl(m, frames, counts, end_secs, end_frac, flush, out, cap, n_out, false);
}

int amb_mlat_process_device(amb_mlat* m, const amb_frame* const* frames_dev, const int* counts, uint64_t end_secs,
                            double end_frac, int flush, amb_mlat_fix* out_dev, int cap, int* n_out)
{
    return mlat_impl(m, frames_dev, counts, end_secs, end_frac, flush, out_dev, cap, n_out, true);
}

int amb_mlat_stats(amb_mlat* m, amb_mlat_counts* out)
{
    if (!m || !out) return AMB_ERR_INVALID;
    *out = m->totals;
    return AMB_OK;
}

const char* amb_mlat_last_error(const amb_mlat* m) { return m ? m->err.c_str() : g_mlat_create_err.c_str(); }

}  // extern "C"
