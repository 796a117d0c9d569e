// Batch field decode (SURVEY.md 8 row f4): kernels + C ABI of amb_decoder (include/airmodes_b200.h).
// The per-message arithmetic is in amb_decode_core.h, the kernels in amb_decode_kernels.cuh and amb_decode_v3.cuh
// (launch-free headers, so that tests/simt can run the same kernel source under a host emulator); this file holds the
// per-aircraft report table and the host orchestration. Compiled with -fmad=false: latitude/longitude follow cpr.py
// operation by operation in IEEE double, nothing may be contracted. Citations are file:line under gr-air-modes/python.
//
// Seven launches per decode, in stream order:
//   amb_fields_kernel   one thread per frame: bit fields, altitude, squawk, ident, velocity; emits the CPR report
//   amb_v3_*            five kernels, cpr_decoder's bookkeeping (cpr.py:206-229): for every position message, the latest
//                       even and odd report of its aircraft as of that message, from the reports partitioned by owner
//                       bucket and a direct-mapped table in HBM (2^26 x 16 B) that carries them from batch to batch
//   amb_resolve_kernel  one thread per frame: global CPR decode, range/bearing.
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
    int have_loc = 0; double lat = 0.0, lon = 0.0;
    AmbCprSlot* table = nullptr;
    double* nl_T = nullptr;              // device copy of the NL transition table
    amb_frame* d_frames = nullptr; amb_fields* d_fields = nullptr; AmbPosRec* d_pos = nullptr; AmbPair* d_pair = nullptr;
    int cap = 0;
    // host <-> device staging: pageable caller arrays go through two pinned bounce buffers per direction so that the
    // copies run at PCIe speed and overlap the memcpy of the next piece
    void* pin[2] = {nullptr, nullptr}; cudaEvent_t pin_ev[2] = {nullptr, nullptr}; size_t pin_bytes = 0;
    AmbV3Bufs v3;                        // scratch of the pairing stage
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
    if (d->d_pos) cudaFree(d->d_pos);
    if (d->d_pair) cudaFree(d->d_pair);
    d->d_frames = nullptr; d->d_fields = nullptr; d->d_pos = nullptr; d->d_pair = nullptr; d->cap = 0;
}

static int ensure_cap(amb_decoder* d, int n)
{
    if (n <= d->cap) return AMB_OK;
    int cap = d->cap ? d->cap : 4096;
    while (cap < n) cap *= 2;
    free_bufs(d);
    DCK(cudaMalloc(&d->d_frames, (size_t)cap * sizeof(amb_frame)));
    DCK(cudaMalloc(&d->d_fields, (size_t)cap * sizeof(amb_fields)));
    DCK(cudaMalloc(&d->d_pos, (size_t)cap * sizeof(AmbPosRec)));
    DCK(cudaMalloc(&d->d_pair, (size_t)cap * sizeof(AmbPair)));
    d->cap = cap;
    return AMB_OK;
}

extern "C" {

int amb_decoder_create(int device, int have_location, double lat, double lon, amb_decoder** out)
{
    static_assert(sizeof(amb_fields) == 144, "amb_fields layout");
    static_assert(sizeof(AmbCprSlot) == 16, "table slot layout");
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
    d->have_loc = have_location ? 1 : 0; d->lat = lat; d->lon = lon;
    int rc = AMB_OK;
    do {
        if (cudaSetDevice(device) != cudaSuccess) { rc = AMB_ERR_NO_DEVICE; break; }
        if (cudaStreamCreateWithFlags(&d->stream, cudaStreamNonBlocking) != cudaSuccess ||
            cudaEventCreate(&d->e0) != cudaSuccess || cudaEventCreate(&d->e1) != cudaSuccess) { rc = AMB_ERR_CUDA; break; }
        cudaError_t e = cudaMalloc(&d->table, AMB_TABLE_SLOTS * sizeof(AmbCprSlot));
        if (e != cudaSuccess) { rc = dfail(d, AMB_ERR_CUDA, "report table (1 GiB)", e); break; }
        if (cudaMalloc(&d->nl_T, AMB_NL_MAX * sizeof(double)) != cudaSuccess) { rc = AMB_ERR_CUDA; break; }
        double T[AMB_NL_MAX];
        amb_build_nl_table(T);                          // cpr.py:46-51 through the host libm, once
        if (cudaMemcpyAsync(d->nl_T, T, sizeof T, cudaMemcpyHostToDevice, d->stream) != cudaSuccess ||
            cudaMemsetAsync(d->table, 0xFF, AMB_TABLE_SLOTS * sizeof(AmbCprSlot), d->stream) != cudaSuccess ||
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
    amb_v3_free(&d->v3);
    for (int k = 0; k < 2; k++) { if (d->pin[k]) cudaFreeHost(d->pin[k]); if (d->pin_ev[k]) cudaEventDestroy(d->pin_ev[k]); }
    if (d->table) cudaFree(d->table);
    if (d->nl_T) cudaFree(d->nl_T);
    if (d->e0) cudaEventDestroy(d->e0);
    if (d->e1) cudaEventDestroy(d->e1);
    if (d->stream) cudaStreamDestroy(d->stream);
    delete d;
}

int amb_decoder_set_location(amb_decoder* d, int have_location, double lat, double lon)
{
    if (!d) return AMB_ERR_INVALID;
    d->have_loc = have_location ? 1 : 0; d->lat = lat; d->lon = lon;
    return AMB_OK;
}

int amb_decoder_reset(amb_decoder* d)
{
    if (!d) return AMB_ERR_INVALID;
    DCK(cudaSetDevice(d->device));
    DCK(cudaMemsetAsync(d->table, 0xFF, AMB_TABLE_SLOTS * sizeof(AmbCprSlot), d->stream));
    DCK(cudaStreamSynchronize(d->stream));
    return AMB_OK;
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
    const int nb = (n + 127) / 128;
    AMB_LAUNCH((amb_fields_kernel), nb, 128, 0, s, src, n, fields, d->d_pos, d->d_pair);
    DCK(cudaGetLastError());
    cudaError_t e = cudaSuccess;
    const int k = amb_v3_launch(&d->v3, d->d_pos, n, d->table, d->d_pair, s, &e);
    if (k < 0) return dfail(d, AMB_ERR_CUDA, "pairing", e);
    AMB_LAUNCH((amb_resolve_kernel), nb, 128, 0, s, fields, d->d_pos, d->d_pair, n, d->have_loc, d->lat, d->lon, d->nl_T);
    DCK(cudaGetLastError());
    d->launches += 2 + (uint64_t)k;
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
