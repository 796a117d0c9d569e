// Text reports (decoder option "reports", DESIGN.md §8 "Text reports"). Runs last, after every other stage, so that
// Comm-B, op-status and local CPR results reach the lines; it reads the frames and the records and writes nothing into
// them. Every queued frame's line (amb_report_line, amb_report_format.h) is written in record order into one packed
// buffer, so that only the byte total crosses PCIe before the copy:
//
//   amb_reports_len    one thread per frame: formats its line into a stack buffer and keeps only the length; the
//                      block's byte count
//   amb_sbs1_scan      one block: the byte offset of every block of lines, and the total (amb_decode_sbs1.cuh)
//   amb_reports_write  one thread per frame: formats its line again, straight to its byte offset in the packed text
//
// The first queued frame after the decoder's creation or last reset is printed at precision 6 (the slicer's first
// message); the flag that says so is one word of device memory. While it is set, the warp's first queued frame looks
// back over the frames before it for an earlier queued one; the write pass's first frame then clears the flag. The
// look-back only runs until the stream's first queued frame has been formatted, and stops at the first queued frame it
// meets, so a pass reads each frame at most once for it.
#pragma once
#include "amb_report_format.h"

// The stage's per-call scratch (n frames); the Beast and AVR feeds (amb_decode_beast.cuh) keep theirs in the same form.
struct AmbReportBufs {
    uint32_t* len = nullptr;             // per record: bytes of its line
    uint32_t* bsum = nullptr;            // per block of 128 records: bytes of its lines
    unsigned long long* boff = nullptr;  // per block: byte offset of its lines; [blocks] = the total
    char* text = nullptr;                // the packed lines, AMB_REP_MAX_LINE bytes per frame of capacity (the feeds:
                                         // AMB_BEAST_MAX_MSG / AMB_AVR_MAX_LINE)
};

// Whether record k is the call's first queued record, for a lane that read the first-message flag as `set`; called by
// every lane of the warp. Only the warp's first queued lane looks back (the others have a queued lane before them).
static __device__ __forceinline__ bool amb_reports_first(const amb_fields* __restrict__ fields, int k, bool queued, bool set)
{
    const unsigned lane = threadIdx.x & 31;
    const unsigned q = __ballot_sync(0xffffffffu, queued);
    if (!set || !queued || (q & ((1u << lane) - 1u))) return false;
    for (int j = k - 1 - (int)lane; j >= 0; j--)
        if (!(fields[j].status & AMB_FS_NOT_QUEUED)) return false;
    return true;
}

// 128 threads per block; __maxnreg__ in place of __launch_bounds__, which leaves ptxas spilling at 72 registers
__global__ void __maxnreg__(128) amb_reports_len(const amb_frame* __restrict__ frames, const amb_fields* __restrict__ fields,
                                                       int n, const unsigned* __restrict__ first, uint32_t* __restrict__ len,
                                                       uint32_t* __restrict__ bsum)
{
    __shared__ unsigned s_w[4];
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    const bool queued = k < n && !(fields[k].status & AMB_FS_NOT_QUEUED);
    const bool f6 = amb_reports_first(fields, k, queued, *first != 0u);
    unsigned L = 0;
    if (queued) {
        char line[AMB_REP_MAX_LINE];
        L = (unsigned)amb_report_line(&frames[k], &fields[k], f6, line);
    }
    if (k < n) len[k] = L;
    unsigned v = L;
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x == 0) bsum[blockIdx.x] = s_w[0] + s_w[1] + s_w[2] + s_w[3];
}

__global__ void __launch_bounds__(128) amb_reports_write(const amb_frame* __restrict__ frames, const amb_fields* __restrict__ fields,
                                                         int n, unsigned* first, const uint32_t* __restrict__ len,
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
    const bool queued = k < n && !(fields[k].status & AMB_FS_NOT_QUEUED);
    // another warp's first frame may clear the flag meanwhile; then this warp holds no first frame and reads 0 or 1
    const bool f6 = amb_reports_first(fields, k, queued, *(volatile const unsigned*)first != 0u);
    if (L) amb_report_line(&frames[k], &fields[k], f6, text + off);
    if (f6) *first = 0u;
}

// Enqueue the stage (three kernels) after every other stage. Returns how many kernels were launched or -1 with *err set.
static int amb_reports_launch(const amb_frame* frames, const amb_fields* fields, int n, unsigned* first,
                              const AmbReportBufs* b, cudaStream_t s, cudaError_t* err)
{
    const int nb = (n + 127) / 128;
    AMB_LAUNCH((amb_reports_len), nb, 128, 0, s, frames, fields, n, first, b->len, b->bsum);
    AMB_LAUNCH((amb_sbs1_scan), 1, 1024, 0, s, b->bsum, nb, b->boff);
    AMB_LAUNCH((amb_reports_write), nb, 128, 0, s, frames, fields, n, first, b->len, b->boff, b->text);
    *err = cudaGetLastError();
    return *err == cudaSuccess ? 3 : -1;
}
