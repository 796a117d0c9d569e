// Beast binary and AVR raw feeds (decoder options "beast" and "avr", DESIGN.md §8 "Beast and AVR feeds"): the wire
// formats dump1090 and readsb exchange raw frames in. Each format runs after the text reports and reads only the frames
// and the records' status; it writes nothing into either. Every queued frame's message is written in record order into
// one packed buffer per format, so that only the byte total crosses PCIe before the copy. Three kernels per format:
//
//   amb_feed_len<F>    one thread per frame: the length of its message; the block's byte count
//   amb_sbs1_scan      one block: the byte offset of every block of messages, and the total (amb_decode_sbs1.cuh)
//   amb_feed_write<F>  one thread per frame: its message, straight to its byte offset in the packed buffer
//
// Nothing is carried from call to call, so the bytes do not depend on how the stream is cut into calls.
#pragma once

#define AMB_BEAST_MAX_MSG 44     // 0x1a, the type byte, then T (6 bytes), S and 14 payload bytes, each written twice
#define AMB_AVR_MAX_LINE 43      // '@', T in 12 hex digits, 28 hex digits of payload, ";\n"

enum { AMB_FEED_BEAST = 0, AMB_FEED_AVR = 1 };

// T of a frame: its stamp as a 48-bit count at 12 MHz (include/airmodes_b200.h rule 2). One fp64 multiply, rint half to
// even; the sum in uint64 wraparound arithmetic is exact modulo 2^48.
AMB_HD uint64_t amb_beast_time(const amb_frame& f)
{
    const double x = f.frac * 12e6;
    if (!(fabs(x) < 4611686018427387904.0)) return 0;   // 2^62; also every NaN and infinity
    return (f.secs * 12000000ull + (uint64_t)(int64_t)rint(x)) & 0xFFFFFFFFFFFFull;
}

// S of a frame: the amplitude of its reference level (a power) on 0 .. 255 (rule 3)
AMB_HD unsigned amb_beast_signal(float ref_level)
{
    const double v = (double)ref_level;
    if (!(v > 0.0)) return 0u;
    if (v >= 1.0) return 255u;
    const int s = (int)rint(255.0 * sqrt(v));
    return s < 1 ? 1u : (unsigned)s;
}

// The message of frame f in format F (the AVR form 1 or 2 in `form`) into out, or only its length when out is NULL;
// returns the length. A frame is long (14 payload bytes) when nbits is 112, else short (7 bytes), as the decoder reads it.
template <int F> AMB_HD unsigned amb_feed_msg(const amb_frame& f, int form, char* out)
{
    const unsigned nb = f.nbits == 112 ? 14u : 7u;
    if (F == AMB_FEED_AVR) {
        const unsigned L = 1u + (form == 2 ? 12u : 0u) + 2u * nb + 2u;
        if (!out) return L;
        const char* hex = "0123456789ABCDEF";
        char* p = out;
        *p++ = form == 2 ? '@' : '*';
        if (form == 2) {
            const uint64_t T = amb_beast_time(f);
            for (int i = 11; i >= 0; i--) *p++ = hex[(T >> (4 * i)) & 15u];
        }
        for (unsigned i = 0; i < nb; i++) { *p++ = hex[f.data[i] >> 4]; *p++ = hex[f.data[i] & 15u]; }
        *p++ = ';'; *p = '\n';
        return L;
    }
    const uint64_t T = amb_beast_time(f);
    const uint8_t S = (uint8_t)amb_beast_signal(f.ref_level);
    if (out) { out[0] = 0x1a; out[1] = nb == 14 ? '3' : '2'; }
    unsigned L = 2;
    for (unsigned i = 0; i < 7 + nb; i++) {             // T, S, payload
        const uint8_t b = i < 6 ? (uint8_t)(T >> (40 - 8 * i)) : i == 6 ? S : f.data[i - 7];
        if (out) out[L] = (char)b;
        L++;
        if (b == 0x1a) { if (out) out[L] = 0x1a; L++; }  // the escape: every 0x1a after the type byte twice
    }
    return L;
}

template <int F>
__global__ void __launch_bounds__(128) amb_feed_len(const amb_frame* __restrict__ frames, const amb_fields* __restrict__ fields,
                                                    int n, int form, uint32_t* __restrict__ len, uint32_t* __restrict__ bsum)
{
    __shared__ unsigned s_w[4];
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned L = k < n && !(fields[k].status & AMB_FS_NOT_QUEUED) ? amb_feed_msg<F>(frames[k], form, nullptr) : 0u;
    if (k < n) len[k] = L;
    unsigned v = L;
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x == 0) bsum[blockIdx.x] = s_w[0] + s_w[1] + s_w[2] + s_w[3];
}

template <int F>
__global__ void __launch_bounds__(128) amb_feed_write(const amb_frame* __restrict__ frames, int n, int form,
                                                      const uint32_t* __restrict__ len,
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
    if (L) amb_feed_msg<F>(frames[k], form, out + off);
}

// Enqueue format F (three kernels) over the n frames into b. Returns how many kernels were launched or -1 with *err set.
template <int F>
static int amb_feed_launch(const amb_frame* frames, const amb_fields* fields, int n, int form, const AmbReportBufs* b,
                           cudaStream_t s, cudaError_t* err)
{
    const int nb = (n + 127) / 128;
    AMB_LAUNCH((amb_feed_len<F>), nb, 128, 0, s, frames, fields, n, form, b->len, b->bsum);
    AMB_LAUNCH((amb_sbs1_scan), 1, 1024, 0, s, b->bsum, nb, b->boff);
    AMB_LAUNCH((amb_feed_write<F>), nb, 128, 0, s, frames, n, form, b->len, b->boff, b->text);
    *err = cudaGetLastError();
    return *err == cudaSuccess ? 3 : -1;
}
