// Beast binary input (amb_beast_reader, include/airmodes_b200.h "Beast binary input", DESIGN.md §8 "Beast input"): the
// byte stream dump1090 and readsb serve on TCP port 30005, and amb_decode_beast.cuh writes, parsed on the device into
// amb_frame records for the batch decoder. The framing looks sequential because every 0x1a inside a message is doubled,
// but whether a byte starts a token depends only on the parity of the 0x1a run in front of it: a byte is a token start
// exactly when the position of the last byte before it that is not 0x1a lies an odd distance back. That position is a
// max-scan, so the parse is two scans and local work. Five kernels per call, whatever the byte count:
//
//   amb_bin_last    one block per tile of 4096 bytes: the position of its last byte that is not 0x1a (-1: none)
//   amb_bin_scan    one block: the exclusive max-scan of those, i.e. the last such byte before every tile
//   amb_bin_count   one block per tile: token starts, then per sync token of type '1' / '2' / '3' a walk of at most 21
//                   data tokens (42 bytes) that decides complete / truncated / still open at the end; the counters, the
//                   tile's frame count, and the start of what is carried (atomicMin)
//   amb_sbs1_scan   one block: the exclusive sum of the tiles' frame counts, the total after them (amb_decode_sbs1.cuh)
//   amb_bin_emit    one block per tile: the same classification again, and every complete Mode S message's frame at its
//                   slot in stream order (assembled in shared memory, stored 16 bytes at a time); block 0 writes the
//                   carry and the stream offset for the next call
//
// The call's bytes B are the carry of the last call (at most AMB_BEAST_CARRY_MAX bytes, kept on the device) followed
// by the new bytes, read in place from device memory or from the staging copy of host bytes. The carry and the stream
// offset live in two device copies that calls alternate between, so that amb_bin_emit can write the next call's while
// its other blocks still read this call's. Only the frame count crosses PCIe.
#pragma once
#include "amb_decode_kernels.cuh"

#define AMB_BIN_TILE 4096        // bytes per block
#define AMB_BIN_THREADS 256
#define AMB_BIN_PER 16           // consecutive bytes per thread: at most one complete Mode S message starts among them
#define AMB_BIN_HALO 64          // bytes past the tile a walk may read: the type byte and 21 data tokens of 2 bytes
#define AMB_BIN_ESC 0x1a

// The stream position the next call starts at, and its first bytes.
struct AmbBinStream {
    unsigned long long base;     // stream offset of B[0] (bytes since create or reset)
    int clen, pad_;              // carried bytes
    uint8_t carry[48];
};

// Device-resident state of one reader: the two alternating stream positions, this call's carry start, and the totals.
struct AmbBinDev {
    AmbBinStream str[2];
    unsigned cs, pad_;           // this call: first carried byte of B (UINT_MAX until a kernel lowers it)
    unsigned long long modes, modeac, other, truncated, skipped, passed;
};

enum { AMB_BIN_COMPLETE = 0, AMB_BIN_TRUNCATED = 1, AMB_BIN_OPEN = 2 };

// Body tokens (rule 2) of the sync token at b[i] whose type asks for `need` of them, b[0 .. L) known: COMPLETE when
// `need` data tokens follow before any sync token, TRUNCATED when a sync token comes first, OPEN when the bytes end
// first (a final lone 0x1a included). *got: the data tokens read; out (when not NULL) receives their values.
AMB_HD int amb_bin_walk(const uint8_t* b, int i, int L, int need, uint8_t* out, int* got)
{
    int p = i + 2, k = 0;
    for (; k < need; k++) {
        if (p >= L) break;
        const uint8_t v = b[p];
        if (v == AMB_BIN_ESC) {
            if (p + 1 >= L) break;
            if (b[p + 1] != AMB_BIN_ESC) { *got = k; return AMB_BIN_TRUNCATED; }
            p += 2;
        } else {
            p += 1;
        }
        if (out) out[k] = v;
    }
    *got = k;
    return k == need ? AMB_BIN_COMPLETE : AMB_BIN_OPEN;
}

// modes_check_crc (modes_crc.cc:55-63) bit by bit: the same polynomial as the table of amb_modes_check_crc
AMB_HD uint32_t amb_bin_crc(const uint8_t* d, int len)
{
    uint32_t c = 0;
    for (int i = 0; i < len; i++) {
        c ^= (uint32_t)d[i] << 16;
        for (int k = 0; k < 8; k++) c = (c & 0x800000u) ? (c << 1) ^ 0xFFF409u : c << 1;
    }
    return c & 0xFFFFFFu;
}

// The frame of a complete Mode S message (rules 3 and 4) into *f, every byte written: body = T (6 bytes), S, then nb
// payload bytes.
AMB_HD void amb_bin_frame(const uint8_t* body, int nb, unsigned long long at, amb_frame* f)
{
    uint64_t T = 0;
    for (int k = 0; k < 6; k++) T = (T << 8) | body[k];
    const unsigned S = body[6];
    // the two divisions first: their slow path is a call, and little is live across it here
    f->frac = (double)(T % 12000000ull) / 12e6;
    f->ref_level = (float)((double)(S * S) / 65025.0);
    f->secs = T / 12000000ull;
    f->sample_index = at;
    const uint8_t* d = body + 7;
    unsigned any = 0;
    for (int k = 0; k < 14; k++) { const uint8_t v = k < nb ? d[k] : 0; f->data[k] = v; any |= v; }
    for (int k = 0; k < 24; k++) f->lowconfbits[k] = 0;
    f->ec = 0; f->ec_flips = 0;
    for (int k = 0; k < 4; k++) f->pad_[k] = 0;
    const int df = d[0] >> 3;
    const uint32_t crc = amb_bin_crc(d, nb - 3) ^ ((uint32_t)d[nb - 3] << 16 | (uint32_t)d[nb - 2] << 8 | d[nb - 1]);
    const int want = df == 16 || df == 17 || df == 20 || df == 21 ? 14 : 7;
    f->crc = crc;
    f->nbits = (uint8_t)(8 * nb);
    f->df = (uint8_t)df;
    f->numlowconf = 0;
    f->passed = any && nb == want && !(crc && (df == 11 || df == 17));
}

AMB_HD int amb_bin_tiles(int n) { return (n + AMB_BEAST_CARRY_MAX + AMB_BIN_TILE - 1) / AMB_BIN_TILE; }

__device__ __forceinline__ uint8_t amb_bin_at(const AmbBinStream& s, const uint8_t* in, int i)
{
    return i < s.clen ? s.carry[i] : in[i - s.clen];
}

__device__ __forceinline__ int amb_bin_max(int a, int b) { return a > b ? a : b; }

__global__ void __launch_bounds__(AMB_BIN_THREADS) amb_bin_last(const AmbBinDev* __restrict__ dv, int cur,
                                                              const uint8_t* __restrict__ in, int n, int* __restrict__ tlast)
{
    __shared__ int s_w[AMB_BIN_THREADS / 32];
    const AmbBinStream& s = dv->str[cur];
    const int L = s.clen + n, t0 = blockIdx.x * AMB_BIN_TILE;
    int m = -1;
    for (int k = threadIdx.x; k < AMB_BIN_TILE; k += AMB_BIN_THREADS)
        if (t0 + k < L && amb_bin_at(s, in, t0 + k) != AMB_BIN_ESC) m = t0 + k;
    for (int o = 16; o; o >>= 1) m = amb_bin_max(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = m;
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < AMB_BIN_THREADS / 32; w++) m = amb_bin_max(m, s_w[w]);
        tlast[blockIdx.x] = amb_bin_max(m, s_w[0]);
    }
}

// tprev[t] = max(-1, tlast[0 .. t)); also opens the call's carry start. One block of 1024 threads.
__global__ void __launch_bounds__(1024) amb_bin_scan(const int* __restrict__ tlast, int nt, int* __restrict__ tprev,
                                                     AmbBinDev* __restrict__ dv)
{
    __shared__ int s_w[32], s_carry;
    const unsigned t = threadIdx.x, lane = t & 31, warp = t >> 5;
    if (t == 0) { s_carry = -1; dv->cs = 0xFFFFFFFFu; }
    __syncthreads();
    for (int i0 = 0; i0 < nt; i0 += 1024) {
        const int i = i0 + (int)t;
        const int x = i < nt ? tlast[i] : -1;
        int v = x;
        for (int o = 1; o < 32; o <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, v, o);
            if (lane >= (unsigned)o) v = amb_bin_max(v, y);
        }
        if (lane == 31) s_w[warp] = v;
        __syncthreads();
        int before = s_carry;
        for (unsigned w = 0; w < warp; w++) before = amb_bin_max(before, s_w[w]);
        const int excl = __shfl_up_sync(0xffffffffu, v, 1);
        if (i < nt) tprev[i] = lane ? amb_bin_max(before, excl) : before;
        __syncthreads();
        if (t == 1023) s_carry = amb_bin_max(before, v);
        __syncthreads();
    }
}

// The tile and its halo into shared memory (0 past L); returns, for the calling thread, the position of the last byte
// before its first one that is not 0x1a (-1: the start of B, which counts as preceded by such a byte).
__device__ __forceinline__ int amb_bin_load(const AmbBinStream& s, const uint8_t* in, int L, int t0, int prev,
                                            uint8_t* sb, int* s_w)
{
    for (int k = threadIdx.x; k < AMB_BIN_TILE + AMB_BIN_HALO; k += AMB_BIN_THREADS)
        sb[k] = t0 + k < L ? amb_bin_at(s, in, t0 + k) : 0;
    __syncthreads();
    const int c0 = threadIdx.x * AMB_BIN_PER;
    int m = -1;
    for (int q = 0; q < AMB_BIN_PER; q++)
        if (t0 + c0 + q < L && sb[c0 + q] != AMB_BIN_ESC) m = t0 + c0 + q;
    const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int v = m;
    for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= (unsigned)o) v = amb_bin_max(v, y);
    }
    const int excl = __shfl_up_sync(0xffffffffu, v, 1);
    if (lane == 31) s_w[warp] = v;
    __syncthreads();
    int before = prev;
    for (unsigned w = 0; w < warp; w++) before = amb_bin_max(before, s_w[w]);
    return lane ? amb_bin_max(before, excl) : before;
}

__global__ void __launch_bounds__(AMB_BIN_THREADS) amb_bin_count(AmbBinDev* __restrict__ dv, int cur,
                                                               const uint8_t* __restrict__ in, int n, int flush,
                                                               const int* __restrict__ tprev, uint32_t* __restrict__ tfr)
{
    __shared__ uint8_t sb[AMB_BIN_TILE + AMB_BIN_HALO];
    __shared__ int s_w[AMB_BIN_THREADS / 32];
    __shared__ unsigned s_c[7];
    const AmbBinStream& s = dv->str[cur];
    const int L = s.clen + n, t0 = blockIdx.x * AMB_BIN_TILE;
    if (threadIdx.x < 7) s_c[threadIdx.x] = 0;
    int j = amb_bin_load(s, in, L, t0, tprev[blockIdx.x], sb, s_w);
    // data tokens, body tokens of Mode S / A/C messages (complete, truncated or open), Mode S, Mode A/C, other, truncated
    unsigned D = 0, used = 0, ms = 0, ac = 0, ot = 0, tr = 0;
    const int Lt = L - t0;
    for (int q = 0; q < AMB_BIN_PER; q++) {
        const int k = threadIdx.x * AMB_BIN_PER + q, i = t0 + k;
        if (i >= L) break;
        const uint8_t b = sb[k];
        const bool start = ((i - 1 - j) & 1) == 0;
        if (b != AMB_BIN_ESC) j = i;
        if (!start) continue;
        if (b != AMB_BIN_ESC) { D++; continue; }
        if (i + 1 >= L) {                                  // a lone final 0x1a: undecided, carried (dropped at flush)
            if (!flush) atomicMin(&dv->cs, (unsigned)i);
            continue;
        }
        const uint8_t ty = sb[k + 1];
        if (ty == AMB_BIN_ESC) { D++; continue; }
        const int need = ty == '1' ? 9 : ty == '2' ? 14 : ty == '3' ? 21 : 0;
        if (!need) { ot++; continue; }
        int got;
        const int o = amb_bin_walk(sb, k, Lt, need, nullptr, &got);
        used += (unsigned)got;
        if (o == AMB_BIN_COMPLETE) { if (need == 9) ac++; else ms++; }
        else if (o == AMB_BIN_TRUNCATED || flush) tr++;
        else atomicMin(&dv->cs, (unsigned)i);                 // still open at the end: carried from its sync byte
    }
    atomicAdd(&s_c[0], D); atomicAdd(&s_c[1], used); atomicAdd(&s_c[2], ms); atomicAdd(&s_c[3], ac);
    atomicAdd(&s_c[4], ot); atomicAdd(&s_c[5], tr);
    __syncthreads();
    if (threadIdx.x == 0) {
        tfr[blockIdx.x] = s_c[2];
        atomicAdd(&dv->skipped, (unsigned long long)((long long)s_c[0] - (long long)s_c[1]));
        atomicAdd(&dv->modes, (unsigned long long)s_c[2]);
        atomicAdd(&dv->modeac, (unsigned long long)s_c[3]);
        atomicAdd(&dv->other, (unsigned long long)s_c[4]);
        atomicAdd(&dv->truncated, (unsigned long long)s_c[5]);
    }
}

__global__ void __launch_bounds__(AMB_BIN_THREADS) amb_bin_emit(AmbBinDev* __restrict__ dv, int cur,
                                                              const uint8_t* __restrict__ in, int n, int flush,
                                                              const int* __restrict__ tprev,
                                                              const unsigned long long* __restrict__ toff,
                                                              amb_frame* __restrict__ frames)
{
    __shared__ uint8_t sb[AMB_BIN_TILE + AMB_BIN_HALO];
    __shared__ int s_w[AMB_BIN_THREADS / 32];
    __shared__ unsigned s_n[AMB_BIN_THREADS / 32], s_pass;
    __shared__ uint8_t s_body[AMB_BIN_THREADS][24];
    __shared__ __align__(16) amb_frame s_fr[AMB_BIN_THREADS];   // the block's frames in slot order, written out whole
    const AmbBinStream& s = dv->str[cur];
    const int L = s.clen + n, t0 = blockIdx.x * AMB_BIN_TILE;
    if (threadIdx.x == 0) s_pass = 0;
    int j = amb_bin_load(s, in, L, t0, tprev[blockIdx.x], sb, s_w);
    const int Lt = L - t0;
    // the complete Mode S messages starting in this thread's bytes (at most one), by tile offset
    int at = -1;
    for (int q = 0; q < AMB_BIN_PER; q++) {
        const int k = threadIdx.x * AMB_BIN_PER + q, i = t0 + k;
        if (i >= L) break;
        const uint8_t b = sb[k];
        const bool start = ((i - 1 - j) & 1) == 0;
        if (b != AMB_BIN_ESC) j = i;
        if (!start || b != AMB_BIN_ESC || i + 1 >= L) continue;
        const uint8_t ty = sb[k + 1];
        if (ty != '2' && ty != '3') continue;
        int got;
        if (amb_bin_walk(sb, k, Lt, ty == '3' ? 21 : 14, nullptr, &got) == AMB_BIN_COMPLETE) at = k;
    }
    const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned mine = __ballot_sync(0xffffffffu, at >= 0);
    if (lane == 0) s_n[warp] = __popc(mine);
    __syncthreads();
    if (at >= 0) {
        unsigned rank = __popc(mine & ((1u << lane) - 1u));
        for (unsigned w = 0; w < warp; w++) rank += s_n[w];
        uint8_t* body = s_body[threadIdx.x];
        int got;
        const int nb = sb[at + 1] == '3' ? 14 : 7;
        amb_bin_walk(sb, at, Lt, 7 + nb, body, &got);
        amb_bin_frame(body, nb, s.base + (unsigned long long)(t0 + at), &s_fr[rank]);
        if (s_fr[rank].passed) atomicAdd(&s_pass, 1u);
    }
    __syncthreads();
    // the block's slots are contiguous from toff[block]: 16-byte stores, coalesced, instead of each thread's narrow ones
    unsigned cnt = 0;
    for (unsigned w = 0; w < AMB_BIN_THREADS / 32; w++) cnt += s_n[w];
    uint4* dst = reinterpret_cast<uint4*>(frames + toff[blockIdx.x]);
    const uint4* src = reinterpret_cast<const uint4*>(s_fr);
    for (unsigned q = threadIdx.x; q < cnt * (sizeof(amb_frame) / 16); q += AMB_BIN_THREADS) dst[q] = src[q];
    if (threadIdx.x == 0 && s_pass) atomicAdd(&dv->passed, (unsigned long long)s_pass);
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        const unsigned cs = flush || dv->cs > (unsigned)L ? (unsigned)L : dv->cs;
        AmbBinStream& nx = dv->str[cur ^ 1];
        nx.base = s.base + cs;
        nx.clen = L - (int)cs;
        for (int k = 0; k < nx.clen; k++) nx.carry[k] = amb_bin_at(s, in, (int)cs + k);
    }
}

// Enqueue one call's five kernels over the n new bytes at `in` (device memory). Returns the launch count or -1 with *err.
static int amb_bin_launch(AmbBinDev* dv, int cur, const uint8_t* in, int n, int flush, int* tlast, int* tprev,
                          uint32_t* tfr, unsigned long long* toff, amb_frame* frames, cudaStream_t st, cudaError_t* err)
{
    const int nt = amb_bin_tiles(n);
    AMB_LAUNCH((amb_bin_last), nt, AMB_BIN_THREADS, 0, st, dv, cur, in, n, tlast);
    AMB_LAUNCH((amb_bin_scan), 1, 1024, 0, st, tlast, nt, tprev, dv);
    AMB_LAUNCH((amb_bin_count), nt, AMB_BIN_THREADS, 0, st, dv, cur, in, n, flush, tprev, tfr);
    AMB_LAUNCH((amb_sbs1_scan), 1, 1024, 0, st, tfr, nt, toff);
    AMB_LAUNCH((amb_bin_emit), nt, AMB_BIN_THREADS, 0, st, dv, cur, in, n, flush, tprev, toff, frames);
    *err = cudaGetLastError();
    return *err == cudaSuccess ? 5 : -1;
}
