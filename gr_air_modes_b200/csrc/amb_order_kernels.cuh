// Device-side drain (amb_drain_device): the frames of the calls that are through, put into STREAM ORDER and STAMPED on
// the device, so that a consumer on the same GPU (amb_decode_frames_device) gets what amb_poll_frames would have handed
// to the host - without the frames crossing PCIe.
//
// The slicer writes a call's frames at frame_base + position in the work list; the work list is ascending inside a
// block of the resolver's second pass and the blocks come in arbitrary order (amb_kernels.cu, amb_walk_par2_kernel), so
// the buffer is a concatenation of sorted runs. Frame starts are unique sample indices: a plain bitonic network over
// (sample_index, slot) pairs puts them in order. n is a few thousand per 2^28 samples of ordinary traffic (ONE launch:
// the whole network runs in shared memory) and 2.4 x 10^5 on dense traffic (34 launches).
//
//   amb_order_keys_kernel    key[i] = frames[i].sample_index (i < n), all ones for the padding up to a power of two
//   amb_order_local_kernel   every compare-exchange stage with a partner distance below the tile, for sequence
//                            lengths k_lo .. k_hi, on a tile held in shared memory
//   amb_order_global_kernel  one stage with a partner distance >= the tile
//   amb_order_gather_kernel  out[i] = frames[val[i]], stamped: tag_to_timestamp (preamble_impl.cc:100-137) against the
//                            rx_time tag in force at the frame - the same expressions, in the same order, as stamp()
//                            in amb_api.cu (uint64 division, one IEEE double division, one addition: nothing the
//                            compiler could contract)
#pragma once

struct AmbTagDev { unsigned long long offset, secs; double frac; };

__global__ void __launch_bounds__(256) amb_order_keys_kernel(const amb_frame* __restrict__ frames, unsigned n, unsigned npad,
                                                             unsigned long long* __restrict__ key, unsigned* __restrict__ val)
{
    const unsigned i = blockIdx.x * 256u + threadIdx.x;
    if (i >= npad) return;
    key[i] = i < n ? (unsigned long long)frames[i].sample_index : ~0ull;
    val[i] = i;
}

// tile = elements per CTA (power of two, >= 2 * blockDim.x is not required: threads stride over the tile's pairs)
__global__ void __launch_bounds__(512) amb_order_local_kernel(unsigned long long* __restrict__ key, unsigned* __restrict__ val,
                                                              unsigned npad, unsigned tile, unsigned k_lo, unsigned k_hi)
{
    AMB_DYN_SMEM(unsigned long long, s_raw, 16);
    unsigned long long* s_key = s_raw;
    unsigned* s_val = reinterpret_cast<unsigned*>(s_raw + tile);
    const unsigned base = blockIdx.x * tile;
    for (unsigned t = threadIdx.x; t < tile; t += blockDim.x) {
        s_key[t] = base + t < npad ? key[base + t] : ~0ull;
        s_val[t] = base + t < npad ? val[base + t] : 0u;
    }
    __syncthreads();
    for (unsigned k = k_lo; k <= k_hi; k <<= 1) {
        for (unsigned j = (k >> 1) < (tile >> 1) ? (k >> 1) : (tile >> 1); j > 0; j >>= 1) {
            for (unsigned p = threadIdx.x; p < (tile >> 1); p += blockDim.x) {
                const unsigned i = ((p & ~(j - 1)) << 1) | (p & (j - 1));      // lower index of pair p at distance j
                const unsigned l = i | j;
                const bool up = ((base + i) & k) == 0;
                const unsigned long long a = s_key[i], b = s_key[l];
                if ((a > b) == up) {
                    s_key[i] = b; s_key[l] = a;
                    const unsigned va = s_val[i]; s_val[i] = s_val[l]; s_val[l] = va;
                }
            }
            __syncthreads();
        }
    }
    for (unsigned t = threadIdx.x; t < tile; t += blockDim.x)
        if (base + t < npad) { key[base + t] = s_key[t]; val[base + t] = s_val[t]; }
}

__global__ void __launch_bounds__(256) amb_order_global_kernel(unsigned long long* __restrict__ key, unsigned* __restrict__ val,
                                                               unsigned npad, unsigned k, unsigned j)
{
    const unsigned p = blockIdx.x * 256u + threadIdx.x;
    if (p >= (npad >> 1)) return;
    const unsigned i = ((p & ~(j - 1)) << 1) | (p & (j - 1));
    const unsigned l = i | j;
    const bool up = (i & k) == 0;
    const unsigned long long a = key[i], b = key[l];
    if ((a > b) == up) {
        key[i] = b; key[l] = a;
        const unsigned va = val[i]; val[i] = val[l]; val[l] = va;
    }
}

__global__ void __launch_bounds__(128) amb_order_gather_kernel(const amb_frame* __restrict__ frames, const unsigned* __restrict__ val,
                                                               unsigned n, amb_frame* __restrict__ out, unsigned long long rate,
                                                               unsigned long long t0_secs, double t0_frac,
                                                               const AmbTagDev* __restrict__ tags, int ntags)
{
    const unsigned i = blockIdx.x * 128u + threadIdx.x;
    if (i >= n) return;
    amb_frame f = frames[val[i]];
    unsigned long long off = 0, t_secs = t0_secs; double t_frac = t0_frac;
    for (int k = ntags; k-- > 0;)
        if (tags[k].offset <= f.sample_index) { off = tags[k].offset; t_secs = tags[k].secs; t_frac = tags[k].frac; break; }
    const unsigned long long cnt = f.sample_index - off;
    f.secs = t_secs + cnt / rate;
    f.frac = t_frac + (double)(cnt % rate) / (double)rate;
    if (f.frac > 1.0f) { f.frac -= 1.0f; f.secs += 1; }
    out[i] = f;
}

// The network alone on key/val (npad entries, a power of two), ascending by key, on stream s. Returns the number of
// kernels launched. Not static: the multilateration stage of the decoder's translation unit sorts with it too.
int amb_launch_bitonic(unsigned long long* key, unsigned* val, unsigned npad, unsigned tile, cudaStream_t s)
{
    int launches = 0;
    if (tile > npad) tile = npad;
    const unsigned tiles = npad / tile;
    const size_t smem = (size_t)tile * (sizeof(unsigned long long) + sizeof(unsigned));
    const unsigned lthreads = tile / 2 < 512 ? (tile / 2 < 32 ? 32 : tile / 2) : 512;
    if (npad > 1) {
        AMB_LAUNCH((amb_order_local_kernel), tiles, lthreads, smem, s, key, val, npad, tile, 2u, tile); launches++;
        for (unsigned k = tile << 1; k <= npad && k; k <<= 1) {
            for (unsigned j = k >> 1; j >= tile; j >>= 1) {
                AMB_LAUNCH((amb_order_global_kernel), (npad / 2 + 255) / 256, 256, 0, s, key, val, npad, k, j); launches++;
            }
            AMB_LAUNCH((amb_order_local_kernel), tiles, lthreads, smem, s, key, val, npad, tile, k, k); launches++;
        }
    }
    return launches;
}

// Enqueue keys -> network -> gather on stream s. key/val hold npad = next power of two >= n entries. Returns the number of
// kernels launched (for the launch counter).
static int amb_launch_order(const amb_frame* frames, unsigned n, unsigned npad, unsigned tile, unsigned long long* key, unsigned* val,
                            amb_frame* out, unsigned long long rate, unsigned long long t0_secs, double t0_frac,
                            const AmbTagDev* tags, int ntags, cudaStream_t s, cudaError_t* err)
{
    int launches = 0;
    AMB_LAUNCH((amb_order_keys_kernel), (npad + 255) / 256, 256, 0, s, frames, n, npad, key, val); launches++;
    launches += amb_launch_bitonic(key, val, npad, tile, s);
    AMB_LAUNCH((amb_order_gather_kernel), (n + 127) / 128, 128, 0, s, frames, val, n, out, rate, t0_secs, t0_frac, tags, ntags); launches++;
    *err = cudaGetLastError();
    return launches;
}
