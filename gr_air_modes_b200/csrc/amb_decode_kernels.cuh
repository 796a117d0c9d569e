// The kernels of the batch field decoder (SURVEY.md 8 row f4): amb_fields_kernel and amb_resolve_kernel here, the CPR
// pairing stage between them in amb_decode_v3.cuh. The host orchestration and the C ABI are in amb_decode.cu, the
// per-message arithmetic in amb_decode_core.h. Kept in headers without any <<< >>> launch so that tests/simt/ can
// compile the very same kernel source for the host under a small SIMT emulator (CPU-side check of the warp-level logic;
// the GPU tests remain the parity gate).
#pragma once
#include "amb_decode_core.h"

#define AMB_TABLE_SLOTS (1ull << 26)     // (24-bit ICAO, surface, even/odd)

struct AmbCprSlot { uint32_t lat, lon; double t; };   // lat == 0xFFFFFFFF: empty

// ---- kernels ------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) amb_fields_kernel(const amb_frame* __restrict__ frames, int n,
                                                         amb_fields* __restrict__ fields, AmbPosRec* __restrict__ pos,
                                                         AmbPair* __restrict__ pair)
{
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    amb_fields r; AmbPosRec p;
    amb_decode_fields(frames[k], &r, &p);
    fields[k] = r;
    pos[k] = p;
    AmbPair z; z.elat = z.elon = z.olat = z.olon = 0; z.have = 0; z.mostrecent = 0;
    pair[k] = z;
}

__global__ void __launch_bounds__(128) amb_resolve_kernel(amb_fields* __restrict__ fields, const AmbPosRec* __restrict__ pos,
                                                          const AmbPair* __restrict__ pair, int n, int have_loc,
                                                          double mylat, double mylon, const double* __restrict__ nl_T)
{
    __shared__ double T[AMB_NL_MAX];
    for (int i = threadIdx.x; i < AMB_NL_MAX; i += blockDim.x) T[i] = nl_T[i];
    __syncthreads();
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    if (pos[k].key == AMB_NO_KEY) return;
    amb_fields r = fields[k];
    amb_resolve_position(&r, pair[k], have_loc, mylat, mylon, T);
    fields[k] = r;
}

#include "amb_decode_v3.cuh"
