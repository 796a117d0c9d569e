// CUDA headers + the two macros through which every kernel launch and every dynamic shared memory declaration of this
// library goes. For nvcc they expand to the usual syntax (the library's SASS is byte-identical with and without them);
// tests/simt defines AMB_SIMT_EMUL and supplies host versions, which is how the CPU test tier runs the kernel source
// and the host orchestration under a SIMT emulator. Then the host helpers of the library's three C ABI objects
// (amb_ctx, amb_decoder, amb_mlat): the last-error text and the device check.
#pragma once
#ifndef AMB_SIMT_EMUL
#include <cuda.h>
#include <cuda_runtime.h>
#define AMB_ID(...) __VA_ARGS__
#define AMB_LAUNCH(kernel, grid, block, smem, stream, ...) AMB_ID kernel<<<(grid), (block), (smem), (stream)>>>(__VA_ARGS__)
#define AMB_DYN_SMEM(type, name, align) extern __shared__ __align__(align) type name[]
#endif
#include <stdio.h>
#include "../../include/airmodes_b200.h"

// Record what failed, and the CUDA error when there is one, as the last error of o (nothing when o is NULL); returns code.
template <typename T> static int fail(T* o, int code, const char* what, cudaError_t e = cudaSuccess)
{
    if (o) {
        char buf[256];
        if (e != cudaSuccess) snprintf(buf, sizeof buf, "%s: %s", what, cudaGetErrorString(e));
        else snprintf(buf, sizeof buf, "%s", what);
        o->err = buf;
    }
    return code;
}
#define CK(o, call)                                                                \
    do { cudaError_t e_ = (call); if (e_ != cudaSuccess) return fail((o), AMB_ERR_CUDA, #call, e_); } while (0)

// AMB_OK, with the device's properties in *prop, when `device` exists and has compute capability 9.0 (the library
// holds sm_90a code only; there is no CPU path); AMB_ERR_NO_DEVICE otherwise.
static inline int amb_check_device(int device, cudaDeviceProp* prop)
{
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0 || device < 0 || device >= ndev) return AMB_ERR_NO_DEVICE;
    if (cudaGetDeviceProperties(prop, device) != cudaSuccess) return AMB_ERR_NO_DEVICE;
    return prop->major == 9 && prop->minor == 0 ? AMB_OK : AMB_ERR_NO_DEVICE;
}
