// TEST INFRASTRUCTURE: host stand-ins for the slice of the CUDA runtime / driver API that this library's host code
// uses, so that amb_api.cu and amb_decode.cu can be compiled into a test-only emulated library (tests/simt/
// library_emul.cc). "Device" memory is host memory; streams and events are inert because an emulated kernel launch
// runs to completion inside AMB_LAUNCH (program order is one valid execution of the stream/event graph the real code
// builds). One emulated device: compute capability 9.0 with two SMs (grids are sized from the SM count).
#pragma once
#include <stdlib.h>
#include <string.h>

struct cudaDeviceProp { int major = 9, minor = 0, multiProcessorCount = 2; };
typedef void* cudaEvent_t;
enum { cudaStreamNonBlocking = 1, cudaEventDisableTiming = 2, cudaEnableDefault = 0 };
enum cudaMemcpyKind { cudaMemcpyHostToHost, cudaMemcpyHostToDevice, cudaMemcpyDeviceToHost, cudaMemcpyDeviceToDevice };
typedef int cudaDriverEntryPointQueryResult;

static inline cudaError_t cudaGetDeviceCount(int* n) { *n = 1; return cudaSuccess; }
static inline cudaError_t cudaGetDeviceProperties(cudaDeviceProp* p, int) { *p = cudaDeviceProp(); return cudaSuccess; }
static inline cudaError_t cudaSetDevice(int) { return cudaSuccess; }
static inline const char* cudaGetErrorString(cudaError_t) { return "emulated CUDA error"; }
static inline cudaError_t cudaStreamCreateWithFlags(cudaStream_t* s, unsigned) { *s = malloc(1); return cudaSuccess; }
static inline cudaError_t cudaStreamDestroy(cudaStream_t s) { free(s); return cudaSuccess; }
static inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
static inline cudaError_t cudaStreamWaitEvent(cudaStream_t, cudaEvent_t, unsigned) { return cudaSuccess; }
static inline cudaError_t cudaEventCreate(cudaEvent_t* e) { *e = malloc(1); return cudaSuccess; }
static inline cudaError_t cudaEventCreateWithFlags(cudaEvent_t* e, unsigned) { *e = malloc(1); return cudaSuccess; }
static inline cudaError_t cudaEventDestroy(cudaEvent_t e) { free(e); return cudaSuccess; }
static inline cudaError_t cudaEventRecord(cudaEvent_t, cudaStream_t) { return cudaSuccess; }
static inline cudaError_t cudaEventElapsedTime(float* ms, cudaEvent_t, cudaEvent_t) { *ms = 0.f; return cudaSuccess; }
template <typename T> static inline cudaError_t cudaMalloc(T** p, size_t n)
{
    void* q = nullptr;
    if (posix_memalign(&q, 1024, n ? n : 1) != 0) return 2;
    *p = static_cast<T*>(q);
    return cudaSuccess;
}
static inline cudaError_t cudaFree(void* p) { free(p); return cudaSuccess; }
static inline cudaError_t cudaMemcpy(void* d, const void* s, size_t n, cudaMemcpyKind) { memmove(d, s, n); return cudaSuccess; }
static inline cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, cudaMemcpyKind, cudaStream_t) { memmove(d, s, n); return cudaSuccess; }
static inline cudaError_t cudaMemset(void* p, int v, size_t n) { memset(p, v, n); return cudaSuccess; }
template <typename T> static inline cudaError_t cudaMallocHost(T** p, size_t n) { return cudaMalloc(p, n); }
static inline cudaError_t cudaFreeHost(void* p) { free(p); return cudaSuccess; }
static inline cudaError_t cudaEventSynchronize(cudaEvent_t) { return cudaSuccess; }
static inline cudaError_t cudaEventQuery(cudaEvent_t) { return cudaSuccess; }
enum { cudaErrorNotReady = 600 };
enum cudaMemoryType { cudaMemoryTypeUnregistered = 0, cudaMemoryTypeHost = 1, cudaMemoryTypeDevice = 2 };
struct cudaPointerAttributes { cudaMemoryType type = cudaMemoryTypeUnregistered; };
static inline cudaError_t cudaPointerGetAttributes(cudaPointerAttributes* a, const void*) { *a = cudaPointerAttributes(); return cudaSuccess; }

// driver API: only cuTensorMapEncodeTiled, reached through cudaGetDriverEntryPoint (amb_api.cu make_tmap)
typedef int CUresult;
enum { CUDA_SUCCESS = 0 };
typedef unsigned long long cuuint64_t;
typedef unsigned int cuuint32_t;
enum CUtensorMapDataType { CU_TENSOR_MAP_DATA_TYPE_FLOAT32 = 7 };
enum CUtensorMapInterleave { CU_TENSOR_MAP_INTERLEAVE_NONE = 0 };
enum CUtensorMapSwizzle { CU_TENSOR_MAP_SWIZZLE_128B = 3 };
enum CUtensorMapL2promotion { CU_TENSOR_MAP_L2_PROMOTION_L2_256B = 3 };
enum CUtensorMapFloatOOBfill { CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE = 0 };
static CUresult simt_encode_tiled(CUtensorMap* m, CUtensorMapDataType dt, cuuint32_t rank, void* base, const cuuint64_t* dims,
                                  const cuuint64_t* strides, const cuuint32_t* box, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle sw, CUtensorMapL2promotion, CUtensorMapFloatOOBfill)
{
    // the one layout the scan kernel uses: 2-D float32, lines of 128 B, box {32 floats, 32 lines}, 128-byte swizzle
    if (dt != CU_TENSOR_MAP_DATA_TYPE_FLOAT32 || rank != 2 || dims[0] != 32 || strides[0] != 128 || box[0] != 32 || box[1] != 32 ||
        sw != CU_TENSOR_MAP_SWIZZLE_128B || ((uintptr_t)base & 15u)) return 1;
    simt_make_tmap(m, base, (size_t)dims[1] * 16);
    return CUDA_SUCCESS;
}
static inline cudaError_t cudaGetDriverEntryPoint(const char* name, void** fn, int, cudaDriverEntryPointQueryResult* qr)
{
    *fn = strcmp(name, "cuTensorMapEncodeTiled") == 0 ? (void*)&simt_encode_tiled : nullptr;
    if (qr) *qr = 0;
    return *fn ? cudaSuccess : 2;
}
