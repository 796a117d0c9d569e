// TEST INFRASTRUCTURE: a small SIMT emulator, enough to run launch-free CUDA kernel headers of this repo on the host.
//
// One kernel launch = blocks run one after the other; the threads of a block are cooperative fibers (ucontext) on one
// OS thread. A fiber runs until it reaches a warp- or block-level collective (__syncthreads, __syncwarp, shuffles,
// votes, match), parks there until every participant has arrived, then continues - i.e. the barrier semantics CUDA
// guarantees, none of its accidental lockstep. `__shared__` becomes a function-local static (one block at a time).
// Supported: full-mask warp collectives with all 32 lanes alive, 1-D grids/blocks (blockDim.x a multiple of 32),
// atomicAdd on unsigned, __ldg/__ldcg/__stcg, bit intrinsics. A launch whose fibers all wait without progress is
// reported as a deadlock (that is how a divergent collective would show up).
#pragma once
#undef _FORTIFY_SOURCE       // fibers switch stacks with _longjmp; the fortified longjmp refuses that (include this header first)
#include <math.h>
#include <stdint.h>
#include <stddef.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <setjmp.h>
#include <ucontext.h>

#include <functional>
#include <utility>
#include <vector>

struct simt_dim3 { unsigned x = 1, y = 1, z = 1; };
struct uint4 { unsigned x, y, z, w; };
static inline uint4 make_uint4(unsigned x, unsigned y, unsigned z, unsigned w) { uint4 v = {x, y, z, w}; return v; }

struct SimtWarp { unsigned arrived = 0, gen = 0, alive = 32; uint64_t slot[32]; unsigned pred[32]; };
struct SimtFiber { ucontext_t ctx; jmp_buf jb; char* stack = nullptr; bool done = false, started = false; simt_dim3 tid; SimtWarp* warp = nullptr; };
struct SimtBlockBar { unsigned arrived = 0, gen = 0, n = 0; };

static ucontext_t simt_sched_ctx;
static jmp_buf simt_sched_jb;
static SimtFiber* simt_cur = nullptr;
static SimtBlockBar simt_block_bar;
static simt_dim3 simt_block_idx, simt_block_dim, simt_grid_dim;
static unsigned long simt_progress = 0;
static std::function<void()> simt_body;
static unsigned long long simt_shuffle_state = [] { const char* e = getenv("SIMT_SHUFFLE"); return e ? strtoull(e, nullptr, 10) * 2 + 1 : 0ull; }();

#define threadIdx (simt_cur->tid)
#define blockIdx simt_block_idx
#define blockDim simt_block_dim
#define gridDim simt_grid_dim
#define __global__ static
#define __device__
#define __host__
#define __forceinline__ inline
#define __restrict__
#define __launch_bounds__(...)
#define __maxnreg__(...)
#define __shared__ static
#define AMB_SIMT_EMUL 1

// switching is _setjmp/_longjmp once a fiber runs (swapcontext costs two sigprocmask system calls per switch)
// every harness is one translation unit, so this is exported once per test library
extern "C" void simt_set_shuffle(unsigned long long seed) { simt_shuffle_state = seed ? seed * 2 + 1 : 0; }

// (-DSIMT_SWAPCONTEXT: plain swapcontext everywhere, for builds with -fsanitize=address, which tracks swapcontext)
#ifdef SIMT_SWAPCONTEXT
static inline void simt_yield() { swapcontext(&simt_cur->ctx, &simt_sched_ctx); }
#else
static inline void simt_yield() { if (!_setjmp(simt_cur->jb)) _longjmp(simt_sched_jb, 1); }
#endif

// every lane of the warp deposits (value, pred), waits for the other 31, then reads; a second rendezvous frees the slots
static inline void simt_warp_exchange(uint64_t value, unsigned pred, uint64_t* vals, unsigned* preds)
{
    SimtWarp* w = simt_cur->warp;
    const unsigned lane = simt_cur->tid.x & 31;
    w->slot[lane] = value; w->pred[lane] = pred;
    unsigned g = w->gen;
    simt_progress++;                                        // an arrival is progress; a parked fiber that stays parked is not
    if (++w->arrived == w->alive) { w->arrived = 0; w->gen++; } else while (w->gen == g) simt_yield();
    for (int i = 0; i < 32; i++) { vals[i] = w->slot[i]; preds[i] = w->pred[i]; }
    g = w->gen;
    simt_progress++;
    if (++w->arrived == w->alive) { w->arrived = 0; w->gen++; } else while (w->gen == g) simt_yield();
}

static inline void __syncwarp(unsigned = 0xffffffffu) { uint64_t v[32]; unsigned p[32]; simt_warp_exchange(0, 0, v, p); }
static inline void __syncthreads()
{
    SimtBlockBar* b = &simt_block_bar;
    const unsigned g = b->gen;
    simt_progress++;
    if (++b->arrived == b->n) { b->arrived = 0; b->gen++; } else while (b->gen == g) simt_yield();
}
static inline void __threadfence_block() {}
static inline unsigned __ballot_sync(unsigned, int pred)
{
    uint64_t v[32]; unsigned p[32]; simt_warp_exchange(0, pred ? 1u : 0u, v, p);
    unsigned m = 0; for (int i = 0; i < 32; i++) m |= (p[i] ? 1u : 0u) << i; return m;
}
static inline int __any_sync(unsigned mask, int pred) { return __ballot_sync(mask, pred) != 0; }
static inline unsigned __match_any_sync(unsigned, unsigned value)
{
    uint64_t v[32]; unsigned p[32]; simt_warp_exchange(value, 0, v, p);
    unsigned m = 0; for (int i = 0; i < 32; i++) m |= (v[i] == (uint64_t)value ? 1u : 0u) << i; return m;
}
template <typename T> static inline T __shfl_sync(unsigned, T var, int src)
{
    static_assert(sizeof(T) <= 8, "shuffle of at most 8 bytes");
    uint64_t bits = 0; memcpy(&bits, &var, sizeof(T));
    uint64_t v[32]; unsigned p[32]; simt_warp_exchange(bits, 0, v, p);
    T out; memcpy(&out, &v[src & 31], sizeof(T)); return out;
}
template <typename T> static inline T __shfl_up_sync(unsigned, T var, unsigned delta)
{
    uint64_t bits = 0; memcpy(&bits, &var, sizeof(T));
    uint64_t v[32]; unsigned p[32]; simt_warp_exchange(bits, 0, v, p);
    const unsigned lane = simt_cur->tid.x & 31;
    T out; memcpy(&out, &v[lane >= delta ? lane - delta : lane], sizeof(T)); return out;
}
static inline unsigned atomicAdd(unsigned* p, unsigned v) { const unsigned o = *p; *p = o + v; return o; }   // fibers never preempt
template <typename T> static inline T __ldg(const T* p) { return *p; }
template <typename T> static inline T __ldcg(const T* p) { return *p; }
template <typename T> static inline void __stcg(T* p, T v) { *p = v; }
static inline int __popc(unsigned x) { return __builtin_popcount(x); }
static inline int __clz(unsigned x) { return x ? __builtin_clz(x) : 32; }
static inline int __ffs(unsigned x) { return __builtin_ffs((int)x); }
static inline double __hiloint2double(int hi, int lo)
{
    const uint64_t b = ((uint64_t)(unsigned)hi << 32) | (unsigned)lo; double d; memcpy(&d, &b, 8); return d;
}
static inline int __double2loint(double d) { uint64_t b; memcpy(&b, &d, 8); return (int)(unsigned)(b & 0xffffffffu); }
static inline int __double2hiint(double d) { uint64_t b; memcpy(&b, &d, 8); return (int)(unsigned)(b >> 32); }


// ---- vector types, runtime stand-ins, launch macros (amb_internal.h skips the CUDA headers under AMB_SIMT_EMUL) ----
struct float2 { float x, y; };
struct short2 { short x, y; };
struct double2 { double x, y; };
static inline float2 make_float2(float x, float y) { float2 v = {x, y}; return v; }
static inline double2 make_double2(double x, double y) { double2 v = {x, y}; return v; }
typedef int cudaError_t;
typedef void* cudaStream_t;
enum { cudaSuccess = 0, cudaErrorInvalidValue = 1, cudaFuncAttributeMaxDynamicSharedMemorySize = 8 };
struct CUtensorMap { alignas(64) unsigned long long opaque[16]; };
#define __constant__ static
#define __grid_constant__
#define __align__(n) __attribute__((aligned(n)))
#define cudaGetLastError() (cudaSuccess)
#define cudaFuncSetAttribute(...) (cudaSuccess)
#define cudaFuncAttributePreferredSharedMemoryCarveout 0
#define cudaMemcpyToSymbol(sym, src, n) (memcpy((void*)&(sym), (src), (n)), cudaSuccess)

static unsigned char* simt_dyn_smem = nullptr;       // dynamic shared memory of the running block
#define AMB_ID(...) __VA_ARGS__
#define AMB_DYN_SMEM(type, name, align) type* name = reinterpret_cast<type*>(simt_dyn_smem)
// every AMB_LAUNCH is counted: the library's kernel_launches statistic must equal simt_launch_count()'s growth
static unsigned long long simt_launches = 0;
extern "C" unsigned long long simt_launch_count() { return simt_launches; }
#define AMB_LAUNCH(kernel, grid, block, smem, stream, ...) \
    (simt_launches++, simt_launch_dyn((unsigned)(grid), (unsigned)(block), (size_t)(smem), [&] { AMB_ID kernel(__VA_ARGS__); }))

template <typename T> static inline T min(T a, T b) { return b < a ? b : a; }
template <typename T> static inline T max(T a, T b) { return a < b ? b : a; }
template <typename T> static inline T __shfl_xor_sync(unsigned, T var, int lanemask)
{
    uint64_t bits = 0; memcpy(&bits, &var, sizeof(T));
    uint64_t v[32]; unsigned p[32]; simt_warp_exchange(bits, 0, v, p);
    T out; memcpy(&out, &v[((simt_cur->tid.x & 31) ^ lanemask) & 31], sizeof(T)); return out;
}
static inline unsigned __reduce_max_sync(unsigned, unsigned x)
{
    uint64_t v[32]; unsigned p[32]; simt_warp_exchange(x, 0, v, p);
    unsigned m = 0; for (int i = 0; i < 32; i++) m = (unsigned)v[i] > m ? (unsigned)v[i] : m; return m;
}
static inline unsigned __reduce_min_sync(unsigned, unsigned x)
{
    uint64_t v[32]; unsigned p[32]; simt_warp_exchange(x, 0, v, p);
    unsigned m = 0xffffffffu; for (int i = 0; i < 32; i++) m = (unsigned)v[i] < m ? (unsigned)v[i] : m; return m;
}
static inline unsigned __brev(unsigned x) { unsigned r = 0; for (int i = 0; i < 32; i++) r |= ((x >> i) & 1u) << (31 - i); return r; }
// n-th set bit of mask counting upward from `base` (fns.b32 with a positive offset; the bit at base counts)
static inline unsigned __fns(unsigned mask, unsigned base, int offset)
{
    if (offset == 0) return ((mask >> base) & 1u) ? base : 0xffffffffu;
    if (offset > 0) { for (unsigned i = base; i < 32; i++) if ((mask >> i) & 1u) { if (--offset == 0) return i; } }
    else { for (int i = (int)base; i >= 0; i--) if ((mask >> i) & 1u) { if (++offset == 0) return (unsigned)i; } }
    return 0xffffffffu;
}
static inline float __fadd_rn(float a, float b) { volatile float r = a + b; return r; }
static inline float __fsub_rn(float a, float b) { volatile float r = a - b; return r; }
static inline float __fmul_rn(float a, float b) { volatile float r = a * b; return r; }
static inline float __fdiv_rn(float a, float b) { volatile float r = a / b; return r; }
static inline int __float2int_rz(float a) { return (int)a; }
static inline unsigned __float_as_uint(float f) { unsigned u; memcpy(&u, &f, 4); return u; }
static inline unsigned atomicOr(unsigned* p, unsigned v) { const unsigned o = *p; *p = o | v; return o; }
static inline unsigned long long atomicAdd(unsigned long long* p, unsigned long long v) { const unsigned long long o = *p; *p = o + v; return o; }
static inline unsigned long long atomicMax(unsigned long long* p, unsigned long long v) { const unsigned long long o = *p; if (v > o) *p = v; return o; }
static inline unsigned long long atomicMin(unsigned long long* p, unsigned long long v) { const unsigned long long o = *p; if (v < o) *p = v; return o; }
static inline unsigned atomicMax(unsigned* p, unsigned v) { const unsigned o = *p; if (v > o) *p = v; return o; }
static inline unsigned atomicMin(unsigned* p, unsigned v) { const unsigned o = *p; if (v < o) *p = v; return o; }

// ---- stand-ins for the six PTX helpers of amb_kernels.cu (mbarrier + TMA tile copy) -------------------------------
// Shared-memory "addresses" are byte offsets into the block's dynamic shared memory. An mbarrier is a counter of
// completed phases; the tile copy happens at issue time and completes the phase (complete_tx), a waiter that finds
// the phase incomplete yields. The copy lands with the 128-byte swizzle of CU_TENSOR_MAP_SWIZZLE_128B (16-byte chunk
// index ^= line index mod 8) and zero-fills lines beyond the tensor, like the hardware. The emulated CUtensorMap
// holds {base pointer, number of 128-byte lines} in opaque[0..1] (see simt_make_tmap).
struct float4 { float x, y, z, w; };
static inline float4 make_float4(float x, float y, float z, float w) { float4 v = {x, y, z, w}; return v; }
static inline void simt_make_tmap(CUtensorMap* m, const void* base, size_t n_samples)
{
    memset(m, 0, sizeof *m);
    m->opaque[0] = (unsigned long long)(uintptr_t)base; m->opaque[1] = (unsigned long long)(n_samples / 16);
}
static inline uint32_t smem_u32(const void* p) { return (uint32_t)((const unsigned char*)p - simt_dyn_smem); }
static inline void mbar_init(uint32_t bar, uint32_t) { *reinterpret_cast<uint64_t*>(simt_dyn_smem + bar) = 0; }
static inline void mbar_expect_tx(uint32_t, uint32_t) {}
static inline bool mbar_try_wait(uint32_t bar, uint32_t parity)
{
    if (((*reinterpret_cast<uint64_t*>(simt_dyn_smem + bar)) & 1u) != parity) return true;
    simt_yield();
    return false;
}
static inline void tma_tile_g2s(uint32_t dst, const void* tmap, int c0, int c1, uint32_t bar)
{
    const CUtensorMap* m = static_cast<const CUtensorMap*>(tmap);
    const unsigned char* base = reinterpret_cast<const unsigned char*>((uintptr_t)m->opaque[0]);
    const long long n_lines = (long long)m->opaque[1];
    if (c0 != 0 || (dst & 1023u)) { fprintf(stderr, "simt: unsupported TMA box\n"); abort(); }
    for (int l = 0; l < 32; l++)
        for (int c = 0; c < 8; c++) {
            unsigned char* d = simt_dyn_smem + dst + l * 128 + ((c ^ (l & 7)) << 4);
            const long long line = (long long)c1 + l;
            if (line >= 0 && line < n_lines) memcpy(d, base + line * 128 + c * 16, 16); else memset(d, 0, 16);
        }
    (*reinterpret_cast<uint64_t*>(simt_dyn_smem + bar))++;
    simt_progress++;
}
static inline bool elect_one() { return (simt_cur->tid.x & 31) == 0; }
static inline void fence_mbar_init() {}

// A thread that has exited no longer takes part in barriers (CUDA semantics for __syncthreads and *_sync with exited lanes)
static void simt_trampoline()
{
    simt_body();
    simt_cur->done = true; simt_progress++;
    SimtWarp* w = simt_cur->warp;
    if (--w->alive && w->arrived == w->alive) { w->arrived = 0; w->gen++; }
    SimtBlockBar* b = &simt_block_bar;
    if (--b->n && b->arrived == b->n) { b->arrived = 0; b->gen++; }
#ifdef SIMT_SWAPCONTEXT
    swapcontext(&simt_cur->ctx, &simt_sched_ctx);
#else
    _longjmp(simt_sched_jb, 1);
#endif
}

// simt_launch(grid, block, [&]{ kernel(args...); })
static inline void simt_launch(unsigned grid, unsigned block, const std::function<void()>& body)
{
    if (block % 32 != 0) { fprintf(stderr, "simt: block size must be a multiple of 32\n"); abort(); }
    simt_body = body;
    simt_grid_dim.x = grid; simt_block_dim.x = block;
    const size_t stack_bytes = 256 * 1024;
    std::vector<SimtFiber> fibers(block);
    std::vector<SimtWarp> warps(block / 32);
    static std::vector<char*> stack_pool;                  // fiber stacks are reused by every later launch
    while (stack_pool.size() < block) stack_pool.push_back((char*)malloc(stack_bytes));
    for (unsigned t = 0; t < block; t++) fibers[t].stack = stack_pool[t];
    for (unsigned b = 0; b < grid; b++) {
        simt_block_idx.x = b;
        simt_block_bar = SimtBlockBar(); simt_block_bar.n = block;
        for (auto& w : warps) w = SimtWarp();
        for (unsigned t = 0; t < block; t++) {
            SimtFiber& f = fibers[t];
            f.done = false; f.started = false; f.tid.x = t; f.warp = &warps[t / 32];
            getcontext(&f.ctx);
            f.ctx.uc_stack.ss_sp = f.stack; f.ctx.uc_stack.ss_size = stack_bytes; f.ctx.uc_link = &simt_sched_ctx;
            makecontext(&f.ctx, simt_trampoline, 0);
        }
        unsigned alive = block;
        std::vector<unsigned> order(block);
        for (unsigned t = 0; t < block; t++) order[t] = t;
        while (alive) {
            const unsigned long before = simt_progress;
            alive = 0;
            if (simt_shuffle_state) {                       // SIMT_SHUFFLE=<seed>: a different thread interleaving every round
                for (unsigned i = block - 1; i > 0; i--) {  // (a kernel that is missing a barrier stops getting away with it)
                    simt_shuffle_state = simt_shuffle_state * 6364136223846793005ull + 1442695040888963407ull;
                    std::swap(order[i], order[(unsigned)((simt_shuffle_state >> 33) % (i + 1))]);
                }
            }
            for (unsigned oi = 0; oi < block; oi++) {
                const unsigned t = order[oi];
                if (fibers[t].done) continue;
                simt_cur = &fibers[t];
#ifdef SIMT_SWAPCONTEXT
                swapcontext(&simt_sched_ctx, &fibers[t].ctx);
#else
                if (!_setjmp(simt_sched_jb)) {
                    if (fibers[t].started) _longjmp(fibers[t].jb, 1);
                    fibers[t].started = true;
                    setcontext(&fibers[t].ctx);             // first entry: onto the fiber's own stack
                }
#endif
                if (!fibers[t].done) alive++;
            }
            if (alive && simt_progress == before) {
                fprintf(stderr, "simt: deadlock in block %u (%u threads wait at a collective that not all reach)\n", b, alive);
                abort();
            }
        }
    }
    simt_cur = nullptr;
}

// launch with `smem` bytes of dynamic shared memory (AMB_LAUNCH)
static inline void simt_launch_dyn(unsigned grid, unsigned block, size_t smem, const std::function<void()>& body)
{
    if (block % 32 != 0) {                              // e.g. <<<1, 1>>>: pad the block with lanes that exit at once
        const unsigned padded = (block + 31) / 32 * 32;
        simt_launch_dyn(grid, padded, smem, [&] { if (threadIdx.x < block) body(); });
        return;
    }
    unsigned char* buf = nullptr;
    if (posix_memalign((void**)&buf, 1024, smem ? smem : 1024) != 0) abort();
    simt_dyn_smem = buf;
    simt_launch(grid, block, body);
    simt_dyn_smem = nullptr;
    free(buf);
}

static inline cudaError_t cudaMemsetAsync(void* p, int v, size_t n, cudaStream_t) { memset(p, v, n); return cudaSuccess; }
#include "simt_cudart.h"
