/*
 * cuda_emu.h — TEST INFRASTRUCTURE.  A small CPU emulation of the CUDA execution model, just large
 * enough to run this repository's kernels (nhd_b200/csrc/nhd_kernels.cuh) and their host side
 * (nhd_api.cu) UNCHANGED on a machine without a GPU, so that the `-m "not gpu"` suite exercises the real
 * kernel logic: warp collectives, the multi-warp hand-off protocol of the sweep, shared-memory caches,
 * mbarrier-staged tiles.  Never part of the product; the product library is built by nvcc only.
 *
 * Model
 *   - every CUDA thread of a block is a fiber (ucontext); blocks of a grid run one after another;
 *   - a fiber runs until it reaches a warp collective (__shfl_sync, __ballot_sync, __all_sync,
 *     __syncwarp), __syncthreads, __nanosleep or an mbarrier wait, where it yields to a round-robin
 *     scheduler; a collective completes when every lane named in its mask has arrived at a collective of
 *     the SAME kind with the SAME mask — anything else (a lane of the mask that has exited, a different
 *     mask or kind: undefined behaviour on the GPU) aborts with a message;
 *   - memory is sequentially consistent (one OS thread), so fences are no-ops: the emulation checks the
 *     logic and the control-flow convergence rules, not the memory model;
 *   - cudaMalloc is calloc, copies are memcpy, streams and events do nothing, one device with 132 SMs (an H100 SXM);
 *   - mbarrier + cp.async.bulk (the TMA staging of filter_kernel) are emulated with a byte-counting
 *     phase barrier and a synchronous memcpy.
 */
#pragma once
#include <math.h>
#include <stddef.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <ucontext.h>

#include <functional>
#include <vector>

/* ------------------------------------------------------------------ language */
#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define EMU_NOINLINE __attribute__((noinline))     /* the build script rewrites __noinline__ (libstdc++ uses that spelling) */
#define __launch_bounds__(...)
#define __align__(n) __attribute__((aligned(n)))

struct alignas(16) uint4 { uint32_t x, y, z, w; };
struct alignas(8) uint2 { uint32_t x, y; };
struct alignas(16) ulonglong2 { unsigned long long x, y; };
static inline ulonglong2 make_ulonglong2(unsigned long long x, unsigned long long y) { ulonglong2 r = {x, y}; return r; }
static inline uint4 make_uint4(uint32_t x, uint32_t y, uint32_t z, uint32_t w) { uint4 r = {x, y, z, w}; return r; }
static inline uint2 make_uint2(uint32_t x, uint32_t y) { uint2 r = {x, y}; return r; }
struct dim3 {
    unsigned x, y, z;
    dim3(unsigned x_ = 1, unsigned y_ = 1, unsigned z_ = 1) : x(x_), y(y_), z(z_) {}
};

/* ------------------------------------------------------------------ runtime (host side) */
typedef int cudaError_t;
enum { cudaSuccess = 0, cudaErrorInvalidValue = 1 };
typedef void* cudaStream_t;
typedef void* cudaEvent_t;
enum cudaMemcpyKind { cudaMemcpyHostToHost, cudaMemcpyHostToDevice, cudaMemcpyDeviceToHost, cudaMemcpyDeviceToDevice, cudaMemcpyDefault };
enum { cudaStreamNonBlocking = 1, cudaHostAllocMapped = 2, cudaHostAllocDefault = 0 };
enum cudaFuncAttribute { cudaFuncAttributeMaxDynamicSharedMemorySize = 8 };
enum cudaMemoryType { cudaMemoryTypeUnregistered = 0, cudaMemoryTypeHost = 1, cudaMemoryTypeDevice = 2, cudaMemoryTypeManaged = 3 };
struct cudaPointerAttributes { cudaMemoryType type; int device; void* devicePointer; void* hostPointer; };
struct cudaDeviceProp {
    char name[256]; int multiProcessorCount; size_t sharedMemPerBlockOptin; size_t sharedMemPerBlock; int major, minor;
    size_t totalGlobalMem;
};

static inline cudaError_t cudaGetDeviceCount(int* n) { *n = 1; return cudaSuccess; }
static inline cudaError_t cudaSetDevice(int) { return cudaSuccess; }
static inline cudaError_t cudaGetDeviceProperties(cudaDeviceProp* p, int)
{
    memset(p, 0, sizeof(*p));
    snprintf(p->name, sizeof(p->name), "CPU emulation (tests/emu)");
    p->multiProcessorCount = 132; p->sharedMemPerBlockOptin = 227 * 1024; p->sharedMemPerBlock = 48 * 1024;
    p->major = 9; p->minor = 0; p->totalGlobalMem = (size_t)80 << 30;
    return cudaSuccess;
}
static inline const char* cudaGetErrorString(cudaError_t e) { return e == cudaSuccess ? "no error" : "emulated CUDA error"; }
static inline cudaError_t cudaGetLastError() { return cudaSuccess; }
/* device memory is NOT zero on allocation: EMU_POISON=1 fills it with 0xA5 to flush out code that assumes so */
static inline cudaError_t cudaMalloc(void** p, size_t n)
{
    *p = calloc(1, n ? n : 1);
    if (*p && getenv("EMU_POISON")) memset(*p, 0xA5, n);
    return *p ? cudaSuccess : cudaErrorInvalidValue;
}
static inline cudaError_t cudaFree(void* p) { free(p); return cudaSuccess; }
static inline cudaError_t cudaMallocHost(void** p, size_t n) { return cudaMalloc(p, n); }
static inline cudaError_t cudaHostAlloc(void** p, size_t n, unsigned) { return cudaMalloc(p, n); }
static inline cudaError_t cudaFreeHost(void* p) { free(p); return cudaSuccess; }
static inline cudaError_t cudaMemcpy(void* d, const void* s, size_t n, cudaMemcpyKind) { memmove(d, s, n); return cudaSuccess; }
static inline cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, cudaMemcpyKind, cudaStream_t = 0) { memmove(d, s, n); return cudaSuccess; }
static inline cudaError_t cudaMemset(void* d, int v, size_t n) { memset(d, v, n); return cudaSuccess; }
static inline cudaError_t cudaMemsetAsync(void* d, int v, size_t n, cudaStream_t = 0) { memset(d, v, n); return cudaSuccess; }
static inline cudaError_t cudaStreamCreateWithFlags(cudaStream_t* s, unsigned) { *s = (void*)1; return cudaSuccess; }
static inline cudaError_t cudaStreamDestroy(cudaStream_t) { return cudaSuccess; }
static inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
static inline cudaError_t cudaDeviceSynchronize() { return cudaSuccess; }
/* events carry the host's monotonic clock: work is synchronous here, so "elapsed" is the emulation's own run time
 * (never a statement about the GPU) */
#include <time.h>
static inline double emu_now_ms() { struct timespec t; clock_gettime(CLOCK_MONOTONIC, &t); return t.tv_sec * 1e3 + t.tv_nsec * 1e-6; }
static inline cudaError_t cudaEventCreate(cudaEvent_t* e) { *e = calloc(1, sizeof(double)); return cudaSuccess; }
static inline cudaError_t cudaEventDestroy(cudaEvent_t e) { free(e); return cudaSuccess; }
static inline cudaError_t cudaEventRecord(cudaEvent_t e, cudaStream_t = 0) { *(double*)e = emu_now_ms(); return cudaSuccess; }
static inline cudaError_t cudaEventSynchronize(cudaEvent_t) { return cudaSuccess; }
static inline cudaError_t cudaEventElapsedTime(float* ms, cudaEvent_t a, cudaEvent_t b) { *ms = (float)(*(double*)b - *(double*)a); return cudaSuccess; }
template <class F> static inline cudaError_t cudaFuncSetAttribute(F, cudaFuncAttribute, int) { return cudaSuccess; }
static inline cudaError_t cudaPointerGetAttributes(cudaPointerAttributes* a, const void*)
{
    memset(a, 0, sizeof(*a)); a->type = cudaMemoryTypeUnregistered; return cudaSuccess;
}

/* ------------------------------------------------------------------ the emulated block */
namespace emu {

enum { ST_RUN = 0, ST_COLL = 1, ST_SYNC = 2, ST_DONE = 3 };
enum { OP_SHFL = 1, OP_SHFL_UP, OP_BALLOT, OP_ALL, OP_SYNCWARP };

struct Fiber { ucontext_t ctx; int state; unsigned tid; int hist[12]; unsigned nhist; };   /* hist: lines of the last collectives */
struct Warp {
    uint32_t waiting, released;
    struct { int op; uint32_t mask; uint64_t val; int arg; int line; } slot[32];
    uint64_t result[32];
};

struct Block {
    std::vector<Fiber> fibers;
    std::vector<Warp> warps;
    std::vector<char> stacks;
    ucontext_t sched;
    int cur = -1, n = 0, live = 0, sync_waiting = 0, completed_warp = -1;
    unsigned sync_gen = 0;
    unsigned long long progress = 0;
    std::function<void()> body;
};

extern Block* g_blk;                 /* the block being executed */
extern const char* g_kernel_name;
extern size_t g_stack_bytes;

[[noreturn]] void fail(const char* fmt, ...);
void yield();
uint64_t collective(int op, uint32_t mask, uint64_t val, int arg, int line);
void syncthreads();
void run_grid(const char* name, dim3 grid, dim3 block, size_t dyn_smem, std::function<void()> body);

}  // namespace emu

extern dim3 threadIdx, blockIdx, blockDim, gridDim;
static const int warpSize = 32;

#define EMU_LAUNCH(kernel, grid, block, smem, stream, ...) \
    emu::run_grid(#kernel, dim3(grid), dim3(block), (size_t)(smem), [=]() { kernel(__VA_ARGS__); })

/* ------------------------------------------------------------------ device intrinsics */
template <class T> static inline T emu_from_bits(uint64_t b) { T v; memcpy(&v, &b, sizeof(T)); return v; }
template <class T> static inline uint64_t emu_to_bits(T v) { static_assert(sizeof(T) <= 8, "shuffle of > 8 bytes"); uint64_t b = 0; memcpy(&b, &v, sizeof(T)); return b; }

/* `line` = source line of the call (GCC evaluates __builtin_LINE() in a default argument at the call site) */
template <class T> static inline T __shfl_sync(unsigned mask, T v, int src, int width = 32, int line = __builtin_LINE())
{
    (void)width;
    return emu_from_bits<T>(emu::collective(emu::OP_SHFL, mask, emu_to_bits(v), src & 31, line));
}
template <class T> static inline T __shfl_up_sync(unsigned mask, T v, unsigned delta, int width = 32, int line = __builtin_LINE())
{
    (void)width;
    return emu_from_bits<T>(emu::collective(emu::OP_SHFL_UP, mask, emu_to_bits(v), (int)delta, line));
}
static inline unsigned __ballot_sync(unsigned mask, int pred, int line = __builtin_LINE()) { return (unsigned)emu::collective(emu::OP_BALLOT, mask, pred ? 1 : 0, 0, line); }
static inline int __all_sync(unsigned mask, int pred, int line = __builtin_LINE()) { return (int)emu::collective(emu::OP_ALL, mask, pred ? 1 : 0, 0, line); }
static inline int __any_sync(unsigned mask, int pred, int line = __builtin_LINE()) { return emu::collective(emu::OP_BALLOT, mask, pred ? 1 : 0, 0, line) != 0; }
static inline void __syncwarp(unsigned mask = 0xFFFFFFFFu, int line = __builtin_LINE()) { emu::collective(emu::OP_SYNCWARP, mask, 0, 0, line); }
static inline void __syncthreads() { emu::syncthreads(); }
static inline void __nanosleep(unsigned) { emu::yield(); }
static inline void __threadfence() { __asm__ volatile("" ::: "memory"); }
static inline void __threadfence_block() { __asm__ volatile("" ::: "memory"); }
static inline void __threadfence_system() { __asm__ volatile("" ::: "memory"); }
[[noreturn]] static inline void __trap() { emu::fail("__trap() in kernel %s", emu::g_kernel_name); }
static inline long long clock64() { return (long long)emu::g_blk->progress; }
template <class T> static inline T __ldcg(const T* p) { return *p; }
template <class T> static inline T __ldg(const T* p) { return *p; }
static inline int __popc(unsigned x) { return __builtin_popcount(x); }
static inline int __popcll(unsigned long long x) { return __builtin_popcountll(x); }
static inline int __ffs(int x) { return __builtin_ffs(x); }
static inline int __ffsll(long long x) { return __builtin_ffsll(x); }
static inline int __clz(int x) { return x ? __builtin_clz((unsigned)x) : 32; }
static inline int __clzll(long long x) { return x ? __builtin_clzll((unsigned long long)x) : 64; }
static inline unsigned __brev(unsigned x)
{
    x = ((x >> 1) & 0x55555555u) | ((x & 0x55555555u) << 1);
    x = ((x >> 2) & 0x33333333u) | ((x & 0x33333333u) << 2);
    x = ((x >> 4) & 0x0F0F0F0Fu) | ((x & 0x0F0F0F0Fu) << 4);
    return __builtin_bswap32(x);
}
static inline size_t __cvta_generic_to_shared(const void* p) { return (size_t)p; }

/* atomics: one OS thread, fibers switch only at yield points -> plain read-modify-write is atomic */
#define EMU_ATOMIC(NAME, EXPR)                                                                    \
    template <class T, class U> static inline T NAME(T* p, U v_) { T old = *p; T v = (T)v_; *p = (EXPR); return old; }
EMU_ATOMIC(atomicAdd, old + v)
EMU_ATOMIC(atomicOr, old | v)
EMU_ATOMIC(atomicAnd, old & v)
EMU_ATOMIC(atomicXor, old ^ v)
EMU_ATOMIC(atomicMax, old > v ? old : v)
EMU_ATOMIC(atomicMin, old < v ? old : v)
EMU_ATOMIC(atomicExch, v)
template <class T, class U, class V> static inline T atomicCAS(T* p, U cmp, V val) { T old = *p; if (old == (T)cmp) *p = (T)val; return old; }

/* mbarrier + 1-D bulk copy (filter_kernel's tile staging).  State word: bit 63 = phase, bits 48..62 = the
 * arrival count given to init, bits 32..47 = arrivals still expected in this phase, bits 0..31 = bytes of
 * bulk copies still in flight.  A phase completes when both counters reach zero. */
static inline void emu_mbar_settle(uint64_t* bar)
{
    uint64_t s = *bar;
    if (((s >> 32) & 0xFFFF) == 0 && (uint32_t)s == 0) {
        const uint64_t init = (s >> 48) & 0x7FFF;
        *bar = ((s ^ (1ull << 63)) & (1ull << 63)) | (init << 48) | (init << 32);
        emu::g_blk->progress++;
    }
}
static inline void emu_mbar_init(uint64_t* bar, uint32_t count) { *bar = ((uint64_t)count << 48) | ((uint64_t)count << 32); }
static inline void emu_mbar_expect_tx(uint64_t* bar, uint32_t bytes)
{
    uint64_t s = *bar;
    if (((s >> 32) & 0xFFFF) == 0) emu::fail("mbarrier: more arrivals than the barrier was initialised for");
    s -= 1ull << 32;                                        /* one arrival ...            */
    s = (s & ~0xFFFFFFFFull) | (uint32_t)((uint32_t)s + bytes);   /* ... expecting `bytes` more  */
    *bar = s;
    emu_mbar_settle(bar);
}
static inline void emu_tma_load_1d(void* dst, const void* src, uint32_t bytes, uint64_t* bar)
{
    if (((uintptr_t)dst | (uintptr_t)src | bytes) & 15) emu::fail("cp.async.bulk: address or size not a multiple of 16");
    memcpy(dst, src, bytes);
    uint64_t s = *bar;
    if ((uint32_t)s < bytes) emu::fail("cp.async.bulk: completes more bytes than the mbarrier expects");
    *bar = (s & ~0xFFFFFFFFull) | (uint32_t)((uint32_t)s - bytes);
    emu_mbar_settle(bar);
}
static inline void emu_mbar_wait(uint64_t* bar, uint32_t parity)
{
    while (((*(volatile uint64_t*)bar) >> 63) == (uint64_t)(parity & 1)) emu::yield();
}
