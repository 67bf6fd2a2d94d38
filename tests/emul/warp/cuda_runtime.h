// TEST INFRASTRUCTURE -- a stand-in for <cuda_runtime.h> that lets g++ compile openhevc_b200/csrc/kernels.cu and engine.cu
// UNCHANGED for the CPU (-DB200_EMUL, this directory first on the include path).  Kernels run as fibers, one per CUDA thread,
// scheduled in warp lock-step (warp_emul.cpp): __shfl_*_sync / __syncwarp / __any_sync / __all_sync / __syncthreads block a
// fiber until every participating lane has arrived, exactly the contract the device gives; everything the runtime API does
// asynchronously on a device (copies, memsets, kernels, events) happens immediately here.  The result is
// oracle/_ref/libb200hevc_emul.so with the same C ABI as libb200hevc.so, loaded ONLY by tests/ (never by the product): the
// CPU suite can run whole work lists and whole streams through the very kernel source that is compiled for sm_90a.
// What it cannot show: memory-model races, stream / event ordering, performance.
#pragma once
#ifndef B200_EMUL
#error "tests/emul/warp/cuda_runtime.h is only for the CPU emulation build (-DB200_EMUL)"
#endif
#include <stddef.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <functional>

// ---- qualifiers -----------------------------------------------------------------------------------------------------
#define __global__
#define __device__
#define __host__
#define __constant__ static const
#define __shared__ static                       /* blocks run one after another: a function-local static is the block's shared memory */
#define __forceinline__ inline __attribute__((always_inline))
#define __noinline__ __attribute__((noinline))
#define __launch_bounds__(...)
#define __align__(n) __attribute__((aligned(n)))

// ---- vector types ---------------------------------------------------------------------------------------------------
struct int2 { int x, y; };
struct int3 { int x, y, z; };
struct __attribute__((aligned(16))) int4 { int x, y, z, w; };
struct __attribute__((aligned(8))) uint2 { unsigned x, y; };
struct uint3 { unsigned x, y, z; };
struct __attribute__((aligned(16))) uint4 { unsigned x, y, z, w; };
struct dim3 {
    unsigned x, y, z;
    dim3(unsigned x_ = 1, unsigned y_ = 1, unsigned z_ = 1) : x(x_), y(y_), z(z_) {}
};
static inline int2 make_int2(int x, int y) { return int2{ x, y }; }
static inline int3 make_int3(int x, int y, int z) { return int3{ x, y, z }; }
static inline int4 make_int4(int x, int y, int z, int w) { return int4{ x, y, z, w }; }
static inline uint2 make_uint2(unsigned x, unsigned y) { return uint2{ x, y }; }
static inline uint4 make_uint4(unsigned x, unsigned y, unsigned z, unsigned w) { return uint4{ x, y, z, w }; }

// ---- built-in variables ---------------------------------------------------------------------------------------------
struct EmuThread { uint3 tid; };
extern EmuThread *emu_self;                      // the fiber that is running
extern uint3 emu_block_idx;
extern dim3 emu_block_dim, emu_grid_dim;
#define threadIdx (emu_self->tid)
#define blockIdx emu_block_idx
#define blockDim emu_block_dim
#define gridDim emu_grid_dim
#define warpSize 32

// ---- warp / block collectives (warp_emul.cpp) --------------------------------------------------------------------------
enum { EMU_SYNCWARP, EMU_SHFL_IDX, EMU_SHFL_XOR, EMU_SHFL_UP, EMU_SHFL_DOWN, EMU_ANY, EMU_ALL, EMU_BALLOT };
uint32_t emu_collective(unsigned mask, int op, uint32_t value, int arg, int width);
void emu_syncthreads();
void emu_yield();                                 // polling loops: let the other warps of the block run

static inline void __syncwarp(unsigned mask = 0xffffffffu) { emu_collective(mask, EMU_SYNCWARP, 0, 0, 32); }
static inline void __syncthreads() { emu_syncthreads(); }
static inline int __any_sync(unsigned mask, int pred) { return (int)emu_collective(mask, EMU_ANY, pred != 0, 0, 32); }
static inline int __all_sync(unsigned mask, int pred) { return (int)emu_collective(mask, EMU_ALL, pred != 0, 0, 32); }
static inline unsigned __ballot_sync(unsigned mask, int pred) { return emu_collective(mask, EMU_BALLOT, pred != 0, 0, 32); }
template <typename T> static inline T emu_shfl(unsigned mask, int op, T v, int arg, int width)
{
    static_assert(sizeof(T) == 4 || sizeof(T) == 8, "shuffle of a 4- or 8-byte value");
    uint32_t w[2] = { 0, 0 };
    memcpy(w, &v, sizeof(T));
    w[0] = emu_collective(mask, op, w[0], arg, width);
    if (sizeof(T) == 8) w[1] = emu_collective(mask, op, w[1], arg, width);
    T r;
    memcpy(&r, w, sizeof(T));
    return r;
}
template <typename T> static inline T __shfl_sync(unsigned mask, T v, int src, int width = 32) { return emu_shfl(mask, EMU_SHFL_IDX, v, src, width); }
template <typename T> static inline T __shfl_xor_sync(unsigned mask, T v, int lane_mask, int width = 32) { return emu_shfl(mask, EMU_SHFL_XOR, v, lane_mask, width); }
template <typename T> static inline T __shfl_up_sync(unsigned mask, T v, unsigned delta, int width = 32) { return emu_shfl(mask, EMU_SHFL_UP, v, (int)delta, width); }
template <typename T> static inline T __shfl_down_sync(unsigned mask, T v, unsigned delta, int width = 32) { return emu_shfl(mask, EMU_SHFL_DOWN, v, (int)delta, width); }

// ---- memory, atomics, time -------------------------------------------------------------------------------------------
template <typename T> static inline T __ldg(const T *p) { return *p; }
// atomics and the relaxed GPU-scope accessors of kernels.cu (inline PTX there) are compiler atomics, so that a thread-sanitizer
// build of the emulation knows them from plain accesses; a polling load is also where a waiting warp yields
static inline unsigned atomicAdd(unsigned *p, unsigned v) { return __atomic_fetch_add(p, v, __ATOMIC_RELAXED); }
static inline int atomicAdd(int *p, int v) { return __atomic_fetch_add(p, v, __ATOMIC_RELAXED); }
static inline unsigned atomicOr(unsigned *p, unsigned v) { return __atomic_fetch_or(p, v, __ATOMIC_RELAXED); }
static inline unsigned atomicMax(unsigned *p, unsigned v) { unsigned o = __atomic_load_n(p, __ATOMIC_RELAXED); while (v > o && !__atomic_compare_exchange_n(p, &o, v, false, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) {} return o; }
static inline void __nanosleep(unsigned) { emu_yield(); }
static inline void __threadfence() { __atomic_thread_fence(__ATOMIC_SEQ_CST); }
static inline void __threadfence_system() { __atomic_thread_fence(__ATOMIC_SEQ_CST); }
static inline unsigned long long gtime() { return 0; }
static inline uint32_t ld_relaxed(const uint32_t *p) { emu_yield(); return __atomic_load_n(p, __ATOMIC_RELAXED); }
static inline void st_relaxed(uint32_t *p, uint32_t v) { __atomic_store_n(p, v, __ATOMIC_RELAXED); }
static inline uint2 ld_edge(const uint2 *p)
{
    emu_yield();
    const uint64_t w = __atomic_load_n(reinterpret_cast<const uint64_t *>(p), __ATOMIC_RELAXED);      // one 8-byte access, as on the device
    uint2 v; v.x = (unsigned)w; v.y = (unsigned)(w >> 32);
    return v;
}
static inline void st_edge(uint2 *p, uint2 v) { __atomic_store_n(reinterpret_cast<uint64_t *>(p), (uint64_t)v.x | ((uint64_t)v.y << 32), __ATOMIC_RELAXED); }

// integer min / max with the device's overload set (the kernels mix int and unsigned like CUDA allows)
static inline int min(int a, int b) { return a < b ? a : b; }
static inline int max(int a, int b) { return a > b ? a : b; }
static inline unsigned min(unsigned a, unsigned b) { return a < b ? a : b; }
static inline unsigned max(unsigned a, unsigned b) { return a > b ? a : b; }
static inline unsigned min(unsigned a, int b) { return min(a, (unsigned)b); }
static inline unsigned min(int a, unsigned b) { return min((unsigned)a, b); }
static inline unsigned max(unsigned a, int b) { return max(a, (unsigned)b); }
static inline unsigned max(int a, unsigned b) { return max((unsigned)a, b); }
static inline long long min(long long a, long long b) { return a < b ? a : b; }
static inline long long max(long long a, long long b) { return a > b ? a : b; }
static inline long min(long a, long b) { return a < b ? a : b; }
static inline long max(long a, long b) { return a > b ? a : b; }

// ---- kernel launch ---------------------------------------------------------------------------------------------------
void emu_run_grid(dim3 grid, dim3 block, const std::function<void()> &thread_body, const char *name);
template <typename F> struct EmuLaunch {
    dim3 grid, block;
    F fn;
    const char *name;
    template <typename... A> void operator()(A... a) const
    {
        emu_run_grid(grid, block, [&]() { fn(a...); }, name);        // every fiber calls the kernel with its own copy of the parameters
    }
};
template <typename F> static inline EmuLaunch<F> emu_make_launch(dim3 g, dim3 b, F fn, const char *name) { return EmuLaunch<F>{ g, b, fn, name }; }
#define B200_LAUNCH(grid, block, smem, stream, ...) emu_make_launch(grid, block, &__VA_ARGS__, #__VA_ARGS__)

// ---- runtime API: everything completes at once ------------------------------------------------------------------------
typedef int cudaError_t;
enum { cudaSuccess = 0, cudaErrorInvalidValue = 1 };
typedef struct EmuStream *cudaStream_t;
typedef struct EmuEvent *cudaEvent_t;
enum cudaMemcpyKind { cudaMemcpyHostToHost, cudaMemcpyHostToDevice, cudaMemcpyDeviceToHost, cudaMemcpyDeviceToDevice, cudaMemcpyDefault };
enum { cudaStreamNonBlocking = 1, cudaEventDisableTiming = 2, cudaHostAllocDefault = 0, cudaHostAllocMapped = 2, cudaHostRegisterDefault = 0 };
enum cudaMemoryType { cudaMemoryTypeUnregistered = 0, cudaMemoryTypeHost = 1, cudaMemoryTypeDevice = 2 };
struct cudaPointerAttributes { cudaMemoryType type; int device; void *devicePointer, *hostPointer; };
struct cudaDeviceProp { char name[256]; int multiProcessorCount; int major, minor; size_t totalGlobalMem; int pciBusID, pciDeviceID, pciDomainID; };

cudaError_t cudaMalloc(void **p, size_t n);
template <typename T> static inline cudaError_t cudaMalloc(T **p, size_t n) { return cudaMalloc((void **)p, n); }
cudaError_t cudaFree(void *p);
cudaError_t cudaHostAlloc(void **p, size_t n, unsigned flags);
template <typename T> static inline cudaError_t cudaHostAlloc(T **p, size_t n, unsigned flags) { return cudaHostAlloc((void **)p, n, flags); }
cudaError_t cudaFreeHost(void *p);
static inline cudaError_t cudaHostGetDevicePointer(void **d, void *h, unsigned) { *d = h; return cudaSuccess; }
static inline cudaError_t cudaHostRegister(void *, size_t, unsigned) { return cudaSuccess; }
static inline cudaError_t cudaHostUnregister(void *) { return cudaSuccess; }
cudaError_t cudaPointerGetAttributes(cudaPointerAttributes *a, const void *p);
static inline cudaError_t cudaMemcpy(void *d, const void *s, size_t n, cudaMemcpyKind) { memmove(d, s, n); return cudaSuccess; }
static inline cudaError_t cudaMemcpyAsync(void *d, const void *s, size_t n, cudaMemcpyKind, cudaStream_t = nullptr) { memmove(d, s, n); return cudaSuccess; }
static inline cudaError_t cudaMemcpy2DAsync(void *d, size_t dp, const void *s, size_t sp, size_t w, size_t h, cudaMemcpyKind, cudaStream_t = nullptr)
{
    for (size_t y = 0; y < h; y++) memmove((uint8_t *)d + y * dp, (const uint8_t *)s + y * sp, w);
    return cudaSuccess;
}
static inline cudaError_t cudaMemset(void *d, int v, size_t n) { memset(d, v, n); return cudaSuccess; }
static inline cudaError_t cudaMemsetAsync(void *d, int v, size_t n, cudaStream_t = nullptr) { memset(d, v, n); return cudaSuccess; }
template <typename T> static inline cudaError_t cudaMemcpyToSymbol(T &sym, const void *src, size_t n) { memcpy((void *)&sym, src, n); return cudaSuccess; }
cudaError_t cudaStreamCreateWithFlags(cudaStream_t *s, unsigned flags);
cudaError_t cudaStreamDestroy(cudaStream_t s);
static inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
static inline cudaError_t cudaStreamWaitEvent(cudaStream_t, cudaEvent_t, unsigned = 0) { return cudaSuccess; }
cudaError_t cudaEventCreateWithFlags(cudaEvent_t *e, unsigned flags);
static inline cudaError_t cudaEventCreate(cudaEvent_t *e) { return cudaEventCreateWithFlags(e, 0); }
cudaError_t cudaEventDestroy(cudaEvent_t e);
static inline cudaError_t cudaEventRecord(cudaEvent_t, cudaStream_t = nullptr) { return cudaSuccess; }
static inline cudaError_t cudaEventSynchronize(cudaEvent_t) { return cudaSuccess; }
static inline cudaError_t cudaEventElapsedTime(float *ms, cudaEvent_t, cudaEvent_t) { *ms = 0.f; return cudaSuccess; }
static inline cudaError_t cudaSetDevice(int) { return cudaSuccess; }
static inline cudaError_t cudaGetDevice(int *d) { *d = 0; return cudaSuccess; }
static inline cudaError_t cudaGetDeviceCount(int *n) { *n = 1; return cudaSuccess; }
static inline cudaError_t cudaDeviceSynchronize() { return cudaSuccess; }
static inline cudaError_t cudaGetLastError() { return cudaSuccess; }
static inline const char *cudaGetErrorString(cudaError_t) { return "emulated CUDA runtime: no error"; }
static inline cudaError_t cudaGetDeviceProperties(cudaDeviceProp *p, int) { memset(p, 0, sizeof(*p)); strcpy(p->name, "warp-lockstep CPU emulation"); p->multiProcessorCount = 132; p->major = 9; return cudaSuccess; }
enum cudaDeviceAttr { cudaDevAttrMultiProcessorCount = 16 };
static inline cudaError_t cudaDeviceGetAttribute(int *v, cudaDeviceAttr a, int) { *v = a == cudaDevAttrMultiProcessorCount ? 132 : 0; return cudaSuccess; }
static inline cudaError_t cudaDeviceGetPCIBusId(char *s, int n, int) { if (n > 0) s[0] = 0; return cudaErrorInvalidValue; }
