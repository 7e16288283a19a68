// cuda_runtime.h -- TEST INFRASTRUCTURE, not a CUDA runtime: the ~45 runtime calls csrc/engine.cu makes, as a synchronous
// single-"device" stand-in in host memory, so that the HOST LOGIC of the engine (node-table builds, directory sizing and growth,
// the bounded-load round protocol, place_batch / check_address_batch flows, every extern "C" entry point) can be compiled with g++
// and exercised on a box without a GPU (tests/test_engine_host_sim.py).  "Device" memory is malloc'ed, every "asynchronous" call
// completes before it returns (so stream order holds trivially), events carry a wall-clock stamp.  The kernels themselves are NOT
// emulated: their launchers are replaced by plain restatements of what each kernel is specified to do (hostsim/launchers.cpp).
// Nothing under rio_rs_b200/ or include/ refers to this directory; the product library is built by nvcc against the real runtime
// and still refuses to start without a GPU (tests/test_abi.py::test_no_gpu_means_loud_failure_not_fallback).
#pragma once
#include <chrono>
#include <cstddef>
#include <cstdint>
#include <cstdlib>
#include <cstring>

#define __align__(n) alignas(n)
#define __host__
#define __device__
#define __forceinline__ inline
#define __restrict__

struct uint2 { uint32_t x, y; };
struct alignas(16) uint4 { uint32_t x, y, z, w; };
inline uint4 make_uint4(uint32_t x, uint32_t y, uint32_t z, uint32_t w) { return uint4{x, y, z, w}; }
inline uint2 make_uint2(uint32_t x, uint32_t y) { return uint2{x, y}; }

typedef int cudaError_t;
constexpr cudaError_t cudaSuccess = 0;
constexpr cudaError_t cudaErrorInvalidValue = 1;
constexpr cudaError_t cudaErrorMisalignedAddress = 716;
struct HostSimStream { int id; };
struct HostSimEvent { std::chrono::steady_clock::time_point t; };
typedef HostSimStream *cudaStream_t;
typedef HostSimEvent *cudaEvent_t;
typedef void *cudaMemPool_t;
enum cudaMemcpyKind { cudaMemcpyHostToHost = 0, cudaMemcpyHostToDevice = 1, cudaMemcpyDeviceToHost = 2, cudaMemcpyDeviceToDevice = 3, cudaMemcpyDefault = 4 };
enum cudaMemPoolAttr { cudaMemPoolAttrReleaseThreshold = 4 };
constexpr unsigned cudaStreamNonBlocking = 1, cudaEventDisableTiming = 2, cudaHostAllocMapped = 2, cudaIpcMemLazyEnablePeerAccess = 1;
struct cudaDeviceProp { char name[256]; size_t totalGlobalMem; int multiProcessorCount; };
struct cudaIpcMemHandle_t { char reserved[64]; };

inline const char *cudaGetErrorString(cudaError_t e) {
    return e == cudaSuccess ? "no error" : e == cudaErrorMisalignedAddress ? "misaligned address" : "host-sim error";
}
// The error a launcher double reported, returned (and cleared) by the next cudaGetLastError of the thread, as the runtime does
inline cudaError_t &hostsim_last_error() { static thread_local cudaError_t e = cudaSuccess; return e; }
inline cudaError_t cudaGetLastError() { const cudaError_t e = hostsim_last_error(); hostsim_last_error() = cudaSuccess; return e; }
// The alignment a kernel assumes of a caller's buffer, as csrc/buffer_align.cuh declares it: HOSTSIM_DECLARED_ALIGN(rio::kAlignTrieKeys).
// Against an engine without that header the doubles check natural alignment only (1 byte: every pointer passes).
#if __has_include("../../../rio_rs_b200/csrc/buffer_align.cuh")
#define HOSTSIM_DECLARED_ALIGN(a) (a)
#else
#define HOSTSIM_DECLARED_ALIGN(a) 1u
#endif
// A launcher double whose kernel reads or writes `p` with loads of `align` bytes calls this first: a pointer the kernel would fault
// on is reported as the launch error a misaligned access gives (the double then computes nothing), instead of being read silently.
inline bool hostsim_misaligned(const void *p, size_t align) {
    if (!p || ((uintptr_t)p & (align - 1)) == 0) return false;
    hostsim_last_error() = cudaErrorMisalignedAddress;
    return true;
}
inline cudaError_t cudaGetDeviceCount(int *n) { *n = 1; return cudaSuccess; }
inline cudaError_t cudaGetDevice(int *d) { *d = 0; return cudaSuccess; }
inline cudaError_t cudaSetDevice(int) { return cudaSuccess; }
inline cudaError_t cudaGetDeviceProperties(cudaDeviceProp *p, int) {
    memset(p, 0, sizeof *p);
    strcpy(p->name, "host-sim (no GPU: engine host logic only)");
    p->totalGlobalMem = (size_t)8 << 30;
    p->multiProcessorCount = 4;
    return cudaSuccess;
}
inline cudaError_t cudaStreamCreateWithFlags(cudaStream_t *s, unsigned) { *s = new HostSimStream{0}; return cudaSuccess; }
inline cudaError_t cudaStreamCreateWithPriority(cudaStream_t *s, unsigned, int) { *s = new HostSimStream{1}; return cudaSuccess; }
inline cudaError_t cudaDeviceGetStreamPriorityRange(int *lo, int *hi) { *lo = 0; *hi = -1; return cudaSuccess; }
inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
inline cudaError_t cudaStreamDestroy(cudaStream_t s) { delete s; return cudaSuccess; }
inline cudaError_t cudaStreamWaitEvent(cudaStream_t, cudaEvent_t, unsigned) { return cudaSuccess; }
inline cudaError_t cudaEventCreate(cudaEvent_t *e) { *e = new HostSimEvent{std::chrono::steady_clock::now()}; return cudaSuccess; }
inline cudaError_t cudaEventCreateWithFlags(cudaEvent_t *e, unsigned) { return cudaEventCreate(e); }
inline cudaError_t cudaEventRecord(cudaEvent_t e, cudaStream_t) { e->t = std::chrono::steady_clock::now(); return cudaSuccess; }
inline cudaError_t cudaEventSynchronize(cudaEvent_t) { return cudaSuccess; }
inline cudaError_t cudaEventElapsedTime(float *ms, cudaEvent_t a, cudaEvent_t b) { *ms = std::chrono::duration<float, std::milli>(b->t - a->t).count(); return cudaSuccess; }
inline cudaError_t cudaEventDestroy(cudaEvent_t e) { delete e; return cudaSuccess; }
// 256-byte aligned, as device allocations are (glibc's malloc gives 16)
inline cudaError_t cudaMalloc(void **p, size_t n) { *p = aligned_alloc(256, ((n ? n : 1) + 255) / 256 * 256); return *p ? cudaSuccess : cudaErrorInvalidValue; }
inline cudaError_t cudaFree(void *p) { free(p); return cudaSuccess; }
inline cudaError_t cudaMallocAsync(void **p, size_t n, cudaStream_t) { return cudaMalloc(p, n); }
inline cudaError_t cudaFreeAsync(void *p, cudaStream_t) { return cudaFree(p); }
inline cudaError_t cudaMallocHost(void **p, size_t n) { return cudaMalloc(p, n); }
inline cudaError_t cudaHostAlloc(void **p, size_t n, unsigned) { return cudaMalloc(p, n); }
inline cudaError_t cudaFreeHost(void *p) { return cudaFree(p); }
inline cudaError_t cudaHostGetDevicePointer(void **d, void *h, unsigned) { *d = h; return cudaSuccess; }
inline cudaError_t cudaMemcpyAsync(void *dst, const void *src, size_t n, cudaMemcpyKind, cudaStream_t) { if (n) memmove(dst, src, n); return cudaSuccess; }
inline cudaError_t cudaMemsetAsync(void *dst, int v, size_t n, cudaStream_t) { if (n) memset(dst, v, n); return cudaSuccess; }
inline cudaError_t cudaMemset(void *dst, int v, size_t n) { if (n) memset(dst, v, n); return cudaSuccess; }
inline cudaError_t cudaDeviceGetDefaultMemPool(cudaMemPool_t *p, int) { *p = nullptr; return cudaSuccess; }
inline cudaError_t cudaMemPoolSetAttribute(cudaMemPool_t, cudaMemPoolAttr, void *) { return cudaSuccess; }
// one process only: the "handle" is the pointer itself
inline cudaError_t cudaIpcGetMemHandle(cudaIpcMemHandle_t *h, void *p) { memset(h, 0, sizeof *h); memcpy(h->reserved, &p, sizeof p); return cudaSuccess; }
inline cudaError_t cudaIpcOpenMemHandle(void **p, cudaIpcMemHandle_t h, unsigned) { memcpy(p, h.reserved, sizeof *p); return cudaSuccess; }
inline cudaError_t cudaIpcCloseMemHandle(void *) { return cudaSuccess; }
