// TEST INFRASTRUCTURE — stands in for <cuda_runtime.h> when the PRODUCT sources are compiled with g++ for the full host
// emulation (tests/host_emu/build.py build_full).  See cuda_host_shim.h.
#pragma once
#define CUP2D_FULL_EMU 1
#include "cuda_host_shim.h"
#include <atomic>
#include <cstdint>
#include <cstdio>

struct cudaDeviceProp { int major = 9, minor = 0, multiProcessorCount = 4; char name[64] = "host emulation (sm_90 semantics)"; };
inline cudaError_t cudaGetDeviceProperties(cudaDeviceProp *p, int) { *p = cudaDeviceProp(); return 0; }
typedef struct EmuEvent *cudaEvent_t;
inline cudaError_t cudaEventCreate(cudaEvent_t *e) { *e = nullptr; return 0; }
enum { cudaEventDisableTiming = 2 };
inline cudaError_t cudaEventCreateWithFlags(cudaEvent_t *e, unsigned) { *e = nullptr; return 0; }
inline cudaError_t cudaStreamWaitEvent(cudaStream_t, cudaEvent_t, unsigned) { return 0; } // streams run in issue order here
inline cudaError_t cudaEventDestroy(cudaEvent_t) { return 0; }
inline cudaError_t cudaEventRecord(cudaEvent_t, cudaStream_t) { return 0; }
inline cudaError_t cudaEventSynchronize(cudaEvent_t) { return 0; }
inline cudaError_t cudaEventElapsedTime(float *ms, cudaEvent_t, cudaEvent_t) { *ms = 0.f; return 0; }
template <class T> cudaError_t cudaMallocHost(T **p, size_t n) { *p = (T *)malloc(n ? n : 1); return 0; }
inline cudaError_t cudaFreeHost(void *p) { free(p); return 0; }
struct cudaIpcMemHandle_t { char reserved[64]; };
enum { cudaIpcMemLazyEnablePeerAccess = 1 };
inline cudaError_t cudaIpcGetMemHandle(cudaIpcMemHandle_t *h, void *p) { memset(h, 0, sizeof *h); memcpy(h, &p, sizeof p); return 0; }
inline cudaError_t cudaIpcOpenMemHandle(void **p, cudaIpcMemHandle_t h, unsigned) { memcpy(p, &h, sizeof *p); return 0; }
inline cudaError_t cudaIpcCloseMemHandle(void *) { return 0; }
inline cudaError_t cudaDeviceSynchronize() { return 0; }
inline cudaError_t cudaStreamCreateWithFlags(cudaStream_t *s, unsigned) { *s = nullptr; return 0; }
enum { cudaStreamNonBlocking = 1 };

// graphs do not exist here: the product code takes its direct-launch path under CUP2D_FULL_EMU; only the types and the
// destructors it names unconditionally are provided
typedef struct EmuGraph *cudaGraph_t;
typedef struct EmuGraphExec *cudaGraphExec_t;
inline cudaError_t cudaGraphExecDestroy(cudaGraphExec_t) { return 0; }
inline cudaError_t cudaGraphDestroy(cudaGraph_t) { return 0; }
#include <chrono>
inline unsigned long long emu_now_ns() {
  return (unsigned long long)std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now().time_since_epoch()).count();
}
inline double __ddiv_rn(double a, double b) { volatile double r = a / b; return r; }
inline unsigned atomicAdd(unsigned *p, unsigned v) { return std::atomic_ref<unsigned>(*p).fetch_add(v); }
inline void __threadfence() { std::atomic_thread_fence(std::memory_order_seq_cst); }
inline void __threadfence_system() { std::atomic_thread_fence(std::memory_order_seq_cst); }
template <class T> T __ldg(const T *p) { return *p; }
inline int __double2hiint(double x) { long long b; memcpy(&b, &x, 8); return (int)(b >> 32); }
inline int __double2loint(double x) { long long b; memcpy(&b, &x, 8); return (int)(b & 0xffffffffll); }
inline long long __double_as_longlong(double x) { long long b; memcpy(&b, &x, 8); return b; }
inline double __longlong_as_double(long long b) { double x; memcpy(&x, &b, 8); return x; }
inline double __dmul_rn(double a, double b) { volatile double r = a * b; return r; }
inline double __dadd_rn(double a, double b) { volatile double r = a + b; return r; }
inline double __dsub_rn(double a, double b) { volatile double r = a - b; return r; }
inline size_t __cvta_generic_to_shared(const void *p) { return (size_t)p; }
using std::max;
using std::min;
inline int min(int a, long b) { return (int)std::min<long>(a, b); }
struct alignas(16) float4 { float x, y, z, w; };
inline float4 make_float4(float x, float y, float z, float w) { return {x, y, z, w}; }
