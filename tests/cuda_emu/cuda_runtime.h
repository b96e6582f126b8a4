// TEST INFRASTRUCTURE (never part of the product): a minimal CUDA-on-CPU shim.  tests/cuda_emu/build.py compiles a few of the
// library's .cu files with g++ against this header so that the DEVICE branches of those kernels (__CUDA_ARCH__ code paths:
// shuffle scans, shared-memory atomics, warp collectives, launch geometry) execute on the CPU: every CTA of a launch runs
// with one OS thread per CUDA thread, __syncthreads is a real barrier, warp collectives rendezvous the 32 lanes of a warp.
// Only what those kernels use is provided.
#pragma once
#include <algorithm>
#include <atomic>
#include <barrier>
#include <cmath>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <memory>
#include <thread>
#include <vector>

#define __CUDA_ARCH__ 900
#define RGBL_CUDA_EMU 1
#define __CUDACC__ 1
#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __noinline__
#define __restrict__
#define __launch_bounds__(...)
#define __align__(n) __attribute__((aligned(n)))
#define __shared__ static                 /* one CTA runs at a time */
#define __constant__ static

struct uint3 { unsigned x, y, z; };
struct dim3 { unsigned x, y, z; dim3(unsigned a = 1, unsigned b = 1, unsigned c = 1) : x(a), y(b), z(c) {} };
struct float4 { float x, y, z, w; };
struct alignas(16) uint4 { unsigned x, y, z, w; };
typedef int cudaError_t;
typedef void* cudaStream_t;
enum { cudaSuccess = 0 };
enum cudaFuncAttribute { cudaFuncAttributeMaxDynamicSharedMemorySize = 8 };
enum cudaDeviceAttr { cudaDevAttrMaxSharedMemoryPerBlockOptin = 97, cudaDevAttrMaxSharedMemoryPerMultiprocessor = 81 };
struct cudaFuncAttributes { size_t sharedSizeBytes = 0; };
template <class F> inline cudaError_t cudaFuncSetAttribute(F, cudaFuncAttribute, int) { return cudaSuccess; }
template <class F> inline cudaError_t cudaFuncGetAttributes(cudaFuncAttributes* a, F) { a->sharedSizeBytes = 0; return cudaSuccess; }
inline cudaError_t cudaGetDevice(int* d) { *d = 0; return cudaSuccess; }
inline cudaError_t cudaDeviceGetAttribute(int* v, cudaDeviceAttr a, int) { *v = a == cudaDevAttrMaxSharedMemoryPerMultiprocessor ? 233472 : 232448; return cudaSuccess; }

namespace emu {
constexpr size_t kDynSmem = 232448;
struct Cta {
    std::unique_ptr<std::barrier<>> bar;
    std::vector<std::unique_ptr<std::barrier<>>> warp_bar;
    std::vector<std::array<unsigned long long, 32>> slot;
    std::atomic<int> nb_count{0}, nb_gen{0};      // named barrier of a subset of the CTA's threads (team_sync)
};
extern Cta* g_cta;
extern thread_local int t_warp, t_lane;
struct Cfg { dim3 grid, block; size_t smem; };
inline Cfg cfg(dim3 g, dim3 b, size_t smem = 0, cudaStream_t = nullptr) { return Cfg{g, b, smem}; }
void run(const Cfg& c, const std::function<void()>& body);
inline double approx64(double v) { unsigned long long u; std::memcpy(&u, &v, 8); u &= 0xffffffff00000000ull; std::memcpy(&v, &u, 8); return v; }
inline void warp_sync() { g_cta->warp_bar[t_warp]->arrive_and_wait(); }
inline void named_barrier(int n) {
    Cta* c = g_cta;
    const int gen = c->nb_gen.load();
    if (c->nb_count.fetch_add(1) + 1 == n) { c->nb_count.store(0); c->nb_gen.fetch_add(1); }
    else while (c->nb_gen.load() == gen) std::this_thread::yield();
}
template <class T> inline T exchange(T v, int src_lane) {       // every lane publishes v, reads lane src_lane's value
    unsigned long long raw = 0;
    std::memcpy(&raw, &v, sizeof(T));
    g_cta->slot[t_warp][t_lane] = raw;
    warp_sync();
    const unsigned long long got = g_cta->slot[t_warp][src_lane & 31];
    warp_sync();
    T out;
    std::memcpy(&out, &got, sizeof(T));
    return out;
}
}  // namespace emu

extern thread_local uint3 threadIdx;
extern uint3 blockIdx;
extern dim3 blockDim, gridDim;

inline void __syncthreads() { emu::g_cta->bar->arrive_and_wait(); }
inline void __syncwarp(unsigned = 0xffffffffu) { emu::warp_sync(); }
template <class T> inline T __shfl_sync(unsigned, T v, int src) { return emu::exchange(v, src); }
template <class T> inline T __shfl_up_sync(unsigned, T v, unsigned d) { const int s = emu::t_lane - (int)d; const T o = emu::exchange(v, s < 0 ? emu::t_lane : s); return s < 0 ? v : o; }
template <class T> inline T __shfl_down_sync(unsigned, T v, unsigned d) { const int s = emu::t_lane + (int)d; const T o = emu::exchange(v, s > 31 ? emu::t_lane : s); return s > 31 ? v : o; }
template <class T> inline T __shfl_xor_sync(unsigned, T v, int m) { return emu::exchange(v, emu::t_lane ^ m); }
inline void emu_gather(unsigned long long v, unsigned long long out[32]) {      // all (live) lanes publish, everybody reads all
    emu::g_cta->slot[emu::t_warp][emu::t_lane] = v;
    emu::warp_sync();
    for (int l = 0; l < 32; ++l) out[l] = emu::g_cta->slot[emu::t_warp][l];
    emu::warp_sync();
}
inline unsigned __ballot_sync(unsigned, int pred) { unsigned long long a[32]; emu_gather(pred ? 1 : 0, a); unsigned r = 0; for (int l = 0; l < 32; ++l) r |= (unsigned)(a[l] & 1) << l; return r; }
inline int __reduce_add_sync(unsigned, int v) { unsigned long long a[32]; emu_gather((unsigned long long)(long long)v, a); int s = 0; for (int l = 0; l < 32; ++l) s += (int)(long long)a[l]; return s; }
inline unsigned __reduce_min_sync(unsigned, unsigned v) { unsigned long long a[32]; emu_gather(v, a); unsigned r = 0xffffffffu; for (int l = 0; l < 32; ++l) r = std::min(r, (unsigned)a[l]); return r; }
inline unsigned __reduce_max_sync(unsigned, unsigned v) { unsigned long long a[32]; emu_gather(v, a); unsigned r = 0; for (int l = 0; l < 32; ++l) r = std::max(r, (unsigned)a[l]); return r; }
inline int __any_sync(unsigned, int pred) { return __ballot_sync(0xffffffffu, pred) != 0; }
inline int __all_sync(unsigned, int pred) { return __ballot_sync(0xffffffffu, pred) == 0xffffffffu; }
inline unsigned __match_any_sync(unsigned, int v) { unsigned long long a[32]; emu_gather((unsigned long long)(unsigned)v, a); unsigned r = 0; for (int l = 0; l < 32; ++l) if ((unsigned)a[l] == (unsigned)v) r |= 1u << l; return r; }
inline int __syncthreads_count(int p) { static std::atomic<int> acc{0}; if (p) acc.fetch_add(1); __syncthreads(); const int r = acc.load(); __syncthreads(); if (threadIdx.x == 0) acc.store(0); __syncthreads(); return r; }
inline int __syncthreads_or(int p) { static std::atomic<int> acc{0}; if (p) acc.store(1); __syncthreads(); const int r = acc.load(); __syncthreads(); if (threadIdx.x == 0) acc.store(0); __syncthreads(); return r; }

template <class T> inline T __ldg(const T* p) { return *p; }
inline int atomicAdd(int* p, int v) { return __atomic_fetch_add(p, v, __ATOMIC_RELAXED); }
inline unsigned atomicAdd(unsigned* p, unsigned v) { return __atomic_fetch_add(p, v, __ATOMIC_RELAXED); }
inline int atomicMin(int* p, int v) { int o = __atomic_load_n(p, __ATOMIC_RELAXED); while (o > v && !__atomic_compare_exchange_n(p, &o, v, true, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) {} return o; }
inline int atomicMax(int* p, int v) { int o = __atomic_load_n(p, __ATOMIC_RELAXED); while (o < v && !__atomic_compare_exchange_n(p, &o, v, true, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) {} return o; }
inline unsigned long long atomicAdd(unsigned long long* p, unsigned long long v) { return __atomic_fetch_add(p, v, __ATOMIC_RELAXED); }
inline float atomicAdd(float* p, float v) { float o = *p, n; do { n = o + v; } while (!__atomic_compare_exchange(p, &o, &n, true, __ATOMIC_RELAXED, __ATOMIC_RELAXED)); return o; }
inline double atomicAdd(double* p, double v) { double o = *p, n; do { n = o + v; } while (!__atomic_compare_exchange(p, &o, &n, true, __ATOMIC_RELAXED, __ATOMIC_RELAXED)); return o; }
inline unsigned atomicExch(unsigned* p, unsigned v) { return __atomic_exchange_n(p, v, __ATOMIC_RELAXED); }
inline unsigned atomicOr(unsigned* p, unsigned v) { return __atomic_fetch_or(p, v, __ATOMIC_RELAXED); }
inline int atomicOr(int* p, int v) { return __atomic_fetch_or(p, v, __ATOMIC_RELAXED); }
inline int atomicExch(int* p, int v) { return __atomic_exchange_n(p, v, __ATOMIC_RELAXED); }
inline unsigned atomicMax(unsigned* p, unsigned v) { unsigned o = __atomic_load_n(p, __ATOMIC_RELAXED); while (o < v && !__atomic_compare_exchange_n(p, &o, v, true, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) {} return o; }
inline void __threadfence() { __atomic_thread_fence(__ATOMIC_SEQ_CST); }
inline int __popc(unsigned v) { return __builtin_popcount(v); }
inline unsigned __funnelshift_l(unsigned lo, unsigned hi, unsigned sh) { sh &= 31; return sh ? (hi << sh) | (lo >> (32 - sh)) : hi; }
inline unsigned __funnelshift_r(unsigned lo, unsigned hi, unsigned sh) { sh &= 31; return sh ? (lo >> sh) | (hi << (32 - sh)) : lo; }
inline int __ffs(int v) { return __builtin_ffs(v); }
inline unsigned __byte_perm(unsigned a, unsigned b, unsigned sel) {
    const unsigned long long src = (unsigned long long)a | ((unsigned long long)b << 32);
    unsigned r = 0;
    for (int i = 0; i < 4; ++i) r |= (unsigned)((src >> (8 * ((sel >> (4 * i)) & 7))) & 0xff) << (8 * i);
    return r;
}
inline unsigned emu_pack2(int lo, int hi) { return (unsigned)(uint16_t)lo | ((unsigned)(uint16_t)hi << 16); }
inline unsigned __vmins2(unsigned a, unsigned b) { return emu_pack2(std::min((int16_t)a, (int16_t)b), std::min((int16_t)(a >> 16), (int16_t)(b >> 16))); }
inline unsigned __vmaxs2(unsigned a, unsigned b) { return emu_pack2(std::max((int16_t)a, (int16_t)b), std::max((int16_t)(a >> 16), (int16_t)(b >> 16))); }
inline unsigned __vsub2(unsigned a, unsigned b) { return emu_pack2((int)(uint16_t)a - (int)(uint16_t)b, (int)(a >> 16) - (int)(b >> 16)); }
inline float __frcp_rn(float a) { return 1.0f / a; }
inline float __fmul_rn(float a, float b) { return a * b; }
inline float __fadd_rn(float a, float b) { return a + b; }
inline float __fsub_rn(float a, float b) { return a - b; }
inline float __fdiv_rn(float a, float b) { return a / b; }
inline double __dmul_rn(double a, double b) { return a * b; }
inline double __dadd_rn(double a, double b) { return a + b; }
inline double __dsub_rn(double a, double b) { return a - b; }
inline double __ddiv_rn(double a, double b) { return a / b; }
inline double __dsqrt_rn(double a) { return std::sqrt(a); }
inline float __fsqrt_rn(float a) { return std::sqrt(a); }
inline int __float2int_rd(float v) { return (int)floorf(v); }
inline int __float2int_rz(float v) { return (int)v; }
inline int __double2int_rn(double v) { return (int)lrint(v); }
inline float __int2float_rn(int v) { return (float)v; }
inline unsigned __brev(unsigned v) { unsigned r = 0; for (int i = 0; i < 32; ++i) r |= ((v >> i) & 1u) << (31 - i); return r; }
inline int __clz(int v) { return v ? __builtin_clz((unsigned)v) : 32; }
inline int __popcll(unsigned long long v) { return __builtin_popcountll(v); }
inline int __float2int_rn(float v) { return (int)lrintf(v); }
inline float __fmaf_rn(float a, float b, float c) { return fmaf(a, b, c); }
inline float __uint_as_float(unsigned u) { float f; std::memcpy(&f, &u, 4); return f; }
inline unsigned __float_as_uint(float f) { unsigned u; std::memcpy(&u, &f, 4); return u; }
inline double rsqrt(double x) { return 1.0 / std::sqrt(x); }
inline void sincos(double x, double* s, double* c) { *s = std::sin(x); *c = std::cos(x); }
using std::isfinite;
using ::fmaxf;
using std::min;
using std::max;

// ---- host-side runtime API: everything is synchronous (a launch returns when the grid has run), memory is host memory ----------
typedef struct EmuEvent { double t; }* cudaEvent_t;
typedef void* cudaGraph_t;
typedef void* cudaGraphExec_t;
enum cudaMemcpyKind { cudaMemcpyHostToHost = 0, cudaMemcpyHostToDevice = 1, cudaMemcpyDeviceToHost = 2, cudaMemcpyDeviceToDevice = 3 };
enum { cudaStreamNonBlocking = 1, cudaEventDisableTiming = 2 };
enum cudaStreamCaptureMode { cudaStreamCaptureModeRelaxed = 2 };
enum { cudaErrorMemoryAllocation = 2, cudaErrorNotSupported = 801 };
inline const char* cudaGetErrorString(cudaError_t e) { return e == cudaSuccess ? "no error" : "emulated CUDA error"; }
inline cudaError_t cudaGetLastError() { return cudaSuccess; }
inline cudaError_t cudaSetDevice(int) { return cudaSuccess; }
inline cudaError_t cudaDeviceGetStreamPriorityRange(int* lo, int* hi) { *lo = 0; *hi = -1; return cudaSuccess; }
// allocation-failure injection: emu_fail_allocation(k) makes the k-th cudaMalloc / cudaMallocHost from now on fail (once; -1: none) and
// returns the countdown it replaces (-1: the previous one has fired, or none was set)
extern "C" int emu_fail_allocation(int nth);
namespace emu { bool allocation_fails(); }
template <class T> inline cudaError_t cudaMalloc(T** p, size_t n) {
    if (emu::allocation_fails()) return cudaErrorMemoryAllocation;
    *p = (T*)calloc(n + 256, 1); return *p ? cudaSuccess : cudaErrorMemoryAllocation;
}
template <class T> inline cudaError_t cudaMallocHost(T** p, size_t n) { return cudaMalloc(p, n); }
inline cudaError_t cudaFree(void* p) { free(p); return cudaSuccess; }
inline cudaError_t cudaFreeHost(void* p) { free(p); return cudaSuccess; }
inline cudaError_t cudaMemcpy(void* d, const void* s, size_t n, cudaMemcpyKind) { memmove(d, s, n); return cudaSuccess; }
inline cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, cudaMemcpyKind, cudaStream_t = nullptr) { memmove(d, s, n); return cudaSuccess; }
inline cudaError_t cudaMemcpy2DAsync(void* d, size_t dp, const void* s, size_t sp, size_t w, size_t h, cudaMemcpyKind, cudaStream_t = nullptr) {
    for (size_t y = 0; y < h; ++y) memmove((char*)d + y * dp, (const char*)s + y * sp, w);
    return cudaSuccess;
}
inline cudaError_t cudaMemset(void* d, int v, size_t n) { memset(d, v, n); return cudaSuccess; }
inline cudaError_t cudaMemsetAsync(void* d, int v, size_t n, cudaStream_t = nullptr) { memset(d, v, n); return cudaSuccess; }
inline cudaError_t cudaStreamCreateWithFlags(cudaStream_t* s, unsigned) { *s = malloc(8); return cudaSuccess; }
inline cudaError_t cudaStreamCreateWithPriority(cudaStream_t* s, unsigned, int) { *s = malloc(8); return cudaSuccess; }
inline cudaError_t cudaStreamDestroy(cudaStream_t s) { free(s); return cudaSuccess; }
inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
inline cudaError_t cudaStreamWaitEvent(cudaStream_t, cudaEvent_t, unsigned = 0) { return cudaSuccess; }
inline double emu_now_ms() { timespec ts; clock_gettime(CLOCK_MONOTONIC, &ts); return ts.tv_sec * 1e3 + ts.tv_nsec * 1e-6; }
inline cudaError_t cudaEventCreate(cudaEvent_t* e) { *e = new EmuEvent{0}; return cudaSuccess; }
inline cudaError_t cudaEventCreateWithFlags(cudaEvent_t* e, unsigned) { *e = new EmuEvent{0}; return cudaSuccess; }
inline cudaError_t cudaEventDestroy(cudaEvent_t e) { delete e; return cudaSuccess; }
inline cudaError_t cudaEventRecord(cudaEvent_t e, cudaStream_t = nullptr) { e->t = emu_now_ms(); return cudaSuccess; }
inline cudaError_t cudaEventSynchronize(cudaEvent_t) { return cudaSuccess; }
inline cudaError_t cudaEventElapsedTime(float* ms, cudaEvent_t a, cudaEvent_t b) { *ms = (float)(b->t - a->t); return cudaSuccess; }
// cudaLaunchKernelEx: the launch attributes (programmatic dependent launch) mean nothing to a synchronous emulation
enum cudaLaunchAttributeID { cudaLaunchAttributeProgrammaticStreamSerialization = 6 };
struct cudaLaunchAttributeValue { int programmaticStreamSerializationAllowed; };
struct cudaLaunchAttribute { cudaLaunchAttributeID id; cudaLaunchAttributeValue val; };
struct cudaLaunchConfig_t { dim3 gridDim, blockDim; size_t dynamicSmemBytes = 0; cudaStream_t stream = nullptr; cudaLaunchAttribute* attrs = nullptr; unsigned numAttrs = 0; };
template <class... KArgs, class... Args>
inline cudaError_t cudaLaunchKernelEx(const cudaLaunchConfig_t* cfg, void (*kernel)(KArgs...), Args&&... args) {
    emu::run(emu::Cfg{cfg->gridDim, cfg->blockDim, cfg->dynamicSmemBytes}, [&]() { kernel(args...); });
    return cudaSuccess;
}
// CUDA graphs are not emulated: capture is refused (the library replays the chain launch by launch when RGBL_CHAIN_GRAPH=0)
inline cudaError_t cudaStreamBeginCapture(cudaStream_t, cudaStreamCaptureMode) { return cudaErrorNotSupported; }
inline cudaError_t cudaStreamEndCapture(cudaStream_t, cudaGraph_t* g) { *g = nullptr; return cudaErrorNotSupported; }
inline cudaError_t cudaGraphInstantiate(cudaGraphExec_t* e, cudaGraph_t, unsigned long long = 0) { *e = nullptr; return cudaErrorNotSupported; }
inline cudaError_t cudaGraphInstantiate(cudaGraphExec_t* e, cudaGraph_t, void*, void*, size_t) { *e = nullptr; return cudaErrorNotSupported; }
inline cudaError_t cudaGraphLaunch(cudaGraphExec_t, cudaStream_t) { return cudaErrorNotSupported; }
inline cudaError_t cudaGraphDestroy(cudaGraph_t) { return cudaSuccess; }
inline cudaError_t cudaGraphExecDestroy(cudaGraphExec_t) { return cudaSuccess; }
