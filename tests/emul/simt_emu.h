// simt_emu.h -- TEST INFRASTRUCTURE ONLY.  A small SIMT emulator that lets the CPU suite compile the
// library's .cu sources with g++ and run the real kernels (barriers, warp collectives, shared memory,
// atomics, the TMA/mbarrier staging) on tiny scenes, so that kernel changes can be checked against the
// oracle without a GPU.  It is never linked into libh3dgs.so and nothing in the product path includes it:
// tests/emul/build_emu.py rewrites the launch syntax of a COPY of the sources and builds libh3dgs_emu.so
// in a temporary directory.
//
// Model: one OS thread; the threads of a CUDA block are fibers (own stacks, hand-written context switch)
// scheduled round-robin; blocks run one after the other, so `__shared__` becomes `static`.
// __syncthreads and the *_sync warp collectives are rendezvous points of the fibers.  Device memory is
// host memory; streams and events do nothing.
#pragma once
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include <functional>
#include <vector>

// ---- qualifiers ---------------------------------------------------------------------------------------
#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __restrict__
#define __launch_bounds__(...)
#define __shared__ static
#define __align__(n) __attribute__((aligned(n)))
#define __constant__
#define H3_SIMT_EMU 1

// ---- vector types ---------------------------------------------------------------------------------------
struct float2 { float x, y; };
struct alignas(16) float4 { float x, y, z, w; };
struct alignas(8) uint2 { unsigned x, y; };
struct int2 { int x, y; };
struct uint3 { unsigned x, y, z; };
struct dim3 { unsigned x, y, z; dim3(unsigned a = 1, unsigned b = 1, unsigned c = 1) : x(a), y(b), z(c) {} };
static inline float2 make_float2(float x, float y) { return float2{x, y}; }
static inline float4 make_float4(float x, float y, float z, float w) { return float4{x, y, z, w}; }
static inline uint2 make_uint2(unsigned x, unsigned y) { return uint2{x, y}; }
static inline int2 make_int2(int x, int y) { return int2{x, y}; }

// ---- the fiber scheduler (simt_emu.cpp) -------------------------------------------------------------------
namespace simt {
struct Ctx { uint3 tid; int lane, warp, linear; };
extern Ctx* g_cur;                 // the running fiber
extern uint3 g_blockIdx;
extern dim3 g_blockDim, g_gridDim;
extern unsigned char* g_dyn_smem;
void run_grid(dim3 grid, dim3 block, size_t dyn_smem, const std::function<void()>& body);
void fiber_yield();               // let the other threads of the block run (spin-wait loops)
void block_barrier();
int block_count(int pred);
uint64_t warp_exchange(uint64_t mine, int src_lane);                 // value of src_lane (own value if out of range)
uint64_t warp_reduce(uint64_t mine, int op);                         // 0 = ballot(pred) 1 = max(u32) 2 = and(pred) 3 = or(pred)
template <class K, class... A>
struct Launch {
    K k; dim3 g, b; size_t sm;
    template <class... B> void operator()(B... args) const {
        K kk = k;
        run_grid(g, b, sm, [=]() { kk(args...); });
    }
};
template <class K> Launch<K> make_launch(K k, dim3 g, dim3 b, size_t sm) { return Launch<K>{k, g, b, sm}; }
}  // namespace simt
#define SIMT_LAUNCH(k, g, b, sm, st) simt::make_launch(k, dim3(g), dim3(b), (size_t)(sm))
#define threadIdx (simt::g_cur->tid)
#define blockIdx (simt::g_blockIdx)
#define blockDim (simt::g_blockDim)
#define gridDim (simt::g_gridDim)

// ---- intrinsics ---------------------------------------------------------------------------------------
static inline unsigned __float_as_uint(float f) { unsigned u; memcpy(&u, &f, 4); return u; }
static inline int __float_as_int(float f) { int u; memcpy(&u, &f, 4); return u; }
static inline float __uint_as_float(unsigned u) { float f; memcpy(&f, &u, 4); return f; }
static inline float __int_as_float(int u) { float f; memcpy(&f, &u, 4); return f; }
static inline int __ffs(unsigned v) { return v ? __builtin_ctz(v) + 1 : 0; }
static inline int __clz(unsigned v) { return v ? __builtin_clz(v) : 32; }
static inline int __popc(unsigned v) { return __builtin_popcount(v); }
// rn single operations: keep the compiler from contracting them (the emulator is built with -ffp-contract=off)
static inline float __fadd_rn(float a, float b) { volatile float r = a + b; return r; }
static inline float __fmul_rn(float a, float b) { volatile float r = a * b; return r; }
static inline float __fmaf_rn(float a, float b, float c) { return fmaf(a, b, c); }
#define __log2f(x) log2f(x)        /* glibc declares functions of these names */
#define __expf(x) expf(x)
#define __logf(x) logf(x)
template <class T> static inline T __ldg(const T* p) { return *p; }
template <class T> static inline T __ldcg(const T* p) { return *p; }
static inline int min(int a, int b) { return a < b ? a : b; }
static inline int max(int a, int b) { return a > b ? a : b; }
static inline unsigned min(unsigned a, unsigned b) { return a < b ? a : b; }
static inline unsigned max(unsigned a, unsigned b) { return a > b ? a : b; }
static inline long long min(long long a, long long b) { return a < b ? a : b; }
static inline long long max(long long a, long long b) { return a > b ? a : b; }
static inline float min(float a, float b) { return fminf(a, b); }
static inline float max(float a, float b) { return fmaxf(a, b); }

static inline void __syncthreads() { simt::block_barrier(); }
static inline int __syncthreads_count(int pred) { return simt::block_count(pred); }
static inline void __syncwarp(unsigned = 0xffffffffu) { simt::warp_reduce(0, 3); }
static inline void __threadfence() {}
static inline unsigned __ballot_sync(unsigned, int pred) { return (unsigned)simt::warp_reduce(pred ? 1 : 0, 0); }
static inline int __any_sync(unsigned, int pred) { return (int)simt::warp_reduce(pred ? 1 : 0, 3); }
static inline int __all_sync(unsigned, int pred) { return (int)simt::warp_reduce(pred ? 1 : 0, 2); }
static inline unsigned __reduce_max_sync(unsigned, unsigned v) { return (unsigned)simt::warp_reduce(v, 1); }
static inline unsigned __match_any_sync(unsigned, unsigned v) {          // 32 exchanges: slow, but exact
    unsigned m = 0;
    for (int src = 0; src < 32; src++) if ((unsigned)simt::warp_exchange((uint64_t)v, src) == v) m |= 1u << src;
    return m;
}
template <class T> static inline T __shfl_sync(unsigned, T v, int src) {
    uint64_t raw = 0; memcpy(&raw, &v, sizeof(T));
    raw = simt::warp_exchange(raw, src & 31);
    T out; memcpy(&out, &raw, sizeof(T)); return out;
}
template <class T> static inline T __shfl_xor_sync(unsigned m, T v, int lane_mask) { return __shfl_sync(m, v, simt::g_cur->lane ^ lane_mask); }
template <class T> static inline T __shfl_up_sync(unsigned, T v, unsigned delta) {
    uint64_t raw = 0; memcpy(&raw, &v, sizeof(T));
    const int src = simt::g_cur->lane - (int)delta;
    raw = simt::warp_exchange(raw, src);                             // src < 0: own value
    T out; memcpy(&out, &raw, sizeof(T)); return out;
}
template <class T> static inline T __shfl_down_sync(unsigned, T v, unsigned delta) {
    uint64_t raw = 0; memcpy(&raw, &v, sizeof(T));
    raw = simt::warp_exchange(raw, simt::g_cur->lane + (int)delta);  // src > 31: own value
    T out; memcpy(&out, &raw, sizeof(T)); return out;
}

// atomics: one OS thread, fibers only switch at collectives
static inline float atomicAdd(float* p, float v) { float o = *p; *p = o + v; return o; }
static inline double atomicAdd(double* p, double v) { double o = *p; *p = o + v; return o; }
static inline int atomicAdd(int* p, int v) { int o = *p; *p = o + v; return o; }
static inline unsigned atomicAdd(unsigned* p, unsigned v) { unsigned o = *p; *p = o + v; return o; }
static inline float4 atomicAdd(float4* p, float4 v) { float4 o = *p; p->x += v.x; p->y += v.y; p->z += v.z; p->w += v.w; return o; }
static inline float atomicAdd_system(float* p, float v) { return atomicAdd(p, v); }
static inline double atomicAdd_system(double* p, double v) { return atomicAdd(p, v); }
static inline unsigned atomicSub(unsigned* p, unsigned v) { unsigned o = *p; *p = o - v; return o; }
static inline unsigned atomicMax(unsigned* p, unsigned v) { unsigned o = *p; if (v > o) *p = v; return o; }
static inline int atomicMax(int* p, int v) { int o = *p; if (v > o) *p = v; return o; }

// ---- CUDA runtime: streams and events do nothing, copies are immediate -----------------------------------------
typedef int cudaError_t;
typedef void* cudaStream_t;
typedef void* cudaEvent_t;
enum { cudaSuccess = 0 };
enum cudaMemcpyKind { cudaMemcpyHostToDevice, cudaMemcpyDeviceToHost, cudaMemcpyDeviceToDevice, cudaMemcpyDefault };
enum cudaStreamCaptureStatus { cudaStreamCaptureStatusNone = 0, cudaStreamCaptureStatusActive };
enum { cudaEventDisableTiming = 2, cudaStreamNonBlocking = 1, cudaHostAllocDefault = 0, cudaFuncAttributeMaxDynamicSharedMemorySize = 8 };
static inline cudaError_t cudaGetLastError() { return cudaSuccess; }
static inline const char* cudaGetErrorString(cudaError_t) { return "emulated"; }
static inline cudaError_t cudaMemsetAsync(void* p, int v, size_t n, cudaStream_t) { memset(p, v, n); return cudaSuccess; }
static inline cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, cudaMemcpyKind, cudaStream_t) { memcpy(d, s, n); return cudaSuccess; }
static inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
static inline cudaError_t cudaStreamWaitEvent(cudaStream_t, cudaEvent_t, unsigned) { return cudaSuccess; }
static inline cudaError_t cudaEventRecord(cudaEvent_t, cudaStream_t) { return cudaSuccess; }
static inline cudaError_t cudaEventCreate(cudaEvent_t* e) { *e = (void*)1; return cudaSuccess; }
static inline cudaError_t cudaEventCreateWithFlags(cudaEvent_t* e, unsigned) { *e = (void*)1; return cudaSuccess; }
static inline cudaError_t cudaEventSynchronize(cudaEvent_t) { return cudaSuccess; }
static inline cudaError_t cudaEventElapsedTime(float* ms, cudaEvent_t, cudaEvent_t) { *ms = 0.f; return cudaSuccess; }
static inline cudaError_t cudaStreamCreateWithFlags(cudaStream_t* s, unsigned) { *s = (void*)2; return cudaSuccess; }
static inline cudaError_t cudaStreamIsCapturing(cudaStream_t, cudaStreamCaptureStatus* st) { *st = cudaStreamCaptureStatusNone; return cudaSuccess; }
static inline cudaError_t cudaHostAlloc(void** p, size_t n, unsigned) { *p = malloc(n); return cudaSuccess; }
static inline cudaError_t cudaGetDevice(int* d) { *d = 0; return cudaSuccess; }
template <class F> static inline cudaError_t cudaFuncSetAttribute(F, int, int) { return cudaSuccess; }

// ---- the two CUB device algorithms the library calls ---------------------------------------------------------
namespace cub {
struct DeviceScan {
    template <class In, class Out>
    static cudaError_t InclusiveSum(void* temp, size_t& bytes, In in, Out out, int n, cudaStream_t = nullptr) {
        if (!temp) { bytes = 16; return cudaSuccess; }
        long long acc = 0;
        for (int i = 0; i < n; i++) { acc += in[i]; out[i] = (decltype(+out[0]))acc; }
        return cudaSuccess;
    }
};
struct DeviceRadixSort {
    template <class K, class V>
    static cudaError_t SortPairs(void* temp, size_t& bytes, const K* kin, K* kout, const V* vin, V* vout, long long n,
                                 int begin_bit = 0, int end_bit = 8 * (int)sizeof(K), cudaStream_t = nullptr) {
        if (!temp) { bytes = 16; return cudaSuccess; }
        std::vector<long long> idx((size_t)n);
        for (long long i = 0; i < n; i++) idx[(size_t)i] = i;
        const K mask = end_bit >= (int)(8 * sizeof(K)) ? ~(K)0 : (((K)1 << end_bit) - 1);
        std::stable_sort(idx.begin(), idx.end(), [&](long long a, long long b) { return ((kin[a] & mask) >> begin_bit) < ((kin[b] & mask) >> begin_bit); });
        for (long long i = 0; i < n; i++) { kout[i] = kin[idx[(size_t)i]]; vout[i] = vin[idx[(size_t)i]]; }
        return cudaSuccess;
    }
};
}  // namespace cub
