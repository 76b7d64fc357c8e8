// cusim -- a functional simulator for the CUDA subset libb200timg's kernels use, so that kernel LOGIC
// (indexing, scans, shuffles, barriers, byte formatting) can be debugged against the oracle on a box
// without a GPU.  DEVELOPMENT / TEST TOOL ONLY: it is never linked into timg_b200/libb200timg.so and
// the product never loads it.  It says nothing about performance, memory ordering or races.
//
// How it works: every .cu file is compiled by g++ with this header standing in for <cuda_runtime.h>
// (tools/cusim/build.py rewrites  k<<<g,b,s,st>>>(a...)  into  cusim::Launcher{g,b,s,st}.run(k, a...)).
// A launch runs the blocks one after the other in index order; the threads of a block are fibers that
// are switched at __syncthreads / warp collectives / __nanosleep.  __shared__ becomes `static`
// (blocks never overlap in time), device memory is host memory, streams are synchronous.
#pragma once
#define CUSIM 1
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <type_traits>
#include <utility>

// ---- keywords
#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __shared__ static
#define __constant__ static
#define __launch_bounds__(...)
#define __align__(n) __attribute__((aligned(n)))
#ifndef __CUDACC_VER_MAJOR__
#define __CUDACC_VER_MAJOR__ 12
#endif

// ---- vector types
struct uint3 { unsigned x, y, z; };
struct dim3 {
    unsigned x, y, z;
    dim3(unsigned a = 1, unsigned b = 1, unsigned c = 1) : x(a), y(b), z(c) {}
};
struct alignas(8) float2 { float x, y; };
struct alignas(16) float4 { float x, y, z, w; };
struct alignas(8) uint2 { unsigned x, y; };
struct alignas(16) uint4 { unsigned x, y, z, w; };
struct alignas(8) int2 { int x, y; };
struct alignas(16) int4 { int x, y, z, w; };
struct alignas(4) uchar4 { unsigned char x, y, z, w; };
struct alignas(2) uchar2 { unsigned char x, y; };
struct alignas(4) ushort2 { unsigned short x, y; };
struct alignas(16) ulonglong2 { unsigned long long x, y; };
static inline float2 make_float2(float a, float b) { return float2{a, b}; }
static inline float4 make_float4(float a, float b, float c, float d) { return float4{a, b, c, d}; }
static inline uint2 make_uint2(unsigned a, unsigned b) { return uint2{a, b}; }
static inline uint4 make_uint4(unsigned a, unsigned b, unsigned c, unsigned d) { return uint4{a, b, c, d}; }
static inline int2 make_int2(int a, int b) { return int2{a, b}; }
static inline int4 make_int4(int a, int b, int c, int d) { return int4{a, b, c, d}; }
static inline uchar4 make_uchar4(unsigned char a, unsigned char b, unsigned char c, unsigned char d) { return uchar4{a, b, c, d}; }
static inline ulonglong2 make_ulonglong2(unsigned long long a, unsigned long long b) { return ulonglong2{a, b}; }

// ---- runtime API (host memory, synchronous)
typedef int cudaError_t;
enum { cudaSuccess = 0, cudaErrorMemoryAllocation = 2, cudaErrorInvalidValue = 1 };
typedef struct cusim_stream *cudaStream_t;
typedef struct cusim_event *cudaEvent_t;
enum cudaMemcpyKind { cudaMemcpyHostToHost = 0, cudaMemcpyHostToDevice = 1, cudaMemcpyDeviceToHost = 2, cudaMemcpyDeviceToDevice = 3, cudaMemcpyDefault = 4 };
enum { cudaStreamNonBlocking = 1, cudaEventDisableTiming = 2, cudaEventDefault = 0 };
enum cudaFuncAttribute { cudaFuncAttributeMaxDynamicSharedMemorySize = 8, cudaFuncAttributePreferredSharedMemoryCarveout = 9 };
struct cudaDeviceProp { char name[256]; int multiProcessorCount; int major, minor; size_t totalGlobalMem; };

static inline cudaError_t cudaGetDeviceCount(int *n) { *n = 1; return cudaSuccess; }
static inline cudaError_t cudaSetDevice(int) { return cudaSuccess; }
static inline cudaError_t cudaGetDevice(int *d) { *d = 0; return cudaSuccess; }
static inline cudaError_t cudaGetLastError() { return cudaSuccess; }
static inline cudaError_t cudaPeekAtLastError() { return cudaSuccess; }
static inline const char *cudaGetErrorString(cudaError_t) { return "cusim"; }
static inline cudaError_t cudaGetDeviceProperties(cudaDeviceProp *p, int) {
    memset(p, 0, sizeof *p); strcpy(p->name, "cusim"); p->multiProcessorCount = 132; p->major = 9; p->minor = 0;
    return cudaSuccess;
}
static inline cudaError_t cudaMalloc(void **p, size_t n) { *p = aligned_alloc(256, (n + 255) / 256 * 256 + 256); return *p ? cudaSuccess : cudaErrorMemoryAllocation; }
template <class T> static inline cudaError_t cudaMalloc(T **p, size_t n) { return cudaMalloc(reinterpret_cast<void **>(p), n); }
static inline cudaError_t cudaFree(void *p) { free(p); return cudaSuccess; }
static inline cudaError_t cudaMallocHost(void **p, size_t n) { return cudaMalloc(p, n); }
template <class T> static inline cudaError_t cudaMallocHost(T **p, size_t n) { return cudaMalloc(reinterpret_cast<void **>(p), n); }
static inline cudaError_t cudaFreeHost(void *p) { free(p); return cudaSuccess; }
static inline cudaError_t cudaMemcpyAsync(void *d, const void *s, size_t n, cudaMemcpyKind, cudaStream_t = nullptr) { memmove(d, s, n); return cudaSuccess; }
static inline cudaError_t cudaMemcpy(void *d, const void *s, size_t n, cudaMemcpyKind) { memmove(d, s, n); return cudaSuccess; }
static inline cudaError_t cudaMemsetAsync(void *d, int v, size_t n, cudaStream_t = nullptr) { memset(d, v, n); return cudaSuccess; }
static inline cudaError_t cudaMemset(void *d, int v, size_t n) { memset(d, v, n); return cudaSuccess; }
static inline cudaError_t cudaMemset2DAsync(void *d, size_t pitch, int v, size_t w, size_t h, cudaStream_t = nullptr) {
    for (size_t r = 0; r < h; ++r) memset(static_cast<char *>(d) + r * pitch, v, w);
    return cudaSuccess;
}
static inline cudaError_t cudaMemcpy2DAsync(void *d, size_t dp, const void *s, size_t sp, size_t w, size_t h, cudaMemcpyKind, cudaStream_t = nullptr) {
    for (size_t r = 0; r < h; ++r) memmove(static_cast<char *>(d) + r * dp, static_cast<const char *>(s) + r * sp, w);
    return cudaSuccess;
}
static inline cudaError_t cudaStreamCreateWithFlags(cudaStream_t *s, unsigned) { *s = reinterpret_cast<cudaStream_t>(malloc(8)); return cudaSuccess; }
static inline cudaError_t cudaStreamCreate(cudaStream_t *s) { return cudaStreamCreateWithFlags(s, 0); }
static inline cudaError_t cudaDeviceGetStreamPriorityRange(int *least, int *greatest) { *least = 0; *greatest = -5; return cudaSuccess; }
static inline cudaError_t cudaStreamCreateWithPriority(cudaStream_t *s, unsigned f, int) { return cudaStreamCreateWithFlags(s, f); }
static inline cudaError_t cudaStreamDestroy(cudaStream_t s) { free(s); return cudaSuccess; }
static inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
static inline cudaError_t cudaDeviceSynchronize() { return cudaSuccess; }
static inline cudaError_t cudaStreamWaitEvent(cudaStream_t, cudaEvent_t, unsigned = 0) { return cudaSuccess; }
static inline cudaError_t cudaEventCreate(cudaEvent_t *e) { *e = reinterpret_cast<cudaEvent_t>(malloc(8)); return cudaSuccess; }
static inline cudaError_t cudaEventCreateWithFlags(cudaEvent_t *e, unsigned) { return cudaEventCreate(e); }
static inline cudaError_t cudaEventDestroy(cudaEvent_t e) { free(e); return cudaSuccess; }
static inline cudaError_t cudaEventRecord(cudaEvent_t, cudaStream_t = nullptr) { return cudaSuccess; }
static inline cudaError_t cudaEventSynchronize(cudaEvent_t) { return cudaSuccess; }
static inline cudaError_t cudaEventElapsedTime(float *ms, cudaEvent_t, cudaEvent_t) { *ms = 0.0f; return cudaSuccess; }
template <class F> static inline cudaError_t cudaFuncSetAttribute(F, cudaFuncAttribute, int) { return cudaSuccess; }

// ---- the scheduler (cusim.cc)
namespace cusim {
struct Fiber {
    uint3 tid;
    int linear, lane, warp;
    void *sp;
    int state;          // 0 runnable, 1 done
};
extern Fiber *cur;
extern uint3 g_blockIdx;
extern dim3 g_blockDim, g_gridDim;
void yield();
void barrier(int pred, int *out_or, int *out_and, int *out_count);
unsigned long long warp_exchange(unsigned mask, unsigned long long v, int kind, int arg);   // kind: 0 shfl idx, 1 up, 2 down, 3 xor, 4 ballot, 5 match_any, 6 sync
void run_grid(dim3 grid, dim3 block, size_t smem, void (*thunk)(void *), void *closure);

struct Launcher {
    dim3 grid, block;
    size_t smem;
    cudaStream_t stream;
    Launcher(dim3 g, dim3 b, size_t s = 0, cudaStream_t st = nullptr) : grid(g), block(b), smem(s), stream(st) {}
    template <class K, class... A>
    void run(K kernel, A &&...args) {
        auto call = [&]() { kernel(args...); };
        using C = decltype(call);
        run_grid(grid, block, smem, [](void *c) { (*static_cast<C *>(c))(); }, &call);
    }
};
}  // namespace cusim

#define threadIdx (cusim::cur->tid)
#define blockIdx (cusim::g_blockIdx)
#define blockDim (cusim::g_blockDim)
#define gridDim (cusim::g_gridDim)
static const int warpSize = 32;

// ---- synchronisation and warp collectives
static inline void __syncthreads() { cusim::barrier(0, nullptr, nullptr, nullptr); }
static inline int __syncthreads_or(int p) { int r; cusim::barrier(p, &r, nullptr, nullptr); return r; }
static inline int __syncthreads_and(int p) { int r; cusim::barrier(p, nullptr, &r, nullptr); return r; }
static inline int __syncthreads_count(int p) { int r; cusim::barrier(p, nullptr, nullptr, &r); return r; }
static inline void __syncwarp(unsigned mask = 0xffffffffu) { cusim::warp_exchange(mask, 0, 6, 0); }
static inline void __threadfence() {}
static inline void __threadfence_block() {}
static inline void __threadfence_system() {}
static inline void __nanosleep(unsigned) { cusim::yield(); }
static inline unsigned __activemask() { return 0xffffffffu; }

template <class T> static inline unsigned long long cusim_bits(T v) {
    static_assert(sizeof(T) <= 8, "shuffle of > 8 bytes");
    unsigned long long b = 0; memcpy(&b, &v, sizeof(T)); return b;
}
template <class T> static inline T cusim_unbits(unsigned long long b) { T v; memcpy(&v, &b, sizeof(T)); return v; }
template <class T> static inline T __shfl_sync(unsigned m, T v, int src, int = 32) { return cusim_unbits<T>(cusim::warp_exchange(m, cusim_bits(v), 0, src)); }
template <class T> static inline T __shfl_up_sync(unsigned m, T v, unsigned d, int = 32) { return cusim_unbits<T>(cusim::warp_exchange(m, cusim_bits(v), 1, (int)d)); }
template <class T> static inline T __shfl_down_sync(unsigned m, T v, unsigned d, int = 32) { return cusim_unbits<T>(cusim::warp_exchange(m, cusim_bits(v), 2, (int)d)); }
template <class T> static inline T __shfl_xor_sync(unsigned m, T v, int x, int = 32) { return cusim_unbits<T>(cusim::warp_exchange(m, cusim_bits(v), 3, x)); }
static inline unsigned __ballot_sync(unsigned m, int p) { return (unsigned)cusim::warp_exchange(m, p ? 1 : 0, 4, 0); }
static inline int __any_sync(unsigned m, int p) { return __ballot_sync(m, p) != 0; }
static inline int __all_sync(unsigned m, int p) { return __ballot_sync(m, !p) == 0; }
template <class T> static inline unsigned __match_any_sync(unsigned m, T v) { return (unsigned)cusim::warp_exchange(m, cusim_bits(v), 5, 0); }
template <class T> static inline T cusim_reduce(unsigned m, T v, int op) {   // redux.sync: 0 add 1 min 2 max 3 or 4 and
    T r = v;
    for (int d = 1; d < 32; d <<= 1) {   // butterfly over all lanes of the mask (mask must be full or lanes symmetric)
        T o = __shfl_xor_sync(m, r, d);
        switch (op) { case 0: r = r + o; break; case 1: r = o < r ? o : r; break; case 2: r = o > r ? o : r; break; case 3: r = r | o; break; default: r = r & o; }
    }
    return r;
}
static inline unsigned __reduce_add_sync(unsigned m, unsigned v) { return cusim_reduce(m, v, 0); }
static inline unsigned __reduce_min_sync(unsigned m, unsigned v) { return cusim_reduce(m, v, 1); }
static inline unsigned __reduce_max_sync(unsigned m, unsigned v) { return cusim_reduce(m, v, 2); }
static inline int __reduce_add_sync(unsigned m, int v) { return cusim_reduce(m, v, 0); }
static inline int __reduce_min_sync(unsigned m, int v) { return cusim_reduce(m, v, 1); }
static inline int __reduce_max_sync(unsigned m, int v) { return cusim_reduce(m, v, 2); }
static inline unsigned __reduce_or_sync(unsigned m, unsigned v) { return cusim_reduce(m, v, 3); }
static inline unsigned __reduce_and_sync(unsigned m, unsigned v) { return cusim_reduce(m, v, 4); }

// ---- atomics (one OS thread: plain read-modify-write)
template <class T, class U> static inline T atomicAdd(T *p, U v) { T o = *p; *p = (T)(o + (T)v); return o; }
template <class T, class U> static inline T atomicSub(T *p, U v) { T o = *p; *p = (T)(o - (T)v); return o; }
template <class T, class U> static inline T atomicOr(T *p, U v) { T o = *p; *p = (T)(o | (T)v); return o; }
template <class T, class U> static inline T atomicAnd(T *p, U v) { T o = *p; *p = (T)(o & (T)v); return o; }
template <class T, class U> static inline T atomicXor(T *p, U v) { T o = *p; *p = (T)(o ^ (T)v); return o; }
template <class T, class U> static inline T atomicMin(T *p, U v) { T o = *p; if ((T)v < o) *p = (T)v; return o; }
template <class T, class U> static inline T atomicMax(T *p, U v) { T o = *p; if ((T)v > o) *p = (T)v; return o; }
template <class T, class U> static inline T atomicExch(T *p, U v) { T o = *p; *p = (T)v; return o; }
template <class T, class U, class V> static inline T atomicCAS(T *p, U c, V v) { T o = *p; if (o == (T)c) *p = (T)v; return o; }
template <class T, class U> static inline T atomicAdd(volatile T *p, U v) { T o = *p; *p = (T)(o + (T)v); return o; }
template <class T, class U> static inline T atomicMax(volatile T *p, U v) { T o = *p; if ((T)v > o) *p = (T)v; return o; }

// ---- arithmetic intrinsics (x86-64 SSE2 float ops are IEEE round-to-nearest; build with -ffp-contract=off)
static inline float __fmul_rn(float a, float b) { return a * b; }
static inline float __fadd_rn(float a, float b) { return a + b; }
static inline float __fsub_rn(float a, float b) { return a - b; }
static inline float __fdiv_rn(float a, float b) { return a / b; }
static inline float __frcp_rn(float a) { return 1.0f / a; }
static inline float __fsqrt_rn(float a) { return sqrtf(a); }
static inline float __fmaf_rn(float a, float b, float c) { return fmaf(a, b, c); }
static inline double __dmul_rn(double a, double b) { return a * b; }
static inline double __dadd_rn(double a, double b) { return a + b; }
static inline float __saturatef(float a) { return a != a ? 0.0f : (a < 0.0f ? 0.0f : (a > 1.0f ? 1.0f : a)); }
static inline unsigned __float2uint_rz(float f) { if (f != f || f <= 0.0f) return 0u; if (f >= 4294967296.0f) return 0xffffffffu; return (unsigned)f; }
static inline int __float2int_rz(float f) { if (f != f) return 0; if (f >= 2147483648.0f) return 0x7fffffff; if (f <= -2147483648.0f) return (int)0x80000000; return (int)f; }
static inline int __float2int_rn(float f) { if (f != f) return 0; return (int)lrintf(f); }
static inline unsigned __float2uint_rn(float f) { if (f != f || f <= 0.0f) return 0u; return (unsigned)llrintf(f); }
static inline float __int2float_rn(int v) { return (float)v; }
static inline float __uint2float_rn(unsigned v) { return (float)v; }
static inline float __uint_as_float(unsigned u) { float f; memcpy(&f, &u, 4); return f; }
static inline unsigned __float_as_uint(float f) { unsigned u; memcpy(&u, &f, 4); return u; }
static inline float __int_as_float(int u) { float f; memcpy(&f, &u, 4); return f; }
static inline int __float_as_int(float f) { int u; memcpy(&u, &f, 4); return u; }
static inline int __popc(unsigned v) { return __builtin_popcount(v); }
static inline int __popcll(unsigned long long v) { return __builtin_popcountll(v); }
static inline int __ffs(int v) { return __builtin_ffs(v); }
static inline int __ffsll(long long v) { return __builtin_ffsll(v); }
static inline int __clz(int v) { return v ? __builtin_clz((unsigned)v) : 32; }
static inline int __clzll(long long v) { return v ? __builtin_clzll((unsigned long long)v) : 64; }
static inline unsigned __brev(unsigned v) { unsigned r = 0; for (int i = 0; i < 32; ++i) r |= ((v >> i) & 1u) << (31 - i); return r; }
static inline unsigned __umulhi(unsigned a, unsigned b) { return (unsigned)(((unsigned long long)a * b) >> 32); }
static inline int __mulhi(int a, int b) { return (int)(((long long)a * b) >> 32); }
static inline unsigned __funnelshift_r(unsigned lo, unsigned hi, unsigned s) { const unsigned long long v = ((unsigned long long)hi << 32) | lo; return (unsigned)(v >> (s & 31)); }
static inline unsigned __funnelshift_l(unsigned lo, unsigned hi, unsigned s) { const unsigned long long v = ((unsigned long long)hi << 32) | lo; return (unsigned)((v << (s & 31)) >> 32); }
static inline unsigned __byte_perm(unsigned a, unsigned b, unsigned s) {
    const unsigned long long v = ((unsigned long long)b << 32) | a;
    unsigned r = 0;
    for (int i = 0; i < 4; ++i) {
        const unsigned sel = (s >> (4 * i)) & 0xf;
        unsigned byte = (unsigned)(v >> (8 * (sel & 7))) & 0xff;
        if (sel & 8) byte = (byte & 0x80) ? 0xff : 0x00;
        r |= byte << (8 * i);
    }
    return r;
}
template <class T> static inline T __ldg(const T *p) { return *p; }
template <class T> static inline T __ldcg(const T *p) { return *p; }
template <class T> static inline T __ldcs(const T *p) { return *p; }
template <class T> static inline T __ldca(const T *p) { return *p; }
template <class T> static inline T __ldcv(const T *p) { return *p; }
template <class T> static inline void __stcg(T *p, T v) { *p = v; }
template <class T> static inline void __stcs(T *p, T v) { *p = v; }
template <class T> static inline void __stwt(T *p, T v) { *p = v; }
static inline size_t __cvta_generic_to_shared(const void *p) { return (size_t)p; }

// DPX / SIMD-in-a-word
static inline int cusim_s16(unsigned v) { return (int)(short)(v & 0xffff); }
static inline int __viaddmin_s32_relu(int a, int b, int c) { int s = a + b; s = s < c ? s : c; return s > 0 ? s : 0; }
static inline int __viaddmax_s32_relu(int a, int b, int c) { int s = a + b; s = s > c ? s : c; return s > 0 ? s : 0; }
static inline int __viaddmin_s32(int a, int b, int c) { int s = a + b; return s < c ? s : c; }
static inline int __viaddmax_s32(int a, int b, int c) { int s = a + b; return s > c ? s : c; }
static inline int __vimax3_s32(int a, int b, int c) { int m = a > b ? a : b; return m > c ? m : c; }
static inline int __vimin3_s32(int a, int b, int c) { int m = a < b ? a : b; return m < c ? m : c; }
static inline int __vimax_s32_relu(int a, int b) { int m = a > b ? a : b; return m > 0 ? m : 0; }
static inline int __vimin_s32_relu(int a, int b) { int m = a < b ? a : b; return m > 0 ? m : 0; }
static inline unsigned __viaddmin_s16x2_relu(unsigned a, unsigned b, unsigned c) {
    unsigned r = 0;
    for (int h = 0; h < 2; ++h) {
        int s = (int)(short)(cusim_s16(a >> (16 * h)) + cusim_s16(b >> (16 * h)));   // 16-bit wrap-around add
        const int lim = cusim_s16(c >> (16 * h));
        s = s < lim ? s : lim; s = s > 0 ? s : 0;
        r |= ((unsigned)s & 0xffff) << (16 * h);
    }
    return r;
}
static inline unsigned __vabsdiffu4(unsigned a, unsigned b) {
    unsigned r = 0;
    for (int k = 0; k < 4; ++k) { const int x = (a >> (8 * k)) & 255, y = (b >> (8 * k)) & 255; r |= (unsigned)(x > y ? x - y : y - x) << (8 * k); }
    return r;
}
static inline unsigned __dp4a(unsigned a, unsigned b, unsigned c) {
    for (int k = 0; k < 4; ++k) c += ((a >> (8 * k)) & 255) * ((b >> (8 * k)) & 255);
    return c;
}
static inline unsigned __vadd2(unsigned a, unsigned b) { return (((a & 0xffff) + (b & 0xffff)) & 0xffff) | (((a >> 16) + (b >> 16)) << 16); }
static inline unsigned __vsub2(unsigned a, unsigned b) { return (((a & 0xffff) - (b & 0xffff)) & 0xffff) | (((a >> 16) - (b >> 16)) << 16); }

// ---- min / max overloads (CUDA's global-namespace set)
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
static inline unsigned long long min(unsigned long long a, unsigned long long b) { return a < b ? a : b; }
static inline unsigned long long max(unsigned long long a, unsigned long long b) { return a > b ? a : b; }
static inline long min(long a, long b) { return a < b ? a : b; }
static inline long max(long a, long b) { return a > b ? a : b; }
static inline unsigned long min(unsigned long a, unsigned long b) { return a < b ? a : b; }
static inline unsigned long max(unsigned long a, unsigned long b) { return a > b ? a : b; }
static inline float min(float a, float b) { return fminf(a, b); }
static inline float max(float a, float b) { return fmaxf(a, b); }
