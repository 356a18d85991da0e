// TEST INFRASTRUCTURE: a minimal stand-in for <cuda_runtime.h> that lets the SIMT (CUDA-core) kernels of libcolddiff be
// compiled by g++ and EXECUTED ON THE CPU, one thread block at a time, every CUDA thread a fiber (tests/simt_cpu/simt.cpp).
// Barriers and warp shuffles are scheduling points; between two of them a thread runs alone, which is one of the legal
// interleavings of a race-free kernel.  Not supported (the build script turns them into aborts): inline PTX, TMA, wgmma.
// Purpose: check indexing / reductions / launch geometry of the SIMT kernels without a GPU.
#pragma once
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <algorithm>
#include <functional>

#ifndef __CUDACC__
#define __CUDACC__ 1
#endif
#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __noinline__
#define __launch_bounds__(...)
// statically sized shared arrays live in their own section so that the scheduler can poison them (NaN pattern) before every
// block: shared memory is uninitialised on the GPU, and a kernel that reads it before writing it then fails the parity tests
#define __shared__ static __attribute__((section("simt_shared")))
#define __constant__ static
#define __align__(n) alignas(n)
#ifndef __restrict__
#define __restrict__ __restrict
#endif

struct uint3 { unsigned x, y, z; };
struct dim3 {
  unsigned x, y, z;
  dim3(unsigned a = 1, unsigned b = 1, unsigned c = 1) : x(a), y(b), z(c) {}
  dim3(long long a) : x((unsigned)a), y(1), z(1) {}
  dim3(int a) : x((unsigned)a), y(1), z(1) {}
};
extern uint3 threadIdx, blockIdx;
extern dim3 blockDim, gridDim;
static const int warpSize = 32;

struct alignas(8) float2 { float x, y; };
struct float3 { float x, y, z; };
struct alignas(16) float4 { float x, y, z, w; };
struct alignas(8) int2 { int x, y; };
struct alignas(16) int4 { int x, y, z, w; };
struct alignas(16) uint4 { unsigned x, y, z, w; };
struct alignas(8) uint2 { unsigned x, y; };
struct uchar4 { unsigned char x, y, z, w; };
static inline float2 make_float2(float a, float b) { return float2{a, b}; }
static inline float4 make_float4(float a, float b, float c, float d) { return float4{a, b, c, d}; }
static inline int2 make_int2(int a, int b) { return int2{a, b}; }
static inline int4 make_int4(int a, int b, int c, int d) { return int4{a, b, c, d}; }
static inline uint4 make_uint4(unsigned a, unsigned b, unsigned c, unsigned d) { return uint4{a, b, c, d}; }
static inline uint2 make_uint2(unsigned a, unsigned b) { return uint2{a, b}; }

// ---- host runtime subset -----------------------------------------------------------------------------------------
typedef void* cudaStream_t;
typedef int cudaError_t;
enum { cudaSuccess = 0 };
enum cudaFuncAttribute { cudaFuncAttributeMaxDynamicSharedMemorySize = 8, cudaFuncAttributePreferredSharedMemoryCarveout = 9 };
enum cudaDeviceAttr { cudaDevAttrMultiProcessorCount = 16, cudaDevAttrMaxSharedMemoryPerBlockOptin = 97 };
enum cudaMemcpyKind { cudaMemcpyHostToHost = 0, cudaMemcpyHostToDevice = 1, cudaMemcpyDeviceToHost = 2, cudaMemcpyDeviceToDevice = 3, cudaMemcpyDefault = 4 };
static inline cudaError_t cudaGetLastError() { return cudaSuccess; }
static inline cudaError_t cudaPeekAtLastError() { return cudaSuccess; }
static inline const char* cudaGetErrorString(cudaError_t) { return "simt-cpu"; }
static inline cudaError_t cudaMemsetAsync(void* p, int v, size_t n, cudaStream_t = nullptr) { memset(p, v, n); return cudaSuccess; }
static inline cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, cudaMemcpyKind, cudaStream_t = nullptr) { memmove(d, s, n); return cudaSuccess; }
static inline cudaError_t cudaGetDevice(int* d) { *d = 0; return cudaSuccess; }
static inline cudaError_t cudaDeviceGetAttribute(int* v, cudaDeviceAttr a, int) {
  *v = (a == cudaDevAttrMultiProcessorCount) ? 132 : 232448; return cudaSuccess; }
template <class F> static inline cudaError_t cudaFuncSetAttribute(F, cudaFuncAttribute, int) { return cudaSuccess; }
int simt_occupancy();                                                    // settable from the test (default 2)
template <class F> static inline cudaError_t cudaOccupancyMaxActiveBlocksPerMultiprocessor(int* n, F, int, size_t) {
  *n = simt_occupancy(); return cudaSuccess; }
static inline cudaError_t cudaMemset2DAsync(void* p, size_t pitch, int v, size_t width, size_t height, cudaStream_t = nullptr) {
  for (size_t r = 0; r < height; ++r) memset((char*)p + r * pitch, v, width);
  return cudaSuccess; }
// driver-API corner used by the library (cuMemsetD32Async through cudaGetDriverEntryPoint)
typedef int CUresult;
typedef unsigned long long CUdeviceptr;
typedef void* CUstream;
enum { CUDA_SUCCESS = 0 };
enum cudaDriverEntryPointQueryResult { cudaDriverEntryPointSuccess = 0, cudaDriverEntryPointSymbolNotFound = 1 };
enum { cudaEnableDefault = 0 };
static inline CUresult simt_cuMemsetD32Async(CUdeviceptr p, unsigned v, size_t n, CUstream) {
  unsigned* q = reinterpret_cast<unsigned*>(p); for (size_t i = 0; i < n; ++i) q[i] = v; return CUDA_SUCCESS; }
static inline cudaError_t cudaGetDriverEntryPoint(const char* name, void** fn, int, cudaDriverEntryPointQueryResult* q) {
  if (strcmp(name, "cuMemsetD32Async") == 0) { *fn = (void*)&simt_cuMemsetD32Async; *q = cudaDriverEntryPointSuccess; return cudaSuccess; }
  *fn = nullptr; *q = cudaDriverEntryPointSymbolNotFound; return cudaSuccess; }
static inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
static inline cudaError_t cudaDeviceSynchronize() { return cudaSuccess; }

// ---- execution model -----------------------------------------------------------------------------------------------
namespace simt {
void launch(dim3 grid, dim3 block, size_t dyn_smem, const std::function<void()>& body);
void block_barrier();
void warp_barrier();
void* dyn_smem();
unsigned long long* warp_slot(int lane);        // exchange buffer of the calling thread's warp
int lane_id();
bool lane_alive(int lane);                      // lane exists in this block and has not returned
[[noreturn]] void unsupported(const char* what);
}
static inline void __syncthreads() { simt::block_barrier(); }
static inline void __syncwarp(unsigned = 0xffffffffu) { simt::warp_barrier(); }
static inline void __threadfence() {}
static inline void __threadfence_block() {}
static inline unsigned __activemask() { unsigned m = 0; for (int l = 0; l < 32; ++l) if (simt::lane_alive(l)) m |= 1u << l; return m; }

template <class T> static inline T simt_exchange(T v, int src) {
  static_assert(sizeof(T) <= 8, "shuffle of > 8 bytes");
  unsigned long long bits = 0; memcpy(&bits, &v, sizeof(T));
  *simt::warp_slot(simt::lane_id()) = bits;
  simt::warp_barrier();
  T r = v;
  if (src >= 0 && src < 32 && simt::lane_alive(src)) { unsigned long long b = *simt::warp_slot(src); memcpy(&r, &b, sizeof(T)); }
  simt::warp_barrier();
  return r;
}
template <class T> static inline T __shfl_xor_sync(unsigned, T v, int m, int width = 32) { (void)width; return simt_exchange(v, simt::lane_id() ^ m); }
template <class T> static inline T __shfl_down_sync(unsigned, T v, unsigned d, int width = 32) {
  const int l = simt::lane_id(), s = l + (int)d; return simt_exchange(v, (s / width == l / width) ? s : l); }
template <class T> static inline T __shfl_up_sync(unsigned, T v, unsigned d, int width = 32) {
  const int l = simt::lane_id(), s = l - (int)d; return simt_exchange(v, (s >= 0 && s / width == l / width) ? s : l); }
template <class T> static inline T __shfl_sync(unsigned, T v, int src, int width = 32) {
  const int l = simt::lane_id(); return simt_exchange(v, (l / width) * width + (src % width)); }
static inline unsigned __ballot_sync(unsigned, int pred) {
  unsigned m = 0; for (int l = 0; l < 32; ++l) { const int p = simt_exchange(pred, l); if (simt::lane_alive(l) && p) m |= 1u << l; } return m; }
static inline int __any_sync(unsigned m, int pred) { return __ballot_sync(m, pred) != 0; }
static inline int __all_sync(unsigned m, int pred) { return __ballot_sync(m, !pred) == 0; }

// atomics: one OS thread, so plain read-modify-write
template <class T> static inline T atomicAdd(T* p, T v) { T o = *p; *p = o + v; return o; }
static inline float atomicAdd(float* p, double v) { float o = *p; *p = o + (float)v; return o; }
template <class T> static inline T atomicMax(T* p, T v) { T o = *p; if (v > o) *p = v; return o; }
template <class T> static inline T atomicMin(T* p, T v) { T o = *p; if (v < o) *p = v; return o; }
template <class T> static inline T atomicExch(T* p, T v) { T o = *p; *p = v; return o; }
template <class T> static inline T atomicCAS(T* p, T c, T v) { T o = *p; if (o == c) *p = v; return o; }
template <class T> static inline T atomicOr(T* p, T v) { T o = *p; *p = o | v; return o; }

// math / bit intrinsics
// (glibc declares __expf & co. itself, hence macros)
#define __expf(x) expf(x)
#define __logf(x) logf(x)
#define __log2f(x) log2f(x)
#define __exp2f(x) exp2f(x)
#define __sinf(x) sinf(x)
#define __cosf(x) cosf(x)
#define __powf(x, y) powf(x, y)
#define __sincosf(x, s, c) sincosf(x, s, c)
static inline float __fdividef(float a, float b) { return a / b; }
static inline float __frcp_rn(float a) { return 1.0f / a; }
static inline float __fsqrt_rn(float a) { return sqrtf(a); }
static inline float rsqrtf(float x) { return 1.0f / sqrtf(x); }
static inline float __frsqrt_rn(float x) { return 1.0f / sqrtf(x); }
static inline float __fmaf_rn(float a, float b, float c) { return fmaf(a, b, c); }
static inline double __dmul_rn(double a, double b) { volatile double r = a * b; return r; }    // volatile: no contraction into an FMA
static inline double __dadd_rn(double a, double b) { volatile double r = a + b; return r; }
static inline double __dsub_rn(double a, double b) { volatile double r = a - b; return r; }
static inline float __fmul_rn(float a, float b) { return a * b; }
static inline float __fadd_rn(float a, float b) { return a + b; }
static inline float __saturatef(float x) { return x < 0.f ? 0.f : (x > 1.f ? 1.f : x); }
static inline int __float2int_rn(float x) { return (int)lrintf(x); }
static inline int __float2int_rd(float x) { return (int)floorf(x); }
static inline int __float2int_rz(float x) { return (int)x; }
static inline unsigned __float2uint_rn(float x) { return (unsigned)lrintf(x); }
static inline float __int2float_rn(int x) { return (float)x; }
static inline float __uint2float_rn(unsigned x) { return (float)x; }
static inline float __uint_as_float(unsigned u) { float f; memcpy(&f, &u, 4); return f; }
static inline unsigned __float_as_uint(float f) { unsigned u; memcpy(&u, &f, 4); return u; }
static inline float __int_as_float(int u) { float f; memcpy(&f, &u, 4); return f; }
static inline int __float_as_int(float f) { int u; memcpy(&u, &f, 4); return u; }
static inline int __popc(unsigned x) { return __builtin_popcount(x); }
static inline int __clz(int x) { return x ? __builtin_clz((unsigned)x) : 32; }
static inline int __ffs(int x) { return __builtin_ffs(x); }
static inline unsigned __umulhi(unsigned a, unsigned b) { return (unsigned)(((unsigned long long)a * b) >> 32); }
template <class T> static inline T __ldg(const T* p) { return *p; }
template <class T> static inline T __ldcs(const T* p) { return *p; }
template <class T> static inline void __stcs(T* p, T v) { *p = v; }
static inline size_t __cvta_generic_to_shared(const void* p) { return (size_t)p; }
#include <type_traits>
template <class A, class B> static inline typename std::common_type<A, B>::type min(A a, B b) {
  typedef typename std::common_type<A, B>::type T; return (T)b < (T)a ? (T)b : (T)a; }
template <class A, class B> static inline typename std::common_type<A, B>::type max(A a, B b) {
  typedef typename std::common_type<A, B>::type T; return (T)a < (T)b ? (T)b : (T)a; }
