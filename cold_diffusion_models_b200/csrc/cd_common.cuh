// Internal helpers shared by the libcolddiff translation units (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include "../../include/colddiff.h"

#ifndef CD_HOST_ONLY
#if !defined(__CUDA_ARCH__) || (__CUDA_ARCH__ >= 900)
#else
#error "libcolddiff is written for sm_90a only"
#endif
#endif

// ---- error plumbing (thread-local text, negative return codes) --------------------------------
void cd_set_error(const char* fmt, ...);
#define CD_FAIL(...) do { cd_set_error(__VA_ARGS__); return -1; } while (0)
#define CD_REQUIRE(cond, ...) do { if (!(cond)) { cd_set_error(__VA_ARGS__); return -1; } } while (0)
#define CD_CUDA(expr) do { cudaError_t e__ = (expr); if (e__ != cudaSuccess) { \
    cd_set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__), __FILE__, __LINE__); return -2; } } while (0)
#define CD_LAUNCH_CHECK() CD_CUDA(cudaGetLastError())

static inline int cd_cdiv(long long a, long long b) { return (int)((a + b - 1) / b); }

// SM count of the current device for the grid sizes and grid-size heuristics of every kernel (queried once; 132 = H100 SXM if
// the query fails, which only changes how work is split)
static inline int cd_num_sms() {
  static int n = 0;
  if (n <= 0) {
    int dev = 0, v = 0;
    n = (cudaGetDevice(&dev) == cudaSuccess && cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && v > 0)
            ? v : 132;
  }
  return n;
}

// final_proj.cu: the final 1x1 projection through a shared-memory tile; returns 1 when not taken
int cd_conv1x1_to_nchw_tiled(const float* x, int ld, long long npix, int HW, int C, const float* w, const float* bias, int Co,
                             const float* resid, float* out, cudaStream_t st);
// layernorm_multi.cu: C <= 128 LayerNorm forward with several pixels per lane group in flight; returns 1 when not taken
int cd_layernorm_fwd_multi(const float* x, int x_ld, long long npix, int C, const float* g, const float* beta, float eps,
                           float* y, int y_ld, float* stats, int round_tf32, cudaStream_t st);
// linattn_small.cu: shared-memory-staged variants of the two per-(batch element, head) LinearAttention kernels, taken when
// cd_linattn_aligned(a, b) (both pointers 16-byte aligned; a null pointer counts as aligned)
int cd_linattn_aligned(const void* a, const void* b);
int cd_linattn_weff_staged(const float* ctx, const float* ksum, const float* w_out, int B, int dim, float scale,
                           int round_tf32, float* weff, cudaStream_t st);
int cd_linattn_bwd_small_staged(const float* dweff, const float* ctx, const float* ksum, const float* w_out, int B, int dim,
                                float scale, float* dw_out, float* dctxn, float* rowdot, cudaStream_t st);

// elementwise.cu: split-plane GroupNorm, taken by cd_groupnorm_fwd / cd_groupnorm_bwd for planes of more than
// CD_GN_SPLIT_MIN_HW pixels (smaller planes keep one CTA per image; both take their statistics from cd_gn_chunk_stats below).
// A chunk is GN_SPLIT_ITERS pixels per pixel lane of a 512-thread CTA.  cd_gn_workspace returns a cached per-(device, stream)
// device buffer of at least `bytes`.  cd_gn_split_stats leaves the per-chunk (mean, M2) partials in part[B][nch][groups][2]
// and (mean, rstd) of x + cond in stats[B][groups][2].
constexpr long long CD_GN_SPLIT_MIN_HW = 128 * 128;
constexpr int GN_SPLIT_ITERS = 16;
int cd_gn_split_chunk(int C);
int cd_gn_workspace(size_t bytes, cudaStream_t st, float** ws);
int cd_gn_split_stats(const float* x, int x_ld, int B, long long HW, int C, int groups, const float* cond, int cond_ld, float eps,
                      float* part, float* stats, cudaStream_t st);

// linattn_bwd.cu: per-pixel LinearAttention backward on mma.sync; returns 1 when the CUDA-core kernel should run
int cd_linattn_bwd_kv_mma(const float* qkv, int ld, int B, int n, const float* kmax, const float* ksum, const float* dctxn,
                          const float* rowdot, float* dqkv, int dld, cudaStream_t st);

#ifdef __CUDACC__
// ---- small device helpers ---------------------------------------------------------------------
__device__ __forceinline__ float cd_gelu(float x) {           // exact erf GELU == nn.GELU()
  return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f));
}
__device__ __forceinline__ float cd_gelu_grad(float x) {
  const float cdf = 0.5f * (1.0f + erff(x * 0.70710678118654752440f));
  const float pdf = 0.39894228040143267794f * __expf(-0.5f * x * x);
  return cdf + x * pdf;
}
__device__ __forceinline__ float cd_round_tf32(float x) {     // RN (ties away), as cvt.rna.tf32.f32
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}
// asynchronous 4-byte global->shared copy (LDGSTS); !valid zero-fills the destination (src-size 0)
__device__ __forceinline__ void cd_cp_async4(float* smem_dst, const float* gsrc, bool valid) {
  const unsigned d = static_cast<unsigned>(__cvta_generic_to_shared(smem_dst));
  const int sz = valid ? 4 : 0;
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" :: "r"(d), "l"(gsrc), "r"(sz) : "memory");
}
// asynchronous 16-byte global->shared copy (LDGSTS.128, L2 only); !valid zero-fills the destination
__device__ __forceinline__ void cd_cp_async16(float* smem_dst, const float* gsrc, bool valid) {
  const unsigned d = static_cast<unsigned>(__cvta_generic_to_shared(smem_dst));
  const int sz = valid ? 16 : 0;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" :: "r"(d), "l"(gsrc), "r"(sz) : "memory");
}
__device__ __forceinline__ void cd_cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }
__device__ __forceinline__ float cd_warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
// GroupNorm: pixels of chunk k (cp pixels from k * cp; ragged last chunk) that pixel lane pl of np visits (pl, pl + np, ...)
__device__ __forceinline__ int cd_gn_lane_count(long long HW, int k, int cp, int pl, int np) {
  const long long rem = HW - static_cast<long long>(k) * cp;
  const int n = rem < cp ? static_cast<int>(rem) : cp;
  return pl < n ? (n - pl + np - 1) / np : 0;
}
// merge (nb, meanb, m2b) into (n, mean, m2) (Chan's formula for counts, means and sums of squared deviations)
__device__ __forceinline__ void cd_chan_merge(float& n, float& mean, float& m2, float nb, float meanb, float m2b) {
  if (nb == 0.f) return;
  const float nn = n + nb, d = meanb - mean;
  mean += d * (nb / nn);
  m2 += m2b + d * d * (n * nb / nn);
  n = nn;
}
// fixed-order tree over the lanes of a warp; lane 0 ends with the merge of all 32
__device__ __forceinline__ void cd_chan_warp_merge(float& n, float& mean, float& m2) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float nb = __shfl_down_sync(0xffffffffu, n, o), mb = __shfl_down_sync(0xffffffffu, mean, o);
    const float qb = __shfl_down_sync(0xffffffffu, m2, o);
    if ((threadIdx.x & 31) + o < 32 && ((threadIdx.x & 31) & (2 * o - 1)) == 0) cd_chan_merge(n, mean, m2, nb, mb, qb);
  }
}
// GroupNorm statistics of x + cond over chunk k of image b (pixels [k * cp, min((k + 1) * cp, HW))), by a CTA of at most 512
// threads mapped thread -> (pixel lane, channel quad) as in groupnorm_kernel (elementwise.cu).  Each thread keeps shifted sums
// about its first value, formed per block of GN_SPLIT_ITERS values and then added up: a one-CTA plane gives a thread up to
// 128² / np values (16384 at C = 2048), and the two levels keep the fp32 rounding of those sums near that of the split path's
// 16-value chunks.  One warp per group then merges the thread-channel (count, mean, M2) triples with Chan's formula in a
// fixed order (no E[x^2] - mean^2 cancellation for inputs with a large mean, no float atomics, the same bits whatever order the
// threads run in), and its lane 0 calls out(g, count, mean, M2).  tm / tq are [4][512] shared scratch.  The split-plane path
// runs it per chunk; the one-CTA kernels pass the whole plane as chunk 0 through cd_gn_plane_stats.
template <class Out>
__device__ __forceinline__ void cd_gn_chunk_stats(const float* __restrict__ x, int x_ld, long long HW, int C, int groups,
                                                  const float* __restrict__ cond, int cond_ld, int b, int k, int cp,
                                                  float (*tm)[512], float (*tq)[512], Out out) {
  const int nq = C >> 2, cg = C / groups;
  const int q = threadIdx.x % nq, pl = threadIdx.x / nq, np = blockDim.x / nq;
  const long long base = static_cast<long long>(b) * HW + static_cast<long long>(k) * cp;
  if (pl < np) {
    float4 cadd = make_float4(0.f, 0.f, 0.f, 0.f);
    if (cond) cadd = *reinterpret_cast<const float4*>(cond + static_cast<long long>(b) * cond_ld + q * 4);
    const int cnt = cd_gn_lane_count(HW, k, cp, pl, np);
    float sh[4] = {0.f, 0.f, 0.f, 0.f}, s[4] = {0.f, 0.f, 0.f, 0.f}, s2[4] = {0.f, 0.f, 0.f, 0.f};
    for (int i0 = 0; i0 < cnt; i0 += GN_SPLIT_ITERS) {     // a split chunk is one block
      const int m = cnt - i0 < GN_SPLIT_ITERS ? cnt - i0 : GN_SPLIT_ITERS;
      float bs[4] = {0.f, 0.f, 0.f, 0.f}, bs2[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll 4
      for (int i = i0; i < i0 + m; ++i) {
        float4 v = *reinterpret_cast<const float4*>(x + (base + pl + static_cast<long long>(i) * np) * x_ld + q * 4);
        const float w[4] = {v.x + cadd.x, v.y + cadd.y, v.z + cadd.z, v.w + cadd.w};
        if (i == 0) for (int j = 0; j < 4; ++j) sh[j] = w[j];
#pragma unroll
        for (int j = 0; j < 4; ++j) { const float d = w[j] - sh[j]; bs[j] += d; bs2[j] += d * d; }
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) { s[j] += bs[j]; s2[j] += bs2[j]; }
    }
    const float inv = cnt > 0 ? 1.f / static_cast<float>(cnt) : 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      tm[j][threadIdx.x] = sh[j] + s[j] * inv;
      tq[j][threadIdx.x] = fmaxf(s2[j] - s[j] * s[j] * inv, 0.f);
    }
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  for (int g = warp; g < groups; g += nw) {
    float n = 0.f, mean = 0.f, m2 = 0.f;
    for (int e = lane; e < cg * np; e += 32) {           // entry e: channel g*cg + e/np of pixel lane e%np
      const int c = g * cg + e / np, pp = e % np, t = pp * nq + (c >> 2);
      cd_chan_merge(n, mean, m2, static_cast<float>(cd_gn_lane_count(HW, k, cp, pp, np)), tm[c & 3][t], tq[c & 3][t]);
    }
    cd_chan_warp_merge(n, mean, m2);
    if (lane == 0) out(g, n, mean, m2);
  }
}
// the one-CTA GroupNorm kernels (planes of at most CD_GN_SPLIT_MIN_HW pixels, one CTA per image): (mean, rstd) of x + cond per
// group of image b -> gst[g][2].  The forward and the backward both call this, so their statistics are bit-identical.  The
// caller synchronises before reading gst.
__device__ __forceinline__ void cd_gn_plane_stats(const float* __restrict__ x, int x_ld, int HW, int C, int groups,
                                                  const float* __restrict__ cond, int cond_ld, float eps, int b,
                                                  float (*tm)[512], float (*tq)[512], float* gst) {
  cd_gn_chunk_stats(x, x_ld, HW, C, groups, cond, cond_ld, b, 0, HW, tm, tq, [&](int g, float n, float mean, float m2) {
    gst[2 * g] = mean;
    gst[2 * g + 1] = rsqrtf(m2 / n + eps);
  });
}
__device__ __forceinline__ float cd_warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
#endif
