// Channel LayerNorm forward for C <= 128 (C / 4 a power of two) with PP = 4 pixels per lane group in flight, on 4096 pixels or more.
// layernorm_kernel<1> (elementwise.cu), which serves the other shapes, gives every thread ONE float4 load before two shuffle
// reductions: 2048 resident threads x 16 bytes = 32 KB in flight per SM, about what HBM latency x bandwidth needs.  Here a lane
// group loads PP pixels up front (PP x 16 bytes per thread in flight), then normalises them with the same per-pixel arithmetic in
// the same order (sum over the group by xor-shuffles, mean, centred sum of squares, rstd) -- bit-identical results.
#include "cd_common.cuh"

namespace {

constexpr int PP = 4;                 // pixels per lane group

__global__ void __launch_bounds__(256)
layernorm_multi_kernel(const float* __restrict__ x, int x_ld, long long npix, int C, const float* __restrict__ g,
                       const float* __restrict__ beta, float eps, float* __restrict__ y, int y_ld,
                       float* __restrict__ stats, int round_tf32) {
  const int lane = threadIdx.x & 31;
  const int nq = C >> 2;                         // <= 32, power of two
  const int G = nq;
  const int ppw = 32 / G, sub = lane / G, gl = lane % G;
  const long long base = (static_cast<long long>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5)) * ppw * PP + sub;
  float4 v[PP];
  bool valid[PP];
#pragma unroll
  for (int k = 0; k < PP; ++k) {
    const long long pix = base + static_cast<long long>(k) * ppw;
    valid[k] = pix < npix;
    v[k] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (valid[k]) v[k] = *reinterpret_cast<const float4*>(x + pix * x_ld + gl * 4);
  }
  const float4 gv = *reinterpret_cast<const float4*>(g + gl * 4);
  const float4 bv = *reinterpret_cast<const float4*>(beta + gl * 4);
#pragma unroll
  for (int k = 0; k < PP; ++k) {
    const long long pix = base + static_cast<long long>(k) * ppw;
    float s = 0.f;
    if (valid[k]) s += v[k].x + v[k].y + v[k].z + v[k].w;
    for (int o = G >> 1; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float mean = s / C;
    float s2 = 0.f;
    if (valid[k]) {
      const float a = v[k].x - mean, b = v[k].y - mean, c = v[k].z - mean, d = v[k].w - mean;
      s2 += a * a + b * b + c * c + d * d;
    }
    for (int o = G >> 1; o > 0; o >>= 1) s2 += __shfl_xor_sync(0xffffffffu, s2, o);
    const float rstd = rsqrtf(s2 / C + eps);
    if (valid[k]) {
      float4 o;
      o.x = (v[k].x - mean) * rstd * gv.x + bv.x; o.y = (v[k].y - mean) * rstd * gv.y + bv.y;
      o.z = (v[k].z - mean) * rstd * gv.z + bv.z; o.w = (v[k].w - mean) * rstd * gv.w + bv.w;
      if (round_tf32) { o.x = cd_round_tf32(o.x); o.y = cd_round_tf32(o.y); o.z = cd_round_tf32(o.z); o.w = cd_round_tf32(o.w); }
      *reinterpret_cast<float4*>(y + pix * y_ld + gl * 4) = o;
      if (stats && gl == 0) { stats[pix * 2] = mean; stats[pix * 2 + 1] = rstd; }
    }
  }
}

}  // namespace

// 1: shape not eligible -> the caller launches layernorm_kernel<N>
int cd_layernorm_fwd_multi(const float* x, int x_ld, long long npix, int C, const float* g, const float* beta, float eps,
                           float* y, int y_ld, float* stats, int round_tf32, cudaStream_t st) {
  const int nq = C / 4;
  if (nq > 32 || (nq & (nq - 1)) != 0 || npix < 4096) return 1;
  const int ppw = 32 / nq;
  layernorm_multi_kernel<<<cd_cdiv(npix, 8 * ppw * PP), 256, 0, st>>>(x, x_ld, npix, C, g, beta, eps, y, y_ld, stats, round_tf32);
  CD_LAUNCH_CHECK();
  return 0;
}
