// Backward / training-mode pieces of the DDPM-style `Model` (deblurring-diffusion-pytorch/deblurring_diffusion_pytorch/
// Model2.py, "M2"): GroupNorm(+swish) backward (M2:32-33,116-125), dropout (M2:125), row-softmax backward of the AttnBlock
// (M2:172-175), nearest-2x upsample backward (M2:47-48), swish and its derivative for the time-embedding MLP (M2:27-29,
// 295-299), the sinusoidal embedding (M2:6-24) and a small dense layer.  The dense convolutions and the batched matmuls of the
// AttnBlock reuse cd_conv_fwd / cd_conv_wgrad (per-batch weights).
//
// tests/test_model2_train_gpu.py checks every parameter gradient against tests/golden/model2_grads_small.npz.
#include "cd_common.cuh"

namespace {

__device__ __forceinline__ float sigmoidf_(float z) { return 1.f / (1.f + __expf(-z)); }
__device__ __forceinline__ float swish_grad(float z) { const float s = sigmoidf_(z); return s * (1.f + z * (1.f - s)); }

// per-channel sum over the pixel lanes of a CTA in lane order: v[j][pp * nq + c / 4] holds channel c of pixel lane pp
__device__ __forceinline__ float gn_lane_sum(const float (*v)[512], int c, int nq, int np) {
  float a = 0.f;
  for (int pp = 0; pp < np; ++pp) a += v[c & 3][pp * nq + (c >> 2)];
  return a;
}

// one block per batch element (same thread -> (pixel lane, channel quad) mapping as groupnorm_kernel in elementwise.cu)
//   z = gamma * xh + beta, xh = (x + cond - mean_g) * rstd_g, y = swish ? z*sigmoid(z) : z
//   dz = dy * (swish ? swish'(z) : 1);  dgamma_c += sum dz*xh;  dbeta_c += sum dz
//   dx = rstd_g * (dz*gamma - mean_g(dz*gamma) - xh * mean_g(dz*gamma*xh));  dcond[b][c] = sum_pixels dx
// mean_g and rstd_g come from cd_gn_plane_stats, as in the forward (the same bits); every sum within the CTA is added in a fixed
// order (gn_lane_sum), so the result does not depend on the order the threads run in.
// kParams = false (dgamma = dbeta = NULL, frozen gamma and beta): the parameter accumulation is compiled out; dx and dcond are
// the same bits as with it.
template <bool kParams>
__global__ void __launch_bounds__(512)
groupnorm_bwd_kernel(const float* __restrict__ x, int x_ld, int HW, int C, int groups, const float* __restrict__ cond, int cond_ld,
                     const float* __restrict__ gamma, const float* __restrict__ beta, float eps, int swish,
                     const float* __restrict__ dy, int dy_ld, float* __restrict__ dx, int dx_ld,
                     float* __restrict__ dgamma, float* __restrict__ dbeta, float* __restrict__ dcond, int dcond_ld) {
  __shared__ float ta[4][512], tb[4][512];   // statistics scratch, then per-thread sums of dz | dz*xh, then of dx
  extern __shared__ float sm[];               // gst[G][2] (mean, rstd) | gab[G][2] | cdz[C] | cdzx[C]
  float* gst = sm; float* gab = gst + 2 * groups; float* cdz = gab + 2 * groups; float* cdzx = cdz + C;
  const int b = blockIdx.x;
  const int nq = C >> 2, cg = C / groups;
  cd_gn_plane_stats(x, x_ld, HW, C, groups, cond, cond_ld, eps, b, ta, tb, gst);
  __syncthreads();
  const long long base = static_cast<long long>(b) * HW;
  const int q = threadIdx.x % nq, pl = threadIdx.x / nq, np = blockDim.x / nq;
  const bool act = pl < np;
  float cadd[4] = {0.f, 0.f, 0.f, 0.f};
  if (cond && act) { const float4 cv = *reinterpret_cast<const float4*>(cond + static_cast<long long>(b) * cond_ld + q * 4); cadd[0] = cv.x; cadd[1] = cv.y; cadd[2] = cv.z; cadd[3] = cv.w; }
  const float inv_n = 1.f / (static_cast<float>(HW) * cg);
  float mean[4], rstd[4], gm[4] = {0.f, 0.f, 0.f, 0.f}, bt[4] = {0.f, 0.f, 0.f, 0.f};
  if (act) {
    for (int j = 0; j < 4; ++j) {
      const int g = (q * 4 + j) / cg;
      mean[j] = gst[2 * g]; rstd[j] = gst[2 * g + 1];
      gm[j] = gamma[q * 4 + j]; bt[j] = beta[q * 4 + j];
    }
    // ---- per-channel sums of dz and dz*xh
    float sdz[4] = {0.f, 0.f, 0.f, 0.f}, sdzx[4] = {0.f, 0.f, 0.f, 0.f};
    for (int p = pl; p < HW; p += np) {
      const float4 v4 = *reinterpret_cast<const float4*>(x + (base + p) * x_ld + q * 4);
      const float4 d4 = *reinterpret_cast<const float4*>(dy + (base + p) * dy_ld + q * 4);
      const float v[4] = {v4.x + cadd[0], v4.y + cadd[1], v4.z + cadd[2], v4.w + cadd[3]};
      const float d[4] = {d4.x, d4.y, d4.z, d4.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float xh = (v[j] - mean[j]) * rstd[j];
        const float dz = swish ? d[j] * swish_grad(xh * gm[j] + bt[j]) : d[j];
        sdz[j] += dz; sdzx[j] += dz * xh;
      }
    }
    for (int j = 0; j < 4; ++j) { ta[j][threadIdx.x] = sdz[j]; tb[j][threadIdx.x] = sdzx[j]; }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    cdz[c] = gn_lane_sum(ta, c, nq, np); cdzx[c] = gn_lane_sum(tb, c, nq, np);
    if constexpr (kParams) {
      atomicAdd(dgamma + c, cdzx[c]);
      atomicAdd(dbeta + c, cdz[c]);
    }
  }
  __syncthreads();
  for (int g = threadIdx.x; g < groups; g += blockDim.x) {
    float a = 0.f, a2 = 0.f;
    for (int c = g * cg; c < (g + 1) * cg; ++c) { a += gamma[c] * cdz[c]; a2 += gamma[c] * cdzx[c]; }
    gab[2 * g] = a * inv_n; gab[2 * g + 1] = a2 * inv_n;
  }
  __syncthreads();
  // ---- dx (+ per-channel sums for the conditioning gradient)
  if (act) {
    float ma[4], mb[4], sdx[4] = {0.f, 0.f, 0.f, 0.f};
    for (int j = 0; j < 4; ++j) { const int g = (q * 4 + j) / cg; ma[j] = gab[2 * g]; mb[j] = gab[2 * g + 1]; }
    for (int p = pl; p < HW; p += np) {
      const float4 v4 = *reinterpret_cast<const float4*>(x + (base + p) * x_ld + q * 4);
      const float4 d4 = *reinterpret_cast<const float4*>(dy + (base + p) * dy_ld + q * 4);
      const float v[4] = {v4.x + cadd[0], v4.y + cadd[1], v4.z + cadd[2], v4.w + cadd[3]};
      const float d[4] = {d4.x, d4.y, d4.z, d4.w};
      float o[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float xh = (v[j] - mean[j]) * rstd[j];
        const float dz = swish ? d[j] * swish_grad(xh * gm[j] + bt[j]) : d[j];
        o[j] = rstd[j] * (dz * gm[j] - ma[j] - xh * mb[j]);
        sdx[j] += o[j];
      }
      *reinterpret_cast<float4*>(dx + (base + p) * dx_ld + q * 4) = make_float4(o[0], o[1], o[2], o[3]);
    }
    for (int j = 0; j < 4; ++j) ta[j][threadIdx.x] = sdx[j];
  }
  if (dcond) {
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += blockDim.x) dcond[static_cast<long long>(b) * dcond_ld + c] = gn_lane_sum(ta, c, nq, np);
  }
}

// ---- split-plane backward (planes above CD_GN_SPLIT_MIN_HW pixels; the (chunk x image) grid and thread mapping of the
// forward's gn_split_* kernels in elementwise.cu).  Every per-channel sum is formed per chunk and the chunks are added in a
// fixed order: no float atomics, run-to-run identical results.
// out[c] = sum over k < nch of src[k * stride + c] in a fixed order: slice s of nsl = max(1, blockDim / C) adds k = s, s + nsl,
// ..., then the slices are added in order.  scratch holds nsl * C <= 2048 floats.
__device__ void gn_chunk_colsum(const float* __restrict__ src, long long stride, int nch, int C, float* scratch, float* out) {
  const int nsl = C < static_cast<int>(blockDim.x) ? blockDim.x / C : 1;
  for (int i = threadIdx.x; i < nsl * C; i += blockDim.x) {
    const int c = i % C, s = i / C;
    float a = 0.f;
    for (int k = s; k < nch; k += nsl) a += src[k * stride + c];
    scratch[i] = a;
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float a = 0.f;
    for (int s = 0; s < nsl; ++s) a += scratch[s * C + c];
    out[c] = a;
  }
  __syncthreads();
}

// per-(image, chunk, channel) sums of dz and dz*xh -> bpart[b][k][2][C]
__global__ void __launch_bounds__(512)
gn_split_bwd_sums_kernel(const float* __restrict__ x, int x_ld, long long HW, int C, int groups, const float* __restrict__ cond,
                         int cond_ld, const float* __restrict__ gamma, const float* __restrict__ beta, int swish,
                         const float* __restrict__ dy, int dy_ld, int cp, const float* __restrict__ stats, float* __restrict__ bpart) {
  __shared__ float tz[4][512], tzx[4][512];
  const int k = blockIdx.x, b = blockIdx.y, nch = gridDim.x;
  const int nq = C >> 2, cg = C / groups;
  const int q = threadIdx.x % nq, pl = threadIdx.x / nq, np = blockDim.x / nq;
  if (pl < np) {
    float cadd[4] = {0.f, 0.f, 0.f, 0.f}, mean[4], rstd[4], gm[4], bt[4];
    if (cond) { const float4 cv = *reinterpret_cast<const float4*>(cond + static_cast<long long>(b) * cond_ld + q * 4); cadd[0] = cv.x; cadd[1] = cv.y; cadd[2] = cv.z; cadd[3] = cv.w; }
    for (int j = 0; j < 4; ++j) {
      const float* st = stats + (static_cast<long long>(b) * groups + (q * 4 + j) / cg) * 2;
      mean[j] = st[0]; rstd[j] = st[1]; gm[j] = gamma[q * 4 + j]; bt[j] = beta[q * 4 + j];
    }
    float sdz[4] = {0.f, 0.f, 0.f, 0.f}, sdzx[4] = {0.f, 0.f, 0.f, 0.f};
    const long long base = static_cast<long long>(b) * HW + static_cast<long long>(k) * cp + pl;
    const int cnt = cd_gn_lane_count(HW, k, cp, pl, np);
    for (int i = 0; i < cnt; ++i) {
      const long long p = base + static_cast<long long>(i) * np;
      const float4 v4 = *reinterpret_cast<const float4*>(x + p * x_ld + q * 4);
      const float4 d4 = *reinterpret_cast<const float4*>(dy + p * dy_ld + q * 4);
      const float v[4] = {v4.x + cadd[0], v4.y + cadd[1], v4.z + cadd[2], v4.w + cadd[3]};
      const float d[4] = {d4.x, d4.y, d4.z, d4.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float xh = (v[j] - mean[j]) * rstd[j];
        const float dz = swish ? d[j] * swish_grad(xh * gm[j] + bt[j]) : d[j];
        sdz[j] += dz; sdzx[j] += dz * xh;
      }
    }
    for (int j = 0; j < 4; ++j) { tz[j][threadIdx.x] = sdz[j]; tzx[j][threadIdx.x] = sdzx[j]; }
  }
  __syncthreads();
  float* o = bpart + (static_cast<long long>(b) * nch + k) * 2 * C;
  for (int c = threadIdx.x; c < C; c += blockDim.x) { o[c] = gn_lane_sum(tz, c, nq, np); o[C + c] = gn_lane_sum(tzx, c, nq, np); }
}

// per image: chunk sums -> csum[b][2][C] (dz, dz*xh) and the group means of gamma*dz and gamma*dz*xh -> gab[b][groups][2]
__global__ void __launch_bounds__(512)
gn_split_bwd_reduce_kernel(const float* __restrict__ bpart, int nch, int C, int groups, const float* __restrict__ gamma, float inv_n,
                           float* __restrict__ csum, float* __restrict__ gab) {
  __shared__ float scratch[2048], cz[2048], czx[2048];
  const int b = blockIdx.x, cg = C / groups;
  const float* src = bpart + static_cast<long long>(b) * nch * 2 * C;
  gn_chunk_colsum(src, 2LL * C, nch, C, scratch, cz);
  gn_chunk_colsum(src + C, 2LL * C, nch, C, scratch, czx);
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    csum[static_cast<long long>(b) * 2 * C + c] = cz[c];
    csum[static_cast<long long>(b) * 2 * C + C + c] = czx[c];
  }
  for (int g = threadIdx.x; g < groups; g += blockDim.x) {
    float a = 0.f, a2 = 0.f;
    for (int c = g * cg; c < (g + 1) * cg; ++c) { a += gamma[c] * cz[c]; a2 += gamma[c] * czx[c]; }
    gab[(static_cast<long long>(b) * groups + g) * 2] = a * inv_n;
    gab[(static_cast<long long>(b) * groups + g) * 2 + 1] = a2 * inv_n;
  }
}

// dx over the (chunk x image) grid; with dpart, also the per-(image, chunk, channel) sums of dx -> dpart[b][k][C]
__global__ void __launch_bounds__(512)
gn_split_bwd_dx_kernel(const float* __restrict__ x, int x_ld, long long HW, int C, int groups, const float* __restrict__ cond,
                       int cond_ld, const float* __restrict__ gamma, const float* __restrict__ beta, int swish,
                       const float* __restrict__ dy, int dy_ld, int cp, const float* __restrict__ stats,
                       const float* __restrict__ gab, float* __restrict__ dx, int dx_ld, float* __restrict__ dpart) {
  __shared__ float tdx[4][512];
  const int k = blockIdx.x, b = blockIdx.y, nch = gridDim.x;
  const int nq = C >> 2, cg = C / groups;
  const int q = threadIdx.x % nq, pl = threadIdx.x / nq, np = blockDim.x / nq;
  if (pl < np) {
    float cadd[4] = {0.f, 0.f, 0.f, 0.f}, mean[4], rstd[4], gm[4], bt[4], ma[4], mb[4], sdx[4] = {0.f, 0.f, 0.f, 0.f};
    if (cond) { const float4 cv = *reinterpret_cast<const float4*>(cond + static_cast<long long>(b) * cond_ld + q * 4); cadd[0] = cv.x; cadd[1] = cv.y; cadd[2] = cv.z; cadd[3] = cv.w; }
    for (int j = 0; j < 4; ++j) {
      const long long g = static_cast<long long>(b) * groups + (q * 4 + j) / cg;
      mean[j] = stats[g * 2]; rstd[j] = stats[g * 2 + 1]; ma[j] = gab[g * 2]; mb[j] = gab[g * 2 + 1];
      gm[j] = gamma[q * 4 + j]; bt[j] = beta[q * 4 + j];
    }
    const long long base = static_cast<long long>(b) * HW + static_cast<long long>(k) * cp + pl;
    const int cnt = cd_gn_lane_count(HW, k, cp, pl, np);
#pragma unroll 4
    for (int i = 0; i < cnt; ++i) {
      const long long p = base + static_cast<long long>(i) * np;
      const float4 v4 = *reinterpret_cast<const float4*>(x + p * x_ld + q * 4);
      const float4 d4 = *reinterpret_cast<const float4*>(dy + p * dy_ld + q * 4);
      const float v[4] = {v4.x + cadd[0], v4.y + cadd[1], v4.z + cadd[2], v4.w + cadd[3]};
      const float d[4] = {d4.x, d4.y, d4.z, d4.w};
      float o[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float xh = (v[j] - mean[j]) * rstd[j];
        const float dz = swish ? d[j] * swish_grad(xh * gm[j] + bt[j]) : d[j];
        o[j] = rstd[j] * (dz * gm[j] - ma[j] - xh * mb[j]);
        sdx[j] += o[j];
      }
      *reinterpret_cast<float4*>(dx + p * dx_ld + q * 4) = make_float4(o[0], o[1], o[2], o[3]);
    }
    for (int j = 0; j < 4; ++j) tdx[j][threadIdx.x] = sdx[j];
  }
  if (!dpart) return;
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) dpart[(static_cast<long long>(b) * nch + k) * C + c] = gn_lane_sum(tdx, c, nq, np);
}

// blocks b < B (with dcond): dcond[b][c] = sum over chunks of dpart; the last block (kParams): dgamma / dbeta += sum over images
// of csum
template <bool kParams>
__global__ void __launch_bounds__(512)
gn_split_bwd_final_kernel(const float* __restrict__ csum, int B, int C, const float* __restrict__ dpart, int nch,
                          float* __restrict__ dcond, int dcond_ld, float* __restrict__ dgamma, float* __restrict__ dbeta) {
  __shared__ float scratch[2048];
  const int b = blockIdx.x;
  if (kParams && b == static_cast<int>(gridDim.x) - 1) {
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
      float a = 0.f, a2 = 0.f;
      for (int i = 0; i < B; ++i) { a += csum[static_cast<long long>(i) * 2 * C + c]; a2 += csum[static_cast<long long>(i) * 2 * C + C + c]; }
      dbeta[c] += a; dgamma[c] += a2;
    }
    return;
  }
  gn_chunk_colsum(dpart + static_cast<long long>(b) * nch * C, C, nch, C, scratch, dcond + static_cast<long long>(b) * dcond_ld);
}

// counter-based mask: keep element i of the call `seed` with probability 1-p (murmur3 finaliser of (seed, i))
__device__ __forceinline__ float uniform01(unsigned long long seed, unsigned long long i) {
  unsigned long long h = seed ^ (i * 0x9E3779B97F4A7C15ull);
  h ^= h >> 33; h *= 0xff51afd7ed558ccdull; h ^= h >> 33; h *= 0xc4ceb9fe1a85ec53ull; h ^= h >> 33;
  return static_cast<float>(h >> 40) * (1.f / 16777216.f);
}
// seed_ptr: the seed is read from device memory (a CUDA graph replays with the seed staged there before each launch), else `seed`
__global__ void dropout_kernel(const float* __restrict__ x, int x_ld, long long npix, int C, float p, unsigned long long seed,
                               const unsigned long long* __restrict__ seed_ptr, float* __restrict__ y, int y_ld) {
  if (seed_ptr) seed = *seed_ptr;
  const long long n = npix * C;
  const float scale = 1.f / (1.f - p);
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long pix = i / C; const int c = static_cast<int>(i - pix * C);
    const float keep = uniform01(seed, static_cast<unsigned long long>(i)) >= p ? scale : 0.f;
    y[pix * y_ld + c] = x[pix * x_ld + c] * keep;
  }
}

// ds[row][j] <- s[row][j] * (ds[row][j] - sum_j ds*s) * scale     (s = softmax(scale * logits))
__global__ void softmax_bwd_rows_kernel(const float* __restrict__ s, float* __restrict__ ds, int ld, long long rows, int n, float scale) {
  const long long row = static_cast<long long>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  const float* sr = s + row * ld;
  float* dr = ds + row * ld;
  float dot = 0.f;
  for (int j = lane; j < n; j += 32) dot = fmaf(dr[j], sr[j], dot);
  dot = cd_warp_sum(dot);
  for (int j = lane; j < n; j += 32) dr[j] = sr[j] * (dr[j] - dot) * scale;
}

// dx[b][y][x][c] = sum of the four children of the nearest-neighbour 2x upsample
__global__ void upsample_nearest2x_bwd_kernel(const float* __restrict__ dy, int dy_ld, int B, int H, int W, int C,
                                              float* __restrict__ dx, int dx_ld) {
  const int nq = C >> 2;
  const long long total = static_cast<long long>(B) * H * W * nq;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int q = static_cast<int>(i % nq);
    const long long pix = i / nq;
    const int xx = static_cast<int>(pix % W), yy = static_cast<int>((pix / W) % H), b = static_cast<int>(pix / (static_cast<long long>(W) * H));
    const long long r0 = ((static_cast<long long>(b) * 2 * H + 2 * yy) * 2 * W + 2 * xx);
    const long long r1 = r0 + 2 * W;
    const float4 a = *reinterpret_cast<const float4*>(dy + r0 * dy_ld + q * 4);
    const float4 bq = *reinterpret_cast<const float4*>(dy + (r0 + 1) * dy_ld + q * 4);
    const float4 c = *reinterpret_cast<const float4*>(dy + r1 * dy_ld + q * 4);
    const float4 d = *reinterpret_cast<const float4*>(dy + (r1 + 1) * dy_ld + q * 4);
    *reinterpret_cast<float4*>(dx + pix * dx_ld + q * 4) = make_float4(a.x + bq.x + c.x + d.x, a.y + bq.y + c.y + d.y,
                                                                       a.z + bq.z + c.z + d.z, a.w + bq.w + c.w + d.w);
  }
}

// act_out = swish(pre) (optional);  y = dy * swish'(pre) (optional)
__global__ void swish_kernel(const float* __restrict__ dy, const float* __restrict__ pre, long long n, float* __restrict__ y,
                             float* __restrict__ act_out) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float p = pre[i];
  if (act_out) act_out[i] = p * sigmoidf_(p);
  if (y) y[i] = dy[i] * swish_grad(p);
}

// get_timestep_embedding (M2:6-24): emb[b] = [sin(t*f_i) | cos(t*f_i)], f_i = exp(-i * ln(10000)/(half-1))
__global__ void timestep_embedding_kernel(const long long* __restrict__ t, int B, int dim, float* __restrict__ emb) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int half = dim / 2;
  if (i >= B * half) return;
  const int b = i / half, k = i - b * half;
  const float f = expf(-(logf(10000.f) / (half - 1)) * k);
  const float a = static_cast<float>(t[b]) * f;
  emb[b * dim + k] = sinf(a);
  emb[b * dim + half + k] = cosf(a);
  if ((dim & 1) && k == 0) emb[b * dim + dim - 1] = 0.f;
}

// y[m][n] = bias[n] + sum_k x[m][k] * w[n][k]   (nn.Linear; tiny M = batch)
__global__ void linear_kernel(const float* __restrict__ x, int K, const float* __restrict__ w, const float* __restrict__ bias,
                              int M, int N, float* __restrict__ y) {
  const int lane = threadIdx.x & 31;
  const long long o = static_cast<long long>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5);     // warp per output
  if (o >= static_cast<long long>(M) * N) return;
  const int m = static_cast<int>(o / N), n = static_cast<int>(o % N);
  float a = 0.f;
  for (int k = lane; k < K; k += 32) a = fmaf(x[static_cast<long long>(m) * K + k], w[static_cast<long long>(n) * K + k], a);
  a = cd_warp_sum(a);
  if (lane == 0) y[o] = a + (bias ? bias[n] : 0.f);
}

}  // namespace

// ---------------------------------------------------------------------------------------------------------------------
// Input pipeline (reference Dataset / Dataset_Aug1, DB:983-1026): the decoded, 1.12x-resized uint8 images stay resident in
// HBM; a batch is gathered with a per-sample crop window and horizontal flip and converted like ToTensor()*2-1.
//   out[b][c][y][x] = src[index[b]][oy[b] + y][ox[b] + (flip[b] ? S-1-x : x)][c] / 255 * 2 - 1
// ---------------------------------------------------------------------------------------------------------------------
namespace {
__global__ void augment_u8_kernel(const unsigned char* __restrict__ src, int Hs, int Ws, const long long* __restrict__ index,
                                  const int* __restrict__ oy, const int* __restrict__ ox, const int* __restrict__ flip,
                                  int B, int S, float* __restrict__ out) {
  const long long n = static_cast<long long>(B) * S * S;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int x = static_cast<int>(i % S), y = static_cast<int>((i / S) % S), b = static_cast<int>(i / (static_cast<long long>(S) * S));
    const int sx = ox[b] + (flip[b] ? S - 1 - x : x), sy = oy[b] + y;
    const unsigned char* px = src + ((static_cast<long long>(index[b]) * Hs + sy) * Ws + sx) * 3;
    float* o = out + (static_cast<long long>(b) * 3 * S + y) * S + x;
#pragma unroll
    for (int c = 0; c < 3; ++c) o[static_cast<long long>(c) * S * S] = (static_cast<float>(px[c]) / 255.f) * 2.f - 1.f;
  }
}
}  // namespace

extern "C" int cd_augment_u8(const uint8_t* src, int N, int Hs, int Ws, const int64_t* index, const int32_t* oy, const int32_t* ox,
                             const int32_t* flip, int B, int S, float* out, void* stream) {
  CD_REQUIRE(S <= Hs && S <= Ws && N >= 1 && B >= 1, "cd_augment_u8: crop %d does not fit the %dx%d source images", S, Hs, Ws);
  const long long n = static_cast<long long>(B) * S * S;
  int blocks = cd_cdiv(n, 256); if (blocks > cd_num_sms() * 16) blocks = cd_num_sms() * 16;
  augment_u8_kernel<<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(src, Hs, Ws, reinterpret_cast<const long long*>(index), oy, ox, flip, B, S, out);
  CD_LAUNCH_CHECK();
  return 0;
}

extern "C" int cd_groupnorm_bwd(const float* x, int x_ld, int B, int64_t HW, int C, int groups, const float* cond, int cond_ld,
                                const float* gamma, const float* beta, float eps, int swish, const float* dy, int dy_ld,
                                float* dx, int dx_ld, float* dgamma, float* dbeta, float* dcond, int dcond_ld, void* stream) {
  CD_REQUIRE(C % 4 == 0 && C % groups == 0 && C / 4 <= 512 && x_ld % 4 == 0 && dy_ld % 4 == 0 && dx_ld % 4 == 0 &&
             (!cond || cond_ld % 4 == 0), "cd_groupnorm_bwd: unsupported C=%d groups=%d", C, groups);
  CD_REQUIRE((dgamma == nullptr) == (dbeta == nullptr), "cd_groupnorm_bwd: dgamma and dbeta are both given or both NULL");
  const bool params = dgamma != nullptr;
  if (HW > CD_GN_SPLIT_MIN_HW) {
    CD_REQUIRE(B <= 65535, "cd_groupnorm_bwd: the split-plane path takes at most 65535 images (B=%d)", B);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int cp = cd_gn_split_chunk(C), nch = cd_cdiv(HW, cp);
    // workspace: stats | part | gab | csum | bpart | dpart
    const long long nstat = 2LL * B * groups, nc = static_cast<long long>(B) * C;
    float* ws = nullptr;
    if (int rc = cd_gn_workspace(sizeof(float) * (nstat * (2 + nch) + nc * (2 + 2LL * nch + (dcond ? nch : 0))), st, &ws)) return rc;
    float *stats = ws, *part = stats + nstat, *gab = part + nstat * nch, *csum = gab + nstat, *bpart = csum + 2 * nc;
    float* dpart = dcond ? bpart + 2 * nc * nch : nullptr;
    if (int rc = cd_gn_split_stats(x, x_ld, B, HW, C, groups, cond, cond_ld, eps, part, stats, st)) return rc;
    gn_split_bwd_sums_kernel<<<dim3(nch, B), 512, 0, st>>>(x, x_ld, HW, C, groups, cond, cond_ld, gamma, beta, swish, dy, dy_ld, cp,
                                                           stats, bpart);
    CD_LAUNCH_CHECK();
    gn_split_bwd_reduce_kernel<<<B, 512, 0, st>>>(bpart, nch, C, groups, gamma, 1.f / (static_cast<float>(HW) * (C / groups)), csum, gab);
    CD_LAUNCH_CHECK();
    gn_split_bwd_dx_kernel<<<dim3(nch, B), 512, 0, st>>>(x, x_ld, HW, C, groups, cond, cond_ld, gamma, beta, swish, dy, dy_ld, cp,
                                                         stats, gab, dx, dx_ld, dpart);
    CD_LAUNCH_CHECK();
    const int fin = (dcond ? B : 0) + (params ? 1 : 0);
    if (fin == 0) return 0;
    if (params) gn_split_bwd_final_kernel<true><<<fin, 512, 0, st>>>(csum, B, C, dpart, nch, dcond, dcond_ld, dgamma, dbeta);
    else gn_split_bwd_final_kernel<false><<<fin, 512, 0, st>>>(csum, B, C, dpart, nch, dcond, dcond_ld, dgamma, dbeta);
    CD_LAUNCH_CHECK();
    return 0;
  }
  // dynamic shared memory beyond 48 KB less the kernel's 16 KB of static scratch (4 * groups + 2 * C > 8192, e.g. groups == C
  // above 1365) needs the opt-in; at most 48 KB + 16 KB
  const size_t smem = sizeof(float) * (4 * groups + 2 * C);
  static size_t attr[2] = {0, 0};
  if (smem > 32 * 1024 && smem > attr[params]) {
    CD_CUDA(cudaFuncSetAttribute(params ? groupnorm_bwd_kernel<true> : groupnorm_bwd_kernel<false>,
                                 cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr[params] = smem;
  }
  if (params)
    groupnorm_bwd_kernel<true><<<B, 512, smem, static_cast<cudaStream_t>(stream)>>>(x, x_ld, (int)HW, C, groups, cond, cond_ld, gamma, beta,
                                                                                 eps, swish, dy, dy_ld, dx, dx_ld, dgamma, dbeta, dcond, dcond_ld);
  else
    groupnorm_bwd_kernel<false><<<B, 512, smem, static_cast<cudaStream_t>(stream)>>>(x, x_ld, (int)HW, C, groups, cond, cond_ld, gamma, beta,
                                                                                  eps, swish, dy, dy_ld, dx, dx_ld, dgamma, dbeta, dcond, dcond_ld);
  CD_LAUNCH_CHECK();
  return 0;
}

static int dropout_launch(const float* x, int x_ld, int64_t npix, int C, float p, uint64_t seed, const uint64_t* seed_ptr, float* y,
                          int y_ld, void* stream) {
  const long long n = static_cast<long long>(npix) * C;
  int blocks = cd_cdiv(n, 256); if (blocks > cd_num_sms() * 16) blocks = cd_num_sms() * 16; if (blocks < 1) blocks = 1;
  dropout_kernel<<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(x, x_ld, npix, C, p, seed,
                                                                       reinterpret_cast<const unsigned long long*>(seed_ptr), y, y_ld);
  CD_LAUNCH_CHECK();
  return 0;
}

extern "C" int cd_dropout(const float* x, int x_ld, int64_t npix, int C, float p, uint64_t seed, float* y, int y_ld, void* stream) {
  CD_REQUIRE(p >= 0.f && p < 1.f, "cd_dropout: p must be in [0, 1)");
  return dropout_launch(x, x_ld, npix, C, p, seed, nullptr, y, y_ld, stream);
}

extern "C" int cd_dropout_seed_dev(const float* x, int x_ld, int64_t npix, int C, float p, const uint64_t* seed, float* y, int y_ld,
                                   void* stream) {
  CD_REQUIRE(p >= 0.f && p < 1.f, "cd_dropout_seed_dev: p must be in [0, 1)");
  CD_REQUIRE(seed != nullptr, "cd_dropout_seed_dev: seed must point to device memory");
  return dropout_launch(x, x_ld, npix, C, p, 0, seed, y, y_ld, stream);
}

extern "C" int cd_softmax_bwd_rows(const float* s, float* ds, int ld, int64_t rows, int n, float scale, void* stream) {
  softmax_bwd_rows_kernel<<<cd_cdiv(rows, 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(s, ds, ld, rows, n, scale);
  CD_LAUNCH_CHECK();
  return 0;
}

extern "C" int cd_upsample_nearest2x_bwd(const float* dy, int dy_ld, int B, int H, int W, int C, float* dx, int dx_ld, void* stream) {
  CD_REQUIRE(C % 4 == 0 && dy_ld % 4 == 0 && dx_ld % 4 == 0, "cd_upsample_nearest2x_bwd: C must be a multiple of 4");
  const long long total = static_cast<long long>(B) * H * W * (C / 4);
  int blocks = cd_cdiv(total, 256); if (blocks > cd_num_sms() * 16) blocks = cd_num_sms() * 16; if (blocks < 1) blocks = 1;
  upsample_nearest2x_bwd_kernel<<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(dy, dy_ld, B, H, W, C, dx, dx_ld);
  CD_LAUNCH_CHECK();
  return 0;
}

extern "C" int cd_swish(const float* dy, const float* pre, int64_t n, float* y, float* act_out, void* stream) {
  swish_kernel<<<cd_cdiv(n, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(dy, pre, n, y, act_out);
  CD_LAUNCH_CHECK();
  return 0;
}

extern "C" int cd_timestep_embedding(const int64_t* t, int B, int dim, float* emb, void* stream) {
  CD_REQUIRE(dim >= 4, "cd_timestep_embedding: dim must be >= 4");
  timestep_embedding_kernel<<<cd_cdiv(B * (dim / 2), 128), 128, 0, static_cast<cudaStream_t>(stream)>>>(reinterpret_cast<const long long*>(t), B, dim, emb);
  CD_LAUNCH_CHECK();
  return 0;
}

extern "C" int cd_linear_fwd(const float* x, int K, const float* w, const float* bias, int M, int N, float* y, void* stream) {
  const long long outs = static_cast<long long>(M) * N;
  linear_kernel<<<cd_cdiv(outs, 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(x, K, w, bias, M, N, y);
  CD_LAUNCH_CHECK();
  return 0;
}
