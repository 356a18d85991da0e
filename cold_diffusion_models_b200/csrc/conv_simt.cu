// fp32 CUDA-core implementation of the tap-list convolution contract in colddiff.h.
// Used (a) where channel counts are not tensor-core shaped (3-channel image edges), (b) as the
// on-device fp32 cross-check of the tensor-core path, (c) for the weight gradient until the tensor-core
// wgrad lands.  64 pixels x 64 out-channels per CTA, 4x4 register tile per thread.
#include "cd_common.cuh"

namespace {

struct SimtSrc {
  const float* src; int ld, C, H, W, ntaps, wpb;
  const float* w;
  int dy[CD_MAX_TAPS], dx[CD_MAX_TAPS];
};
struct SimtParams {
  int B, Hg, Wg, sy, sx, Cout, nsrc;
  SimtSrc s[2];
  float* out; int out_ld, Ho, Wo, oys, oxs, oy0, ox0;
  const float* bias; const float* resid; int resid_ld; int act, round_tf32;
  float* out2; int out2_ld;
  const float* aux; int aux_ld;
  int tiles_per_img;
};

constexpr int TM = 64, TNc = 64, TK = 16;

__global__ void __launch_bounds__(256)
conv_simt_kernel(const SimtParams p) {
  __shared__ float As[TK][TM + 4];
  __shared__ float Bs[TK][TNc + 4];
  const int tid = threadIdx.x;
  const int b = blockIdx.x / p.tiles_per_img;
  const int m0 = (blockIdx.x % p.tiles_per_img) * TM;
  const int co0 = blockIdx.y * TNc;
  const int npix = p.Hg * p.Wg;
  const int tx = tid % 16, ty = tid / 16;
  float acc[4][4] = {};

  // loader mapping: element (row = tid / 4, k-quad = tid % 4)
  const int lrow = tid >> 2, lk = (tid & 3) * 4;
  const int lm = m0 + lrow;
  const bool lvalid = lm < npix;
  const int lgy = lvalid ? lm / p.Wg : 0, lgx = lvalid ? lm % p.Wg : 0;

  for (int s = 0; s < p.nsrc; ++s) {
    const SimtSrc& S = p.s[s];
    for (int tap = 0; tap < S.ntaps; ++tap) {
      const int iy = lgy * p.sy + S.dy[tap], ix = lgx * p.sx + S.dx[tap];
      const bool inb = lvalid && iy >= 0 && iy < S.H && ix >= 0 && ix < S.W;
      const float* arow = S.src + ((static_cast<long long>(b) * S.H + iy) * S.W + ix) * S.ld;
      const float* wrow = S.w + ((static_cast<long long>(S.wpb ? b : 0) * S.ntaps + tap) * p.Cout + (co0 + lrow)) * S.C;
      const bool wvalid = (co0 + lrow) < p.Cout;
      for (int k0 = 0; k0 < S.C; k0 += TK) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int k = k0 + lk + j;
          As[lk + j][lrow] = (inb && k < S.C) ? arow[k] : 0.f;
          Bs[lk + j][lrow] = (wvalid && k < S.C) ? wrow[k] : 0.f;
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < TK; ++k) {
          float a[4], w[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) { a[i] = As[k][ty * 4 + i]; w[i] = Bs[k][tx * 4 + i]; }
#pragma unroll
          for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], w[j], acc[i][j]);
        }
        __syncthreads();
      }
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty * 4 + i;
    if (m >= npix) continue;
    const int gy = m / p.Wg, gx = m % p.Wg;
    const long long pix = (static_cast<long long>(b) * p.Ho + (gy * p.oys + p.oy0)) * p.Wo + (gx * p.oxs + p.ox0);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int co = co0 + tx * 4 + j;
      if (co >= p.Cout) continue;
      float v = acc[i][j];
      if (p.bias) v += p.bias[co];
      if (p.resid) v += p.resid[pix * p.resid_ld + co];
      if (p.out2) p.out2[pix * p.out2_ld + co] = v;
      if (p.act == CD_ACT_GELU) v = cd_gelu(v);
      else if (p.act == CD_ACT_GELU_BWD) v *= cd_gelu_grad(p.aux[pix * p.aux_ld + co]);
      if (p.round_tf32) v = cd_round_tf32(v);
      p.out[pix * p.out_ld + co] = v;
    }
  }
}

// Image-edge convolution (Cin <= 4, e.g. the 3-channel input of the first ConvNextBlock): one thread per pixel keeps the
// whole receptive field (taps x Cin <= 36 values) in registers; weights [K][Cout] are broadcast from shared memory.
constexpr int kSmallK = 36;
__global__ void __launch_bounds__(128)
conv_smallc_kernel(const SimtParams p) {
  extern __shared__ float ws[];                    // [K][Cout]
  const SimtSrc& S = p.s[0];
  const int K = S.ntaps * S.C;
  for (int i = threadIdx.x; i < K * p.Cout; i += blockDim.x) {
    const int co = i % p.Cout, k = i / p.Cout, tap = k / S.C, c = k % S.C;
    ws[i] = S.w[(static_cast<long long>(tap) * p.Cout + co) * S.C + c];
  }
  __syncthreads();
  const long long gp = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long total = static_cast<long long>(p.B) * p.Hg * p.Wg;
  if (gp >= total) return;
  const int gx = static_cast<int>(gp % p.Wg);
  const int gy = static_cast<int>((gp / p.Wg) % p.Hg);
  const int b = static_cast<int>(gp / (static_cast<long long>(p.Wg) * p.Hg));
  float patch[kSmallK];
#pragma unroll
  for (int k = 0; k < kSmallK; ++k) patch[k] = 0.f;
  for (int tap = 0; tap < S.ntaps; ++tap) {
    const int iy = gy * p.sy + S.dy[tap], ix = gx * p.sx + S.dx[tap];
    if (iy < 0 || iy >= S.H || ix < 0 || ix >= S.W) continue;
    const float* row = S.src + ((static_cast<long long>(b) * S.H + iy) * S.W + ix) * S.ld;
    for (int c = 0; c < S.C; ++c) patch[tap * S.C + c] = row[c];
  }
  const long long pix = (static_cast<long long>(b) * p.Ho + (gy * p.oys + p.oy0)) * p.Wo + (gx * p.oxs + p.ox0);
  for (int co = 0; co < p.Cout; co += 4) {
    float a[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int k = 0; k < kSmallK; ++k) {
      if (k < K) {
        const float4 wv = *reinterpret_cast<const float4*>(&ws[k * p.Cout + co]);
        a[0] = fmaf(patch[k], wv.x, a[0]); a[1] = fmaf(patch[k], wv.y, a[1]);
        a[2] = fmaf(patch[k], wv.z, a[2]); a[3] = fmaf(patch[k], wv.w, a[3]);
      }
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float v = a[j];
      if (p.bias) v += p.bias[co + j];
      if (p.resid) v += p.resid[pix * p.resid_ld + co + j];
      if (p.out2) p.out2[pix * p.out2_ld + co + j] = v;
      if (p.act == CD_ACT_GELU) v = cd_gelu(v);
      else if (p.act == CD_ACT_GELU_BWD) v *= cd_gelu_grad(p.aux[pix * p.aux_ld + co + j]);
      if (p.round_tf32) v = cd_round_tf32(v);
      a[j] = v;
    }
    *reinterpret_cast<float4*>(p.out + pix * p.out_ld + co) = make_float4(a[0], a[1], a[2], a[3]);
  }
}

// Register-tiled variant (Cout % 4 == 0, Cout <= 128, Cout/4 a power of two): thread = 4 output channels with their
// K = ntaps*C weights in registers; 256 threads cover 256/(Cout/4) pixels at a time, the receptive fields of a 64-pixel
// chunk are staged in shared memory and read as broadcast LDS.128; a warp writes whole contiguous output rows.
// (16*KQ FMAs per KQ LDS.128 instead of 4 per LDS.128, and coalesced stores instead of one pixel row per thread.)
// The register-tiled image-edge kernels run ONE block of 8 warps per SM (~185-227 registers per thread), so nothing hides the
// memory latency of a staging loop; stage_patches_preload loads the (at most three) receptive-field entries a thread stages per
// 64-pixel chunk before it stores the first one.  stage_patches (same values in the same places) serves tap counts above 12.
__device__ __forceinline__ void stage_patches_preload(float* patch_f, int KP, long long q0, long long pend, const float* __restrict__ src,
                                                      int ld, int C, int H, int W, int Hg, int Wg, int sy, int sx, int ntaps,
                                                      const int* dyv, const int* dxv) {
  const int hw = Hg * Wg;
  float v[3][4];
#pragma unroll
  for (int u = 0; u < 3; ++u) {
    const int i = threadIdx.x + u * 256;
    v[u][0] = v[u][1] = v[u][2] = v[u][3] = 0.f;
    if (i < 64 * ntaps) {
      const int pp = i / ntaps, tap = i - pp * ntaps;
      const long long q = q0 + pp;
      if (q < pend) {
        const int qi = static_cast<int>(q);
        const int b = qi / hw, rem = qi - b * hw;
        const int gy = rem / Wg, gx = rem - gy * Wg;
        const int iy = gy * sy + dyv[tap], ix = gx * sx + dxv[tap];
        if (iy >= 0 && iy < H && ix >= 0 && ix < W) {
          const float* row = src + ((static_cast<long long>(b) * H + iy) * W + ix) * ld;
          for (int c = 0; c < C; ++c) v[u][c] = row[c];
        }
      }
    }
  }
#pragma unroll
  for (int u = 0; u < 3; ++u) {
    const int i = threadIdx.x + u * 256;
    if (i < 64 * ntaps) {
      const int pp = i / ntaps, tap = i - pp * ntaps;
      for (int c = 0; c < C; ++c) patch_f[pp * KP + tap * C + c] = v[u][c];
    }
  }
}

__device__ __forceinline__ void stage_patches(float* patch_f, int KP, long long q0, long long pend, const float* __restrict__ src,
                                              int ld, int C, int H, int W, int Hg, int Wg, int sy, int sx, int ntaps,
                                              const int* dyv, const int* dxv) {
  const int hw = Hg * Wg;
  for (int i = threadIdx.x; i < 64 * ntaps; i += blockDim.x) {
    const int pp = i / ntaps, tap = i - pp * ntaps;
    const long long q = q0 + pp;
    float v[4] = {0.f, 0.f, 0.f, 0.f};
    if (q < pend) {
      const int qi = static_cast<int>(q);                  // callers guarantee B*Hg*Wg < 2^31
      const int b = qi / hw, rem = qi - b * hw;
      const int gy = rem / Wg, gx = rem - gy * Wg;
      const int iy = gy * sy + dyv[tap], ix = gx * sx + dxv[tap];
      if (iy >= 0 && iy < H && ix >= 0 && ix < W) {
        const float* row = src + ((static_cast<long long>(b) * H + iy) * W + ix) * ld;
        for (int c = 0; c < C; ++c) v[c] = row[c];
      }
    }
    for (int c = 0; c < C; ++c) patch_f[pp * KP + tap * C + c] = v[c];
  }
}

template <int KQ>
__global__ void __launch_bounds__(256, 1)
conv_smallc4_kernel(const SimtParams p, int chunks_per_block, int preload) {
  constexpr int KP = 4 * KQ;
  __shared__ float4 patch[64][KQ];
  const SimtSrc& S = p.s[0];
  const int K = S.ntaps * S.C;
  const int CQ = p.Cout >> 2, PG = 256 / CQ;
  const int cq = threadIdx.x % CQ, pg = threadIdx.x / CQ;
  float* patch_f = reinterpret_cast<float*>(&patch[0][0]);
  for (int i = threadIdx.x; i < 64 * KP; i += 256) patch_f[i] = 0.f;       // padding entries k >= K stay zero
  float w[4][KP];
#pragma unroll
  for (int c = 0; c < 4; ++c)
#pragma unroll
    for (int k = 0; k < KP; ++k)
      w[c][k] = k < K ? S.w[(static_cast<long long>(k / S.C) * p.Cout + cq * 4 + c) * S.C + (k % S.C)] : 0.f;
  float4 bv = make_float4(0.f, 0.f, 0.f, 0.f);
  if (p.bias) bv = *reinterpret_cast<const float4*>(p.bias + cq * 4);
  const long long total = static_cast<long long>(p.B) * p.Hg * p.Wg;
  const int hw = p.Hg * p.Wg;
  const long long cbeg = static_cast<long long>(blockIdx.x) * chunks_per_block;
  for (long long ch = cbeg; ch < cbeg + chunks_per_block; ++ch) {
    const long long q0 = ch * 64;
    if (q0 >= total) break;
    const long long pend = q0 + 64 < total ? q0 + 64 : total;
    __syncthreads();
    if (preload) stage_patches_preload(patch_f, KP, q0, pend, S.src, S.ld, S.C, S.H, S.W, p.Hg, p.Wg, p.sy, p.sx, S.ntaps, S.dy, S.dx);
    else stage_patches(patch_f, KP, q0, pend, S.src, S.ld, S.C, S.H, S.W, p.Hg, p.Wg, p.sy, p.sx, S.ntaps, S.dy, S.dx);
    __syncthreads();
    const int np = static_cast<int>(pend - q0);
    for (int pp = pg; pp < np; pp += PG) {
      float a0 = bv.x, a1 = bv.y, a2 = bv.z, a3 = bv.w;
#pragma unroll
      for (int kq = 0; kq < KQ; ++kq) {
        const float4 x = patch[pp][kq];
        a0 = fmaf(x.x, w[0][4 * kq], a0); a0 = fmaf(x.y, w[0][4 * kq + 1], a0); a0 = fmaf(x.z, w[0][4 * kq + 2], a0); a0 = fmaf(x.w, w[0][4 * kq + 3], a0);
        a1 = fmaf(x.x, w[1][4 * kq], a1); a1 = fmaf(x.y, w[1][4 * kq + 1], a1); a1 = fmaf(x.z, w[1][4 * kq + 2], a1); a1 = fmaf(x.w, w[1][4 * kq + 3], a1);
        a2 = fmaf(x.x, w[2][4 * kq], a2); a2 = fmaf(x.y, w[2][4 * kq + 1], a2); a2 = fmaf(x.z, w[2][4 * kq + 2], a2); a2 = fmaf(x.w, w[2][4 * kq + 3], a2);
        a3 = fmaf(x.x, w[3][4 * kq], a3); a3 = fmaf(x.y, w[3][4 * kq + 1], a3); a3 = fmaf(x.z, w[3][4 * kq + 2], a3); a3 = fmaf(x.w, w[3][4 * kq + 3], a3);
      }
      const long long q = q0 + pp;
      const int b = static_cast<int>(q / hw);
      const int rem = static_cast<int>(q - static_cast<long long>(b) * hw);
      const int gy = rem / p.Wg, gx = rem - gy * p.Wg;
      const long long pix = (static_cast<long long>(b) * p.Ho + (gy * p.oys + p.oy0)) * p.Wo + (gx * p.oxs + p.ox0);
      float4 v = make_float4(a0, a1, a2, a3);
      if (p.resid) { const float4 r = *reinterpret_cast<const float4*>(p.resid + pix * p.resid_ld + cq * 4); v.x += r.x; v.y += r.y; v.z += r.z; v.w += r.w; }
      if (p.out2) *reinterpret_cast<float4*>(p.out2 + pix * p.out2_ld + cq * 4) = v;
      if (p.act == CD_ACT_GELU) { v.x = cd_gelu(v.x); v.y = cd_gelu(v.y); v.z = cd_gelu(v.z); v.w = cd_gelu(v.w); }
      else if (p.act == CD_ACT_GELU_BWD) {
        const float4 g = *reinterpret_cast<const float4*>(p.aux + pix * p.aux_ld + cq * 4);
        v.x *= cd_gelu_grad(g.x); v.y *= cd_gelu_grad(g.y); v.z *= cd_gelu_grad(g.z); v.w *= cd_gelu_grad(g.w);
      }
      if (p.round_tf32) { v.x = cd_round_tf32(v.x); v.y = cd_round_tf32(v.y); v.z = cd_round_tf32(v.z); v.w = cd_round_tf32(v.w); }
      *reinterpret_cast<float4*>(p.out + pix * p.out_ld + cq * 4) = v;
    }
  }
}

// dW[tap][co][ci] += sum_pix dout[pix][co] * src[pix(tap)][ci]
struct WgradParams {
  int B, Hg, Wg, sy, sx, Cout, C, H, W, ld, ntaps;
  int dy[CD_MAX_TAPS], dx[CD_MAX_TAPS];
  const float* src; const float* dout; int dout_ld, Ho, Wo, oys, oxs, oy0, ox0;
  float* dw;
  int splits, pix_per_split;
  int per_batch;   // splits never cross images; dw indexed [b][tap][co][ci]
};

__global__ void __launch_bounds__(256)
wgrad_simt_kernel(const WgradParams p) {
  __shared__ float As[TK][TM + 4];   // dout chunk  [pix][co]
  __shared__ float Bs[TK][TNc + 4];  // src chunk   [pix][ci]
  const int tid = threadIdx.x;
  const int co0 = blockIdx.x * TM, ci0 = blockIdx.y * TNc;
  const int tap = blockIdx.z / p.splits, split = blockIdx.z % p.splits;
  const int tx = tid % 16, ty = tid / 16;
  long long total = static_cast<long long>(p.B) * p.Hg * p.Wg;
  long long pbeg = static_cast<long long>(split) * p.pix_per_split;
  long long pend = pbeg + p.pix_per_split;
  int wb = 0;
  if (p.per_batch) {                       // split = b * splits_per_img + s
    const long long per_img = static_cast<long long>(p.Hg) * p.Wg;
    const int spi = p.splits / p.B;
    wb = split / spi;
    pbeg = wb * per_img + static_cast<long long>(split % spi) * p.pix_per_split;
    pend = pbeg + p.pix_per_split;
    total = (wb + 1) * per_img;
  }
  if (pend > total) pend = total;
  float acc[4][4] = {};
  // loader: pixel row = tid / 16 (16 pixels per chunk), channel quad = (tid % 16) * 4
  const int lp = tid >> 4, lc = (tid & 15) * 4;
  for (long long q0 = pbeg; q0 < pend; q0 += TK) {
    const long long q = q0 + lp;
    float a[4] = {0, 0, 0, 0}, s[4] = {0, 0, 0, 0};
    if (q < pend) {
      const int gx = static_cast<int>(q % p.Wg);
      const long long r = q / p.Wg;
      const int gy = static_cast<int>(r % p.Hg), b = static_cast<int>(r / p.Hg);
      const long long opix = (static_cast<long long>(b) * p.Ho + (gy * p.oys + p.oy0)) * p.Wo + (gx * p.oxs + p.ox0);
      const float* drow = p.dout + opix * p.dout_ld;
#pragma unroll
      for (int j = 0; j < 4; ++j) if (co0 + lc + j < p.Cout) a[j] = drow[co0 + lc + j];
      const int iy = gy * p.sy + p.dy[tap], ix = gx * p.sx + p.dx[tap];
      if (iy >= 0 && iy < p.H && ix >= 0 && ix < p.W) {
        const float* srow = p.src + ((static_cast<long long>(b) * p.H + iy) * p.W + ix) * p.ld;
#pragma unroll
        for (int j = 0; j < 4; ++j) if (ci0 + lc + j < p.C) s[j] = srow[ci0 + lc + j];
      }
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) { As[lp][lc + j] = a[j]; Bs[lp][lc + j] = s[j]; }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < TK; ++k) {
      float av[4], sv[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) { av[i] = As[k][ty * 4 + i]; sv[i] = Bs[k][tx * 4 + i]; }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], sv[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int co = co0 + ty * 4 + i;
    if (co >= p.Cout) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int ci = ci0 + tx * 4 + j;
      if (ci >= p.C) continue;
      atomicAdd(p.dw + ((static_cast<long long>(wb) * p.ntaps + tap) * p.Cout + co) * p.C + ci, acc[i][j]);
    }
  }
}

// weight gradient for image-edge convolutions (Cin <= 4): thread = output channel, the receptive fields of a chunk of
// pixels are staged in shared memory and broadcast; dout reads are coalesced over channels.
__global__ void __launch_bounds__(128)
wgrad_smallc_kernel(const WgradParams p) {
  __shared__ float patch[64][kSmallK + 1];
  __shared__ long long opix_s[64];
  const int co = blockIdx.y * 128 + threadIdx.x;
  const int K = p.ntaps * p.C;
  const long long total = static_cast<long long>(p.B) * p.Hg * p.Wg;
  const long long pbeg = static_cast<long long>(blockIdx.x) * p.pix_per_split;
  long long pend = pbeg + p.pix_per_split; if (pend > total) pend = total;
  float acc[kSmallK];
#pragma unroll
  for (int k = 0; k < kSmallK; ++k) acc[k] = 0.f;
  const int hw = p.Hg * p.Wg;
  for (long long q0 = pbeg; q0 < pend; q0 += 64) {
    __syncthreads();
    // stage the receptive fields: thread -> (pixel pp, tap group); 64 pixels x ntaps taps over 128 threads
    for (int i = threadIdx.x; i < 64 * p.ntaps; i += blockDim.x) {
      const int pp = i & 63, tap = i >> 6;
      const long long q = q0 + pp;
      const bool valid = q < pend;
      const int b = valid ? static_cast<int>(q / hw) : 0;
      const int rem = valid ? static_cast<int>(q - static_cast<long long>(b) * hw) : 0;
      const int gy = rem / p.Wg, gx = rem - gy * p.Wg;
      if (tap == 0) opix_s[pp] = (static_cast<long long>(b) * p.Ho + (gy * p.oys + p.oy0)) * p.Wo + (gx * p.oxs + p.ox0);
      const int iy = gy * p.sy + p.dy[tap], ix = gx * p.sx + p.dx[tap];
      const bool inb = valid && iy >= 0 && iy < p.H && ix >= 0 && ix < p.W;
      const float* row = p.src + ((static_cast<long long>(b) * p.H + iy) * p.W + ix) * p.ld;
      for (int c = 0; c < p.C; ++c) patch[pp][tap * p.C + c] = inb ? row[c] : 0.f;
    }
    __syncthreads();
    if (co < p.Cout) {
      const int np = static_cast<int>(pend - q0 < 64 ? pend - q0 : 64);
      for (int pp0 = 0; pp0 < np; pp0 += 8) {          // 8 independent dout loads in flight per thread
        float d[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) d[u] = (pp0 + u < np) ? p.dout[opix_s[pp0 + u] * p.dout_ld + co] : 0.f;
#pragma unroll
        for (int u = 0; u < 8; ++u) {
#pragma unroll
          for (int k = 0; k < kSmallK; ++k) if (k < K) acc[k] = fmaf(d[u], patch[(pp0 + u) & 63][k], acc[k]);
        }
      }
    }
  }
  if (co < p.Cout) {
#pragma unroll
    for (int k = 0; k < kSmallK; ++k)
      if (k < K) atomicAdd(p.dw + (static_cast<long long>(k / p.C) * p.Cout + co) * p.C + (k % p.C), acc[k]);
  }
}

// Register-tiled variant for Cout % 4 == 0, Cout <= 128: thread = 4 output channels x all K = ntaps*C (padded to 4*KQ)
// taps, one float4 of dY per pixel per thread (a warp reads whole 512-byte dY rows), the receptive field comes from shared
// memory as broadcast LDS.128 -- 16*KQ FMAs per (1 LDG.128 + KQ LDS.128).  Pixel groups of one block are reduced through
// shared memory so that each block issues one atomicAdd per weight.  (The first kernel above issued one LDS per FMA and
// ran ~9x off the HBM roofline on the 3->128 3x3 / 3->64 1x1 image-edge convolutions of the Unet.)
template <int KQ>
__global__ void __launch_bounds__(256, 1)
wgrad_smallc4_kernel(const WgradParams p, int preload) {
  constexpr int KP = 4 * KQ;
  __shared__ float4 patch[64][KQ];
  __shared__ float red[256 * 4 * 4];                       // [pixel group][cq][4 co][4 k] of one k-quad
  const int CQ = p.Cout >> 2;                              // threads per pixel (<= 32)
  const int PG = 256 / CQ;                                 // pixel groups per block
  const int cq = threadIdx.x % CQ, pg = threadIdx.x / CQ;
  const int K = p.ntaps * p.C;
  const long long total = static_cast<long long>(p.B) * p.Hg * p.Wg;
  const long long pbeg = static_cast<long long>(blockIdx.x) * p.pix_per_split;
  long long pend = pbeg + p.pix_per_split; if (pend > total) pend = total;
  float acc[4][KP];
#pragma unroll
  for (int c = 0; c < 4; ++c)
#pragma unroll
    for (int k = 0; k < KP; ++k) acc[c][k] = 0.f;
  const int hw = p.Hg * p.Wg;
  float* patch_f = reinterpret_cast<float*>(&patch[0][0]);
  for (int i = threadIdx.x; i < 64 * KP; i += 256) patch_f[i] = 0.f;       // padding entries k >= K stay zero
  const int NPT = 64 / PG;                                 // pixels per thread per 64-pixel chunk (<= 8)
  for (long long q0 = pbeg; q0 < pend; q0 += 64) {
    // all dY rows of this thread for the chunk are requested first: one exposed DRAM latency per chunk, overlapped with
    // the staging of the receptive fields (two-pixel trips left every trip latency-bound at one block per SM)
    float4 d[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      d[u] = make_float4(0.f, 0.f, 0.f, 0.f);
      const long long q = q0 + pg + u * PG;
      if (u < NPT && q < pend) {
        const int qi = static_cast<int>(q);
        const int b = qi / hw, rem = qi - b * hw;
        const int gy = rem / p.Wg, gx = rem - gy * p.Wg;
        const long long o = (static_cast<long long>(b) * p.Ho + (gy * p.oys + p.oy0)) * p.Wo + (gx * p.oxs + p.ox0);
        d[u] = __ldg(reinterpret_cast<const float4*>(p.dout + o * p.dout_ld + cq * 4));
      }
    }
    __syncthreads();
    if (preload) stage_patches_preload(patch_f, KP, q0, pend, p.src, p.ld, p.C, p.H, p.W, p.Hg, p.Wg, p.sy, p.sx, p.ntaps, p.dy, p.dx);
    else stage_patches(patch_f, KP, q0, pend, p.src, p.ld, p.C, p.H, p.W, p.Hg, p.Wg, p.sy, p.sx, p.ntaps, p.dy, p.dx);
    __syncthreads();
    const int np = static_cast<int>(pend - q0 < 64 ? pend - q0 : 64);
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const int pp = pg + u * PG;
      if (u < NPT && pp < np) {
        const float4 dv = d[u];
#pragma unroll
        for (int kq = 0; kq < KQ; ++kq) {
          const float4 x = patch[pp][kq];
          acc[0][4 * kq] = fmaf(dv.x, x.x, acc[0][4 * kq]); acc[0][4 * kq + 1] = fmaf(dv.x, x.y, acc[0][4 * kq + 1]);
          acc[0][4 * kq + 2] = fmaf(dv.x, x.z, acc[0][4 * kq + 2]); acc[0][4 * kq + 3] = fmaf(dv.x, x.w, acc[0][4 * kq + 3]);
          acc[1][4 * kq] = fmaf(dv.y, x.x, acc[1][4 * kq]); acc[1][4 * kq + 1] = fmaf(dv.y, x.y, acc[1][4 * kq + 1]);
          acc[1][4 * kq + 2] = fmaf(dv.y, x.z, acc[1][4 * kq + 2]); acc[1][4 * kq + 3] = fmaf(dv.y, x.w, acc[1][4 * kq + 3]);
          acc[2][4 * kq] = fmaf(dv.z, x.x, acc[2][4 * kq]); acc[2][4 * kq + 1] = fmaf(dv.z, x.y, acc[2][4 * kq + 1]);
          acc[2][4 * kq + 2] = fmaf(dv.z, x.z, acc[2][4 * kq + 2]); acc[2][4 * kq + 3] = fmaf(dv.z, x.w, acc[2][4 * kq + 3]);
          acc[3][4 * kq] = fmaf(dv.w, x.x, acc[3][4 * kq]); acc[3][4 * kq + 1] = fmaf(dv.w, x.y, acc[3][4 * kq + 1]);
          acc[3][4 * kq + 2] = fmaf(dv.w, x.z, acc[3][4 * kq + 2]); acc[3][4 * kq + 3] = fmaf(dv.w, x.w, acc[3][4 * kq + 3]);
        }
      }
    }
  }
  // block reduction over the pixel groups, one k-quad at a time: red[pg][cq*4 + c][4]
  for (int kq = 0; kq < KQ; ++kq) {
    __syncthreads();
#pragma unroll
    for (int c = 0; c < 4; ++c)
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float v = 0.f;
#pragma unroll
        for (int q = 0; q < KQ; ++q) if (q == kq) v = acc[c][4 * q + j];        // static register indexing
        red[((pg * CQ + cq) * 4 + c) * 4 + j] = v;
      }
    __syncthreads();
    for (int i = threadIdx.x; i < p.Cout * 4; i += 256) {                       // i = co*4 + j
      float s = 0.f;
      for (int g = 0; g < PG; ++g) s += red[g * p.Cout * 4 + i];
      const int co = i >> 2, k = 4 * kq + (i & 3);
      if (k < K) atomicAdd(p.dw + (static_cast<long long>(k / p.C) * p.Cout + co) * p.C + (k % p.C), s);
    }
  }
}

// column sums: out[c] += sum_rows x[row*ld + c]
__global__ void colsum_kernel(const float* x, int ld, long long rows, int C, float* out, long long rows_per_block) {
  const int c = blockIdx.x * 32 + (threadIdx.x & 31);
  const int ry = threadIdx.x >> 5;   // 8 row lanes
  const long long r0 = blockIdx.y * rows_per_block;
  long long r1 = r0 + rows_per_block; if (r1 > rows) r1 = rows;
  float s = 0.f;
  if (c < C) for (long long r = r0 + ry; r < r1; r += 8) s += x[r * ld + c];
  __shared__ float sm[8][33];
  sm[ry][threadIdx.x & 31] = s;
  __syncthreads();
  if (ry == 0 && c < C) {
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) t += sm[i][threadIdx.x & 31];
    atomicAdd(out + c, t);
  }
}

// vectorised column sums (C % 4 == 0): a warp covers 32/G rows x G float4 channel-quads (G = min(32, C/4) rounded up to a
// power of two), four independent 16-byte loads in flight per thread; partial sums meet in shared memory.
__global__ void __launch_bounds__(256)
colsum_vec_kernel(const float* __restrict__ x, int ld, long long rows, int C, float* __restrict__ out, long long rows_per_block, int G) {
  extern __shared__ float red[];                 // [C]
  const int nq = C >> 2;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarp = blockDim.x >> 5;
  const int rpw = 32 / G;                        // rows per warp pass
  const int gl = lane % G, sub = lane / G;
  const int qd = blockIdx.x * G + gl;            // channel quad handled by this lane
  const long long r0 = blockIdx.y * rows_per_block;
  long long r1 = r0 + rows_per_block; if (r1 > rows) r1 = rows;
  float4 a0 = make_float4(0, 0, 0, 0), a1 = a0, a2 = a0, a3 = a0;
  const long long stride = static_cast<long long>(nwarp) * rpw;
  if (qd < nq) {
    long long r = r0 + static_cast<long long>(warp) * rpw + sub;
    for (; r + 3 * stride < r1; r += 4 * stride) {
      const float4 v0 = *reinterpret_cast<const float4*>(x + r * ld + qd * 4);
      const float4 v1 = *reinterpret_cast<const float4*>(x + (r + stride) * ld + qd * 4);
      const float4 v2 = *reinterpret_cast<const float4*>(x + (r + 2 * stride) * ld + qd * 4);
      const float4 v3 = *reinterpret_cast<const float4*>(x + (r + 3 * stride) * ld + qd * 4);
      a0.x += v0.x; a0.y += v0.y; a0.z += v0.z; a0.w += v0.w;  a1.x += v1.x; a1.y += v1.y; a1.z += v1.z; a1.w += v1.w;
      a2.x += v2.x; a2.y += v2.y; a2.z += v2.z; a2.w += v2.w;  a3.x += v3.x; a3.y += v3.y; a3.z += v3.z; a3.w += v3.w;
    }
    for (; r < r1; r += stride) {
      const float4 v0 = *reinterpret_cast<const float4*>(x + r * ld + qd * 4);
      a0.x += v0.x; a0.y += v0.y; a0.z += v0.z; a0.w += v0.w;
    }
  }
  a0.x += a1.x + a2.x + a3.x; a0.y += a1.y + a2.y + a3.y; a0.z += a1.z + a2.z + a3.z; a0.w += a1.w + a2.w + a3.w;
  for (int i = threadIdx.x; i < G * 4; i += blockDim.x) red[i] = 0.f;
  __syncthreads();
  if (qd < nq) {
    atomicAdd(&red[gl * 4 + 0], a0.x); atomicAdd(&red[gl * 4 + 1], a0.y); atomicAdd(&red[gl * 4 + 2], a0.z); atomicAdd(&red[gl * 4 + 3], a0.w);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < G * 4; i += blockDim.x) {
    const int c = blockIdx.x * G * 4 + i;
    if (c < C) atomicAdd(out + c, red[i]);
  }
}

static int launch_colsum(const float* x, int ld, long long rows, int C, float* out, cudaStream_t st) {
  if (C % 4 == 0 && ld % 4 == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0 && rows >= 64) {
    const int nq = C / 4;
    int G = 1; while (G < nq && G < 32) G <<= 1;
    // rows per block: at most 1024, but aim for >= 4 blocks per SM (8192 rows x 512 channels gave 32 blocks)
    const int xb = cd_cdiv(nq, G);
    long long rpb = rows * xb / (cd_num_sms() * 4);
    if (rpb > 1024) rpb = 1024;
    if (rpb < 64) rpb = 64;
    dim3 g2(xb, cd_cdiv(rows, rpb));
    colsum_vec_kernel<<<g2, 256, sizeof(float) * G * 4, st>>>(x, ld, rows, C, out, rpb, G);
  } else {
    const long long rpb = 4096;
    dim3 g2(cd_cdiv(C, 32), cd_cdiv(rows, rpb));
    colsum_kernel<<<g2, 256, 0, st>>>(x, ld, rows, C, out, rpb);
  }
  return 0;
}

// weight repack kernels -----------------------------------------------------------------------
struct TapList { int ky[CD_MAX_TAPS], kx[CD_MAX_TAPS]; };
__global__ void pack_weight_kernel(const float* w, int O, int I, int KH, int KW, int transposed_conv, int mode,
                                   const TapList tl, int ntaps, int round_tf32, float* packed) {
  const int* ky = tl.ky; const int* kx = tl.kx;
  // forward operand: packed[t][o][i] ; dgrad operand: packed[t][i][o]
  const int N = mode == 0 ? O : I, K = mode == 0 ? I : O;
  const long long total = static_cast<long long>(ntaps) * N * K;
  for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int k = static_cast<int>(idx % K);
    const int n = static_cast<int>((idx / K) % N);
    const int t = static_cast<int>(idx / (static_cast<long long>(K) * N));
    const int o = mode == 0 ? n : k, i = mode == 0 ? k : n;
    // reference storage: Conv2d (O,I,KH,KW); ConvTranspose2d (I,O,KH,KW)
    const long long src = transposed_conv ? ((static_cast<long long>(i) * O + o) * KH + ky[t]) * KW + kx[t]
                                          : ((static_cast<long long>(o) * I + i) * KH + ky[t]) * KW + kx[t];
    float v = w[src];
    if (round_tf32) v = cd_round_tf32(v);
    packed[idx] = v;
  }
}
__global__ void unpack_wgrad_kernel(const float* packed, int O, int I, int KH, int KW, int transposed_conv,
                                    const TapList tl, int ntaps, float* wg, int accumulate) {
  const int* ky = tl.ky; const int* kx = tl.kx;
  const long long total = static_cast<long long>(ntaps) * O * I;
  for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int i = static_cast<int>(idx % I);
    const int o = static_cast<int>((idx / I) % O);
    const int t = static_cast<int>(idx / (static_cast<long long>(I) * O));
    const long long dst = transposed_conv ? ((static_cast<long long>(i) * O + o) * KH + ky[t]) * KW + kx[t]
                                          : ((static_cast<long long>(o) * I + i) * KH + ky[t]) * KW + kx[t];
    if (accumulate) wg[dst] += packed[idx]; else wg[dst] = packed[idx];
  }
}

// Conv2d (O,I,KH,KW) <-> packed [tap][O][I] through a shared-memory tile of 256 (o,i) rows x KH*KW taps, so that both the
// reference-layout side (contiguous KH*KW-float rows) and the packed side (contiguous (o,i) runs per tap) are coalesced.
// The element-wise kernels above touch one side with a stride of KH*KW floats (9x sector inflation on the read-modify-write).
constexpr int kMaxKHW = 16;
__global__ void __launch_bounds__(256)
unpack_wgrad_tiled_kernel(const float* __restrict__ packed, long long rows, int KHW, int KW, const TapList tl, int ntaps,
                          float* __restrict__ wg, int accumulate) {
  __shared__ float tile[256 * (kMaxKHW + 1)];
  __shared__ int covered[kMaxKHW];
  const int stride = KHW | 1;
  const long long r0 = static_cast<long long>(blockIdx.x) * 256;
  if (threadIdx.x < KHW) covered[threadIdx.x] = 0;
  __syncthreads();
  if (threadIdx.x < ntaps) covered[tl.ky[threadIdx.x] * KW + tl.kx[threadIdx.x]] = 1;
  const long long r = r0 + threadIdx.x;
  for (int t = 0; t < ntaps; ++t)
    tile[threadIdx.x * stride + tl.ky[t] * KW + tl.kx[t]] = r < rows ? packed[static_cast<long long>(t) * rows + r] : 0.f;
  __syncthreads();
  const int nrows = static_cast<int>(rows - r0 < 256 ? rows - r0 : 256);
  float* dst = wg + r0 * KHW;
  for (int idx = threadIdx.x; idx < nrows * KHW; idx += 256) {
    const int rr = idx / KHW, k = idx - rr * KHW;
    if (covered[k]) {
      const float v = tile[rr * stride + k];
      dst[idx] = accumulate ? dst[idx] + v : v;
    }
  }
}
__global__ void __launch_bounds__(256)
pack_weight_tiled_kernel(const float* __restrict__ w, long long rows, int KHW, int KW, const TapList tl, int ntaps,
                         int round_tf32, float* __restrict__ packed) {
  __shared__ float tile[256 * (kMaxKHW + 1)];
  const int stride = KHW | 1;
  const long long r0 = static_cast<long long>(blockIdx.x) * 256;
  const int nrows = static_cast<int>(rows - r0 < 256 ? rows - r0 : 256);
  const float* src = w + r0 * KHW;
  for (int idx = threadIdx.x; idx < nrows * KHW; idx += 256) {
    const int rr = idx / KHW, k = idx - rr * KHW;
    tile[rr * stride + k] = src[idx];
  }
  __syncthreads();
  const long long r = r0 + threadIdx.x;
  if (r < rows)
    for (int t = 0; t < ntaps; ++t) {
      float v = tile[threadIdx.x * stride + tl.ky[t] * KW + tl.kx[t]];
      if (round_tf32) v = cd_round_tf32(v);
      packed[static_cast<long long>(t) * rows + r] = v;
    }
}

}  // namespace

int cd_conv_fwd_tc(const CdConvDesc* d, cudaStream_t st);
int cd_conv_wgrad_tc(const CdConvDesc* d, const float* dout, int dout_ld, float* dw, float* db, int* bias_done, cudaStream_t st);

static int conv_fwd_simt(const CdConvDesc* d, cudaStream_t st) {
  SimtParams p{};
  p.B = d->B; p.Hg = d->Hg; p.Wg = d->Wg; p.sy = d->sy; p.sx = d->sx; p.Cout = d->Cout; p.nsrc = d->nsrc;
  for (int s = 0; s < d->nsrc; ++s) {
    const CdConvSrc& c = d->s[s];
    CD_REQUIRE(c.ntaps >= 1 && c.ntaps <= CD_MAX_TAPS, "conv_simt: bad ntaps");
    p.s[s].src = c.src; p.s[s].ld = c.ld; p.s[s].C = c.C; p.s[s].H = c.H; p.s[s].W = c.W;
    p.s[s].ntaps = c.ntaps; p.s[s].wpb = c.w_per_batch; p.s[s].w = c.w;
    for (int t = 0; t < c.ntaps; ++t) { p.s[s].dy[t] = c.dy[t]; p.s[s].dx[t] = c.dx[t]; }
  }
  p.out = d->out; p.out_ld = d->out_ld; p.Ho = d->Ho; p.Wo = d->Wo; p.oys = d->oys; p.oxs = d->oxs; p.oy0 = d->oy0; p.ox0 = d->ox0;
  p.bias = d->bias; p.resid = d->resid; p.resid_ld = d->resid_ld; p.act = d->act; p.round_tf32 = d->round_tf32;
  p.out2 = d->out2; p.out2_ld = d->out2_ld; p.aux = d->aux; p.aux_ld = d->aux_ld;
  CD_REQUIRE(d->act != CD_ACT_GELU_BWD || d->aux, "conv_simt: GELU_BWD needs aux");
  const CdConvSrc& c0 = d->s[0];
  if (d->nsrc == 1 && c0.C <= 4 && c0.ntaps * c0.C <= kSmallK && !c0.w_per_batch && d->Cout % 4 == 0 && d->Cout <= 512 &&
      d->out_ld % 4 == 0 && (reinterpret_cast<uintptr_t>(d->out) & 15) == 0) {
    const long long total = static_cast<long long>(d->B) * d->Hg * d->Wg;
    const int cq = d->Cout >> 2;
    const bool vec_ok = d->Cout <= 128 && (cq & (cq - 1)) == 0 && total >= 1024 && total < (1ll << 31) &&
                        (!d->bias || (reinterpret_cast<uintptr_t>(d->bias) & 15) == 0) &&
                        (!d->resid || (d->resid_ld % 4 == 0 && (reinterpret_cast<uintptr_t>(d->resid) & 15) == 0)) &&
                        (!d->out2 || (d->out2_ld % 4 == 0 && (reinterpret_cast<uintptr_t>(d->out2) & 15) == 0)) &&
                        (!d->aux || (d->aux_ld % 4 == 0 && (reinterpret_cast<uintptr_t>(d->aux) & 15) == 0));
    if (vec_ok) {
      const long long chunks = cd_cdiv(total, 64);
      long long blocks = cd_num_sms() * 2; if (blocks > chunks) blocks = chunks;
      const int cpb = cd_cdiv(chunks, blocks);
      const int grid = cd_cdiv(chunks, cpb);
      const int KQ = cd_cdiv(c0.ntaps * c0.C, 4);
      const int pre = 64 * c0.ntaps <= 768 ? 1 : 0;
      if (KQ <= 1) conv_smallc4_kernel<1><<<grid, 256, 0, st>>>(p, cpb, pre);
      else if (KQ <= 3) conv_smallc4_kernel<3><<<grid, 256, 0, st>>>(p, cpb, pre);
      else if (KQ <= 7) conv_smallc4_kernel<7><<<grid, 256, 0, st>>>(p, cpb, pre);
      else conv_smallc4_kernel<9><<<grid, 256, 0, st>>>(p, cpb, pre);
      CD_LAUNCH_CHECK();
      return 0;
    }
    const size_t smem = sizeof(float) * c0.ntaps * c0.C * d->Cout;
    static size_t attr = 0;
    if (smem > 48 * 1024 && smem > attr) { CD_CUDA(cudaFuncSetAttribute(conv_smallc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); attr = smem; }
    conv_smallc_kernel<<<cd_cdiv(total, 128), 128, smem, st>>>(p);
    CD_LAUNCH_CHECK();
    return 0;
  }
  p.tiles_per_img = cd_cdiv(d->Hg * d->Wg, TM);
  dim3 grid(d->B * p.tiles_per_img, cd_cdiv(d->Cout, TNc));
  conv_simt_kernel<<<grid, 256, 0, st>>>(p);
  CD_LAUNCH_CHECK();
  return 0;
}

extern "C" int cd_conv_fwd(const CdConvDesc* d, int impl, void* stream) {
  CD_REQUIRE(d != nullptr, "cd_conv_fwd: null descriptor");
  CD_REQUIRE(d->nsrc >= 1 && d->nsrc <= 2, "cd_conv_fwd: nsrc must be 1 or 2");
  CD_REQUIRE(d->B > 0 && d->Hg > 0 && d->Wg > 0 && d->Cout > 0, "cd_conv_fwd: empty problem");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (impl == CD_CONV_TC) return cd_conv_fwd_tc(d, st);
  if (impl == CD_CONV_SIMT) return conv_fwd_simt(d, st);
  CD_FAIL("cd_conv_fwd: unknown impl %d", impl);
}

extern "C" int cd_conv_wgrad(const CdConvDesc* d, const float* dout, int dout_ld, float* dw, float* db,
                             int impl, void* stream) {
  CD_REQUIRE(d && d->nsrc == 1, "cd_conv_wgrad: single source only");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const CdConvSrc& c = d->s[0];
  bool done = false;
  int bias_done = 0;
  if (impl == CD_CONV_TC) {
    const int rc = cd_conv_wgrad_tc(d, dout, dout_ld, dw, db, &bias_done, st);
    if (rc < 0) return rc;
    done = (rc == 0);                       // rc == 1: not tensor-core shaped -> fp32 CUDA-core kernel below
  }
  if (!done) {
  WgradParams p{};
  p.B = d->B; p.Hg = d->Hg; p.Wg = d->Wg; p.sy = d->sy; p.sx = d->sx; p.Cout = d->Cout;
  p.C = c.C; p.H = c.H; p.W = c.W; p.ld = c.ld; p.ntaps = c.ntaps;
  for (int t = 0; t < c.ntaps; ++t) { p.dy[t] = c.dy[t]; p.dx[t] = c.dx[t]; }
  p.src = c.src; p.dout = dout; p.dout_ld = dout_ld; p.Ho = d->Ho; p.Wo = d->Wo;
  p.oys = d->oys; p.oxs = d->oxs; p.oy0 = d->oy0; p.ox0 = d->ox0; p.dw = dw;
  const long long total = static_cast<long long>(d->B) * d->Hg * d->Wg;
  const int Ksm = c.ntaps * c.C;
  const bool pow2_cq = d->Cout >= 4 && ((d->Cout >> 2) & ((d->Cout >> 2) - 1)) == 0;
  if (c.C <= 4 && Ksm <= kSmallK && !c.w_per_batch && d->Cout % 4 == 0 && d->Cout <= 128 && pow2_cq &&
      dout_ld % 4 == 0 && (reinterpret_cast<uintptr_t>(dout) & 15) == 0 && total >= 1024 && total < (1ll << 31)) {
    int blocks = cd_num_sms() * 2; if (blocks > cd_cdiv(total, 256)) blocks = cd_cdiv(total, 256);
    p.pix_per_split = cd_cdiv(total, blocks);
    const int grid = cd_cdiv(total, p.pix_per_split);
    const int KQ = cd_cdiv(Ksm, 4);
    const int wpre = 64 * c.ntaps <= 768 ? 1 : 0;
    if (KQ <= 1) wgrad_smallc4_kernel<1><<<grid, 256, 0, st>>>(p, wpre);
    else if (KQ <= 3) wgrad_smallc4_kernel<3><<<grid, 256, 0, st>>>(p, wpre);
    else if (KQ <= 7) wgrad_smallc4_kernel<7><<<grid, 256, 0, st>>>(p, wpre);
    else wgrad_smallc4_kernel<9><<<grid, 256, 0, st>>>(p, wpre);
    CD_LAUNCH_CHECK();
  } else if (c.C <= 4 && c.ntaps * c.C <= kSmallK && !c.w_per_batch) {
    int splits = cd_cdiv(total, 512); if (splits > cd_num_sms() * 16) splits = cd_num_sms() * 16; if (splits < 1) splits = 1;
    p.pix_per_split = cd_cdiv(total, splits);
    dim3 grid(cd_cdiv(total, p.pix_per_split), cd_cdiv(d->Cout, 128));
    wgrad_smallc_kernel<<<grid, 128, 0, st>>>(p);
    CD_LAUNCH_CHECK();
  } else {
  const int tiles = cd_cdiv(d->Cout, TM) * cd_cdiv(c.C, TNc) * c.ntaps;
  int splits = cd_cdiv(cd_num_sms() * 4, tiles);
  const int max_splits = cd_cdiv(total, 256);
  if (splits > max_splits) splits = max_splits;
  if (splits < 1) splits = 1;
  p.per_batch = c.w_per_batch;
  if (c.w_per_batch) {
    const long long per_img = static_cast<long long>(d->Hg) * d->Wg;
    int spi = cd_cdiv(splits, d->B); if (spi < 1) spi = 1;
    p.pix_per_split = cd_cdiv(cd_cdiv(per_img, spi), TK) * TK;
    spi = cd_cdiv(per_img, p.pix_per_split);
    splits = spi * d->B;
  } else {
    p.pix_per_split = cd_cdiv(cd_cdiv(total, splits), TK) * TK;
    splits = cd_cdiv(total, p.pix_per_split);
  }
  p.splits = splits;
  dim3 grid(cd_cdiv(d->Cout, TM), cd_cdiv(c.C, TNc), c.ntaps * splits);
  wgrad_simt_kernel<<<grid, 256, 0, st>>>(p);
  CD_LAUNCH_CHECK();
  }
  }
  if (db && !bias_done) {
    const long long rows = static_cast<long long>(d->B) * d->Ho * d->Wo;
    CD_REQUIRE(d->oys == 1 && d->oxs == 1, "cd_conv_wgrad: bias gradient needs a dense output grid");
    launch_colsum(dout, dout_ld, rows, d->Cout, db, st);
    CD_LAUNCH_CHECK();
  }
  return 0;
}

extern "C" int cd_colsum(const float* x, int ld, int64_t rows, int C, float* out, void* stream) {
  launch_colsum(x, ld, rows, C, out, static_cast<cudaStream_t>(stream));
  CD_LAUNCH_CHECK();
  return 0;
}

extern "C" int cd_pack_weight(const float* w, int O, int I, int KH, int KW, int transposed_conv, int mode,
                              const int32_t* ky, const int32_t* kx, int ntaps, int round_tf32,
                              float* packed, void* stream) {
  CD_REQUIRE(ntaps >= 1 && ntaps <= CD_MAX_TAPS, "cd_pack_weight: bad ntaps");
  TapList tl{}; for (int t = 0; t < ntaps; ++t) { tl.ky[t] = ky[t]; tl.kx[t] = kx[t]; }
  const long long total = static_cast<long long>(ntaps) * O * I;
  if (!transposed_conv && mode == 0 && KH * KW <= kMaxKHW) {
    const long long rows = static_cast<long long>(O) * I;
    pack_weight_tiled_kernel<<<cd_cdiv(rows, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(w, rows, KH * KW, KW, tl, ntaps,
                                                                                              round_tf32, packed);
    CD_LAUNCH_CHECK();
    return 0;
  }
  int blocks = cd_cdiv(total, 256); if (blocks > cd_num_sms() * 8) blocks = cd_num_sms() * 8;
  pack_weight_kernel<<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(w, O, I, KH, KW, transposed_conv, mode,
                                                                          tl, ntaps, round_tf32, packed);
  CD_LAUNCH_CHECK();
  return 0;
}

extern "C" int cd_unpack_wgrad(const float* packed, int O, int I, int KH, int KW, int transposed_conv,
                               const int32_t* ky, const int32_t* kx, int ntaps, float* w_grad, int accumulate,
                               void* stream) {
  CD_REQUIRE(ntaps >= 1 && ntaps <= CD_MAX_TAPS, "cd_unpack_wgrad: bad ntaps");
  TapList tl{}; for (int t = 0; t < ntaps; ++t) { tl.ky[t] = ky[t]; tl.kx[t] = kx[t]; }
  const long long total = static_cast<long long>(ntaps) * O * I;
  if (!transposed_conv && KH * KW <= kMaxKHW) {
    const long long rows = static_cast<long long>(O) * I;
    unpack_wgrad_tiled_kernel<<<cd_cdiv(rows, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(packed, rows, KH * KW, KW, tl, ntaps,
                                                                                               w_grad, accumulate);
    CD_LAUNCH_CHECK();
    return 0;
  }
  int blocks = cd_cdiv(total, 256); if (blocks > cd_num_sms() * 8) blocks = cd_num_sms() * 8;
  unpack_wgrad_kernel<<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(packed, O, I, KH, KW, transposed_conv,
                                                                            tl, ntaps, w_grad, accumulate);
  CD_LAUNCH_CHECK();
  return 0;
}
