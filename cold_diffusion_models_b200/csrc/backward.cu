// Backward kernels of the HBM-bound Unet pieces (the dense-conv gradients reuse the tap-list
// convolution contract: dgrad = cd_conv_fwd with transposed/flipped packed weights, wgrad =
// cd_conv_wgrad).  Everything here is fp32 on NHWC activations.
#include "cd_common.cuh"

namespace {

// ---------------------------------------------------------------------------------------------
// channel LayerNorm backward (DB:111-121): warp per pixel.
//   xhat = (h - mean) * rstd ; dxh = dy * g ; dh = rstd * (dxh - mean_c(dxh) - xhat * mean_c(dxh * xhat)) (+ addend)
//   dg[c] += sum_pix dy * xhat ; dbeta[c] += sum_pix dy
// ---------------------------------------------------------------------------------------------
// lanes are split into groups of G = min(32, C/4) (a power of two): each group owns one pixel per iteration, each lane
// C/(4G) float4 slots; two iterations are in flight per warp so the load->reduce->store chain is not latency-bound.
// kParams = false (dg = dbeta = NULL, frozen g and b): dh only, the parameter sums and their block reduction are compiled out.
template <int NQ, int PP, bool kParams>     // float4 slots per lane, pixel groups per trip, parameter gradients
__global__ void __launch_bounds__(256, NQ == 1 ? 3 : 1)
layernorm_bwd_kernel(const float* __restrict__ dy, int dy_ld, const float* __restrict__ h, int h_ld,
                     const float* __restrict__ stats, const float* __restrict__ g, long long npix, int C,
                     const float* __restrict__ addend, int addend_ld, float* __restrict__ dh, int dh_ld,
                     float* __restrict__ dg, float* __restrict__ dbeta, int pix_per_block) {
  extern __shared__ float red[];   // [2][C]
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarp = blockDim.x >> 5;
  const int nq = C >> 2;
  const int G = nq < 32 ? nq : 32;               // lanes per pixel
  const int ppw = 32 / G;                         // pixels per warp iteration
  const int sub = lane / G, gl = lane % G;
  float4 ag[NQ], ab[NQ], gv[NQ];
#pragma unroll
  for (int i = 0; i < NQ; ++i) {
    ag[i] = make_float4(0, 0, 0, 0); ab[i] = make_float4(0, 0, 0, 0);
    const int qd = gl + i * G;
    gv[i] = qd < nq ? *reinterpret_cast<const float4*>(g + qd * 4) : make_float4(0, 0, 0, 0);
  }
  const long long p0 = static_cast<long long>(blockIdx.x) * pix_per_block;
  long long p1 = p0 + pix_per_block; if (p1 > npix) p1 = npix;
  // PP pixel groups per trip: all 2 * PP * NQ 16-byte loads of a trip are requested before the first use (one load pair per
  // thread in flight left the kernel at 0.67 of the HBM rate); pixels are visited in the same order as with PP = 1, so the
  // parameter-gradient partial sums and dh are bit-identical
  const long long stride = static_cast<long long>(nwarp) * ppw;
  for (long long base = p0 + static_cast<long long>(warp) * ppw; base < p1; base += stride * PP) {
    float4 dl[PP][NQ], hl[PP][NQ];
    float mean[PP], rstd[PP];
    bool valid[PP];
#pragma unroll
    for (int k = 0; k < PP; ++k) {
      const long long pix = base + k * stride + sub;
      valid[k] = (base + k * stride < p1) && pix < p1;
      mean[k] = 0.f; rstd[k] = 0.f;
      if (valid[k]) { mean[k] = stats[pix * 2]; rstd[k] = stats[pix * 2 + 1]; }
#pragma unroll
      for (int i = 0; i < NQ; ++i) {
        const int qd = gl + i * G;
        dl[k][i] = make_float4(0, 0, 0, 0); hl[k][i] = make_float4(0, 0, 0, 0);
        if (valid[k] && qd < nq) {
          dl[k][i] = *reinterpret_cast<const float4*>(dy + pix * dy_ld + qd * 4);
          hl[k][i] = *reinterpret_cast<const float4*>(h + pix * h_ld + qd * 4);
        }
      }
    }
#pragma unroll
    for (int k = 0; k < PP; ++k) {
      if (base + k * stride >= p1) continue;                // warp-uniform (`continue`, not `break`: the unrolled loop keeps static indices)
      const long long pix = base + k * stride + sub;
      float4 dv[NQ], xh[NQ];
      float s1 = 0.f, s2 = 0.f;
#pragma unroll
      for (int i = 0; i < NQ; ++i) {
        const int qd = gl + i * G;
        dv[i] = make_float4(0, 0, 0, 0); xh[i] = make_float4(0, 0, 0, 0);
        if (valid[k] && qd < nq) {
          const float4 d = dl[k][i];
          const float4 hv = hl[k][i];
          xh[i] = make_float4((hv.x - mean[k]) * rstd[k], (hv.y - mean[k]) * rstd[k], (hv.z - mean[k]) * rstd[k], (hv.w - mean[k]) * rstd[k]);
          if constexpr (kParams) {
            ag[i].x += d.x * xh[i].x; ag[i].y += d.y * xh[i].y; ag[i].z += d.z * xh[i].z; ag[i].w += d.w * xh[i].w;
            ab[i].x += d.x; ab[i].y += d.y; ab[i].z += d.z; ab[i].w += d.w;
          }
          dv[i] = make_float4(d.x * gv[i].x, d.y * gv[i].y, d.z * gv[i].z, d.w * gv[i].w);
          s1 += dv[i].x + dv[i].y + dv[i].z + dv[i].w;
          s2 += dv[i].x * xh[i].x + dv[i].y * xh[i].y + dv[i].z * xh[i].z + dv[i].w * xh[i].w;
        }
      }
      for (int o = G >> 1; o > 0; o >>= 1) { s1 += __shfl_xor_sync(0xffffffffu, s1, o); s2 += __shfl_xor_sync(0xffffffffu, s2, o); }
      s1 /= C; s2 /= C;
#pragma unroll
      for (int i = 0; i < NQ; ++i) {
        const int qd = gl + i * G;
        if (valid[k] && qd < nq) {
          float4 o;
          o.x = rstd[k] * (dv[i].x - s1 - xh[i].x * s2); o.y = rstd[k] * (dv[i].y - s1 - xh[i].y * s2);
          o.z = rstd[k] * (dv[i].z - s1 - xh[i].z * s2); o.w = rstd[k] * (dv[i].w - s1 - xh[i].w * s2);
          if (addend) {
            const float4 a = *reinterpret_cast<const float4*>(addend + pix * addend_ld + qd * 4);
            o.x += a.x; o.y += a.y; o.z += a.z; o.w += a.w;
          }
          *reinterpret_cast<float4*>(dh + pix * dh_ld + qd * 4) = o;
        }
      }
    }
  }
  if constexpr (kParams) {
    // block reduction of the parameter gradients, one atomicAdd per channel per block
    for (int i = threadIdx.x; i < 2 * C; i += blockDim.x) red[i] = 0.f;
    __syncthreads();
#pragma unroll
    for (int i = 0; i < NQ; ++i) {
      const int qd = gl + i * G;
      if (qd < nq) {
        atomicAdd(&red[qd * 4 + 0], ag[i].x); atomicAdd(&red[qd * 4 + 1], ag[i].y);
        atomicAdd(&red[qd * 4 + 2], ag[i].z); atomicAdd(&red[qd * 4 + 3], ag[i].w);
        atomicAdd(&red[C + qd * 4 + 0], ab[i].x); atomicAdd(&red[C + qd * 4 + 1], ab[i].y);
        atomicAdd(&red[C + qd * 4 + 2], ab[i].z); atomicAdd(&red[C + qd * 4 + 3], ab[i].w);
      }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < C; i += blockDim.x) { atomicAdd(dg + i, red[i]); atomicAdd(dbeta + i, red[C + i]); }
  }
}

// ---------------------------------------------------------------------------------------------
// depthwise 7x7 weight gradient: dw[c][ky*7+kx] += sum_{b,y,x} dh[b,y,x,c] * x[b,y+ky-3,x+kx-3,c]
// block = (b, TY x TX pixel tile, 32-channel slab): the dh tile and the x tile with its 3-pixel halo are staged in
// shared memory once; warp ky (7 warps, lane = channel) slides along x with a 7-wide register window of input row
// y+ky-3, so every pixel costs two conflict-free LDS and 7 FMAs.
// ---------------------------------------------------------------------------------------------
constexpr int kDwSeg = 4;                        // x segments per tile row: 7 ky x 4 segments = 28 warps per block
constexpr int kDwTilesPerBlock = 8;              // consecutive tiles reduced in registers before touching global memory
__global__ void __launch_bounds__(224 * kDwSeg)
dwconv7_wgrad_kernel(const float* __restrict__ dh, int dh_ld, const float* __restrict__ x, int x_ld,
                     int B, int H, int W, int C, float* __restrict__ dw, int TY, int TX) {
  extern __shared__ float sm[];                  // xs[(TY+6)][(TX+6)][32] | ds[TY][TX][32]
  __shared__ float red[49][32];
  const int XW = TX + 6;
  float* xs = sm;
  float* ds = sm + (TY + 6) * XW * 32;
  const int lane = threadIdx.x & 31, ky = (threadIdx.x >> 5) % 7, seg = (threadIdx.x >> 5) / 7;
  const int wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const int c0 = blockIdx.x * 32;
  const int tiles_x = W / TX, tiles_y = H / TY;
  const int ntiles = B * tiles_x * tiles_y;
  const bool cvalid = c0 + lane < C;
  const int TS = TX / kDwSeg, px0 = seg * TS;       // this warp's pixel columns [px0, px0 + TS)
  float acc[7] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  for (int tile = blockIdx.y * kDwTilesPerBlock; tile < min(ntiles, (static_cast<int>(blockIdx.y) + 1) * kDwTilesPerBlock); ++tile) {
    const int tx = tile % tiles_x, ty = (tile / tiles_x) % tiles_y, b = tile / (tiles_x * tiles_y);
    const int x0 = tx * TX, y0 = ty * TY;
    __syncthreads();                                // previous tile fully consumed
    // staging: one warp per tile row (lane = channel, 128-byte coalesced LDGSTS), whole tile in flight before the wait
    for (int ry = wid; ry < TY + 6; ry += nw) {
      const int iy = y0 + ry - 3;
      const bool rowok = cvalid && iy >= 0 && iy < H;
      const float* src = x + ((static_cast<long long>(b) * H + (rowok ? iy : 0)) * W) * x_ld + c0 + (cvalid ? lane : 0);
      float* dst = xs + (ry * XW) * 32 + lane;
      for (int px = 0; px < XW; ++px) {
        const int ix = x0 + px - 3;
        const bool ok = rowok && ix >= 0 && ix < W;
        cd_cp_async4(dst + px * 32, src + static_cast<long long>(ok ? ix : 0) * x_ld, ok);
      }
    }
    for (int ry = wid; ry < TY; ry += nw) {
      const float* src = dh + ((static_cast<long long>(b) * H + y0 + ry) * W + x0) * dh_ld + c0 + (cvalid ? lane : 0);
      float* dst = ds + (ry * TX) * 32 + lane;
      for (int px = 0; px < TX; ++px) cd_cp_async4(dst + px * 32, src + static_cast<long long>(px) * dh_ld, cvalid);
    }
    cd_cp_async_wait_all();
    __syncthreads();
    for (int ry = 0; ry < TY; ++ry) {
      const float* xr = xs + ((ry + ky) * XW + px0) * 32 + lane;  // input row y0+ry+ky-3, starting at x0+px0-3
      const float* dr = ds + (ry * TX + px0) * 32 + lane;
      float w0 = xr[0], w1 = xr[32], w2 = xr[64], w3 = xr[96], w4 = xr[128], w5 = xr[160], w6;
#pragma unroll 4
      for (int px = 0; px < TS; ++px) {
        w6 = xr[(px + 6) * 32];
        const float d = dr[px * 32];
        acc[0] = fmaf(d, w0, acc[0]); acc[1] = fmaf(d, w1, acc[1]); acc[2] = fmaf(d, w2, acc[2]); acc[3] = fmaf(d, w3, acc[3]);
        acc[4] = fmaf(d, w4, acc[4]); acc[5] = fmaf(d, w5, acc[5]); acc[6] = fmaf(d, w6, acc[6]);
        w0 = w1; w1 = w2; w2 = w3; w3 = w4; w4 = w5; w5 = w6;
      }
    }
  }
  // block reduction over the x segments, then ONE atomic per (channel, tap) per block
  for (int i = threadIdx.x; i < 49 * 32; i += blockDim.x) red[i / 32][i % 32] = 0.f;
  __syncthreads();
#pragma unroll
  for (int kx = 0; kx < 7; ++kx) atomicAdd(&red[ky * 7 + kx][lane], acc[kx]);
  __syncthreads();
  for (int i = threadIdx.x; i < 49 * 32; i += blockDim.x) {
    const int tap = i / 32, cl = i % 32;
    if (c0 + cl < C) atomicAdd(dw + (c0 + cl) * 49 + tap, red[tap][cl]);
  }
}

// ---------------------------------------------------------------------------------------------
// batched column sums: out[b*out_ld + c] += sum_{rows of image b} x[(b*rows + r)*ld + c]
// ---------------------------------------------------------------------------------------------
__global__ void colsum_batched_kernel(const float* __restrict__ x, int ld, long long rows, int C, float* __restrict__ out,
                                      int out_ld, long long rows_per_block) {
  const int c = blockIdx.x * 32 + (threadIdx.x & 31);
  const int ry = threadIdx.x >> 5;
  const int b = blockIdx.z;
  const long long r0 = blockIdx.y * rows_per_block;
  long long r1 = r0 + rows_per_block; if (r1 > rows) r1 = rows;
  float s = 0.f;
  if (c < C) for (long long r = r0 + ry; r < r1; r += 8) s += x[(static_cast<long long>(b) * rows + r) * ld + c];
  __shared__ float smr[8][33];
  smr[ry][threadIdx.x & 31] = s;
  __syncthreads();
  if (ry == 0 && c < C) {
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) t += smr[i][threadIdx.x & 31];
    atomicAdd(out + static_cast<long long>(b) * out_ld + c, t);
  }
}

// float4 variant (C % 4 == 0, 16-byte aligned rows, rows >= 256; colsum_batched_kernel above serves the rest): a warp covers 32/G rows x
// G channel quads (G = min(32, C/4) rounded up to a power of two), four independent 16-byte loads per thread in flight, partial
// sums meet in shared memory, one atomicAdd per channel and block.  Different summation order than the scalar kernel: results agree to fp32 rounding.
__global__ void __launch_bounds__(256)
colsum_batched_vec_kernel(const float* __restrict__ x, int ld, long long rows, int C, float* __restrict__ out, int out_ld,
                          long long rows_per_block, int G) {
  extern __shared__ float redv[];                // [G * 4]
  const int b = blockIdx.z;
  x += static_cast<long long>(b) * rows * ld;
  out += static_cast<long long>(b) * out_ld;
  const int nq = C >> 2;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int rpw = 32 / G, gl = lane % G, sub = lane / G;
  const int qd = blockIdx.x * G + gl;
  const long long r0 = blockIdx.y * rows_per_block;
  long long r1 = r0 + rows_per_block; if (r1 > rows) r1 = rows;
  float4 a0 = make_float4(0.f, 0.f, 0.f, 0.f), a1 = a0, a2 = a0, a3 = a0;
  const long long stride = 8LL * rpw;
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
  for (int i = threadIdx.x; i < G * 4; i += blockDim.x) redv[i] = 0.f;
  __syncthreads();
  if (qd < nq) {
    atomicAdd(&redv[gl * 4 + 0], a0.x); atomicAdd(&redv[gl * 4 + 1], a0.y); atomicAdd(&redv[gl * 4 + 2], a0.z); atomicAdd(&redv[gl * 4 + 3], a0.w);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < G * 4; i += blockDim.x) {
    const int c = blockIdx.x * G * 4 + i;
    if (c < C) atomicAdd(out + c, redv[i]);
  }
}

// ---------------------------------------------------------------------------------------------
// LinearAttention backward, small per-(b) part.  Inputs: dweff[b][co][hd], ctx (un-normalised), ksum, w_out.
//   ctxn[h][d][e] = ctx / ksum[h*32+d]
//   dW_out[co][h*32+e] += scale * sum_d dweff[b][co][h*32+d] * ctxn[b][h][d][e]         (atomic over b)
//   dctxn[b][h][d][e]   = scale * sum_co dweff[b][co][h*32+d] * w_out[co][h*32+e]
//   rowdot[b][h*32+d]   = sum_e dctxn * ctxn
// grid = B, block = 256
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
attn_bwd_small_kernel(const float* __restrict__ dweff, const float* __restrict__ ctx, const float* __restrict__ ksum,
                      const float* __restrict__ w_out, int dim, float scale, float* __restrict__ dw_out,
                      float* __restrict__ dctxn, float* __restrict__ rowdot) {
  // one block per (head, batch element)
  __shared__ float cn[32][33];     // ctxn[d][e]
  __shared__ float dcs[32][33];    // dctxn[d][e]
  const int h = blockIdx.x, b = blockIdx.y;
  const float* dwe = dweff + static_cast<long long>(b) * dim * 128 + h * 32;     // [co][d], row stride 128
  const float* wo = w_out + h * 32;                                              // [co][e], row stride 128
  const float* cb = ctx + (static_cast<long long>(b) * 4 + h) * 1024;
  for (int i = threadIdx.x; i < 1024; i += blockDim.x) {
    const int d = i >> 5, e = i & 31;
    cn[d][e] = cb[i] / ksum[b * 128 + h * 32 + d];
  }
  __syncthreads();
  // dctxn[d][e] = scale * sum_co dweff[co][d] * w_out[co][e]  : thread -> (d, e quad)
  {
    const int d = threadIdx.x >> 3, e4 = (threadIdx.x & 7) * 4;
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
    for (int co = 0; co < dim; ++co) {
      const float dv = dwe[co * 128 + d];
      const float4 wv = *reinterpret_cast<const float4*>(wo + co * 128 + e4);
      a0 = fmaf(dv, wv.x, a0); a1 = fmaf(dv, wv.y, a1); a2 = fmaf(dv, wv.z, a2); a3 = fmaf(dv, wv.w, a3);
    }
    dcs[d][e4] = a0 * scale; dcs[d][e4 + 1] = a1 * scale; dcs[d][e4 + 2] = a2 * scale; dcs[d][e4 + 3] = a3 * scale;
  }
  __syncthreads();
  float* dout = dctxn + (static_cast<long long>(b) * 4 + h) * 1024;
  for (int i = threadIdx.x; i < 1024; i += blockDim.x) dout[i] = dcs[i >> 5][i & 31];
  if (threadIdx.x < 32) {
    float a = 0.f;
    for (int e = 0; e < 32; ++e) a = fmaf(dcs[threadIdx.x][e], cn[threadIdx.x][e], a);
    rowdot[b * 128 + h * 32 + threadIdx.x] = a;
  }
  // dW_out[co][h*32+e] += scale * sum_d dweff[co][d] * ctxn[d][e]
  for (int o = threadIdx.x; o < dim * 32; o += blockDim.x) {
    const int co = o >> 5, e = o & 31;
    float a = 0.f;
#pragma unroll 8
    for (int d = 0; d < 32; ++d) a = fmaf(dwe[co * 128 + d], cn[d][e], a);
    atomicAdd(dw_out + co * 128 + h * 32 + e, a * scale);
  }
}

// per-pixel part: dk[n][hd] = P * (sum_e dctxn[hd][e] v[n][h,e] - rowdot[hd]),  P = exp(k-kmax)/ksum
//                 dv[n][he] = sum_d P[n][h,d] dctxn[h,d][e]
// Two 32x32 GEMMs per head and pixel.  Block = kKvTiles tiles of 32 pixels of one image; dctxn is staged once per block in
// both orientations, P and v of a tile transposed ([channel][pixel]) so that a thread owning 4 pixels x 4 channels feeds
// 32 FMAs from 4 LDS.128 per step (2 scalar LDS per FMA would make the kernel shared-memory-issue bound).
constexpr int kKvPix = 32;
constexpr int kKvTiles = 8;
constexpr int kKvStride = 36;         // floats per channel row of the transposed tiles (16-byte aligned, 4-way store conflicts)
// A warp owns ONE head and 4 pixel quads (lane = 8 channel quads x 4 pixel quads).  The heads' rows of every shared array are a
// multiple of 32 floats apart, so a warp spanning the four heads of one pixel quad would hit the same banks: each of the four
// LDS.128 of a step would cost 4 wavefronts (16 per 32 FMAs, shared-memory bound at one wavefront per clock and SM); with one
// head per warp each is one 64- or 128-byte wavefront.
// This CUDA-core kernel serves the operands the mma.sync kernel (linattn_bwd.cu) refuses: ld % 4 != 0 or unaligned qkv.
__global__ void __launch_bounds__(256)
attn_bwd_kv_kernel(const float* __restrict__ qkv, int ld, int n, const float* __restrict__ kmax,
                   const float* __restrict__ ksum, const float* __restrict__ dctxn, const float* __restrict__ rowdot,
                   float* __restrict__ dqkv, int dld, int tiles) {
  extern __shared__ float smkv[];
  float* dcA = smkv;                         // [h*32+d][e]
  float* dcB = dcA + 4096;                   // [h*32+e][d]
  float* psT = dcB + 4096;                   // [h*32+d][pixel], stride kKvStride
  float* vsT = psT + 128 * kKvStride;        // [h*32+e][pixel]
  const int b = blockIdx.y;
  const int tid = threadIdx.x;
  for (int i = tid; i < 4096; i += 256) {
    const float v = dctxn[static_cast<long long>(b) * 4096 + i];
    const int hd = i >> 5, e = i & 31;
    dcA[i] = v;
    dcB[((hd & ~31) + e) * 32 + (hd & 31)] = v;
  }
  // head = warp % 4, channel quad j4 = lane % 8, pixel quad = 4 (warp / 4) + lane / 8
  const int h = (tid >> 5) & 3;
  const int j4 = (tid & 7) * 4;
  const int pq = (tid >> 7) * 4 + ((tid & 31) >> 3);
  const int c4 = h * 32 + j4;
  const float4 rd = *reinterpret_cast<const float4*>(rowdot + b * 128 + c4);
  const int lc = tid & 127, lhalf = tid >> 7;
  const float kmx = kmax[b * 128 + lc], kinv = 1.f / ksum[b * 128 + lc];
  for (int tile = 0; tile < tiles; ++tile) {
    const int p0 = (blockIdx.x * tiles + tile) * kKvPix;
    if (p0 >= n) break;
    __syncthreads();                                 // previous tile consumed (and dc staged)
    {                                                // all 32 loads of the tile in flight before the first use
      float kr[kKvPix / 2], vr[kKvPix / 2];
#pragma unroll
      for (int u = 0; u < kKvPix / 2; ++u) {
        const int p = p0 + lhalf + 2 * u;
        kr[u] = 0.f; vr[u] = 0.f;
        if (p < n) {
          const float* row = qkv + (static_cast<long long>(b) * n + p) * ld;
          kr[u] = row[128 + lc];
          vr[u] = row[256 + lc];
        }
      }
#pragma unroll
      for (int u = 0; u < kKvPix / 2; ++u) {
        const int pp = lhalf + 2 * u;
        psT[lc * kKvStride + pp] = (p0 + pp < n) ? __expf(kr[u] - kmx) * kinv : 0.f;
        vsT[lc * kKvStride + pp] = vr[u];
      }
    }
    __syncthreads();
    float dk[4][4] = {}, dv[4][4] = {};               // [pixel][channel]
#pragma unroll 4
    for (int e = 0; e < 32; ++e) {
      const float4 vq = *reinterpret_cast<const float4*>(vsT + (h * 32 + e) * kKvStride + pq * 4);   // v[4 px][h,e]
      const float4 da = *reinterpret_cast<const float4*>(dcB + (h * 32 + e) * 32 + j4);            // dctxn[h, d=j4..][e]
      const float4 pq4 = *reinterpret_cast<const float4*>(psT + (h * 32 + e) * kKvStride + pq * 4);  // P[4 px][h, d=e]
      const float4 db = *reinterpret_cast<const float4*>(dcA + (h * 32 + e) * 32 + j4);            // dctxn[h, d=e][e'=j4..]
      const float vp[4] = {vq.x, vq.y, vq.z, vq.w}, pp_[4] = {pq4.x, pq4.y, pq4.z, pq4.w};
      const float a4[4] = {da.x, da.y, da.z, da.w}, b4[4] = {db.x, db.y, db.z, db.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) { dk[i][j] = fmaf(vp[i], a4[j], dk[i][j]); dv[i][j] = fmaf(pp_[i], b4[j], dv[i][j]); }
    }
    const float rdv[4] = {rd.x, rd.y, rd.z, rd.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int p = p0 + pq * 4 + i;
      if (p < n) {
        float* orow = dqkv + (static_cast<long long>(b) * n + p) * dld;
        float4 ok, ov;
        ok.x = psT[(c4 + 0) * kKvStride + pq * 4 + i] * (dk[i][0] - rdv[0]);
        ok.y = psT[(c4 + 1) * kKvStride + pq * 4 + i] * (dk[i][1] - rdv[1]);
        ok.z = psT[(c4 + 2) * kKvStride + pq * 4 + i] * (dk[i][2] - rdv[2]);
        ok.w = psT[(c4 + 3) * kKvStride + pq * 4 + i] * (dk[i][3] - rdv[3]);
        ov = make_float4(dv[i][0], dv[i][1], dv[i][2], dv[i][3]);
        *reinterpret_cast<float4*>(orow + 128 + c4) = ok;
        *reinterpret_cast<float4*>(orow + 256 + c4) = ov;
      }
    }
  }
}

// transpose per-batch weff [B][dim][128] -> [B][128][dim]
__global__ void transpose_weff_kernel(const float* __restrict__ w, int dim, float* __restrict__ wt) {
  const int b = blockIdx.y;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= dim * 128) return;
  const int co = i >> 7, hd = i & 127;
  wt[(static_cast<long long>(b) * 128 + hd) * dim + co] = w[static_cast<long long>(b) * dim * 128 + i];
}

// ---------------------------------------------------------------------------------------------
// final 1x1 projection backward: dx[pix][c] = sum_co dout[b][co][pix] w[co][c]; dw[co][c], db[co]
// ---------------------------------------------------------------------------------------------
// thread = (pixel group, channel): x reads are coalesced over channels, dout is a warp broadcast.
// Four pixels per trip with their loads issued first: one 4-byte load per thread in flight (8 KB per SM) left the kernel
// latency-bound at ~7x its HBM time.  Pixels are consumed in ascending order per thread; the tail goes one pixel per trip.
// CO > 0 fixes the number of image channels at compile time (3 for RGB): every per-channel array then lives in registers instead
// of local memory (the run-time Co of the CO = 0 instantiation indexes them dynamically).
template <int CO = 0>
__global__ void __launch_bounds__(256)
conv1x1_to_nchw_bwd_kernel(const float* __restrict__ dout, const float* __restrict__ x, int ld, int B, int HW, int C,
                           const float* __restrict__ w, int Co_rt, float* __restrict__ dx, int dx_ld,
                           float* __restrict__ dw, float* __restrict__ db, int pix_per_block) {
  constexpr int U = 4;                // pixels per trip
  const int Co = CO > 0 ? CO : Co_rt;
  extern __shared__ float red[];      // [groups][Co][C]
  const int groups = blockDim.x / C;
  const int c = threadIdx.x % C, gq = threadIdx.x / C;
  const long long npix = static_cast<long long>(B) * HW;
  const long long p0 = static_cast<long long>(blockIdx.x) * pix_per_block;
  long long p1 = p0 + pix_per_block; if (p1 > npix) p1 = npix;
  float wv[8], acc[8], accb[8];
  for (int co = 0; co < Co; ++co) { wv[co] = w[co * C + c]; acc[co] = 0.f; accb[co] = 0.f; }
  if (gq < groups) {
    long long pix = p0 + gq;
    for (; pix + static_cast<long long>(U - 1) * groups < p1; pix += static_cast<long long>(U) * groups) {
      float xv[U], dv[U][8];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const long long pu = pix + static_cast<long long>(u) * groups;
        const int b = static_cast<int>(pu / HW), p = static_cast<int>(pu % HW);
        xv[u] = x[pu * ld + c];
#pragma unroll
        for (int co = 0; co < (CO > 0 ? CO : 8); ++co)
          if (co < Co) dv[u][co] = dout[(static_cast<long long>(b) * Co + co) * HW + p];
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        float d = 0.f;
#pragma unroll
        for (int co = 0; co < (CO > 0 ? CO : 8); ++co) {
          if (co < Co) {
            d = fmaf(dv[u][co], wv[co], d);
            acc[co] = fmaf(dv[u][co], xv[u], acc[co]);
            accb[co] += dv[u][co];
          }
        }
        dx[(pix + static_cast<long long>(u) * groups) * dx_ld + c] = d;
      }
    }
    for (; pix < p1; pix += groups) {
      const int b = static_cast<int>(pix / HW), p = static_cast<int>(pix % HW);
      const float xv = x[pix * ld + c];
      float d = 0.f;
      for (int co = 0; co < Co; ++co) {
        const float dv = dout[(static_cast<long long>(b) * Co + co) * HW + p];
        d = fmaf(dv, wv[co], d);
        acc[co] = fmaf(dv, xv, acc[co]);
        accb[co] += dv;
      }
      dx[pix * dx_ld + c] = d;
    }
    for (int co = 0; co < Co; ++co) red[(gq * Co + co) * C + c] = acc[co];
  }
  __syncthreads();
  if (gq == 0) {
    for (int co = 0; co < Co; ++co) {
      float t = 0.f;
      for (int k = 0; k < groups; ++k) t += red[(k * Co + co) * C + c];
      atomicAdd(dw + co * C + c, t);
    }
  }
  // bias gradient: channel-0 threads of every group hold partial sums over their pixels
  __syncthreads();
  if (c == 0 && gq < groups) for (int co = 0; co < Co; ++co) red[gq * Co + co] = accb[co];
  __syncthreads();
  if (threadIdx.x < Co) {
    float t = 0.f;
    for (int k = 0; k < groups; ++k) t += red[k * Co + threadIdx.x];
    atomicAdd(db + threadIdx.x, t);
  }
}

// ---------------------------------------------------------------------------------------------
// tiny dense helpers for the time-MLP backward
// ---------------------------------------------------------------------------------------------
// C[m][n] (+)= sum_k A(m,k) * B(k,n); A(m,k) = transA ? A[k*lda+m] : A[m*lda+k]; same for B
__global__ void small_gemm_kernel(const float* __restrict__ A, int lda, int transA, const float* __restrict__ Bm, int ldb,
                                  int transB, float* __restrict__ Cm, int ldc, int M, int N, int K, int accumulate) {
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= static_cast<long long>(M) * N) return;
  const int n = static_cast<int>(idx % N), m = static_cast<int>(idx / N);
  float a = 0.f;
  for (int k = 0; k < K; ++k) {
    const float av = transA ? A[static_cast<long long>(k) * lda + m] : A[static_cast<long long>(m) * lda + k];
    const float bv = transB ? Bm[static_cast<long long>(n) * ldb + k] : Bm[static_cast<long long>(k) * ldb + n];
    a = fmaf(av, bv, a);
  }
  float* o = Cm + static_cast<long long>(m) * ldc + n;
  *o = accumulate ? *o + a : a;
}
// long-K variant: grid (ceil(M*N/128), KS); every block reduces a K slice and adds it atomically (C zeroed by the host when
// not accumulating).  The time-embedding backward has M*N = 2048 outputs over K ~ 6000 (all conditioning channels).
__global__ void small_gemm_splitk_kernel(const float* __restrict__ A, int lda, int transA, const float* __restrict__ Bm, int ldb,
                                         int transB, float* __restrict__ Cm, int ldc, int M, int N, int K, int kslice) {
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= static_cast<long long>(M) * N) return;
  const int n = static_cast<int>(idx % N), m = static_cast<int>(idx / N);
  const int k0 = blockIdx.y * kslice;
  int k1 = k0 + kslice; if (k1 > K) k1 = K;
  float a = 0.f;
  for (int k = k0; k < k1; ++k) {
    const float av = transA ? A[static_cast<long long>(k) * lda + m] : A[static_cast<long long>(m) * lda + k];
    const float bv = transB ? Bm[static_cast<long long>(n) * ldb + k] : Bm[static_cast<long long>(k) * ldb + n];
    a = fmaf(av, bv, a);
  }
  atomicAdd(Cm + static_cast<long long>(m) * ldc + n, a);
}
// y[i] = dy[i] * gelu'(pre[i])   (y may alias dy);  act_out (optional) = gelu(pre)
__global__ void gelu_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ pre, long long n,
                                float* __restrict__ y, float* __restrict__ act_out) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float p = pre[i];
  if (act_out) act_out[i] = cd_gelu(p);
  if (y) y[i] = dy[i] * cd_gelu_grad(p);
}

// out[pix][c] = a[pix][c] + b[pix][c]
__global__ void add_kernel(const float* __restrict__ a, int a_ld, const float* __restrict__ b, int b_ld,
                           float* __restrict__ out, int out_ld, long long npix, int C) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= npix * C) return;
  const long long pix = i / C; const int c = static_cast<int>(i % C);
  out[pix * out_ld + c] = a[pix * a_ld + c] + b[pix * b_ld + c];
}

}  // namespace

extern "C" int cd_add(const float* a, int a_ld, const float* b, int b_ld, float* out, int out_ld, int64_t npix, int C,
                      void* stream) {
  add_kernel<<<cd_cdiv(npix * C, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(a, a_ld, b, b_ld, out, out_ld, npix, C);
  CD_LAUNCH_CHECK();
  return 0;
}

extern "C" int cd_layernorm_bwd(const float* dy, int dy_ld, const float* h, int h_ld, const float* stats,
                                const float* g, int64_t npix, int C, const float* addend, int addend_ld,
                                float* dh, int dh_ld, float* dg, float* dbeta, void* stream) {
  CD_REQUIRE(C % 4 == 0 && C <= 1024 && dy_ld % 4 == 0 && h_ld % 4 == 0 && dh_ld % 4 == 0, "cd_layernorm_bwd: unsupported C=%d", C);
  const int nq = C / 4;
  CD_REQUIRE((nq & (nq - 1)) == 0 || nq >= 32, "cd_layernorm_bwd: C/4 must be a power of two below 128 channels (C=%d)", C);
  // pixels per block: at most 512, but never fewer than ~4 blocks per SM (8192 pixels of the 16x16 level gave 16 blocks)
  int ppb = static_cast<int>(npix / (cd_num_sms() * 4));
  if (ppb > 512) ppb = 512;
  if (ppb < 32) ppb = 32;
  const int blocks = cd_cdiv(npix, ppb);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  CD_REQUIRE((dg == nullptr) == (dbeta == nullptr), "cd_layernorm_bwd: dg and dbeta are both given or both NULL");
  const size_t smem = dg ? sizeof(float) * 2 * C : 0;
  const int slots = nq <= 32 ? 1 : cd_cdiv(nq, 32);
#define CD_LNB(N, P) do { \
    if (dg) layernorm_bwd_kernel<N, P, true><<<blocks, 256, smem, st>>>(dy, dy_ld, h, h_ld, stats, g, npix, C, addend, addend_ld, dh, dh_ld, dg, dbeta, ppb); \
    else layernorm_bwd_kernel<N, P, false><<<blocks, 256, smem, st>>>(dy, dy_ld, h, h_ld, stats, g, npix, C, addend, addend_ld, dh, dh_ld, dg, dbeta, ppb); \
  } while (0)
  if (slots == 1) CD_LNB(1, 4); else if (slots == 2) CD_LNB(2, 2); else if (slots <= 4) CD_LNB(4, 1); else CD_LNB(8, 1);
#undef CD_LNB
  CD_LAUNCH_CHECK();
  return 0;
}

int cd_dwconv7_wgrad_pipe(const float* dh, int dh_ld, const float* x, int x_ld, int B, int H, int W, int C, float* dw, cudaStream_t st);

extern "C" int cd_dwconv7_wgrad(const float* dh, int dh_ld, const float* x, int x_ld, int B, int H, int W, int C,
                                float* dw, void* stream) {
  {
    const int rc = cd_dwconv7_wgrad_pipe(dh, dh_ld, x, x_ld, B, H, W, C, dw, static_cast<cudaStream_t>(stream));
    if (rc <= 0) return rc;                           // 1: shape not eligible for the persistent kernel
  }
  // tile: TX = min(W, 32), TY <= 8 so that two blocks (2 x 28 warps) fit one SM (~100 KB of shared memory each)
  int TX = W < 32 ? W : 32;
  while (W % TX) --TX;
  CD_REQUIRE(TX % kDwSeg == 0, "cd_dwconv7_wgrad: image width %d unsupported", W);
  int TY = H < 8 ? H : 8;
  while (H % TY) --TY;
  auto bytes = [&](int ty) { return sizeof(float) * 32 * (size_t(ty + 6) * (TX + 6) + size_t(ty) * TX); };
  while (TY > 1 && bytes(TY) > 110 * 1024) { --TY; while (H % TY) --TY; }
  const size_t smem = bytes(TY);
  CD_REQUIRE(smem <= 200 * 1024, "cd_dwconv7_wgrad: tile does not fit (W=%d)", W);
  static size_t attr = 0;
  if (smem > attr) { CD_CUDA(cudaFuncSetAttribute(dwconv7_wgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); attr = smem; }
  dim3 grid(cd_cdiv(C, 32), cd_cdiv(B * (H / TY) * (W / TX), kDwTilesPerBlock));
  dwconv7_wgrad_kernel<<<grid, 224 * kDwSeg, smem, static_cast<cudaStream_t>(stream)>>>(dh, dh_ld, x, x_ld, B, H, W, C, dw, TY, TX);
  CD_LAUNCH_CHECK();
  return 0;
}

extern "C" int cd_colsum_batched(const float* x, int ld, int B, int64_t rows, int C, float* out, int out_ld, void* stream) {
  if (C % 4 == 0 && ld % 4 == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0 && rows >= 256) {
    const int nq = C / 4;
    int G = 1; while (G < nq && G < 32) G <<= 1;
    const int xb = cd_cdiv(nq, G);
    long long rpbv = rows * xb * B / (cd_num_sms() * 4);          // >= 4 blocks per SM over the whole batch
    if (rpbv > 1024) rpbv = 1024;
    if (rpbv < 64) rpbv = 64;
    dim3 gv(xb, cd_cdiv(rows, rpbv), B);
    colsum_batched_vec_kernel<<<gv, 256, sizeof(float) * G * 4, static_cast<cudaStream_t>(stream)>>>(x, ld, rows, C, out, out_ld, rpbv, G);
    CD_LAUNCH_CHECK();
    return 0;
  }
  const long long rpb = 2048;
  dim3 grid(cd_cdiv(C, 32), cd_cdiv(rows, rpb), B);
  colsum_batched_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(x, ld, rows, C, out, out_ld, rpb);
  CD_LAUNCH_CHECK();
  return 0;
}

extern "C" int cd_linattn_bwd_small(const float* dweff, const float* ctx, const float* ksum, const float* w_out,
                                    int B, int dim, float scale, float* dw_out, float* dctxn, float* rowdot, void* stream) {
  if (cd_linattn_aligned(w_out, dweff))
    return cd_linattn_bwd_small_staged(dweff, ctx, ksum, w_out, B, dim, scale, dw_out, dctxn, rowdot, static_cast<cudaStream_t>(stream));
  attn_bwd_small_kernel<<<dim3(4, B), 256, 0, static_cast<cudaStream_t>(stream)>>>(dweff, ctx, ksum, w_out, dim, scale, dw_out, dctxn, rowdot);
  CD_LAUNCH_CHECK();
  return 0;
}

extern "C" int cd_linattn_bwd_kv(const float* qkv, int ld, int B, int n, const float* kmax, const float* ksum,
                                 const float* dctxn, const float* rowdot, float* dqkv, int dld, void* stream) {
  CD_REQUIRE(dld % 4 == 0 && (reinterpret_cast<uintptr_t>(dqkv) & 15) == 0, "cd_linattn_bwd_kv: dqkv must be 16-byte aligned with dld %% 4 == 0");
  {
    const int rc = cd_linattn_bwd_kv_mma(qkv, ld, B, n, kmax, ksum, dctxn, rowdot, dqkv, dld, static_cast<cudaStream_t>(stream));
    if (rc <= 0) return rc;                      // 1: ld % 4 != 0 or unaligned qkv -> CUDA-core kernel
  }
  const size_t smem = sizeof(float) * (2 * 4096 + 2 * 128 * kKvStride);
  static bool attr = false;
  if (!attr) {
    CD_CUDA(cudaFuncSetAttribute(attn_bwd_kv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr = true;
  }
  // tiles per block: up to kKvTiles (amortises the 32 KB dctxn staging), fewer when that would leave SMs idle
  int tiles = static_cast<int>(static_cast<long long>(cd_cdiv(n, kKvPix)) * B / (cd_num_sms() * 2));
  if (tiles > kKvTiles) tiles = kKvTiles;
  if (tiles < 1) tiles = 1;
  dim3 grid(cd_cdiv(n, kKvPix * tiles), B);
  attn_bwd_kv_kernel<<<grid, 256, smem, static_cast<cudaStream_t>(stream)>>>(qkv, ld, n, kmax, ksum, dctxn, rowdot, dqkv, dld, tiles);
  CD_LAUNCH_CHECK();
  return 0;
}

extern "C" int cd_transpose_weff(const float* weff, int B, int dim, float* weff_t, void* stream) {
  dim3 grid(cd_cdiv(dim * 128, 256), B);
  transpose_weff_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(weff, dim, weff_t);
  CD_LAUNCH_CHECK();
  return 0;
}

extern "C" int cd_conv1x1_to_nchw_bwd(const float* dout_nchw, const float* x, int ld, int B, int H, int W, int C,
                                      const float* w, int Co, float* dx, int dx_ld, float* dw, float* db, void* stream) {
  CD_REQUIRE(Co <= 8 && C <= 256, "cd_conv1x1_to_nchw_bwd: at most 8 image channels / 256 features");
  const long long npix = static_cast<long long>(B) * H * W;
  const int groups = 256 / C;
  const size_t smem = sizeof(float) * size_t(groups) * Co * C;
  const int ppb = 1024;
  if (Co == 3)
    conv1x1_to_nchw_bwd_kernel<3><<<cd_cdiv(npix, ppb), 256, smem, static_cast<cudaStream_t>(stream)>>>(dout_nchw, x, ld, B, H * W, C, w, Co,
                                                                                                      dx, dx_ld, dw, db, ppb);
  else
    conv1x1_to_nchw_bwd_kernel<><<<cd_cdiv(npix, ppb), 256, smem, static_cast<cudaStream_t>(stream)>>>(dout_nchw, x, ld, B, H * W, C, w, Co,
                                                                                                     dx, dx_ld, dw, db, ppb);
  CD_LAUNCH_CHECK();
  return 0;
}

extern "C" int cd_small_gemm(const float* A, int lda, int transA, const float* Bm, int ldb, int transB,
                             float* Cm, int ldc, int M, int N, int K, int accumulate, void* stream) {
  const long long total = static_cast<long long>(M) * N;
  if (K >= 512 && total <= cd_num_sms() * 128) {
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (!accumulate) CD_CUDA(cudaMemset2DAsync(Cm, sizeof(float) * ldc, 0, sizeof(float) * N, M, st));
    const int ks = cd_cdiv(cd_num_sms() * 4, cd_cdiv(total, 128));
    const int kslice = cd_cdiv(K, ks);
    dim3 grid(cd_cdiv(total, 128), cd_cdiv(K, kslice));
    small_gemm_splitk_kernel<<<grid, 128, 0, st>>>(A, lda, transA, Bm, ldb, transB, Cm, ldc, M, N, K, kslice);
    CD_LAUNCH_CHECK();
    return 0;
  }
  small_gemm_kernel<<<cd_cdiv(total, 128), 128, 0, static_cast<cudaStream_t>(stream)>>>(A, lda, transA, Bm, ldb, transB, Cm, ldc, M, N, K, accumulate);
  CD_LAUNCH_CHECK();
  return 0;
}

extern "C" int cd_gelu_bwd(const float* dy, const float* pre, int64_t n, float* y, float* act_out, void* stream) {
  gelu_bwd_kernel<<<cd_cdiv(n, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(dy, pre, n, y, act_out);
  CD_LAUNCH_CHECK();
  return 0;
}
