// HBM-bound pieces of the Unet forward (NHWC fp32): depthwise 7x7 + time-conditioning + channel
// LayerNorm (ConvNextBlock head, DB:145,159-162,111-121), PreNorm LayerNorm (DB:123-131), the time
// MLP (DB:91-103,209-216,140-143), the LinearAttention softmax/context reduction (DB:176-187), the
// final 1x1 projection to image channels (DB:253) and NCHW<->NHWC boundary conversion.
#include "cd_common.cuh"
#include <mutex>
#include <vector>

namespace {

// ---------------------------------------------------------------------------------------------
// dwconv7x7 + bias + cond + LayerNorm.  One thread = 8 consecutive x-pixels x 4 channels.
// blockDim = (C/4) * strips; LN statistics reduced across the C/4 threads of a strip.
// ---------------------------------------------------------------------------------------------
constexpr int kStrip = 8;

template <bool kNorm>
__global__ void __launch_bounds__(256)
dwconv7_ln_kernel(const float* __restrict__ x, int x_ld, int B, int H, int W, int C,
                  const float* __restrict__ wdw, const float* __restrict__ bdw, const float* __restrict__ cond, int cond_ld,
                  const float* __restrict__ g, const float* __restrict__ beta, float eps,
                  float* __restrict__ y, int y_ld, float* __restrict__ stats, float* __restrict__ hpre, int hpre_ld,
                  int round_tf32, int flip, const float* __restrict__ addend, int addend_ld) {
  extern __shared__ float red[];                 // [strips][warps_per_strip][kStrip]
  const int cq = C >> 2;                         // channel quads (threads per strip)
  const int strip_in_block = threadIdx.x / cq;
  const int q = threadIdx.x % cq;
  const int strips_per_block = blockDim.x / cq;
  const int strips_x = W / kStrip;
  const long long strip = static_cast<long long>(blockIdx.x) * strips_per_block + strip_in_block;
  const long long nstrips = static_cast<long long>(B) * H * strips_x;
  const bool active = strip < nstrips;
  const int sx = active ? static_cast<int>(strip % strips_x) : 0;
  const long long rr = active ? strip / strips_x : 0;
  const int yy = static_cast<int>(rr % H), b = static_cast<int>(rr / H);
  const int x0 = sx * kStrip, c0 = q * 4;

  float4 acc[kStrip];
#pragma unroll
  for (int i = 0; i < kStrip; ++i) acc[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  if (active) {
    const float* w0 = wdw + (c0 + 0) * 49; const float* w1 = wdw + (c0 + 1) * 49;
    const float* w2 = wdw + (c0 + 2) * 49; const float* w3 = wdw + (c0 + 3) * 49;
#pragma unroll 1
    for (int ky = 0; ky < 7; ++ky) {
      const int iy = yy + ky - 3;
      if (iy < 0 || iy >= H) continue;
      float4 wv[7];
#pragma unroll
      for (int kx = 0; kx < 7; ++kx) {
        const int wi = flip ? 48 - (ky * 7 + kx) : ky * 7 + kx;
        wv[kx] = make_float4(__ldg(w0 + wi), __ldg(w1 + wi), __ldg(w2 + wi), __ldg(w3 + wi));
      }
      const float* row = x + ((static_cast<long long>(b) * H + iy) * W) * x_ld + c0;
#pragma unroll
      for (int ix = 0; ix < kStrip + 6; ++ix) {
        const int gx = x0 + ix - 3;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (gx >= 0 && gx < W) v = *reinterpret_cast<const float4*>(row + static_cast<long long>(gx) * x_ld);
#pragma unroll
        for (int ox = 0; ox < kStrip; ++ox) {
          const int kx = ix - ox;
          if (kx >= 0 && kx < 7) {
            acc[ox].x = fmaf(v.x, wv[kx].x, acc[ox].x); acc[ox].y = fmaf(v.y, wv[kx].y, acc[ox].y);
            acc[ox].z = fmaf(v.z, wv[kx].z, acc[ox].z); acc[ox].w = fmaf(v.w, wv[kx].w, acc[ox].w);
          }
        }
      }
    }
    float4 add = bdw ? *reinterpret_cast<const float4*>(bdw + c0) : make_float4(0.f, 0.f, 0.f, 0.f);
    if (cond) {
      const float4 cv = *reinterpret_cast<const float4*>(cond + static_cast<long long>(b) * cond_ld + c0);
      add.x += cv.x; add.y += cv.y; add.z += cv.z; add.w += cv.w;
    }
#pragma unroll
    for (int i = 0; i < kStrip; ++i) { acc[i].x += add.x; acc[i].y += add.y; acc[i].z += add.z; acc[i].w += add.w; }
  }
  const long long pix0 = (static_cast<long long>(b) * H + yy) * W + x0;
  if (addend && active) {
#pragma unroll
    for (int i = 0; i < kStrip; ++i) {
      const float4 a = *reinterpret_cast<const float4*>(addend + (pix0 + i) * addend_ld + c0);
      acc[i].x += a.x; acc[i].y += a.y; acc[i].z += a.z; acc[i].w += a.w;
    }
  }
  if (hpre && active) {
#pragma unroll
    for (int i = 0; i < kStrip; ++i) *reinterpret_cast<float4*>(hpre + (pix0 + i) * hpre_ld + c0) = acc[i];
  }
  if (kNorm) {
    // two-pass statistics over the C channels of each of the kStrip pixels
    const int width = cq < 32 ? cq : 32;           // lanes sharing a strip inside a warp
    const int wps = (cq + 31) / 32;                // warps per strip
    const int warp_in_strip = q >> 5;
    float mean[kStrip], rstd[kStrip];
    for (int pass = 0; pass < 2; ++pass) {
      float part[kStrip];
#pragma unroll
      for (int i = 0; i < kStrip; ++i) {
        float s;
        if (pass == 0) s = acc[i].x + acc[i].y + acc[i].z + acc[i].w;
        else {
          const float a = acc[i].x - mean[i], bb = acc[i].y - mean[i], c = acc[i].z - mean[i], d = acc[i].w - mean[i];
          s = a * a + bb * bb + c * c + d * d;
        }
        for (int o = width >> 1; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        part[i] = s;
      }
      if (wps > 1) {
        __syncthreads();
        if ((q & 31) == 0) {
#pragma unroll
          for (int i = 0; i < kStrip; ++i) red[(strip_in_block * wps + warp_in_strip) * kStrip + i] = part[i];
        }
        __syncthreads();
#pragma unroll
        for (int i = 0; i < kStrip; ++i) {
          float s = 0.f;
          for (int w = 0; w < wps; ++w) s += red[(strip_in_block * wps + w) * kStrip + i];
          part[i] = s;
        }
      }
#pragma unroll
      for (int i = 0; i < kStrip; ++i) {
        if (pass == 0) mean[i] = part[i] / C;
        else rstd[i] = rsqrtf(part[i] / C + eps);
      }
    }
    if (active) {
      const float4 gv = *reinterpret_cast<const float4*>(g + c0);
      const float4 bv = *reinterpret_cast<const float4*>(beta + c0);
#pragma unroll
      for (int i = 0; i < kStrip; ++i) {
        float4 o;
        o.x = (acc[i].x - mean[i]) * rstd[i] * gv.x + bv.x; o.y = (acc[i].y - mean[i]) * rstd[i] * gv.y + bv.y;
        o.z = (acc[i].z - mean[i]) * rstd[i] * gv.z + bv.z; o.w = (acc[i].w - mean[i]) * rstd[i] * gv.w + bv.w;
        if (round_tf32) { o.x = cd_round_tf32(o.x); o.y = cd_round_tf32(o.y); o.z = cd_round_tf32(o.z); o.w = cd_round_tf32(o.w); }
        *reinterpret_cast<float4*>(y + (pix0 + i) * y_ld + c0) = o;
        if (stats && q == 0) { stats[(pix0 + i) * 2] = mean[i]; stats[(pix0 + i) * 2 + 1] = rstd[i]; }
      }
    }
  } else if (active) {
#pragma unroll
    for (int i = 0; i < kStrip; ++i) {
      float4 o = acc[i];
      if (round_tf32) { o.x = cd_round_tf32(o.x); o.y = cd_round_tf32(o.y); o.z = cd_round_tf32(o.z); o.w = cd_round_tf32(o.w); }
      *reinterpret_cast<float4*>(y + (pix0 + i) * y_ld + c0) = o;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// depthwise 7x7 (+bias +cond +addend), shared-memory tiled: block = 32-channel slab x (TY x TX) pixel tile whose input
// (with the 3-pixel halo) is staged once; warp = output row, lane = channel.  A thread walks the input columns of its
// row band: each new column (7 LDS) feeds the 7 output pixels in flight (49 FMA); finished pixels leave through a
// 7-deep accumulator shift -- no re-reads, stores are 128-byte coalesced.  FMA-bound (49 FMA / pixel / channel).
// ---------------------------------------------------------------------------------------------
constexpr int kDwTY = 8;
__global__ void __launch_bounds__(32 * kDwTY)
dwconv7_tile_kernel(const float* __restrict__ x, int x_ld, int B, int H, int W, int C,
                    const float* __restrict__ wdw, const float* __restrict__ bdw, const float* __restrict__ cond, int cond_ld,
                    float* __restrict__ out, int out_ld, int flip, const float* __restrict__ addend, int addend_ld, int TX, int TY) {
  extern __shared__ float xs[];                  // [(TY+6)][(TX+6)][32]
  const int XW = TX + 6;
  const int lane = threadIdx.x & 31, ry = threadIdx.x >> 5;
  const int c0 = blockIdx.x * 32, c = c0 + lane;
  const bool cvalid = c < C;
  const int tiles_x = W / TX, tiles_y = H / TY;
  const int tx = blockIdx.y % tiles_x, ty = (blockIdx.y / tiles_x) % tiles_y, b = blockIdx.y / (tiles_x * tiles_y);
  const int x0 = tx * TX, y0 = ty * TY;
  for (int r = ry; r < TY + 6; r += kDwTY) {
    const int iy = y0 + r - 3;
    const bool rowok = cvalid && iy >= 0 && iy < H;
    const float* src = x + ((static_cast<long long>(b) * H + (rowok ? iy : 0)) * W) * x_ld + (cvalid ? c : 0);
    float* dst = xs + (r * XW) * 32 + lane;
    for (int px = 0; px < XW; ++px) {                       // LDGSTS: all copies of the tile are in flight together
      const int ix = x0 + px - 3;
      const bool ok = rowok && ix >= 0 && ix < W;
      cd_cp_async4(dst + px * 32, src + static_cast<long long>(ok ? ix : 0) * x_ld, ok);
    }
  }
  // the 32 x 49 filter slab of this block is one contiguous run of wdw: copy it coalesced (a per-thread gather has a
  // 49-float lane stride, 32 sectors per load, repeated by all 8 warps); row stride 49 is odd -> conflict-free reads
  float* wsm = xs + (TY + 6) * XW * 32;
  {
    const int nw = (C - c0 < 32 ? C - c0 : 32) * 49;
    for (int i = threadIdx.x; i < nw; i += blockDim.x) cd_cp_async4(wsm + i, wdw + static_cast<long long>(c0) * 49 + i, true);
  }
  float add = (cvalid && bdw) ? bdw[c] : 0.f;
  if (cvalid && cond) add += cond[static_cast<long long>(b) * cond_ld + c];
  cd_cp_async_wait_all();
  __syncthreads();
  if (ry >= TY) return;
  float w[49];
#pragma unroll
  for (int k = 0; k < 49; ++k) w[k] = cvalid ? wsm[lane * 49 + (flip ? 48 - k : k)] : 0.f;
  float acc[7] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  const float* band = xs + (ry * XW) * 32 + lane;          // rows ry .. ry+6 of the staged tile = input rows y-3 .. y+3
  const long long orow = (static_cast<long long>(b) * H + y0 + ry) * W + x0;
  for (int cx = 0; cx < XW; ++cx) {                          // staged column cx = input x0 + cx - 3
    float col[7];
#pragma unroll
    for (int ky = 0; ky < 7; ++ky) col[ky] = band[(ky * XW + cx) * 32];
    // slot o holds output pixel (x0 + cx - o); this column is its kx = o tap
#pragma unroll
    for (int o = 0; o < 7; ++o) {
#pragma unroll
      for (int ky = 0; ky < 7; ++ky) acc[o] = fmaf(w[ky * 7 + o], col[ky], acc[o]);
    }
    const int px = cx - 6;                                   // output pixel completed by this column (tile-local)
    if (px >= 0 && cvalid) {
      float v = acc[6] + add;
      if (addend) v += addend[(orow + px) * addend_ld + c];
      out[(orow + px) * out_ld + c] = v;
    }
#pragma unroll
    for (int o = 6; o > 0; --o) acc[o] = acc[o - 1];
    acc[0] = 0.f;
  }
}

// ---------------------------------------------------------------------------------------------
// Persistent, double-buffered variant (C % 32 == 0, H >= 16): one block per SM walks (32-channel slab, TY x TX tile) work
// items; while the 16 row-warps compute tile i from one shared-memory buffer, tile i+1 streams into the other with 16-byte
// LDGSTS (zero-filled outside the image).  The one-tile-per-block kernel above exposed every tile's load latency (two
// resident blocks per SM cannot cover it) and ran at ~22 % of the FMA rate it is bound by.
// ---------------------------------------------------------------------------------------------
constexpr int kDwPTY = 16;
// stage one (TY+6) x (TX+6) x 32-channel input tile (zero outside the image) with 16-byte LDGSTS; 8 lanes per pixel
template <int TX>
__device__ __forceinline__ void dw_issue_tile(float* buf, const float* __restrict__ base, int x_ld, int H, int W, int x0, int y0) {
  constexpr int XW = TX + 6, YH = kDwPTY + 6;
  for (int i = threadIdx.x; i < YH * XW * 8; i += 32 * kDwPTY) {
    const int q = i & 7, cell = i >> 3;
    const int r = cell / XW, px = cell - r * XW;        // XW is a compile-time constant: multiply-shift, no division
    const int iy = y0 + r, ix = x0 + px;
    const bool ok = static_cast<unsigned>(iy) < static_cast<unsigned>(H) && static_cast<unsigned>(ix) < static_cast<unsigned>(W);
    cd_cp_async16(buf + cell * 32 + q * 4, base + (static_cast<long long>(ok ? iy : 0) * W + (ok ? ix : 0)) * x_ld + q * 4, ok);
  }
}

template <int TX>
__global__ void __launch_bounds__(32 * kDwPTY, 1)
dwconv7_pipe_kernel(const float* __restrict__ x, int x_ld, int B, int H, int W, int C,
                    const float* __restrict__ wdw, const float* __restrict__ bdw, const float* __restrict__ cond, int cond_ld,
                    float* __restrict__ out, int out_ld, int flip, const float* __restrict__ addend, int addend_ld) {
  extern __shared__ __align__(16) float xsp[];       // 2 x [(TY+6)][(TX+6)][32]
  constexpr int TY = kDwPTY, XW = TX + 6, YH = TY + 6;
  constexpr int tile_floats = YH * XW * 32;
  const int lane = threadIdx.x & 31, ry = threadIdx.x >> 5;
  const int tiles_x = W / TX, tiles_y = H / TY;
  const int ntiles = B * tiles_x * tiles_y;
  const int total = (C / 32) * ntiles;                 // slab-major: consecutive items of a block mostly share the filter slab

  auto issue = [&](int item, float* buf) {
    const int slab = item / ntiles, t = item - slab * ntiles;
    const int tx = t % tiles_x, ty = (t / tiles_x) % tiles_y, b = t / (tiles_x * tiles_y);
    dw_issue_tile<TX>(buf, x + static_cast<long long>(b) * H * W * x_ld + slab * 32, x_ld, H, W, tx * TX - 3, ty * TY - 3);
    asm volatile("cp.async.commit_group;" ::: "memory");
  };

  int item = blockIdx.x;
  if (item >= total) return;
  int bufi = 0;
  issue(item, xsp);
  float w[49];
  int cur_slab = -1;
  for (; item < total; item += gridDim.x) {
    const int nxt = item + gridDim.x;
    const float* buf = xsp + bufi * tile_floats;
    if (nxt < total) {
      issue(nxt, xsp + (bufi ^ 1) * tile_floats);
      asm volatile("cp.async.wait_group 1;" ::: "memory");
    } else {
      asm volatile("cp.async.wait_group 0;" ::: "memory");
    }
    __syncthreads();
    const int slab = item / ntiles, t = item - slab * ntiles;
    const int tx = t % tiles_x, ty = (t / tiles_x) % tiles_y, b = t / (tiles_x * tiles_y);
    const int c = slab * 32 + lane;
    if (slab != cur_slab) {
      cur_slab = slab;
#pragma unroll
      for (int k = 0; k < 49; ++k) w[k] = __ldg(wdw + static_cast<long long>(c) * 49 + (flip ? 48 - k : k));
    }
    {
      float add = bdw ? bdw[c] : 0.f;
      if (cond) add += cond[static_cast<long long>(b) * cond_ld + c];
      float acc[7] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
      const float* band = buf + (ry * XW) * 32 + lane;
      const long long opix = (static_cast<long long>(b) * H + ty * TY + ry) * W + tx * TX;
      float* outp = out + opix * out_ld + c;
      const float* addp = addend ? addend + opix * addend_ld + c : nullptr;
      // fully unrolled: every LDS has an immediate offset, the 7-slot accumulator shift is register renaming
#pragma unroll
      for (int cx = 0; cx < XW; ++cx) {
        float col[7];
#pragma unroll
        for (int ky = 0; ky < 7; ++ky) col[ky] = band[(ky * XW + cx) * 32];
#pragma unroll
        for (int o = 0; o < 7; ++o) {
#pragma unroll
          for (int ky = 0; ky < 7; ++ky) acc[o] = fmaf(w[ky * 7 + o], col[ky], acc[o]);
        }
        if (cx >= 6) {
          float v = acc[6] + add;
          if (addp) { v += *addp; addp += addend_ld; }
          *outp = v; outp += out_ld;
        }
#pragma unroll
        for (int o = 6; o > 0; --o) acc[o] = acc[o - 1];
        acc[0] = 0.f;
      }
    }
    __syncthreads();                                   // buffer fully read before the next iteration's prefetch overwrites it
    bufi ^= 1;
  }
}

// Weight gradient with the same structure (the mirror image of the forward: 49 accumulators per channel, a 7x7 input window
// slides along the row of the warp, one new column (7 LDS) + one dY value per pixel feed 49 FMAs).  Tiles of 16 x 16 outputs:
// input tile + dY tile = 94 KB, double-buffered; accumulators live across all items of a slab and leave through one
// shared-memory reduction over the 16 row-warps and one atomicAdd per (channel, tap) per block and slab.
constexpr int kDwWTX = 16;
__global__ void __launch_bounds__(32 * kDwPTY, 1)
dwconv7_wgrad_pipe_kernel(const float* __restrict__ dh, int dh_ld, const float* __restrict__ x, int x_ld,
                          int B, int H, int W, int C, float* __restrict__ dw) {
  extern __shared__ __align__(16) float xsw[];       // 2 x ( [(TY+6)][(TX+6)][32] | [TY][TX][32] )
  constexpr int TX = kDwWTX, TY = kDwPTY, XW = TX + 6, YH = TY + 6;
  constexpr int x_floats = YH * XW * 32, d_floats = TY * TX * 32, buf_floats = x_floats + d_floats;
  __shared__ float red[49][32];
  const int lane = threadIdx.x & 31, ry = threadIdx.x >> 5;
  const int tiles_x = W / TX, tiles_y = H / TY;
  const int ntiles = B * tiles_x * tiles_y;
  const int total = (C / 32) * ntiles;

  auto issue = [&](int item, float* buf) {
    const int slab = item / ntiles, t = item - slab * ntiles;
    const int tx = t % tiles_x, ty = (t / tiles_x) % tiles_y, b = t / (tiles_x * tiles_y);
    dw_issue_tile<TX>(buf, x + static_cast<long long>(b) * H * W * x_ld + slab * 32, x_ld, H, W, tx * TX - 3, ty * TY - 3);
    const float* dbase = dh + ((static_cast<long long>(b) * H + ty * TY) * W + tx * TX) * dh_ld + slab * 32;
    float* dbuf = buf + x_floats;
    for (int i = threadIdx.x; i < TY * TX * 8; i += 32 * kDwPTY) {
      const int q = i & 7, cell = i >> 3;
      const int r = cell / TX, px = cell - r * TX;
      cd_cp_async16(dbuf + cell * 32 + q * 4, dbase + (static_cast<long long>(r) * W + px) * dh_ld + q * 4, true);
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };
  auto flush = [&](float (&acc)[49], int slab) {        // all threads of the block
    for (int i = threadIdx.x; i < 49 * 32; i += blockDim.x) red[i >> 5][i & 31] = 0.f;
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 49; ++k) { atomicAdd(&red[k][lane], acc[k]); acc[k] = 0.f; }
    __syncthreads();
    for (int i = threadIdx.x; i < 49 * 32; i += blockDim.x)
      atomicAdd(dw + static_cast<long long>(slab * 32 + (i & 31)) * 49 + (i >> 5), red[i >> 5][i & 31]);
    __syncthreads();
  };

  int item = blockIdx.x;
  if (item >= total) return;
  int bufi = 0;
  issue(item, xsw);
  float acc[49];
#pragma unroll
  for (int k = 0; k < 49; ++k) acc[k] = 0.f;
  int cur_slab = item / ntiles;
  for (; item < total; item += gridDim.x) {
    const int nxt = item + gridDim.x;
    const float* buf = xsw + bufi * buf_floats;
    if (nxt < total) {
      issue(nxt, xsw + (bufi ^ 1) * buf_floats);
      asm volatile("cp.async.wait_group 1;" ::: "memory");
    } else {
      asm volatile("cp.async.wait_group 0;" ::: "memory");
    }
    __syncthreads();
    const int slab = item / ntiles;
    if (slab != cur_slab) { flush(acc, cur_slab); cur_slab = slab; }
    {
      const float* band = buf + (ry * XW) * 32 + lane;            // input rows ry .. ry+6 (image rows y-3 .. y+3)
      const float* drow = buf + x_floats + (ry * TX) * 32 + lane;
      float win[7][7];                                            // win[ky][kx] = x[y+ky-3][px+kx-3]
#pragma unroll
      for (int kx = 1; kx < 7; ++kx)
#pragma unroll
        for (int ky = 0; ky < 7; ++ky) win[ky][kx] = band[(ky * XW + kx - 1) * 32];
#pragma unroll
      for (int px = 0; px < TX; ++px) {
#pragma unroll
        for (int ky = 0; ky < 7; ++ky) {
#pragma unroll
          for (int kx = 0; kx < 6; ++kx) win[ky][kx] = win[ky][kx + 1];
          win[ky][6] = band[(ky * XW + px + 6) * 32];
        }
        const float d = drow[px * 32];
#pragma unroll
        for (int ky = 0; ky < 7; ++ky)
#pragma unroll
          for (int kx = 0; kx < 7; ++kx) acc[ky * 7 + kx] = fmaf(d, win[ky][kx], acc[ky * 7 + kx]);
      }
    }
    __syncthreads();
    bufi ^= 1;
  }
  flush(acc, cur_slab);
}

// generic (any C, e.g. the 1/3-channel image): one thread per pixel, loops channels; LN optional.
__global__ void dwconv7_small_kernel(const float* __restrict__ x, int x_ld, int B, int H, int W, int C,
                                     const float* __restrict__ wdw, const float* __restrict__ bdw,
                                     const float* __restrict__ cond, int cond_ld, const float* __restrict__ g,
                                     const float* __restrict__ beta, float eps, float* __restrict__ y, int y_ld,
                                     float* __restrict__ stats, float* __restrict__ hpre, int hpre_ld, int round_tf32,
                                     int flip, const float* __restrict__ addend, int addend_ld) {
  const long long pix = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long npix = static_cast<long long>(B) * H * W;
  if (pix >= npix) return;
  const int xx = static_cast<int>(pix % W);
  const int yy = static_cast<int>((pix / W) % H);
  const int b = static_cast<int>(pix / (static_cast<long long>(W) * H));
  float hbuf[16];
  float mean = 0.f;
  for (int c = 0; c < C; ++c) {
    float a = (bdw ? bdw[c] : 0.f) + (cond ? cond[static_cast<long long>(b) * cond_ld + c] : 0.f);
    if (addend) a += addend[pix * addend_ld + c];
    for (int ky = 0; ky < 7; ++ky) {
      const int iy = yy + ky - 3;
      if (iy < 0 || iy >= H) continue;
      for (int kx = 0; kx < 7; ++kx) {
        const int ix = xx + kx - 3;
        if (ix < 0 || ix >= W) continue;
        a = fmaf(x[((static_cast<long long>(b) * H + iy) * W + ix) * x_ld + c], wdw[c * 49 + (flip ? 48 - (ky * 7 + kx) : ky * 7 + kx)], a);
      }
    }
    hbuf[c] = a; mean += a;
    if (hpre) hpre[pix * hpre_ld + c] = a;
  }
  if (g) {
    mean /= C;
    float var = 0.f;
    for (int c = 0; c < C; ++c) var += (hbuf[c] - mean) * (hbuf[c] - mean);
    const float rstd = rsqrtf(var / C + eps);
    for (int c = 0; c < C; ++c) hbuf[c] = (hbuf[c] - mean) * rstd * g[c] + beta[c];
    if (stats) { stats[pix * 2] = mean; stats[pix * 2 + 1] = rstd; }
  }
  for (int c = 0; c < C; ++c) y[pix * y_ld + c] = round_tf32 ? cd_round_tf32(hbuf[c]) : hbuf[c];
}

// ---------------------------------------------------------------------------------------------
// channel LayerNorm: lanes are split into groups of G = min(32, C/4) (power of two); each group owns one pixel,
// each lane NQ float4 slots (C <= 1024, C % 4 == 0).  In place (y == x) is allowed.
// ---------------------------------------------------------------------------------------------
template <int NQ>
__global__ void __launch_bounds__(256)
layernorm_kernel(const float* __restrict__ x, int x_ld, long long npix, int C, const float* __restrict__ g,
                 const float* __restrict__ beta, float eps, float* __restrict__ y, int y_ld,
                 float* __restrict__ stats, int round_tf32) {
  const int lane = threadIdx.x & 31;
  const int nq = C >> 2;
  const int G = nq < 32 ? nq : 32;
  const int ppw = 32 / G, sub = lane / G, gl = lane % G;
  const long long pix = (static_cast<long long>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5)) * ppw + sub;
  const bool valid = pix < npix;
  float4 v[NQ];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < NQ; ++i) {
    const int qd = gl + i * G;
    v[i] = make_float4(0, 0, 0, 0);
    if (valid && qd < nq) { v[i] = *reinterpret_cast<const float4*>(x + pix * x_ld + qd * 4); s += v[i].x + v[i].y + v[i].z + v[i].w; }
  }
  for (int o = G >> 1; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float mean = s / C;
  float s2 = 0.f;
#pragma unroll
  for (int i = 0; i < NQ; ++i) {
    const int qd = gl + i * G;
    if (valid && qd < nq) {
      const float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
      s2 += a * a + b * b + c * c + d * d;
    }
  }
  for (int o = G >> 1; o > 0; o >>= 1) s2 += __shfl_xor_sync(0xffffffffu, s2, o);
  const float rstd = rsqrtf(s2 / C + eps);
#pragma unroll
  for (int i = 0; i < NQ; ++i) {
    const int qd = gl + i * G;
    if (valid && qd < nq) {
      const float4 gv = *reinterpret_cast<const float4*>(g + qd * 4);
      const float4 bv = *reinterpret_cast<const float4*>(beta + qd * 4);
      float4 o;
      o.x = (v[i].x - mean) * rstd * gv.x + bv.x; o.y = (v[i].y - mean) * rstd * gv.y + bv.y;
      o.z = (v[i].z - mean) * rstd * gv.z + bv.z; o.w = (v[i].w - mean) * rstd * gv.w + bv.w;
      if (round_tf32) { o.x = cd_round_tf32(o.x); o.y = cd_round_tf32(o.y); o.z = cd_round_tf32(o.z); o.w = cd_round_tf32(o.w); }
      *reinterpret_cast<float4*>(y + pix * y_ld + qd * 4) = o;
    }
  }
  if (stats && valid && gl == 0) { stats[pix * 2] = mean; stats[pix * 2 + 1] = rstd; }
}

// ---------------------------------------------------------------------------------------------
// time MLP: one block per batch element
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
time_mlp_kernel(const long long* __restrict__ t, int dim, const float* __restrict__ w1, const float* __restrict__ b1,
                const float* __restrict__ w2, const float* __restrict__ b2, const float* __restrict__ wc,
                const float* __restrict__ bc, int sumC, float* __restrict__ sinemb, float* __restrict__ hid_pre,
                float* __restrict__ temb, float* __restrict__ cond_all) {
  extern __shared__ float sm[];          // emb[dim] | hid[4dim] | gt[dim]
  float* emb = sm; float* hid = sm + dim; float* gt = hid + 4 * dim;
  const int b = blockIdx.x;
  const float tv = static_cast<float>(t[b]);
  const int half = dim / 2;
  const float k = logf(10000.f) / (half - 1);
  for (int i = threadIdx.x; i < half; i += blockDim.x) {
    const float f = expf(-k * i);
    const float a = tv * f;
    emb[i] = sinf(a); emb[i + half] = cosf(a);
  }
  __syncthreads();
  if (sinemb) for (int i = threadIdx.x; i < dim; i += blockDim.x) sinemb[b * dim + i] = emb[i];
  for (int o = threadIdx.x; o < 4 * dim; o += blockDim.x) {
    float a = b1[o];
    for (int i = 0; i < dim; ++i) a = fmaf(w1[o * dim + i], emb[i], a);
    if (hid_pre) hid_pre[b * 4 * dim + o] = a;
    hid[o] = cd_gelu(a);
  }
  __syncthreads();
  for (int o = threadIdx.x; o < dim; o += blockDim.x) {
    float a = b2[o];
    for (int i = 0; i < 4 * dim; ++i) a = fmaf(w2[o * 4 * dim + i], hid[i], a);
    temb[b * dim + o] = a;
    gt[o] = cd_gelu(a);
  }
}

// conditioning rows of every ConvNextBlock (GELU -> Linear(dim, block_dim), DB:143-146) for all batch elements:
// cond_all[b][o] = bc[o] + sum_i wc[o][i] * act(temb[b][i]), act = GELU (ConvNeXt Unet) or swish (DDPM Model, M2:121).
// grid (row chunks, B); one warp per output row, lanes stride the (coalesced) weight row, so the ~6000 rows
// are spread over the GPU instead of running serially inside the one-block-per-sample kernel above.
constexpr int kCondRows = 64;
__global__ void __launch_bounds__(256)
cond_proj_kernel(const float* __restrict__ temb, int dim, const float* __restrict__ wc, const float* __restrict__ bc, int sumC,
                 float* __restrict__ cond_all, int swish) {
  extern __shared__ float gt[];          // [dim]
  const int b = blockIdx.y;
  for (int i = threadIdx.x; i < dim; i += blockDim.x) {
    const float a = temb[b * dim + i];
    gt[i] = swish ? a / (1.f + expf(-a)) : cd_gelu(a);
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const int o0 = blockIdx.x * kCondRows;
  const int o1 = o0 + kCondRows < sumC ? o0 + kCondRows : sumC;
  for (int o = o0 + warp; o < o1; o += nw) {
    const float* wr = wc + static_cast<long long>(o) * dim;
    float a = 0.f;
    for (int i = lane; i < dim; i += 32) a = fmaf(wr[i], gt[i], a);
    a = cd_warp_sum(a);
    if (lane == 0) cond_all[static_cast<long long>(b) * sumC + o] = a + bc[o];
  }
}

// ---------------------------------------------------------------------------------------------
// LinearAttention: effective output weights from the context (linattn_ctx.cu computes kmax / ksum / ctx).
// ---------------------------------------------------------------------------------------------
// weff[b][co][h*32+d] = scale * sum_e w_out[co][h*32+e] * ctx[b][h][d][e] / ksum[b][h*32+d]
// block = (head, batch element): the normalised 32x32 context is staged in shared memory.
__global__ void __launch_bounds__(256)
weff_kernel(const float* __restrict__ ctx, const float* __restrict__ ksum, const float* __restrict__ w_out,
            int dim, float scale, int round_tf32, float* __restrict__ weff) {
  __shared__ float cn[32][33];
  const int h = blockIdx.x, b = blockIdx.y;
  const float* cb = ctx + (static_cast<long long>(b) * 4 + h) * 1024;
  for (int i = threadIdx.x; i < 1024; i += blockDim.x) {
    const int d = i >> 5, e = i & 31;
    cn[d][e] = cb[i] * scale / ksum[b * 128 + h * 32 + d];
  }
  __syncthreads();
  for (int o = threadIdx.x; o < dim * 32; o += blockDim.x) {
    const int co = o >> 5, d = o & 31;
    const float* wrow = w_out + co * 128 + h * 32;
    float a = 0.f;
#pragma unroll 8
    for (int e = 0; e < 32; ++e) a = fmaf(__ldg(wrow + e), cn[d][e], a);
    weff[(static_cast<long long>(b) * dim + co) * 128 + h * 32 + d] = round_tf32 ? cd_round_tf32(a) : a;
  }
}

// ---------------------------------------------------------------------------------------------
// final 1x1 conv to image channels, NHWC -> NCHW; and NCHW -> NHWC (padded ld) input conversion
// ---------------------------------------------------------------------------------------------
__global__ void conv1x1_to_nchw_kernel(const float* __restrict__ x, int ld, int B, int HW, int C,
                                       const float* __restrict__ w, const float* __restrict__ bias, int Co,
                                       const float* __restrict__ resid, float* __restrict__ out) {
  const long long pix = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (pix >= static_cast<long long>(B) * HW) return;
  const int b = static_cast<int>(pix / HW), p = static_cast<int>(pix % HW);
  const float* row = x + pix * ld;
  for (int co = 0; co < Co; ++co) {
    float a = bias ? bias[co] : 0.f;
    for (int c = 0; c < C; c += 4) {
      const float4 v = *reinterpret_cast<const float4*>(row + c);
      const float4 wv = *reinterpret_cast<const float4*>(w + co * C + c);
      a = fmaf(v.x, wv.x, a); a = fmaf(v.y, wv.y, a); a = fmaf(v.z, wv.z, a); a = fmaf(v.w, wv.w, a);
    }
    const long long o = (static_cast<long long>(b) * Co + co) * HW + p;
    if (resid) a += resid[o];
    out[o] = a;
  }
}

__global__ void nchw_to_nhwc_kernel(const float* __restrict__ x, int B, int C, int HW, float* __restrict__ out, int ld) {
  const long long pix = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (pix >= static_cast<long long>(B) * HW) return;
  const int b = static_cast<int>(pix / HW), p = static_cast<int>(pix % HW);
  for (int c = 0; c < ld; ++c) out[pix * ld + c] = c < C ? x[(static_cast<long long>(b) * C + c) * HW + p] : 0.f;
}

}  // namespace

extern "C" int cd_dwconv7_ln_fwd(const float* x, int x_ld, int B, int H, int W, int C,
                                 const float* w_dw, const float* b_dw, const float* cond, int cond_ld,
                                 const float* g, const float* beta, float eps, float* y, int y_ld,
                                 float* stats, float* hpre, int hpre_ld, int round_tf32, int flip,
                                 const float* addend, int addend_ld, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int cq = C / 4;
  const bool fast = (C % 4 == 0) && cq >= 8 && cq <= 256 && (cq & (cq - 1)) == 0 && (W % kStrip == 0) &&
                    (x_ld % 4 == 0) && (y_ld % 4 == 0) && (!hpre || hpre_ld % 4 == 0) && (!addend || addend_ld % 4 == 0);
  if (fast) {
    const int strips_per_block = 256 / cq;
    const long long nstrips = static_cast<long long>(B) * H * (W / kStrip);
    const int blocks = cd_cdiv(nstrips, strips_per_block);
    const size_t smem = sizeof(float) * strips_per_block * ((cq + 31) / 32) * kStrip;
    if (g) dwconv7_ln_kernel<true><<<blocks, 256, smem, st>>>(x, x_ld, B, H, W, C, w_dw, b_dw, cond, cond_ld, g, beta, eps, y, y_ld, stats, hpre, hpre_ld, round_tf32, flip, addend, addend_ld);
    else dwconv7_ln_kernel<false><<<blocks, 256, smem, st>>>(x, x_ld, B, H, W, C, w_dw, b_dw, cond, cond_ld, g, beta, eps, y, y_ld, stats, hpre, hpre_ld, round_tf32, flip, addend, addend_ld);
  } else {
    CD_REQUIRE(C <= 16, "cd_dwconv7_ln_fwd: unsupported channel count %d (W=%d)", C, W);
    const long long npix = static_cast<long long>(B) * H * W;
    dwconv7_small_kernel<<<cd_cdiv(npix, 128), 128, 0, st>>>(x, x_ld, B, H, W, C, w_dw, b_dw, cond, cond_ld, g, beta, eps, y, y_ld, stats, hpre, hpre_ld, round_tf32, flip, addend, addend_ld);
  }
  CD_LAUNCH_CHECK();
  return 0;
}

extern "C" int cd_layernorm_fwd(const float* x, int x_ld, int64_t npix, int C, const float* g, const float* beta,
                                float eps, float* y, int y_ld, float* stats, int round_tf32, void* stream) {
  CD_REQUIRE(C % 4 == 0 && C <= 1024 && x_ld % 4 == 0 && y_ld % 4 == 0, "cd_layernorm_fwd: unsupported C=%d", C);
  const int nq = C / 4;
  CD_REQUIRE((nq & (nq - 1)) == 0 || nq >= 32, "cd_layernorm_fwd: C/4 must be a power of two below 128 channels (C=%d)", C);
  const int G = nq < 32 ? nq : 32, ppw = 32 / G, slots = nq <= 32 ? 1 : cd_cdiv(nq, 32);
  const int blocks = cd_cdiv(npix, 8 * ppw);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (slots == 1 && g != nullptr && beta != nullptr) {
    const int rc = cd_layernorm_fwd_multi(x, x_ld, npix, C, g, beta, eps, y, y_ld, stats, round_tf32, st);   // layernorm_multi.cu
    if (rc <= 0) return rc;
  }
#define CD_LNF(N) layernorm_kernel<N><<<blocks, 256, 0, st>>>(x, x_ld, npix, C, g, beta, eps, y, y_ld, stats, round_tf32)
  if (slots == 1) CD_LNF(1); else if (slots == 2) CD_LNF(2); else if (slots <= 4) CD_LNF(4); else CD_LNF(8);
#undef CD_LNF
  CD_LAUNCH_CHECK();
  return 0;
}

// returns 1 when the shape is not eligible (caller falls back to dwconv7_wgrad_kernel in backward.cu)
int cd_dwconv7_wgrad_pipe(const float* dh, int dh_ld, const float* x, int x_ld, int B, int H, int W, int C, float* dw, cudaStream_t st);
static int g_dw_pipe = 1;     // 1: persistent double-buffered depthwise kernels where eligible; 0: one tile per block
extern "C" int cd_dwconv7_set_pipe(int enable) { g_dw_pipe = enable; return 0; }

// dwconv_tma.cu: the same kernels with TMA-staged tiles; 1 = not eligible / switched off
int cd_dwconv7_fwd_tma(const float* x, int x_ld, int B, int H, int W, int C, const float* w_dw, const float* b_dw,
                       const float* cond, int cond_ld, float* out, int out_ld, int flip, const float* addend, int addend_ld,
                       cudaStream_t st);
int cd_dwconv7_wgrad_tma(const float* dh, int dh_ld, const float* x, int x_ld, int B, int H, int W, int C, float* dw, cudaStream_t st);

int cd_dwconv7_wgrad_pipe(const float* dh, int dh_ld, const float* x, int x_ld, int B, int H, int W, int C, float* dw, cudaStream_t st) {
  if (g_dw_pipe) {
    const int rc = cd_dwconv7_wgrad_tma(dh, dh_ld, x, x_ld, B, H, W, C, dw, st);
    if (rc <= 0) return rc;
  }
  if (!g_dw_pipe || C % 32 != 0 || H % kDwPTY != 0 || W % kDwWTX != 0 || x_ld % 4 != 0 || dh_ld % 4 != 0 ||
      (reinterpret_cast<uintptr_t>(x) & 15) != 0 || (reinterpret_cast<uintptr_t>(dh) & 15) != 0) return 1;
  const size_t smem = sizeof(float) * 2 * 32 * (size_t(kDwPTY + 6) * (kDwWTX + 6) + size_t(kDwPTY) * kDwWTX);
  static bool attr = false;
  if (!attr) { CD_CUDA(cudaFuncSetAttribute(dwconv7_wgrad_pipe_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); attr = true; }
  const long long total = static_cast<long long>(C / 32) * B * (H / kDwPTY) * (W / kDwWTX);
  const int grid = total < cd_num_sms() ? static_cast<int>(total) : cd_num_sms();
  dwconv7_wgrad_pipe_kernel<<<grid, 32 * kDwPTY, smem, st>>>(dh, dh_ld, x, x_ld, B, H, W, C, dw);
  CD_LAUNCH_CHECK();
  return 0;
}

extern "C" int cd_dwconv7_fwd(const float* x, int x_ld, int B, int H, int W, int C, const float* w_dw, const float* b_dw,
                              const float* cond, int cond_ld, float* out, int out_ld, int flip, const float* addend,
                              int addend_ld, void* stream) {
  if (g_dw_pipe) {
    const int rc = cd_dwconv7_fwd_tma(x, x_ld, B, H, W, C, w_dw, b_dw, cond, cond_ld, out, out_ld, flip, addend, addend_ld,
                                      static_cast<cudaStream_t>(stream));
    if (rc <= 0) return rc;
  }
  if (C % 32 == 0 && H % kDwPTY == 0 && W % 16 == 0 && x_ld % 4 == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0 && g_dw_pipe) {
    const int TXp = W % 32 == 0 ? 32 : 16;
    const size_t smem = sizeof(float) * 2 * 32 * size_t(kDwPTY + 6) * (TXp + 6);
    static bool attr_p = false;
    if (!attr_p) {
      CD_CUDA(cudaFuncSetAttribute(dwconv7_pipe_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(sizeof(float) * 2 * 32 * (kDwPTY + 6) * 38)));
      CD_CUDA(cudaFuncSetAttribute(dwconv7_pipe_kernel<16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(sizeof(float) * 2 * 32 * (kDwPTY + 6) * 22)));
      attr_p = true;
    }
    const long long total = static_cast<long long>(C / 32) * B * (H / kDwPTY) * (W / TXp);
    const int grid = total < cd_num_sms() ? static_cast<int>(total) : cd_num_sms();
    if (TXp == 32)
      dwconv7_pipe_kernel<32><<<grid, 32 * kDwPTY, smem, static_cast<cudaStream_t>(stream)>>>(x, x_ld, B, H, W, C, w_dw, b_dw, cond, cond_ld,
                                                                                            out, out_ld, flip, addend, addend_ld);
    else
      dwconv7_pipe_kernel<16><<<grid, 32 * kDwPTY, smem, static_cast<cudaStream_t>(stream)>>>(x, x_ld, B, H, W, C, w_dw, b_dw, cond, cond_ld,
                                                                                            out, out_ld, flip, addend, addend_ld);
    CD_LAUNCH_CHECK();
    return 0;
  }
  int TX = W < 32 ? W : 32;
  int TY = H < kDwTY ? H : kDwTY;
  CD_REQUIRE(W % TX == 0 && H % TY == 0, "cd_dwconv7_fwd: unsupported image size %dx%d", H, W);
  const size_t smem = sizeof(float) * 32 * (size_t(TY + 6) * (TX + 6) + 49);
  static size_t attr = 0;
  if (smem > 48 * 1024 && smem > attr) { CD_CUDA(cudaFuncSetAttribute(dwconv7_tile_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); attr = smem; }
  dim3 grid(cd_cdiv(C, 32), B * (H / TY) * (W / TX));
  dwconv7_tile_kernel<<<grid, 32 * kDwTY, smem, static_cast<cudaStream_t>(stream)>>>(x, x_ld, B, H, W, C, w_dw, b_dw, cond, cond_ld,
                                                                                  out, out_ld, flip, addend, addend_ld, TX, TY);
  CD_LAUNCH_CHECK();
  return 0;
}

extern "C" int cd_time_mlp_fwd(const int64_t* t, int B, int dim, const float* w1, const float* b1,
                               const float* w2, const float* b2, const float* wc, const float* bc, int sumC,
                               float* sinemb, float* hid_pre, float* temb, float* cond_all, void* stream) {
  const size_t smem = sizeof(float) * 6 * dim;
  time_mlp_kernel<<<B, 256, smem, static_cast<cudaStream_t>(stream)>>>(reinterpret_cast<const long long*>(t), dim, w1, b1, w2, b2,
                                                                     wc, bc, sumC, sinemb, hid_pre, temb, cond_all);
  CD_LAUNCH_CHECK();
  if (sumC > 0) {
    cond_proj_kernel<<<dim3(cd_cdiv(sumC, kCondRows), B), 256, sizeof(float) * dim, static_cast<cudaStream_t>(stream)>>>(temb, dim, wc, bc, sumC, cond_all, 0);
    CD_LAUNCH_CHECK();
  }
  return 0;
}

extern "C" int cd_linattn_weff(const float* ctx, const float* ksum, const float* w_out, int B, int dim, float scale,
                               int round_tf32, float* weff, void* stream) {
  if (cd_linattn_aligned(w_out, nullptr))
    return cd_linattn_weff_staged(ctx, ksum, w_out, B, dim, scale, round_tf32, weff, static_cast<cudaStream_t>(stream));
  weff_kernel<<<dim3(4, B), 256, 0, static_cast<cudaStream_t>(stream)>>>(ctx, ksum, w_out, dim, scale, round_tf32, weff);
  CD_LAUNCH_CHECK();
  return 0;
}

extern "C" int cd_conv1x1_to_nchw(const float* x, int ld, int B, int H, int W, int C, const float* w,
                                  const float* b, int Co, const float* resid_nchw, float* out_nchw, void* stream) {
  CD_REQUIRE(C % 4 == 0 && ld % 4 == 0, "cd_conv1x1_to_nchw: C must be a multiple of 4");
  const long long npix = static_cast<long long>(B) * H * W;
  {                                                      // tile through shared memory (final_proj.cu) where eligible
    const int rc = cd_conv1x1_to_nchw_tiled(x, ld, npix, H * W, C, w, b, Co, resid_nchw, out_nchw, static_cast<cudaStream_t>(stream));
    if (rc <= 0) return rc;
  }
  conv1x1_to_nchw_kernel<<<cd_cdiv(npix, 128), 128, 0, static_cast<cudaStream_t>(stream)>>>(x, ld, B, H * W, C, w, b, Co, resid_nchw, out_nchw);
  CD_LAUNCH_CHECK();
  return 0;
}

extern "C" int cd_nchw_to_nhwc(const float* x, int B, int C, int H, int W, float* out, int ld, void* stream) {
  const long long npix = static_cast<long long>(B) * H * W;
  nchw_to_nhwc_kernel<<<cd_cdiv(npix, 128), 128, 0, static_cast<cudaStream_t>(stream)>>>(x, B, C, H * W, out, ld);
  CD_LAUNCH_CHECK();
  return 0;
}

// =============================================================================================================
// DDPM-style `Model` (Model2.py, "M2") forward pieces: GroupNorm(32, eps 1e-6) [+ per-(b,c) time-embedding add]
// [+ swish] (M2:27-33,114-123), row softmax of the AttnBlock (M2:172-175), nearest 2x upsample (M2:47-48), batched
// transpose (value matrix of the AttnBlock, M2:178-181) and NHWC -> NCHW for the 3-channel output.
// =============================================================================================================
namespace {
// one block per batch element: (mean, rstd) per group from cd_gn_plane_stats (cd_common.cuh: shifted per-thread sums merged
// with Chan's formula in a fixed order), then y = (x + cond - mean) * rstd * gamma + beta [swish].
__global__ void __launch_bounds__(512)
groupnorm_kernel(const float* __restrict__ x, int x_ld, int HW, int C, int groups, const float* __restrict__ cond, int cond_ld,
                 const float* __restrict__ gamma, const float* __restrict__ beta, float eps, int swish,
                 float* __restrict__ y, int y_ld) {
  __shared__ float tm[4][512], tq[4][512];
  extern __shared__ float gst[];                // (mean, rstd)[groups]
  const int b = blockIdx.x;
  const int nq = C >> 2, cg = C / groups;
  const long long base = static_cast<long long>(b) * HW;
  // thread -> (pixel lane, channel quad): consecutive threads walk consecutive quads of one pixel (coalesced)
  const int q = threadIdx.x % nq, pl = threadIdx.x / nq, np = blockDim.x / nq;
  cd_gn_plane_stats(x, x_ld, HW, C, groups, cond, cond_ld, eps, b, tm, tq, gst);
  __syncthreads();
  if (pl < np) {
    float4 cadd = make_float4(0.f, 0.f, 0.f, 0.f);
    if (cond) cadd = *reinterpret_cast<const float4*>(cond + static_cast<long long>(b) * cond_ld + q * 4);
    float mean[4], rstd[4];
    for (int j = 0; j < 4; ++j) {
      const int g = (q * 4 + j) / cg;
      mean[j] = gst[2 * g]; rstd[j] = gst[2 * g + 1];
    }
    const float4 gm = *reinterpret_cast<const float4*>(gamma + q * 4);
    const float4 bt = *reinterpret_cast<const float4*>(beta + q * 4);
    for (int p = pl; p < HW; p += np) {
      float4 v = *reinterpret_cast<const float4*>(x + (base + p) * x_ld + q * 4);
      float o[4] = {(v.x + cadd.x - mean[0]) * rstd[0] * gm.x + bt.x, (v.y + cadd.y - mean[1]) * rstd[1] * gm.y + bt.y,
                    (v.z + cadd.z - mean[2]) * rstd[2] * gm.z + bt.z, (v.w + cadd.w - mean[3]) * rstd[3] * gm.w + bt.w};
      if (swish) for (int j = 0; j < 4; ++j) o[j] = o[j] / (1.f + __expf(-o[j]));
      *reinterpret_cast<float4*>(y + (base + p) * y_ld + q * 4) = make_float4(o[0], o[1], o[2], o[3]);
    }
  }
}

// softmax over the last dimension of [rows][n] (row stride ld), scale applied first; warp per row
__global__ void softmax_rows_kernel(float* __restrict__ s, int ld, long long rows, int n, float scale) {
  const long long row = static_cast<long long>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  float* r = s + row * ld;
  float m = -INFINITY;
  for (int j = lane; j < n; j += 32) m = fmaxf(m, r[j] * scale);
  m = cd_warp_max(m);
  float sum = 0.f;
  for (int j = lane; j < n; j += 32) { const float e = expf(r[j] * scale - m); r[j] = e; sum += e; }
  sum = cd_warp_sum(sum);
  const float inv = 1.f / sum;
  for (int j = lane; j < n; j += 32) r[j] *= inv;
}

// [B][R][Cc] (row stride ld) -> [B][Cc][R]
__global__ void transpose_batched_kernel(const float* __restrict__ src, int ld, int R, int Cc, float* __restrict__ dst) {
  __shared__ float t[32][33];
  const int b = blockIdx.z, r0 = blockIdx.y * 32, c0 = blockIdx.x * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int r = r0 + i, c = c0 + threadIdx.x;
    t[i][threadIdx.x] = (r < R && c < Cc) ? src[(static_cast<long long>(b) * R + r) * ld + c] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int c = c0 + i, r = r0 + threadIdx.x;
    if (r < R && c < Cc) dst[(static_cast<long long>(b) * Cc + c) * R + r] = t[threadIdx.x][i];
  }
}

__global__ void upsample_nearest2x_kernel(const float* __restrict__ x, int x_ld, int B, int H, int W, int C, float* __restrict__ y, int y_ld) {
  const int nq = C >> 2;
  const long long total = static_cast<long long>(B) * 4 * H * W * nq;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int q = static_cast<int>(i % nq);
    const long long op = i / nq;
    const int ox = static_cast<int>(op % (2 * W)), oy = static_cast<int>((op / (2 * W)) % (2 * H)), b = static_cast<int>(op / (4LL * H * W));
    const float4 v = *reinterpret_cast<const float4*>(x + ((static_cast<long long>(b) * H + oy / 2) * W + ox / 2) * x_ld + q * 4);
    *reinterpret_cast<float4*>(y + op * y_ld + q * 4) = v;
  }
}

// out (NCHW) = x (NHWC, row stride ld) [+ add (NCHW, same shape as out)]
__global__ void nhwc_to_nchw_kernel(const float* __restrict__ x, int ld, int B, int HW, int C, const float* __restrict__ add,
                                    float* __restrict__ out) {
  const long long pix = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (pix >= static_cast<long long>(B) * HW) return;
  const int b = static_cast<int>(pix / HW), p = static_cast<int>(pix % HW);
  for (int c = 0; c < C; ++c) {
    const long long o = (static_cast<long long>(b) * C + c) * HW + p;
    out[o] = add ? x[pix * ld + c] + add[o] : x[pix * ld + c];
  }
}

// generalised time MLP: emb(dim) -> hid (act) -> tdim ; cond_all = Wc act(temb) + bc.  act: 0 gelu, 1 swish
__global__ void __launch_bounds__(256)
time_mlp2_kernel(const long long* __restrict__ t, int dim, int hid, int tdim, int act, const float* __restrict__ w1,
                 const float* __restrict__ b1, const float* __restrict__ w2, const float* __restrict__ b2,
                 const float* __restrict__ wc, const float* __restrict__ bc, int sumC, float* __restrict__ temb,
                 float* __restrict__ cond_all) {
  extern __shared__ float sm[];          // emb[dim] | h[hid] | gt[tdim]
  float* emb = sm; float* h = sm + dim; float* gt = h + hid;
  const int b = blockIdx.x;
  const float tv = static_cast<float>(t[b]);
  const int half = dim / 2;
  const float k = logf(10000.f) / (half - 1);
  for (int i = threadIdx.x; i < half; i += blockDim.x) { const float a = tv * expf(-k * i); emb[i] = sinf(a); emb[i + half] = cosf(a); }
  if ((dim & 1) && threadIdx.x == 0) emb[dim - 1] = 0.f;
  __syncthreads();
  for (int o = threadIdx.x; o < hid; o += blockDim.x) {
    float a = b1[o];
    for (int i = 0; i < dim; ++i) a = fmaf(w1[o * dim + i], emb[i], a);
    h[o] = act ? a / (1.f + expf(-a)) : cd_gelu(a);
  }
  __syncthreads();
  for (int o = threadIdx.x; o < tdim; o += blockDim.x) {
    float a = b2[o];
    for (int i = 0; i < hid; ++i) a = fmaf(w2[o * hid + i], h[i], a);
    if (temb) temb[b * tdim + o] = a;
    gt[o] = act ? a / (1.f + expf(-a)) : cd_gelu(a);
  }
  __syncthreads();
  for (int o = threadIdx.x; o < sumC; o += blockDim.x) {
    float a = bc[o];
    for (int i = 0; i < tdim; ++i) a = fmaf(wc[static_cast<long long>(o) * tdim + i], gt[i], a);
    cond_all[static_cast<long long>(b) * sumC + o] = a;
  }
}
// the two dense layers of the same MLP with one warp per output (lanes stride the weight row: coalesced), writing temb; the
// conditioning rows then come from cond_proj_kernel across the whole grid
__global__ void __launch_bounds__(256)
time_mlp2_dense_kernel(const long long* __restrict__ t, int dim, int hid, int tdim, int act, const float* __restrict__ w1,
                       const float* __restrict__ b1, const float* __restrict__ w2, const float* __restrict__ b2,
                       float* __restrict__ temb) {
  extern __shared__ float sm[];          // emb[dim] | h[hid]
  float* emb = sm; float* h = sm + dim;
  const int b = blockIdx.x;
  const float tv = static_cast<float>(t[b]);
  const int half = dim / 2;
  const float k = logf(10000.f) / (half - 1);
  for (int i = threadIdx.x; i < half; i += blockDim.x) { const float a = tv * expf(-k * i); emb[i] = sinf(a); emb[i + half] = cosf(a); }
  if ((dim & 1) && threadIdx.x == 0) emb[dim - 1] = 0.f;
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  for (int o = warp; o < hid; o += nw) {
    const float* wr = w1 + static_cast<long long>(o) * dim;
    float a = 0.f;
    for (int i = lane; i < dim; i += 32) a = fmaf(wr[i], emb[i], a);
    a = cd_warp_sum(a) + b1[o];
    if (lane == 0) h[o] = act ? a / (1.f + expf(-a)) : cd_gelu(a);
  }
  __syncthreads();
  for (int o = warp; o < tdim; o += nw) {
    const float* wr = w2 + static_cast<long long>(o) * hid;
    float a = 0.f;
    for (int i = lane; i < hid; i += 32) a = fmaf(wr[i], h[i], a);
    a = cd_warp_sum(a) + b2[o];
    if (lane == 0) temb[b * tdim + o] = a;
  }
}

// ---- GroupNorm split-plane path (planes above CD_GN_SPLIT_MIN_HW pixels): a (chunk x image) grid of CTAs with the thread ->
// (pixel lane, channel quad) mapping of groupnorm_kernel; chunk k of image b covers pixels [k * cp, (k + 1) * cp), cp =
// cd_gn_split_chunk(C) = GN_SPLIT_ITERS pixels per active thread.  Statistics are (count, mean, M2) triples merged with Chan's
// formula in a fixed order (no E[x^2] - mean^2 cancellation for inputs with a large mean, no float atomics).
// pass 1: per-(image, chunk, group) (mean, M2) of x + cond -> part[b][k][g][2] (cd_gn_chunk_stats); the count is implied by
// the chunk geometry
__global__ void __launch_bounds__(512)
gn_split_stats_kernel(const float* __restrict__ x, int x_ld, long long HW, int C, int groups, const float* __restrict__ cond,
                      int cond_ld, int cp, float* __restrict__ part) {
  __shared__ float tm[4][512], tq[4][512];
  const int k = blockIdx.x, b = blockIdx.y, nch = gridDim.x;
  cd_gn_chunk_stats(x, x_ld, HW, C, groups, cond, cond_ld, b, k, cp, tm, tq, [&](int g, float, float mean, float m2) {
    float* o = part + ((static_cast<long long>(b) * nch + k) * groups + g) * 2;
    o[0] = mean; o[1] = m2;
  });
}

// pass 2: merge the chunks of each (image, group) in a fixed order -> stats[b][g] = (mean, rstd); one warp per group
__global__ void __launch_bounds__(256)
gn_split_combine_kernel(const float* __restrict__ part, long long HW, int cg, int groups, int cp, int nch, float eps,
                        float* __restrict__ stats) {
  const int b = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  for (int g = warp; g < groups; g += nw) {
    float n = 0.f, mean = 0.f, m2 = 0.f;
    for (int k = lane; k < nch; k += 32) {
      const float* p = part + ((static_cast<long long>(b) * nch + k) * groups + g) * 2;
      const long long pix = HW - static_cast<long long>(k) * cp < cp ? HW - static_cast<long long>(k) * cp : cp;
      cd_chan_merge(n, mean, m2, static_cast<float>(pix * cg), p[0], p[1]);
    }
    cd_chan_warp_merge(n, mean, m2);
    if (lane == 0) {
      stats[(static_cast<long long>(b) * groups + g) * 2] = mean;
      stats[(static_cast<long long>(b) * groups + g) * 2 + 1] = rsqrtf(m2 / n + eps);
    }
  }
}

// pass 3: y = (x + cond - mean) * rstd * gamma + beta [swish] over the (chunk x image) grid
__global__ void __launch_bounds__(512)
gn_split_norm_kernel(const float* __restrict__ x, int x_ld, long long HW, int C, int groups, const float* __restrict__ cond,
                     int cond_ld, const float* __restrict__ gamma, const float* __restrict__ beta, int swish, int cp,
                     const float* __restrict__ stats, float* __restrict__ y, int y_ld) {
  const int k = blockIdx.x, b = blockIdx.y;
  const int nq = C >> 2, cg = C / groups;
  const int q = threadIdx.x % nq, pl = threadIdx.x / nq, np = blockDim.x / nq;
  if (pl >= np) return;
  float4 cadd = make_float4(0.f, 0.f, 0.f, 0.f);
  if (cond) cadd = *reinterpret_cast<const float4*>(cond + static_cast<long long>(b) * cond_ld + q * 4);
  float mean[4], rstd[4];
  for (int j = 0; j < 4; ++j) {
    const float* st = stats + (static_cast<long long>(b) * groups + (q * 4 + j) / cg) * 2;
    mean[j] = st[0]; rstd[j] = st[1];
  }
  const float4 gm = *reinterpret_cast<const float4*>(gamma + q * 4);
  const float4 bt = *reinterpret_cast<const float4*>(beta + q * 4);
  const long long base = static_cast<long long>(b) * HW + static_cast<long long>(k) * cp;
  const int cnt = cd_gn_lane_count(HW, k, cp, pl, np);
#pragma unroll 4
  for (int i = 0; i < cnt; ++i) {
    const long long p = base + pl + static_cast<long long>(i) * np;
    float4 v = *reinterpret_cast<const float4*>(x + p * x_ld + q * 4);
    float o[4] = {(v.x + cadd.x - mean[0]) * rstd[0] * gm.x + bt.x, (v.y + cadd.y - mean[1]) * rstd[1] * gm.y + bt.y,
                  (v.z + cadd.z - mean[2]) * rstd[2] * gm.z + bt.z, (v.w + cadd.w - mean[3]) * rstd[3] * gm.w + bt.w};
    if (swish) for (int j = 0; j < 4; ++j) o[j] = o[j] / (1.f + __expf(-o[j]));
    *reinterpret_cast<float4*>(y + p * y_ld + q * 4) = make_float4(o[0], o[1], o[2], o[3]);
  }
}
}  // namespace

int cd_gn_split_chunk(int C) { return (512 / (C / 4)) * GN_SPLIT_ITERS; }

int cd_gn_workspace(size_t bytes, cudaStream_t st, float** ws) {
#ifdef CD_HOST_ONLY
  static std::vector<float> buf;
  if (buf.size() * sizeof(float) < bytes) buf.resize(bytes / sizeof(float) + 1);
  *ws = buf.data();
  return 0;
#else
  // one buffer per (device, stream), grown in stream order and never shrunk.  A buffer a CUDA graph has captured stays
  // allocated for the life of the process (the graph may be replayed); growing one during a capture is refused.
  struct Entry { int dev; cudaStream_t st; void* p; size_t bytes; bool captured; };
  static std::mutex mu;
  static std::vector<Entry> cache;
  int dev = 0;
  CD_CUDA(cudaGetDevice(&dev));
  cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
  CD_CUDA(cudaStreamIsCapturing(st, &cs));
  std::lock_guard<std::mutex> lock(mu);
  Entry* e = nullptr;
  for (Entry& c : cache) if (c.dev == dev && c.st == st) e = &c;
  if (!e) { cache.push_back(Entry{dev, st, nullptr, 0, false}); e = &cache.back(); }
  if (e->bytes < bytes) {
    CD_REQUIRE(cs == cudaStreamCaptureStatusNone, "cd_groupnorm: the split-plane path needs a %zu-byte workspace on this stream; "
               "run the same shape once outside CUDA-graph capture first", bytes);
    if (e->p && !e->captured) CD_CUDA(cudaFreeAsync(e->p, st));
    e->p = nullptr; e->bytes = 0; e->captured = false;
    CD_CUDA(cudaMallocAsync(&e->p, bytes, st));
    e->bytes = bytes;
  }
  if (cs != cudaStreamCaptureStatusNone) e->captured = true;
  *ws = static_cast<float*>(e->p);
  return 0;
#endif
}

int cd_gn_split_stats(const float* x, int x_ld, int B, long long HW, int C, int groups, const float* cond, int cond_ld, float eps,
                      float* part, float* stats, cudaStream_t st) {
  const int cp = cd_gn_split_chunk(C), nch = cd_cdiv(HW, cp);
  gn_split_stats_kernel<<<dim3(nch, B), 512, 0, st>>>(x, x_ld, HW, C, groups, cond, cond_ld, cp, part);
  CD_LAUNCH_CHECK();
  gn_split_combine_kernel<<<B, 256, 0, st>>>(part, HW, C / groups, groups, cp, nch, eps, stats);
  CD_LAUNCH_CHECK();
  return 0;
}

extern "C" int cd_groupnorm_fwd(const float* x, int x_ld, int B, int64_t HW, int C, int groups, const float* cond, int cond_ld,
                                const float* gamma, const float* beta, float eps, int swish, float* y, int y_ld, void* stream) {
  CD_REQUIRE(C % 4 == 0 && C % groups == 0 && C / 4 <= 512 && x_ld % 4 == 0 && y_ld % 4 == 0 && (!cond || cond_ld % 4 == 0),
             "cd_groupnorm_fwd: unsupported C=%d groups=%d", C, groups);
  if (HW > CD_GN_SPLIT_MIN_HW) {
    CD_REQUIRE(B <= 65535, "cd_groupnorm_fwd: the split-plane path takes at most 65535 images (B=%d)", B);
    const long long nch = cd_cdiv(HW, cd_gn_split_chunk(C)), nstat = 2LL * B * groups;
    float* ws = nullptr;
    if (int rc = cd_gn_workspace(sizeof(float) * (nstat + nstat * nch), static_cast<cudaStream_t>(stream), &ws)) return rc;
    if (int rc = cd_gn_split_stats(x, x_ld, B, HW, C, groups, cond, cond_ld, eps, ws + nstat, ws, static_cast<cudaStream_t>(stream))) return rc;
    gn_split_norm_kernel<<<dim3(nch, B), 512, 0, static_cast<cudaStream_t>(stream)>>>(x, x_ld, HW, C, groups, cond, cond_ld, gamma, beta,
                                                                                        swish, cd_gn_split_chunk(C), ws, y, y_ld);
    CD_LAUNCH_CHECK();
    return 0;
  }
  groupnorm_kernel<<<B, 512, sizeof(float) * 2 * groups, static_cast<cudaStream_t>(stream)>>>(x, x_ld, (int)HW, C, groups, cond, cond_ld,
                                                                                           gamma, beta, eps, swish, y, y_ld);
  CD_LAUNCH_CHECK();
  return 0;
}
extern "C" int cd_softmax_rows(float* s, int ld, int64_t rows, int n, float scale, void* stream) {
  softmax_rows_kernel<<<cd_cdiv(rows, 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(s, ld, rows, n, scale);
  CD_LAUNCH_CHECK();
  return 0;
}
extern "C" int cd_transpose_batched(const float* src, int ld, int B, int R, int C, float* dst, void* stream) {
  dim3 grid(cd_cdiv(C, 32), cd_cdiv(R, 32), B), block(32, 8);
  transpose_batched_kernel<<<grid, block, 0, static_cast<cudaStream_t>(stream)>>>(src, ld, R, C, dst);
  CD_LAUNCH_CHECK();
  return 0;
}
extern "C" int cd_upsample_nearest2x(const float* x, int x_ld, int B, int H, int W, int C, float* y, int y_ld, void* stream) {
  CD_REQUIRE(C % 4 == 0 && x_ld % 4 == 0 && y_ld % 4 == 0, "cd_upsample_nearest2x: C must be a multiple of 4");
  const long long total = static_cast<long long>(B) * 4 * H * W * (C / 4);
  int blocks = cd_cdiv(total, 256); if (blocks > cd_num_sms() * 16) blocks = cd_num_sms() * 16;
  upsample_nearest2x_kernel<<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(x, x_ld, B, H, W, C, y, y_ld);
  CD_LAUNCH_CHECK();
  return 0;
}
extern "C" int cd_nhwc_to_nchw_add(const float* x, int ld, int B, int H, int W, int C, const float* add, float* out, void* stream) {
  const long long npix = static_cast<long long>(B) * H * W;
  nhwc_to_nchw_kernel<<<cd_cdiv(npix, 128), 128, 0, static_cast<cudaStream_t>(stream)>>>(x, ld, B, H * W, C, add, out);
  CD_LAUNCH_CHECK();
  return 0;
}
extern "C" int cd_nhwc_to_nchw(const float* x, int ld, int B, int H, int W, int C, float* out, void* stream) {
  return cd_nhwc_to_nchw_add(x, ld, B, H, W, C, nullptr, out, stream);
}
extern "C" int cd_time_mlp2_fwd(const int64_t* t, int B, int dim, int hid, int tdim, int act, const float* w1, const float* b1,
                                const float* w2, const float* b2, const float* wc, const float* bc, int sumC, float* temb,
                                float* cond_all, void* stream) {
  if (temb) {        // with a temb buffer: dense layers per sample, conditioning rows over the whole grid (2 launches)
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    time_mlp2_dense_kernel<<<B, 256, sizeof(float) * (dim + hid), st>>>(reinterpret_cast<const long long*>(t), dim, hid, tdim, act, w1, b1,
                                                                     w2, b2, temb);
    CD_LAUNCH_CHECK();
    if (sumC > 0) {
      cond_proj_kernel<<<dim3(cd_cdiv(sumC, kCondRows), B), 256, sizeof(float) * tdim, st>>>(temb, tdim, wc, bc, sumC, cond_all, act);
      CD_LAUNCH_CHECK();
    }
    return 0;
  }
  const size_t smem = sizeof(float) * (dim + hid + tdim);
  time_mlp2_kernel<<<B, 256, smem, static_cast<cudaStream_t>(stream)>>>(reinterpret_cast<const long long*>(t), dim, hid, tdim, act, w1, b1,
                                                                     w2, b2, wc, bc, sumC, temb, cond_all);
  CD_LAUNCH_CHECK();
  return 0;
}
