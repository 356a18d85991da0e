// Depthwise 7x7 forward / data gradient / weight gradient with the input tiles staged by TMA.
//
// Same arithmetic, tile shapes and per-thread loops as dwconv7_pipe_kernel / dwconv7_wgrad_pipe_kernel (elementwise.cu; the
// ConvNext depthwise convolution DB:145 and its backward).  Those kernels stage every (TY+6) x (TX+6) x 32-channel tile with
// 16-byte LDGSTS: 13 copies per thread and item, each with its own row / column / bounds arithmetic -- ~490 of the ~3000
// instructions a warp issues per item, in kernels that are instruction-issue bound.  Here ONE thread
// issues ONE cp.async.bulk.tensor per tile: the 4-D box {32 channels, TX+6, TY+6, 1 image} lands densely in shared memory in
// exactly the layout the LDGSTS version builds, the image border (zero padding of the convolution) is the tensor map's
// out-of-bounds zero fill, and completion is an mbarrier the whole block waits on.
#include "tc_common.cuh"

namespace {

constexpr int kTY = 16;            // output rows per tile = warps per block
constexpr int kWTX = 16;           // weight gradient: output columns per tile

__device__ __forceinline__ float* align128(uint8_t* raw) {      // bulk tensor copies need a 128-byte aligned destination
  return reinterpret_cast<float*>(raw + ((128u - (smem_u32(raw) & 127u)) & 127u));
}

template <int TX>
__global__ void __launch_bounds__(32 * kTY, 1)
dwconv7_tma_kernel(const __grid_constant__ CUtensorMap mapX, int B, int H, int W, int C,
                   const float* __restrict__ wdw, const float* __restrict__ bdw, const float* __restrict__ cond, int cond_ld,
                   float* __restrict__ out, int out_ld, int flip, const float* __restrict__ addend, int addend_ld) {
  extern __shared__ uint8_t dw_smem_raw[];
  float* xsp = align128(dw_smem_raw);                // 2 x [(TY+6)][(TX+6)][32]
  __shared__ uint64_t full[2];
  constexpr int TY = kTY, XW = TX + 6, YH = TY + 6;
  constexpr int tile_floats = YH * XW * 32;
  const int lane = threadIdx.x & 31, ry = threadIdx.x >> 5;
  const int tiles_x = W / TX, tiles_y = H / TY;
  const int ntiles = B * tiles_x * tiles_y;
  const int total = (C / 32) * ntiles;                 // slab-major: consecutive items of a block mostly share the filter slab

  if (threadIdx.x == 0) {
    mbar_init(&full[0], 1); mbar_init(&full[1], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  auto issue = [&](int item, int bi) {                 // one thread
    const int slab = item / ntiles, t = item - slab * ntiles;
    const int tx = t % tiles_x, ty = (t / tiles_x) % tiles_y, b = t / (tiles_x * tiles_y);
    fence_proxy_async();                               // the block's reads of this buffer (before the last __syncthreads) precede the bulk write
    mbar_expect_tx(&full[bi], tile_floats * 4);
    tma_load_4d(smem_u32(xsp + bi * tile_floats), &mapX, &full[bi], slab * 32, tx * TX - 3, ty * TY - 3, b);
  };

  int item = blockIdx.x;
  if (item >= total) return;
  int bufi = 0;
  uint32_t phases = 0;
  if (threadIdx.x == 0) issue(item, 0);
  float w[49];
  int cur_slab = -1;
  for (; item < total; item += gridDim.x) {
    const int nxt = item + gridDim.x;
    if (threadIdx.x == 0 && nxt < total) issue(nxt, bufi ^ 1);
    const float* buf = xsp + bufi * tile_floats;
    const int slab = item / ntiles, t = item - slab * ntiles;
    const int tx = t % tiles_x, ty = (t / tiles_x) % tiles_y, b = t / (tiles_x * tiles_y);
    const int c = slab * 32 + lane;
    if (slab != cur_slab) {
      cur_slab = slab;
#pragma unroll
      for (int k = 0; k < 49; ++k) w[k] = __ldg(wdw + static_cast<long long>(c) * 49 + (flip ? 48 - k : k));
    }
    mbar_wait(&full[bufi], (phases >> bufi) & 1u);
    phases ^= 1u << bufi;
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
    __syncthreads();                                   // buffer fully read before the next iteration's bulk copy overwrites it
    bufi ^= 1;
  }
}

// weight gradient: 49 accumulators per channel and thread, a 7x7 input window slides along the warp's row; the dY tile
// ({32, TX, TY, 1} box) rides on the same mbarrier as the input tile
__global__ void __launch_bounds__(32 * kTY, 1)
dwconv7_wgrad_tma_kernel(const __grid_constant__ CUtensorMap mapX, const __grid_constant__ CUtensorMap mapD,
                         int B, int H, int W, int C, float* __restrict__ dw) {
  extern __shared__ uint8_t dw_smem_raw[];
  float* xsw = align128(dw_smem_raw);                // 2 x ( [(TY+6)][(TX+6)][32] | [TY][TX][32] )
  constexpr int TX = kWTX, TY = kTY, XW = TX + 6, YH = TY + 6;
  constexpr int x_floats = YH * XW * 32, d_floats = TY * TX * 32, buf_floats = x_floats + d_floats;
  __shared__ float red[49][32];
  __shared__ uint64_t full[2];
  const int lane = threadIdx.x & 31, ry = threadIdx.x >> 5;
  const int tiles_x = W / TX, tiles_y = H / TY;
  const int ntiles = B * tiles_x * tiles_y;
  const int total = (C / 32) * ntiles;

  if (threadIdx.x == 0) {
    mbar_init(&full[0], 1); mbar_init(&full[1], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  auto issue = [&](int item, int bi) {                 // one thread
    const int slab = item / ntiles, t = item - slab * ntiles;
    const int tx = t % tiles_x, ty = (t / tiles_x) % tiles_y, b = t / (tiles_x * tiles_y);
    fence_proxy_async();
    mbar_expect_tx(&full[bi], buf_floats * 4);
    tma_load_4d(smem_u32(xsw + bi * buf_floats), &mapX, &full[bi], slab * 32, tx * TX - 3, ty * TY - 3, b);
    tma_load_4d(smem_u32(xsw + bi * buf_floats + x_floats), &mapD, &full[bi], slab * 32, tx * TX, ty * TY, b);
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
  uint32_t phases = 0;
  if (threadIdx.x == 0) issue(item, 0);
  float acc[49];
#pragma unroll
  for (int k = 0; k < 49; ++k) acc[k] = 0.f;
  int cur_slab = item / ntiles;
  for (; item < total; item += gridDim.x) {
    const int nxt = item + gridDim.x;
    if (threadIdx.x == 0 && nxt < total) issue(nxt, bufi ^ 1);
    const float* buf = xsw + bufi * buf_floats;
    const int slab = item / ntiles;
    if (slab != cur_slab) { flush(acc, cur_slab); cur_slab = slab; }
    mbar_wait(&full[bufi], (phases >> bufi) & 1u);
    phases ^= 1u << bufi;
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

int g_dw_tma = 1;

// plain fp32 tiles, no swizzle, zero fill outside the image
bool make_map(CUtensorMap* m, const float* p, int ld, int B, int H, int W, int C, int bx, int by) {
  const cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
  const cuuint64_t strides[3] = {(cuuint64_t)ld * 4, (cuuint64_t)ld * 4 * W, (cuuint64_t)ld * 4 * W * H};
  const cuuint32_t box[4] = {32, (cuuint32_t)bx, (cuuint32_t)by, 1};
  const cuuint32_t estr[4] = {1, 1, 1, 1};
  return encode_tiled(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, p, dims, strides, box, estr, CU_TENSOR_MAP_SWIZZLE_NONE,
                      CU_TENSOR_MAP_L2_PROMOTION_L2_128B, "dwconv7");
}

}  // namespace

extern "C" int cd_dwconv7_set_tma(int enable) { g_dw_tma = enable ? 1 : 0; return 0; }

// both return 1 when the caller should use the LDGSTS kernels of elementwise.cu (switch off, shape / alignment not eligible)
int cd_dwconv7_fwd_tma(const float* x, int x_ld, int B, int H, int W, int C, const float* w_dw, const float* b_dw,
                       const float* cond, int cond_ld, float* out, int out_ld, int flip, const float* addend, int addend_ld,
                       cudaStream_t st) {
  if (!g_dw_tma || C % 32 != 0 || H % kTY != 0 || W % 16 != 0 || x_ld % 4 != 0 || (reinterpret_cast<uintptr_t>(x) & 15) != 0) return 1;
  const int TX = W % 32 == 0 ? 32 : 16;
  CUtensorMap mapX;
  if (!make_map(&mapX, x, x_ld, B, H, W, C, TX + 6, kTY + 6)) return 1;
  const size_t smem = sizeof(float) * 2 * 32 * size_t(kTY + 6) * (TX + 6) + 128;
  CD_CUDA(TX == 32 ? smem_limit_once<dwconv7_tma_kernel<32>>(smem) : smem_limit_once<dwconv7_tma_kernel<16>>(smem));
  const long long total = static_cast<long long>(C / 32) * B * (H / kTY) * (W / TX);
  const int grid = total < cd_num_sms() ? static_cast<int>(total) : cd_num_sms();
  auto kern = TX == 32 ? dwconv7_tma_kernel<32> : dwconv7_tma_kernel<16>;
  kern<<<grid, 32 * kTY, smem, st>>>(mapX, B, H, W, C, w_dw, b_dw, cond, cond_ld, out, out_ld, flip, addend, addend_ld);
  CD_LAUNCH_CHECK();
  return 0;
}

int cd_dwconv7_wgrad_tma(const float* dh, int dh_ld, const float* x, int x_ld, int B, int H, int W, int C, float* dw, cudaStream_t st) {
  if (!g_dw_tma || C % 32 != 0 || H % kTY != 0 || W % kWTX != 0 || x_ld % 4 != 0 || dh_ld % 4 != 0 ||
      (reinterpret_cast<uintptr_t>(x) & 15) != 0 || (reinterpret_cast<uintptr_t>(dh) & 15) != 0) return 1;
  CUtensorMap mapX, mapD;
  if (!make_map(&mapX, x, x_ld, B, H, W, C, kWTX + 6, kTY + 6) || !make_map(&mapD, dh, dh_ld, B, H, W, C, kWTX, kTY)) return 1;
  const size_t smem = sizeof(float) * 2 * 32 * (size_t(kTY + 6) * (kWTX + 6) + size_t(kTY) * kWTX) + 128;
  CD_CUDA(smem_limit_once<dwconv7_wgrad_tma_kernel>(smem));
  const long long total = static_cast<long long>(C / 32) * B * (H / kTY) * (W / kWTX);
  const int grid = total < cd_num_sms() ? static_cast<int>(total) : cd_num_sms();
  dwconv7_wgrad_tma_kernel<<<grid, 32 * kTY, smem, st>>>(mapX, mapD, B, H, W, C, dw);
  CD_LAUNCH_CHECK();
  return 0;
}
