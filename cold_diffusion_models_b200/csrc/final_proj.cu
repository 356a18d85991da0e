// Final 1x1 projection to image channels (NHWC features -> NCHW image, DB:253,279-282) through a shared-memory tile, for C = 32,
// 64 or 128.  conv1x1_to_nchw_kernel (elementwise.cu; the other C) gives every thread one pixel and lets it
// read its own 256-byte feature row with float4 loads: each warp instruction touches 32 different lines (the row-per-lane pattern
// that bounds the row epilogue of the tensor-core convolutions) and the row is read again for every output channel.  Here the
// 128 x C tile of a block is loaded with line-coalesced float4 loads (the rows of consecutive pixels are adjacent in memory when
// ld == C), each thread then takes its pixel's row from shared memory (row stride C + 1: conflict-free) into registers once and
// forms the Co dot products in the SAME order as conv1x1_to_nchw_kernel (bias first, channels ascending) -> bit-identical.
#include "cd_common.cuh"

namespace {

constexpr int kFpPix = 128;

template <int C>
__global__ void __launch_bounds__(kFpPix)
conv1x1_to_nchw_tiled_kernel(const float* __restrict__ x, int ld, long long npix, int HW, const float* __restrict__ w,
                             const float* __restrict__ bias, int Co, const float* __restrict__ resid, float* __restrict__ out) {
  extern __shared__ float tile[];                       // [kFpPix][C + 1]
  const long long p0 = static_cast<long long>(blockIdx.x) * kFpPix;
  const int np = static_cast<int>(npix - p0 < kFpPix ? npix - p0 : kFpPix);
  constexpr int Q = C / 4;                              // float4 per pixel row
  for (int i = threadIdx.x; i < kFpPix * Q; i += kFpPix) {
    const int r = i / Q, q = i - r * Q;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (r < np) v = *reinterpret_cast<const float4*>(x + (p0 + r) * ld + q * 4);
    float* t = tile + r * (C + 1) + q * 4;
    t[0] = v.x; t[1] = v.y; t[2] = v.z; t[3] = v.w;
  }
  __syncthreads();
  if (threadIdx.x >= np) return;
  float row[C];
#pragma unroll
  for (int c = 0; c < C; ++c) row[c] = tile[threadIdx.x * (C + 1) + c];
  const long long pix = p0 + threadIdx.x;
  const int b = static_cast<int>(pix / HW), p = static_cast<int>(pix % HW);
  for (int co = 0; co < Co; ++co) {
    float a = bias ? bias[co] : 0.f;
#pragma unroll
    for (int c = 0; c < C; ++c) a = fmaf(row[c], __ldg(w + co * C + c), a);
    const long long o = (static_cast<long long>(b) * Co + co) * HW + p;
    if (resid) a += resid[o];
    out[o] = a;
  }
}

}  // namespace

// 1: not taken (the caller launches conv1x1_to_nchw_kernel)
int cd_conv1x1_to_nchw_tiled(const float* x, int ld, long long npix, int HW, int C, const float* w, const float* bias, int Co,
                             const float* resid, float* out, cudaStream_t st) {
  if ((C != 64 && C != 32 && C != 128) || (reinterpret_cast<uintptr_t>(x) & 15) != 0 || ld % 4 != 0) return 1;
  const int blocks = cd_cdiv(npix, kFpPix);
  const size_t smem = sizeof(float) * kFpPix * (C + 1);
  if (C == 64) {
    conv1x1_to_nchw_tiled_kernel<64><<<blocks, kFpPix, smem, st>>>(x, ld, npix, HW, w, bias, Co, resid, out);
  } else if (C == 32) {
    conv1x1_to_nchw_tiled_kernel<32><<<blocks, kFpPix, smem, st>>>(x, ld, npix, HW, w, bias, Co, resid, out);
  } else {
    static bool attr = false;
    if (!attr) { CD_CUDA(cudaFuncSetAttribute(conv1x1_to_nchw_tiled_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); attr = true; }
    conv1x1_to_nchw_tiled_kernel<128><<<blocks, kFpPix, smem, st>>>(x, ld, npix, HW, w, bias, Co, resid, out);
  }
  CD_LAUNCH_CHECK();
  return 0;
}
