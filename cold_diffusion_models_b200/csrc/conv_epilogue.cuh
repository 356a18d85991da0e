// Line-coalesced epilogue of the tensor-core convolutions (opt-in, cd_conv_tc_set_staged_epilogue).
//
// The default epilogue of conv_tc_kernel stores straight from the wgmma accumulator fragment: a lane holds pairs of adjacent
// channels of two pixels, so every store instruction of a warp touches 8 different pixel rows with 32 bytes each.  The short-K
// convolutions (1x1 projections, K = 64..512) do little MMA work per output byte, and there the number of memory requests,
// not the bytes, can bound the launch.
//
// With this epilogue the accumulator chunk of a warpgroup is first staged so that a lane holds 32 consecutive output channels
// of ITS OWN pixel (conv_tc.cu), and then the 32 x 32 block of a warp goes through a per-warp shared-memory tile (row stride 36 floats: the float4 row
// writes and the float4 transposed reads are both conflict-free per quarter-warp) and leaves as 8 store instructions that
// each cover 4 pixels x 128 contiguous bytes (4 full lines instead of 32 sectors in 32 lines); the residual / GELU'
// operand reads are coalesced the same way.  The arithmetic per element and its order are those of the row epilogue
// (acc + bias + resid -> out2 -> activation -> TF32 rounding -> out): results are bit-identical.
//
// No wgmma / TMA in this header: tests/simt_cpu executes it from source on the CPU (tests/test_conv_epilogue_cpu.py).
#pragma once
#include "cd_common.cuh"

constexpr int kEpiStageStride = 36;                           // floats per staged pixel row (16-byte aligned, 4 banks of skew)
constexpr int kEpiStageFloats = 32 * kEpiStageStride;         // per warp

// P needs: out, out_ld, bias, resid, resid_ld, act, round_tf32, out2, out2_ld, aux, aux_ld (the CdConvDesc epilogue fields).
// r: accumulator columns [col0, col0 + 32) of this lane's pixel; pix: this lane's output pixel index; valid: the pixel exists.
// All 32 lanes must call it (warp shuffles); col0 + 32 <= Cout; every pointer 16-byte aligned, every ld a multiple of 4.
template <class P>
__device__ __forceinline__ void cd_epilogue_staged32(const uint32_t (&r)[32], float* __restrict__ st, int lane, long long pix,
                                                     bool valid, int col0, const P& p) {
#pragma unroll
  for (int j = 0; j < 32; j += 4)
    *reinterpret_cast<float4*>(st + lane * kEpiStageStride + j) =
        make_float4(__uint_as_float(r[j]), __uint_as_float(r[j + 1]), __uint_as_float(r[j + 2]), __uint_as_float(r[j + 3]));
  __syncwarp();
  const int sub = lane >> 3, j4 = (lane & 7) * 4;
  const int col = col0 + j4;
  float4 bb = make_float4(0.f, 0.f, 0.f, 0.f);
  if (p.bias) bb = __ldg(reinterpret_cast<const float4*>(p.bias + col));
#pragma unroll
  for (int it = 0; it < 8; ++it) {
    const int pr = it * 4 + sub;                              // pixel (row of the staged tile) this lane helps to write
    const long long ppix = __shfl_sync(0xffffffffu, pix, pr);
    const int pvalid = __shfl_sync(0xffffffffu, valid ? 1 : 0, pr);
    if (pvalid) {
      float4 v = *reinterpret_cast<const float4*>(st + pr * kEpiStageStride + j4);
      if (p.bias) { v.x += bb.x; v.y += bb.y; v.z += bb.z; v.w += bb.w; }
      if (p.resid) {
        const float4 rr = *reinterpret_cast<const float4*>(p.resid + ppix * p.resid_ld + col);
        v.x += rr.x; v.y += rr.y; v.z += rr.z; v.w += rr.w;
      }
      if (p.out2) *reinterpret_cast<float4*>(p.out2 + ppix * p.out2_ld + col) = v;
      if (p.act == CD_ACT_GELU) { v.x = cd_gelu(v.x); v.y = cd_gelu(v.y); v.z = cd_gelu(v.z); v.w = cd_gelu(v.w); }
      else if (p.act == CD_ACT_GELU_BWD) {
        const float4 a = *reinterpret_cast<const float4*>(p.aux + ppix * p.aux_ld + col);
        v.x *= cd_gelu_grad(a.x); v.y *= cd_gelu_grad(a.y); v.z *= cd_gelu_grad(a.z); v.w *= cd_gelu_grad(a.w);
      }
      if (p.round_tf32) { v.x = cd_round_tf32(v.x); v.y = cd_round_tf32(v.y); v.z = cd_round_tf32(v.z); v.w = cd_round_tf32(v.w); }
      *reinterpret_cast<float4*>(p.out + ppix * p.out_ld + col) = v;
    }
  }
  __syncwarp();                                               // the tile is reused by the next column chunk
}
