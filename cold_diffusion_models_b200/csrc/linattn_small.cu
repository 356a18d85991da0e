// LinearAttention, the two per-(batch element, head) kernels with their operands STAGED through shared memory.
// cd_linattn_weff and cd_linattn_bwd_small (elementwise.cu / backward.cu) run 4 x B blocks whose threads walk the `dim`
// output channels with dependent strided global loads: a few MFLOP per call, bound by load latency.  The kernels below read
// every operand once, 64 channel rows per pass with all loads of a pass in flight (one float4 per thread and array), and keep
// the arithmetic ORDER of the originals (sums over co / d / e ascending, one fmaf per term), so their results are bit-identical
// up to the order of the float atomics that were already there.  The originals serve a w_out (weff) or dweff (backward) that is
// not 16-byte aligned.
#include "cd_common.cuh"

namespace {

constexpr int kRows = 64;            // channel rows (co) staged per pass

// weff[b][co][h*32+d] = sum_e w_out[co][h*32+e] * ctxn[d][e],  ctxn[d][e] = ctx[b][h][d][e] * scale / ksum[b][h*32+d]
__global__ void __launch_bounds__(256)
weff_staged_kernel(const float* __restrict__ ctx, const float* __restrict__ ksum, const float* __restrict__ w_out,
                   int dim, float scale, int round_tf32, float* __restrict__ weff) {
  __shared__ float cn[32][33];
  __shared__ __align__(16) float wos[kRows][32];      // w_out[co0 + r][h*32 + e]
  const int h = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
  const float* cb = ctx + (static_cast<long long>(b) * 4 + h) * 1024;
  for (int i = tid; i < 1024; i += 256) {
    const int d = i >> 5, e = i & 31;
    cn[d][e] = cb[i] * scale / ksum[b * 128 + h * 32 + d];
  }
  const int lane = tid & 31, warp = tid >> 5;
  for (int co0 = 0; co0 < dim; co0 += kRows) {
    const int nco = dim - co0 < kRows ? dim - co0 : kRows;
    __syncthreads();                                   // cn ready / previous pass done with wos
    for (int i = tid; i < kRows * 8; i += 256) {
      const int r = i >> 3, q = i & 7;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (r < nco) v = *reinterpret_cast<const float4*>(w_out + static_cast<long long>(co0 + r) * 128 + h * 32 + q * 4);
      *reinterpret_cast<float4*>(&wos[r][q * 4]) = v;
    }
    __syncthreads();
    // warp w owns rows w, w + 8, ...; lane = d.  wos reads are broadcasts, cn[d][e] is conflict-free (row stride 33)
    for (int r = warp; r < nco; r += 8) {
      float a = 0.f;
#pragma unroll 8
      for (int e = 0; e < 32; ++e) a = fmaf(wos[r][e], cn[lane][e], a);
      weff[(static_cast<long long>(b) * dim + co0 + r) * 128 + h * 32 + lane] = round_tf32 ? cd_round_tf32(a) : a;
    }
  }
}

// the small backward part (backward.cu: attn_bwd_small_kernel has the formulas)
__global__ void __launch_bounds__(256)
attn_bwd_small_staged_kernel(const float* __restrict__ dweff, const float* __restrict__ ctx, const float* __restrict__ ksum,
                             const float* __restrict__ w_out, int dim, float scale, float* __restrict__ dw_out,
                             float* __restrict__ dctxn, float* __restrict__ rowdot) {
  __shared__ float cn[32][33];                         // ctxn[d][e]
  __shared__ float dcs[32][33];                        // dctxn[d][e]
  __shared__ __align__(16) float dws[kRows][32];       // dweff[b][co0 + r][h*32 + d]
  __shared__ __align__(16) float wos[kRows][32];       // w_out[co0 + r][h*32 + e]
  const int h = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
  const float* dwe = dweff + static_cast<long long>(b) * dim * 128 + h * 32;
  const float* wo = w_out + h * 32;
  const float* cb = ctx + (static_cast<long long>(b) * 4 + h) * 1024;
  for (int i = tid; i < 1024; i += 256) {
    const int d = i >> 5, e = i & 31;
    cn[d][e] = cb[i] / ksum[b * 128 + h * 32 + d];
  }
  const int d = tid >> 3, e4 = (tid & 7) * 4;          // dctxn: thread -> (d, e quad)
  const int lane = tid & 31, warp = tid >> 5;          // dW_out: warp -> co row, lane -> e
  float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
  for (int co0 = 0; co0 < dim; co0 += kRows) {
    const int nco = dim - co0 < kRows ? dim - co0 : kRows;
    __syncthreads();                                   // cn ready / previous pass done with dws, wos
    for (int i = tid; i < kRows * 8; i += 256) {
      const int r = i >> 3, q = i & 7;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f), w = v;
      if (r < nco) {
        v = *reinterpret_cast<const float4*>(dwe + static_cast<long long>(co0 + r) * 128 + q * 4);
        w = *reinterpret_cast<const float4*>(wo + static_cast<long long>(co0 + r) * 128 + q * 4);
      }
      *reinterpret_cast<float4*>(&dws[r][q * 4]) = v;
      *reinterpret_cast<float4*>(&wos[r][q * 4]) = w;
    }
    __syncthreads();
    // dctxn[d][e] += sum_co dweff[co][d] * w_out[co][e]   (rows past nco are zero-filled: they add +0 like no term at all
    // would, except that -0 + +0 = +0; the sums start from +0, so nothing changes)
    for (int r = 0; r < nco; ++r) {
      const float dv = dws[r][d];
      const float4 wv = *reinterpret_cast<const float4*>(&wos[r][e4]);
      a0 = fmaf(dv, wv.x, a0); a1 = fmaf(dv, wv.y, a1); a2 = fmaf(dv, wv.z, a2); a3 = fmaf(dv, wv.w, a3);
    }
    // dW_out[co][h*32+e] += scale * sum_d dweff[co][d] * ctxn[d][e]
    for (int r = warp; r < nco; r += 8) {
      float a = 0.f;
#pragma unroll 8
      for (int dd = 0; dd < 32; ++dd) a = fmaf(dws[r][dd], cn[dd][lane], a);
      atomicAdd(dw_out + static_cast<long long>(co0 + r) * 128 + h * 32 + lane, a * scale);
    }
  }
  dcs[d][e4] = a0 * scale; dcs[d][e4 + 1] = a1 * scale; dcs[d][e4 + 2] = a2 * scale; dcs[d][e4 + 3] = a3 * scale;
  __syncthreads();
  float* dout = dctxn + (static_cast<long long>(b) * 4 + h) * 1024;
  for (int i = tid; i < 1024; i += 256) dout[i] = dcs[i >> 5][i & 31];
  if (tid < 32) {
    float a = 0.f;
    for (int e = 0; e < 32; ++e) a = fmaf(dcs[tid][e], cn[tid][e], a);
    rowdot[b * 128 + h * 32 + tid] = a;
  }
}

}  // namespace

// the staged kernels read rows with float4 loads: callers fall back to the original kernels for unaligned operands
int cd_linattn_aligned(const void* a, const void* b) {
  return ((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b)) & 15) == 0;
}

int cd_linattn_weff_staged(const float* ctx, const float* ksum, const float* w_out, int B, int dim, float scale,
                           int round_tf32, float* weff, cudaStream_t st) {
  weff_staged_kernel<<<dim3(4, B), 256, 0, st>>>(ctx, ksum, w_out, dim, scale, round_tf32, weff);
  CD_LAUNCH_CHECK();
  return 0;
}

int cd_linattn_bwd_small_staged(const float* dweff, const float* ctx, const float* ksum, const float* w_out, int B, int dim,
                                float scale, float* dw_out, float* dctxn, float* rowdot, cudaStream_t st) {
  attn_bwd_small_staged_kernel<<<dim3(4, B), 256, 0, st>>>(dweff, ctx, ksum, w_out, dim, scale, dw_out, dctxn, rowdot);
  CD_LAUNCH_CHECK();
  return 0;
}
