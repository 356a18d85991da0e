// LinearAttention context (DB:176-187: k.softmax(dim=-1); context = einsum('bhdn,bhen->bhde', k, v)), DETERMINISTIC and in one
// pass over k and v.
//
//   ctx[b][h][d][e] = sum_n exp(k[b][n][h*32+d] - kmax[b][h*32+d]) * v[b][n][h*32+e],   ksum[b][c] = sum_n exp(k[b][n][c] - kmax[b][c])
//
// A max pass, a CUDA-core outer-product pass and float atomics over the pixel blocks would read k twice and give a result whose
// last bit depends on the order of the atomics -- which the TF32 roundings downstream amplify into run-to-run differences of the
// network output.
//
// Here a block walks a contiguous span of pixels of one image with the flash-attention recurrence: running per-channel max m,
// accumulators rescaled by exp(m_old - m_new) when m grows.  The 32x32 (per head) products E^T V run on the tensor cores with
// warp-level mma.sync.m16n8k8 TF32 in the 3xTF32 split (hi*hi + lo*hi + hi*lo: fp32-grade products, fp32 accumulation) -- the
// whole GEMM is 4 GFLOP per 128x128 micro-batch, so the legacy path is plenty and the kernel stays HBM-bound.  k and v tiles are
// double-buffered through shared memory with 16-byte LDGSTS.  Every block writes ONE partial (m, s, ctx) to a workspace; a second
// kernel merges the partials of an image in block order (fixed summation order => bit-identical results run to run).
#include "cd_common.cuh"

namespace {

constexpr int kP = 32;              // pixels per staged chunk
constexpr int kLd = 136;            // padded row of a staged tile in floats: (pixel*8 + channel) % 32 is conflict-free for the fragments
constexpr int kPart = 4096 + 256;   // floats of one partial: ctx[4][32][32] | m[128] | s[128]

// D(16x8) += A(16x8, row) * B(8x8, col); fragments as in the PTX ISA (groupID g = lane / 4, t = lane % 4):
// a0 = A[g][t], a1 = A[g+8][t], a2 = A[g][t+4], a3 = A[g+8][t+4]; b0 = B[t][g], b1 = B[t+4][g]; d0,d1 = D[g][2t,2t+1], d2,d3 = D[g+8][2t,2t+1]
__device__ __forceinline__ void cd_mma_m16n8k8_tf32(float* d, const float* a, const float* b) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(__float_as_uint(a[0])), "r"(__float_as_uint(a[1])), "r"(__float_as_uint(a[2])), "r"(__float_as_uint(a[3])),
                 "r"(__float_as_uint(b[0])), "r"(__float_as_uint(b[1])));
}

__device__ __forceinline__ void split_tf32(float x, float& hi, float& lo) {
  hi = cd_round_tf32(x);
  lo = cd_round_tf32(x - hi);
}

__global__ void __launch_bounds__(256)
ctx_partial_kernel(const float* __restrict__ qkv, int ld, int n, int ppb, float* __restrict__ ws) {
  extern __shared__ __align__(16) float sm[];          // [2 stages][k tile | v tile][kP][kLd]
  const int b = blockIdx.y, blk = blockIdx.x, nblk = gridDim.x;
  const int p0 = blk * ppb;
  int p1 = p0 + ppb; if (p1 > n) p1 = n;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const int h = warp >> 1, dbase = h * 32 + (warp & 1) * 16;       // this warp: context rows d = dbase + g, dbase + g + 8 of head h
  const float* base = qkv + static_cast<long long>(b) * n * ld + 128;  // k at +0..127, v at +128..255 of every pixel row

  auto issue = [&](int q0, int s) {
    float* kd = sm + s * 2 * kP * kLd;
    float* vd = kd + kP * kLd;
    for (int i = tid; i < kP * 64; i += 256) {
      const int pix = i >> 6, seg = i & 63;
      const int p = q0 + pix;
      const bool ok = p < p1;
      const float* src = base + static_cast<long long>(ok ? p : p0) * ld + seg * 4;
      float* dst = seg < 32 ? kd + pix * kLd + seg * 4 : vd + pix * kLd + (seg - 32) * 4;
      cd_cp_async16(dst, src, ok);
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };

  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  float m0 = -INFINITY, m1 = -INFINITY, s0 = 0.f, s1 = 0.f;        // running max and exp-sum of rows g / g + 8 (this lane's pixels only)

  int stage = 0;
  issue(p0, 0);
  for (int q0 = p0; q0 < p1; q0 += kP) {
    if (q0 + kP < p1) {
      issue(q0 + kP, stage ^ 1);
      asm volatile("cp.async.wait_group 1;" ::: "memory");
    } else {
      asm volatile("cp.async.wait_group 0;" ::: "memory");
    }
    __syncthreads();
    const float* kd = sm + stage * 2 * kP * kLd;
    const float* vd = kd + kP * kLd;
#pragma unroll
    for (int ks = 0; ks < kP / 8; ++ks) {
      const float* kt = kd + (ks * 8) * kLd + dbase + g;
      const int pa = q0 + ks * 8 + t, pb = pa + 4;
      float k00 = kt[t * kLd], k10 = kt[t * kLd + 8], k01 = kt[(t + 4) * kLd], k11 = kt[(t + 4) * kLd + 8];
      if (pa >= p1) { k00 = -INFINITY; k10 = -INFINITY; }
      if (pb >= p1) { k01 = -INFINITY; k11 = -INFINITY; }
      // max of the step's 8 pixels per row: the four lanes of a quad hold them
      float mg = fmaxf(k00, k01), mh = fmaxf(k10, k11);
      mg = fmaxf(mg, __shfl_xor_sync(0xffffffffu, mg, 1)); mg = fmaxf(mg, __shfl_xor_sync(0xffffffffu, mg, 2));
      mh = fmaxf(mh, __shfl_xor_sync(0xffffffffu, mh, 1)); mh = fmaxf(mh, __shfl_xor_sync(0xffffffffu, mh, 2));
      const float n0 = fmaxf(m0, mg), n1 = fmaxf(m1, mh);
      if (__any_sync(0xffffffffu, n0 > m0 || n1 > m1)) {
        const float f0 = (n0 == m0) ? 1.f : __expf(m0 - n0), f1 = (n1 == m1) ? 1.f : __expf(m1 - n1);
        s0 *= f0; s1 *= f1;
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) { acc[nt][0] *= f0; acc[nt][1] *= f0; acc[nt][2] *= f1; acc[nt][3] *= f1; }
        m0 = n0; m1 = n1;
      }
      float a[4], ahi[4], alo[4];
      a[0] = (k00 == -INFINITY) ? 0.f : __expf(k00 - m0);
      a[1] = (k10 == -INFINITY) ? 0.f : __expf(k10 - m1);
      a[2] = (k01 == -INFINITY) ? 0.f : __expf(k01 - m0);
      a[3] = (k11 == -INFINITY) ? 0.f : __expf(k11 - m1);
      s0 += a[0] + a[2]; s1 += a[1] + a[3];
#pragma unroll
      for (int i = 0; i < 4; ++i) split_tf32(a[i], ahi[i], alo[i]);
      const float* vt = vd + (ks * 8) * kLd + h * 32 + g;
#pragma unroll
      for (int nt = 0; nt < 4; ++nt) {
        float bhi[2], blo[2];
        split_tf32(vt[t * kLd + nt * 8], bhi[0], blo[0]);
        split_tf32(vt[(t + 4) * kLd + nt * 8], bhi[1], blo[1]);
        cd_mma_m16n8k8_tf32(acc[nt], alo, bhi);
        cd_mma_m16n8k8_tf32(acc[nt], ahi, blo);
        cd_mma_m16n8k8_tf32(acc[nt], ahi, bhi);
      }
    }
    __syncthreads();                                   // tile fully read before the next prefetch overwrites it
    stage ^= 1;
  }
  // exp-sums of a row: add the quad's four lanes (fixed order)
  s0 += __shfl_xor_sync(0xffffffffu, s0, 1); s0 += __shfl_xor_sync(0xffffffffu, s0, 2);
  s1 += __shfl_xor_sync(0xffffffffu, s1, 1); s1 += __shfl_xor_sync(0xffffffffu, s1, 2);
  float* part = ws + (static_cast<long long>(b) * nblk + blk) * kPart;
  const int d0 = (warp & 1) * 16 + g;
#pragma unroll
  for (int nt = 0; nt < 4; ++nt) {
    *reinterpret_cast<float2*>(part + (h * 32 + d0) * 32 + nt * 8 + 2 * t) = make_float2(acc[nt][0], acc[nt][1]);
    *reinterpret_cast<float2*>(part + (h * 32 + d0 + 8) * 32 + nt * 8 + 2 * t) = make_float2(acc[nt][2], acc[nt][3]);
  }
  if (t == 0) {
    part[4096 + dbase + g] = m0; part[4096 + dbase + g + 8] = m1;
    part[4224 + dbase + g] = s0; part[4224 + dbase + g + 8] = s1;
  }
}

// merge the partials of (image b, head h) in block order: kmax = max_blk m, ksum = sum_blk exp(m - kmax) s, ctx likewise
__global__ void __launch_bounds__(256)
ctx_merge_kernel(const float* __restrict__ ws, int nblk, float* __restrict__ kmax, float* __restrict__ ksum, float* __restrict__ ctx) {
  extern __shared__ float f[];                         // [nblk][32] rescaling factors of this head's rows
  const int h = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
  const float* part = ws + static_cast<long long>(b) * nblk * kPart;
  if (tid < 32) {
    const int c = h * 32 + tid;
    float M = -INFINITY;
    for (int i = 0; i < nblk; ++i) M = fmaxf(M, part[static_cast<long long>(i) * kPart + 4096 + c]);
    float S = 0.f;
    for (int i = 0; i < nblk; ++i) {
      const float fi = __expf(part[static_cast<long long>(i) * kPart + 4096 + c] - M);
      f[i * 32 + tid] = fi;
      S += fi * part[static_cast<long long>(i) * kPart + 4224 + c];
    }
    kmax[b * 128 + c] = M;
    ksum[b * 128 + c] = S;
  }
  __syncthreads();
  float* out = ctx + (static_cast<long long>(b) * 4 + h) * 1024;
  for (int i = tid; i < 1024; i += 256) {
    const int d = i >> 5;
    float a = 0.f;
    for (int j = 0; j < nblk; ++j) a += f[j * 32 + d] * part[static_cast<long long>(j) * kPart + h * 1024 + i];
    out[i] = a;
  }
}

}  // namespace

// The caller cuts the pixel axis of one image into nblk = ceil(n / ppb) spans of ppb pixels (a multiple of 32) and owns the
// workspace ws[B][nblk][4352]; about one wave of resident blocks (3 per SM: 69.6 KB of shared memory each) is the sweet spot.
extern "C" int cd_linattn_context_det(const float* qkv, int ld, int B, int n, int nblk, int ppb, float* ws, float* kmax,
                                      float* ksum, float* ctx, void* stream) {
  CD_REQUIRE(ld % 4 == 0 && (reinterpret_cast<uintptr_t>(qkv) & 15) == 0, "cd_linattn_context_det: qkv rows must be 16-byte aligned (ld=%d)", ld);
  CD_REQUIRE(ppb > 0 && ppb % kP == 0 && nblk == cd_cdiv(n, ppb) && nblk <= 1024, "cd_linattn_context_det: plan (nblk=%d, ppb=%d) does not cover n=%d", nblk, ppb, n);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const size_t smem = sizeof(float) * 2 * 2 * kP * kLd;
  static bool attr = false;
  if (!attr) { CD_CUDA(cudaFuncSetAttribute(ctx_partial_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); attr = true; }
  ctx_partial_kernel<<<dim3(nblk, B), 256, smem, st>>>(qkv, ld, n, ppb, ws);
  CD_LAUNCH_CHECK();
  // the merge keeps 32 weights per span: above 384 spans (one 512^2 image at the finest level) that passes the 48 KB a launch
  // gets without opting in
  const size_t msmem = sizeof(float) * nblk * 32;
  static size_t mattr = 48 * 1024;
  if (msmem > mattr) { CD_CUDA(cudaFuncSetAttribute(ctx_merge_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)msmem)); mattr = msmem; }
  ctx_merge_kernel<<<dim3(4, B), 256, msmem, st>>>(ws, nblk, kmax, ksum, ctx);
  CD_LAUNCH_CHECK();
  return 0;
}
