// Degradation operators D(x,t) for the Gaussian-blur family and the Algorithm-2 update, the loss
// and the fused Adam+EMA step (all HBM / on-chip bound fp32).
//
// Reference: every blur step is nn.Conv2d(C,C,k,groups=C,padding_mode=circular|reflect) with a
// separable Gaussian (DB:348-389); q_sample applies steps 0..t_b sequentially on the whole batch and
// stacks all of them (DB:927-953); x0_step_down sampling recomputes D(xhat,t) and D(xhat,t-1) from
// scratch every step (DB:436-451).  Because each step is linear, separable and boundary-closed, the
// cumulative degradation of one S x S plane is  A_t X A_t^T  with a precomputed S x S operator A_t
// (host side: cold_diffusion_models_b200/degradation.py builds A_t in float64 from the fp32 taps).
// One CTA owns one (b,c) plane: X, A_t and the intermediate live in shared memory, so HBM traffic is
// the algorithmic minimum (read plane + operator, write plane) and D(x,t) costs two S^3 fp32 matmuls
// regardless of t -- instead of t sequential 2-D stencils.
#include "cd_common.cuh"

namespace {

// C(S x S) = A(S x S, row-major, ld = S) * Bm(S x S, row stride ldb), each thread 4x4 micro-tiles.
// Result micro-tile (i..i+3, j..j+3) is handed to `sink(i, j, acc)`.
template <typename Sink>
__device__ __forceinline__ void matmul_tiles(const float* __restrict__ A, const float* __restrict__ Bm, int ldb,
                                             int S, Sink sink) {
  const int tj_n = S >> 2;
  const int ntiles = tj_n * tj_n;
  for (int tile = threadIdx.x; tile < ntiles; tile += blockDim.x) {
    const int i0 = (tile / tj_n) * 4, j0 = (tile % tj_n) * 4;
    float acc[4][4] = {};
#pragma unroll 4
    for (int k = 0; k < S; ++k) {
      const float4 bv = *reinterpret_cast<const float4*>(Bm + k * ldb + j0);
      const float a0 = A[(i0 + 0) * S + k], a1 = A[(i0 + 1) * S + k], a2 = A[(i0 + 2) * S + k], a3 = A[(i0 + 3) * S + k];
      acc[0][0] = fmaf(a0, bv.x, acc[0][0]); acc[0][1] = fmaf(a0, bv.y, acc[0][1]); acc[0][2] = fmaf(a0, bv.z, acc[0][2]); acc[0][3] = fmaf(a0, bv.w, acc[0][3]);
      acc[1][0] = fmaf(a1, bv.x, acc[1][0]); acc[1][1] = fmaf(a1, bv.y, acc[1][1]); acc[1][2] = fmaf(a1, bv.z, acc[1][2]); acc[1][3] = fmaf(a1, bv.w, acc[1][3]);
      acc[2][0] = fmaf(a2, bv.x, acc[2][0]); acc[2][1] = fmaf(a2, bv.y, acc[2][1]); acc[2][2] = fmaf(a2, bv.z, acc[2][2]); acc[2][3] = fmaf(a2, bv.w, acc[2][3]);
      acc[3][0] = fmaf(a3, bv.x, acc[3][0]); acc[3][1] = fmaf(a3, bv.y, acc[3][1]); acc[3][2] = fmaf(a3, bv.z, acc[3][2]); acc[3][3] = fmaf(a3, bv.w, acc[3][3]);
    }
    sink(i0, j0, acc);
  }
}

__device__ __forceinline__ void load_plane(float* dst, int ldd, const float* __restrict__ src, int S) {
  const int nv = (S * S) >> 2;
  const int per_row = S >> 2;
  for (int i = threadIdx.x; i < nv; i += blockDim.x) {
    const int r = i / per_row, c = (i % per_row) * 4;
    *reinterpret_cast<float4*>(dst + r * ldd + c) = __ldg(reinterpret_cast<const float4*>(src) + i);
  }
}

// dst[c][r] = src[r][c] (ld S both): thread i reads a float4 of row i % S, so a warp stores 32 consecutive floats of a dst row
__device__ __forceinline__ void load_plane_transposed(float* dst, const float* __restrict__ src, int S) {
  const int nv = (S * S) >> 2;
  for (int i = threadIdx.x; i < nv; i += blockDim.x) {
    const int r = i % S, c = (i / S) * 4;
    const float4 v = __ldg(reinterpret_cast<const float4*>(src + r * S + c));
    dst[(c + 0) * S + r] = v.x; dst[(c + 1) * S + r] = v.y; dst[(c + 2) * S + r] = v.z; dst[(c + 3) * S + r] = v.w;
  }
}

__device__ __forceinline__ float block_sum(float v, float* scratch) {
  v = cd_warp_sum(v);
  const int w = threadIdx.x >> 5, nw = blockDim.x >> 5;
  __syncthreads();
  if ((threadIdx.x & 31) == 0) scratch[w] = v;
  __syncthreads();
  float t = 0.f;
  for (int i = 0; i < nw; ++i) t += scratch[i];
  return t;
}

// Z = A X A^T for one plane, result left in Zs (row stride ldp) as Z (not transposed).
//   step 1: Yt[j][i] = (A X)[i][j]            (written transposed, padded stride)
//   step 2: Z^T[j][i] = sum_k A[j][k] Yt[k][i] -> Zs[i][j]
__device__ __forceinline__ void plane_apply(const float* As, const float* Xs, float* Yt, float* Zs, int S, int ldp) {
  matmul_tiles(As, Xs, ldp, S, [&](int i0, int j0, float (&acc)[4][4]) {
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
      for (int b = 0; b < 4; ++b) Yt[(j0 + b) * ldp + i0 + a] = acc[a][b];
  });
  __syncthreads();
  matmul_tiles(As, Yt, ldp, S, [&](int j0, int i0, float (&acc)[4][4]) {
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
      for (int b = 0; b < 4; ++b) Zs[(i0 + b) * ldp + j0 + a] = acc[a][b];
  });
  __syncthreads();
}

// smem layout: As[S*S] | Xs[S*ldp] | Yt[S*ldp] | scratch[32]   (Zs aliases Xs after step 1... no: Xs is
// read only in step 1, Zs written in step 2 -> Zs = Xs)
// kAdj: the adjoint A^T G A of the same operator (the gradient of A X A^T): A_idx is loaded transposed into As, and the
// collapse at T-1 comes first -- the adjoint of X -> mean(A X A^T) 11^T is G -> A^T (mean(G) 11^T) A.
// kEpi (guided restoration; collapse_last and quantize are then 0): kEpiNone = the plain product; kEpiAxpy = A X A^T - w g
// (the guided `default` update, and with w = 1, g = y the residual of the two-pass guidance gradient); kEpiGuide = the guidance
// gradient A^T (A X A^T - g) A in one pass: the residual stays in shared memory and A is reloaded transposed over the used As.
constexpr int kEpiNone = 0, kEpiAxpy = 1, kEpiGuide = 2;
template <bool kAdj, int kEpi = kEpiNone>
__global__ void __launch_bounds__(256)
blur_apply_kernel(const float* __restrict__ x, float* __restrict__ out, const float* __restrict__ ops,
                  const long long* __restrict__ t, int t_scalar, int S, int T, int collapse_last, int quantize,
                  const float* __restrict__ g, float w) {
  extern __shared__ __align__(16) float sm[];
  const int ldp = S + 4;
  float* As = sm; float* Xs = As + S * S; float* Yt = Xs + S * ldp; float* scratch = Yt + S * ldp;
  const int plane = blockIdx.x;            // b * C + c
  const int b = blockIdx.y;                // grid = (C, B): plane index = b * C + blockIdx.x
  const long long pl = static_cast<long long>(b) * gridDim.x + plane;
  const float* xp = x + pl * S * S;
  float* op = out + pl * S * S;
  const int idx = t ? static_cast<int>(t[b]) : t_scalar;
  load_plane(Xs, ldp, xp, S);
  if (idx >= 0) {
    if (kAdj) load_plane_transposed(As, ops + static_cast<long long>(idx) * S * S, S);
    else load_plane(As, S, ops + static_cast<long long>(idx) * S * S, S);
  }
  __syncthreads();
  float mean = 0.f;
  const bool collapse = collapse_last && idx == T - 1;
  if (kAdj && collapse) {
    float s = 0.f;
    for (int i = threadIdx.x; i < S * S; i += blockDim.x) s += Xs[(i / S) * ldp + (i % S)];
    mean = block_sum(s, scratch) / (S * S);
    for (int i = threadIdx.x; i < S * S; i += blockDim.x) Xs[(i / S) * ldp + (i % S)] = mean;
    __syncthreads();
  }
  if (idx >= 0) plane_apply(As, Xs, Yt, Xs, S, ldp);
  if (!kAdj && collapse) {
    float s = 0.f;
    for (int i = threadIdx.x; i < S * S; i += blockDim.x) s += Xs[(i / S) * ldp + (i % S)];
    mean = block_sum(s, scratch) / (S * S);
  }
  const int per_row = S >> 2;
  if constexpr (kEpi == kEpiGuide) {
    // each thread rewrites the float4 slots it stores below; plane_apply ended with a barrier, so As is free
    for (int i = threadIdx.x; i < (S * S) >> 2; i += blockDim.x) {
      const int r = i / per_row, c = (i % per_row) * 4;
      float4* z = reinterpret_cast<float4*>(Xs + r * ldp + c);
      const float4 yv = __ldg(reinterpret_cast<const float4*>(g + pl * S * S) + i);
      *z = make_float4(z->x - yv.x, z->y - yv.y, z->z - yv.z, z->w - yv.w);
    }
    if (idx >= 0) load_plane_transposed(As, ops + static_cast<long long>(idx) * S * S, S);
    __syncthreads();
    if (idx >= 0) plane_apply(As, Xs, Yt, Xs, S, ldp);
  }
  for (int i = threadIdx.x; i < (S * S) >> 2; i += blockDim.x) {
    const int r = i / per_row, c = (i % per_row) * 4;
    float4 v = *reinterpret_cast<const float4*>(Xs + r * ldp + c);
    if constexpr (kEpi == kEpiAxpy) {
      const float4 gv = __ldg(reinterpret_cast<const float4*>(g + pl * S * S) + i);
      v = make_float4(v.x - w * gv.x, v.y - w * gv.y, v.z - w * gv.z, v.w - w * gv.w);
    }
    if (!kAdj && collapse) v = make_float4(mean, mean, mean, mean);
    if (quantize) {
      float* f = reinterpret_cast<float*>(&v);
#pragma unroll
      for (int k = 0; k < 4; ++k) {          // DB:954-958, same op order, truncation toward zero
        float q = (f[k] + 1.f) * 0.5f;
        q = q * 255.f;
        q = static_cast<float>(static_cast<int>(q)) / 255.f;
        f[k] = q * 2.f - 1.f;
      }
    }
    reinterpret_cast<float4*>(op)[i] = v;
  }
}

// out = xt - A_hi xhat A_hi^T + A_lo xhat A_lo^T   (index -1 = identity).
// smem: As | Xs | Yt (Z overwrites Xs; xhat is re-read from L2 for the second term) = 196 KB at S = 128.
// kAxpy: the guided update, out - w g in the epilogue.
template <bool kAxpy = false>
__global__ void __launch_bounds__(256)
blur_step_down_kernel(const float* __restrict__ xt, const float* __restrict__ xhat, float* __restrict__ out,
                      const float* __restrict__ ops, int t_hi, int t_lo, int S, int T, int collapse_last,
                      const float* __restrict__ g, float w) {
  extern __shared__ __align__(16) float sm[];
  const int ldp = S + 4;
  float* As = sm; float* Xs = As + S * S; float* Yt = Xs + S * ldp; float* scratch = Yt + S * ldp;
  const long long pl = static_cast<long long>(blockIdx.y) * gridDim.x + blockIdx.x;
  const float* xh = xhat + pl * S * S;
  const int per_row = S >> 2;
  // ---- high index term: Xs <- A_hi xhat A_hi^T ----
  load_plane(Xs, ldp, xh, S);
  if (t_hi >= 0) load_plane(As, S, ops + static_cast<long long>(t_hi) * S * S, S);
  __syncthreads();
  if (t_hi >= 0) plane_apply(As, Xs, Yt, Xs, S, ldp);
  float mean_hi = 0.f;
  const bool collapse = collapse_last && t_hi == T - 1;
  if (collapse) {
    float s = 0.f;
    for (int i = threadIdx.x; i < S * S; i += blockDim.x) s += Xs[(i / S) * ldp + (i % S)];
    mean_hi = block_sum(s, scratch) / (S * S);
  }
  // d = xt - Zhi   (kept in registers: each thread owns fixed float4 slots; S <= 128 -> <= 16 slots)
  float4 d[16];
  int nslot = 0;
  for (int i = threadIdx.x; i < (S * S) >> 2; i += blockDim.x, ++nslot) {
    const int r = i / per_row, c = (i % per_row) * 4;
    const float4 a = __ldg(reinterpret_cast<const float4*>(xt + pl * S * S) + i);
    float4 z = *reinterpret_cast<const float4*>(Xs + r * ldp + c);
    if (collapse) z = make_float4(mean_hi, mean_hi, mean_hi, mean_hi);
    d[nslot] = make_float4(a.x - z.x, a.y - z.y, a.z - z.z, a.w - z.w);
  }
  __syncthreads();
  // ---- low index term: Xs <- A_lo xhat A_lo^T ----
  load_plane(Xs, ldp, xh, S);
  if (t_lo >= 0) load_plane(As, S, ops + static_cast<long long>(t_lo) * S * S, S);
  __syncthreads();
  if (t_lo >= 0) plane_apply(As, Xs, Yt, Xs, S, ldp);
  nslot = 0;
  for (int i = threadIdx.x; i < (S * S) >> 2; i += blockDim.x, ++nslot) {
    const int r = i / per_row, c = (i % per_row) * 4;
    const float4 z = *reinterpret_cast<const float4*>(Xs + r * ldp + c);
    float4 o = d[nslot];
    o.x += z.x; o.y += z.y; o.z += z.z; o.w += z.w;
    if constexpr (kAxpy) {
      const float4 gv = __ldg(reinterpret_cast<const float4*>(g + pl * S * S) + i);
      o = make_float4(o.x - w * gv.x, o.y - w * gv.y, o.z - w * gv.z, o.w - w * gv.w);
    }
    reinterpret_cast<float4*>(out + pl * S * S)[i] = o;
  }
}

// ---- 128 < S <= 512: one CTA per (plane, strip of kStripR rows) ----------------------------------------------------------
// A plane, its operator and the intermediate no longer fit in shared memory, but a row strip of Z = A X A^T needs only the
// same rows of A:  Z[r0:r0+R, :] = (A[r0:r0+R, :] X) A^T.
//   phase 1: Y = A[r0:r0+R, :] X  (R x S), kept in shared memory transposed (Yt[k][r]);
//   phase 2: Z_strip[r][j] = sum_k Y[r][k] A[j][k].
// X (phase 1) and A^T (phase 2) stream through a double-buffered ring of kStripK-row chunks (cp.async; the A^T chunk is
// transposed by 4-byte copies), so the intermediate never reaches HBM and X / A_t are re-read from L2 once per strip; the
// strips of one plane are adjacent in the grid.  Warp w owns the strip rows 4w..4w+3, lane l the columns 4l + 128q
// (q < NQ = ceil(S / 128)): 16 NQ fp32 FFMA accumulators per thread.  When S is not a multiple of 128 the ring columns
// S .. 128 NQ - 1 are never written: they feed only the accumulators of columns j >= S, which are never stored (neither to Yt
// nor to the output), so whatever they hold does not reach a result.  The caller must not alias out with x / xhat: the
// other strips of a plane still read it.
constexpr int kStripR = 32, kStripK = 16, kStripThreads = 256, kStripLdy = kStripR + 4;

template <int NQ> __host__ __device__ constexpr int strip_ldb() { return 128 * NQ + 4; }
__host__ __device__ __forceinline__ int strip_cdiv(int a, int b) { return (a + b - 1) / b; }

// floats of shared memory: ring 2 x [kStripK][ldb] | A-strip ring 2 x [kStripK][kStripR] | Yt [S rounded up to kStripK][kStripLdy]
// | scratch 32  (the plane-mean path keeps its column sums w[S] where Yt goes)
template <int NQ> size_t strip_smem(int S) {
  return sizeof(float) * (2 * kStripK * strip_ldb<NQ>() + 2 * kStripK * kStripR + size_t(strip_cdiv(S, kStripK)) * kStripK * kStripLdy + 32);
}

__device__ __forceinline__ void fma4x4(float (&acc)[4][4], float4 a, float4 b) {
  const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
}

// f(q, a, offset of Z[r][j] in the plane) for every in-plane float4 this thread owns: r = r0 + 4w + a, j = 4 lane + 128 q
template <int NQ, typename F>
__device__ __forceinline__ void strip_for_each(int S, int r0, F f) {
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int q = 0; q < NQ; ++q)
#pragma unroll
    for (int a = 0; a < 4; ++a) {
      const int r = r0 + 4 * w + a, j = 4 * lane + 128 * q;
      if (r < S && j < S) f(q, a, static_cast<long long>(r) * S + j);
    }
}

// acc <- this thread's part of the strip of A X A^T (rows and columns outside the plane hold garbage).
// kAdj: the strip of A^T X A.  Only the operator loads differ: both chunks of A^T are row segments of A, copied 16 bytes at a time.
template <int NQ, bool kAdj>
__device__ __forceinline__ void strip_product(const float* __restrict__ A, const float* __restrict__ X, int S, int r0, float* sm,
                                              float (&acc)[NQ][4][4]) {
  constexpr int ldb = strip_ldb<NQ>();
  float* ring = sm;
  float* aring = ring + 2 * kStripK * ldb;
  float* Yt = aring + 2 * kStripK * kStripR;
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nk = strip_cdiv(S, kStripK), per_row = S >> 2;
  auto zero = [&] {
#pragma unroll
    for (int q = 0; q < NQ; ++q)
#pragma unroll
      for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b) acc[q][a][b] = 0.f;
  };
  // chunk c: `issue` fills ring buffer c & 1 and commits, then every chunk is waited for, consumed by `compute` and released
  auto run = [&](auto issue, auto compute) {
    issue(0);
    for (int c = 0; c < nk; ++c) {
      if (c + 1 < nk) {
        issue(c + 1);
        asm volatile("cp.async.wait_group 1;" ::: "memory");
      } else {
        asm volatile("cp.async.wait_group 0;" ::: "memory");
      }
      __syncthreads();
      compute(c);
      __syncthreads();
    }
  };
  // phase 1, chunk c: ring[kk][j] = X[k0 + kk][j], aring[kk][r] = A[r0 + r][k0 + kk]  (zero outside the plane)
  auto issue1 = [&](int c) {
    const int k0 = c * kStripK;
    float* rb = ring + (c & 1) * kStripK * ldb;
    for (int i = threadIdx.x; i < kStripK * per_row; i += kStripThreads) {
      const int kk = i / per_row, j = (i - kk * per_row) * 4;
      const bool v = k0 + kk < S;
      cd_cp_async16(rb + kk * ldb + j, X + (v ? static_cast<long long>(k0 + kk) * S + j : 0), v);
    }
    float* ab = aring + (c & 1) * kStripK * kStripR;
    if (kAdj) {                                                 // aring[kk][r] = A^T[r0 + r][k0 + kk] = A[k0 + kk][r0 + r]
      for (int i = threadIdx.x; i < kStripK * (kStripR / 4); i += kStripThreads) {
        const int kk = i / (kStripR / 4), r = (i - kk * (kStripR / 4)) * 4;
        const bool v = r0 + r < S && k0 + kk < S;              // S % 4 == 0: a float4 is wholly inside or outside
        cd_cp_async16(ab + kk * kStripR + r, A + (v ? static_cast<long long>(k0 + kk) * S + r0 + r : 0), v);
      }
    } else {
      for (int i = threadIdx.x; i < kStripK * kStripR; i += kStripThreads) {
        const int r = i / kStripK, kk = i - r * kStripK;          // kk fastest: a warp reads two 64-byte row segments of A
        const bool v = r0 + r < S && k0 + kk < S;
        cd_cp_async4(ab + kk * kStripR + r, A + (v ? static_cast<long long>(r0 + r) * S + k0 + kk : 0), v);
      }
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };
  auto compute1 = [&](int c) {
    const float* rb = ring + (c & 1) * kStripK * ldb + 4 * lane;
    const float* ab = aring + (c & 1) * kStripK * kStripR + 4 * w;
#pragma unroll 4
    for (int kk = 0; kk < kStripK; ++kk) {
      const float4 a = *reinterpret_cast<const float4*>(ab + kk * kStripR);
#pragma unroll
      for (int q = 0; q < NQ; ++q) fma4x4(acc[q], a, *reinterpret_cast<const float4*>(rb + kk * ldb + 128 * q));
    }
  };
  // phase 2, chunk c: ring[kk][j] = A[j][k0 + kk]  (kAdj: (A^T)^T = A, ring[kk][j] = A[k0 + kk][j], the layout of the X chunks)
  auto issue2 = [&](int c) {
    const int k0 = c * kStripK;
    float* rb = ring + (c & 1) * kStripK * ldb;
    if (kAdj) {
      for (int i = threadIdx.x; i < kStripK * per_row; i += kStripThreads) {
        const int kk = i / per_row, j = (i - kk * per_row) * 4;
        const bool v = k0 + kk < S;
        cd_cp_async16(rb + kk * ldb + j, A + (v ? static_cast<long long>(k0 + kk) * S + j : 0), v);
      }
    } else {
      for (int i = threadIdx.x; i < kStripK * S; i += kStripThreads) {
        const int j = i / kStripK, kk = i - j * kStripK;
        const bool v = k0 + kk < S;
        cd_cp_async4(rb + kk * ldb + j, A + (v ? static_cast<long long>(j) * S + k0 + kk : 0), v);
      }
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };
  auto compute2 = [&](int c) {
    const float* rb = ring + (c & 1) * kStripK * ldb + 4 * lane;
    const float* yb = Yt + c * kStripK * kStripLdy + 4 * w;
#pragma unroll 4
    for (int kk = 0; kk < kStripK; ++kk) {
      const float4 y = *reinterpret_cast<const float4*>(yb + kk * kStripLdy);
#pragma unroll
      for (int q = 0; q < NQ; ++q) fma4x4(acc[q], y, *reinterpret_cast<const float4*>(rb + kk * ldb + 128 * q));
    }
  };
  zero();
  run(issue1, compute1);
  // Yt[j][r] = Y[r][j]; the rows past S (the last chunk's tail) are zero, as is the A^T chunk there
#pragma unroll
  for (int q = 0; q < NQ; ++q)
#pragma unroll
    for (int b = 0; b < 4; ++b) {
      const int j = 4 * lane + 128 * q + b;
      if (j < S) *reinterpret_cast<float4*>(Yt + j * kStripLdy + 4 * w) = make_float4(acc[q][0][b], acc[q][1][b], acc[q][2][b], acc[q][3][b]);
    }
  for (int i = S * kStripLdy + threadIdx.x; i < nk * kStripK * kStripLdy; i += kStripThreads) Yt[i] = 0.f;
  zero();
  run(issue2, compute2);                  // its first barrier orders the Yt writes before any read
}

// w = A^T 1 (column sums of A)
__device__ __forceinline__ void column_sums(const float* __restrict__ A, int S, float* w) {
  for (int k = threadIdx.x; k < S; k += blockDim.x) {
    float s = 0.f;
    for (int j = 0; j < S; ++j) s += __ldg(A + static_cast<long long>(j) * S + k);
    w[k] = s;
  }
  __syncthreads();
}

// mean(A X A^T) = w^T X w / S^2 with w = A^T 1: the `discrete` collapse without the strip product
__device__ __forceinline__ float plane_mean_closed_form(const float* __restrict__ A, const float* __restrict__ X, int S,
                                                        float* w, float* scratch) {
  column_sums(A, S, w);
  float s = 0.f;
  for (int i = threadIdx.x; i < S * S; i += blockDim.x) s = fmaf(w[i / S] * __ldg(X + i), w[i % S], s);
  return block_sum(s, scratch) / (static_cast<float>(S) * S);
}

// acc <- this thread's part of the strip of D = A_idx X A_idx^T  (idx < 0: X itself; collapse at idx == T-1: the plane mean).
// kAdj: of the adjoint A^T X A; its collapse is A^T (mean(X) 11^T) A = mean(X) w w^T.
template <int NQ, bool kAdj>
__device__ __forceinline__ void strip_degrade(const float* __restrict__ ops, const float* __restrict__ X, int idx, int S, int T,
                                              int collapse_last, int r0, float* sm, float (&acc)[NQ][4][4]) {
  if (idx < 0) {
    strip_for_each<NQ>(S, r0, [&](int q, int a, long long o) {
      const float4 v = __ldg(reinterpret_cast<const float4*>(X + o));
      acc[q][a][0] = v.x; acc[q][a][1] = v.y; acc[q][a][2] = v.z; acc[q][a][3] = v.w;
    });
    return;
  }
  const float* A = ops + static_cast<long long>(idx) * S * S;
  if (collapse_last && idx == T - 1) {
    float* w = sm + 2 * kStripK * strip_ldb<NQ>() + 2 * kStripK * kStripR;
    float* scratch = w + strip_cdiv(S, kStripK) * kStripK * kStripLdy;
    if (kAdj) {
      column_sums(A, S, w);
      float s = 0.f;
      for (int i = threadIdx.x; i < S * S; i += blockDim.x) s += __ldg(X + i);
      const float mean = block_sum(s, scratch) / (static_cast<float>(S) * S);
      const int wi = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
      for (int q = 0; q < NQ; ++q)
#pragma unroll
        for (int a = 0; a < 4; ++a)
#pragma unroll
          for (int b = 0; b < 4; ++b) {              // w has S entries: rows and columns outside the plane get 0
            const int r = r0 + 4 * wi + a, j = 4 * lane + 128 * q + b;
            acc[q][a][b] = r < S && j < S ? mean * w[r] * w[j] : 0.f;
          }
      return;
    }
    const float mean = plane_mean_closed_form(A, X, S, w, scratch);
#pragma unroll
    for (int q = 0; q < NQ; ++q)
#pragma unroll
      for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b) acc[q][a][b] = mean;
    return;
  }
  strip_product<NQ, kAdj>(A, X, S, r0, sm, acc);
}

// kAdj: the adjoint A^T G A of the same operator (cd_blur_apply_adjoint; quantize is then 0).  kAxpy: out = D x - w g (the
// guided `default` update, and the residual D x - y of the two-pass guidance gradient; quantize is then 0).
template <int NQ, bool kAdj, bool kAxpy = false>
__global__ void __launch_bounds__(kStripThreads, 1)
blur_apply_strip_kernel(const float* __restrict__ x, float* __restrict__ out, const float* __restrict__ ops,
                        const long long* __restrict__ t, int t_scalar, int C, int S, int T, int collapse_last, int quantize,
                        const float* __restrict__ g, float w) {
  extern __shared__ __align__(16) float sm[];
  const int nstrip = strip_cdiv(S, kStripR);
  const int pl = blockIdx.x / nstrip;                     // b * C + c; the strips of one plane are adjacent
  const int r0 = (blockIdx.x - pl * nstrip) * kStripR;
  const float* xp = x + static_cast<long long>(pl) * S * S;
  float* op = out + static_cast<long long>(pl) * S * S;
  const int idx = t ? static_cast<int>(t[pl / C]) : t_scalar;
  float acc[NQ][4][4];
  strip_degrade<NQ, kAdj>(ops, xp, idx, S, T, collapse_last, r0, sm, acc);
  strip_for_each<NQ>(S, r0, [&](int q, int a, long long o) {
    float f[4] = {acc[q][a][0], acc[q][a][1], acc[q][a][2], acc[q][a][3]};
    if (quantize) {
#pragma unroll
      for (int k = 0; k < 4; ++k) {          // DB:954-958, same op order as blur_apply_kernel
        float qv = (f[k] + 1.f) * 0.5f;
        qv = qv * 255.f;
        qv = static_cast<float>(static_cast<int>(qv)) / 255.f;
        f[k] = qv * 2.f - 1.f;
      }
    }
    if constexpr (kAxpy) {
      const float4 gv = __ldg(reinterpret_cast<const float4*>(g + static_cast<long long>(pl) * S * S + o));
      f[0] = f[0] - w * gv.x; f[1] = f[1] - w * gv.y; f[2] = f[2] - w * gv.z; f[3] = f[3] - w * gv.w;
    }
    *reinterpret_cast<float4*>(op + o) = make_float4(f[0], f[1], f[2], f[3]);
  });
}

// out = xt - Z_hi + Z_lo: xt - Z_hi is parked in `out` and read back by the thread that wrote it.  kAxpy: minus w g as well.
template <int NQ, bool kAxpy = false>
__global__ void __launch_bounds__(kStripThreads, 1)
blur_step_down_strip_kernel(const float* __restrict__ xt, const float* __restrict__ xhat, float* out, const float* __restrict__ ops,
                            int t_hi, int t_lo, int S, int T, int collapse_last, const float* __restrict__ g, float w) {
  extern __shared__ __align__(16) float sm[];
  const int nstrip = strip_cdiv(S, kStripR);
  const int pl = blockIdx.x / nstrip;
  const int r0 = (blockIdx.x - pl * nstrip) * kStripR;
  const float* xh = xhat + static_cast<long long>(pl) * S * S;
  const float* xp = xt + static_cast<long long>(pl) * S * S;
  float* op = out + static_cast<long long>(pl) * S * S;
  float acc[NQ][4][4];
  strip_degrade<NQ, false>(ops, xh, t_hi, S, T, collapse_last, r0, sm, acc);
  strip_for_each<NQ>(S, r0, [&](int q, int a, long long o) {
    const float4 v = __ldg(reinterpret_cast<const float4*>(xp + o));
    *reinterpret_cast<float4*>(op + o) = make_float4(v.x - acc[q][a][0], v.y - acc[q][a][1], v.z - acc[q][a][2], v.w - acc[q][a][3]);
  });
  __syncthreads();
  strip_degrade<NQ, false>(ops, xh, t_lo, S, T, 0, r0, sm, acc);
  strip_for_each<NQ>(S, r0, [&](int q, int a, long long o) {
    float4 d = *reinterpret_cast<const float4*>(op + o);
    d.x += acc[q][a][0]; d.y += acc[q][a][1]; d.z += acc[q][a][2]; d.w += acc[q][a][3];
    if constexpr (kAxpy) {
      const float4 gv = __ldg(reinterpret_cast<const float4*>(g + static_cast<long long>(pl) * S * S + o));
      d = make_float4(d.x - w * gv.x, d.y - w * gv.y, d.z - w * gv.z, d.w - w * gv.w);
    }
    *reinterpret_cast<float4*>(op + o) = d;
  });
}

// ---- loss -----------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
loss_kernel(const float* __restrict__ x0, const float* __restrict__ xhat, long long n, int mode, float inv_n,
            float grad_scale, float* __restrict__ loss, float* __restrict__ dxhat) {
  __shared__ float scratch[8];
  float s = 0.f;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float d = xhat[i] - x0[i];
    if (mode == 0) { s += fabsf(d); if (dxhat) dxhat[i] = (d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f)) * inv_n * grad_scale; }
    else { s += d * d; if (dxhat) dxhat[i] = 2.f * d * inv_n * grad_scale; }
  }
  s = block_sum(s, scratch);
  if (threadIdx.x == 0) atomicAdd(loss, s * inv_n);
}

// ---- Adam (+EMA) ------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
adam_ema_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                float* __restrict__ ema, long long n, float lr, float b1, float b2, float eps, float bc1, float bc2_sqrt,
                int ema_mode, float ema_beta, float grad_scale) {
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float gi = g[i] * grad_scale;
    const float mi = b1 * m[i] + (1.f - b1) * gi;          // torch: exp_avg.lerp_(grad, 1-beta1)
    const float vi = b2 * v[i] + (1.f - b2) * gi * gi;
    m[i] = mi; v[i] = vi;
    const float denom = sqrtf(vi) / bc2_sqrt + eps;
    const float pi = p[i] - (lr / bc1) * (mi / denom);
    p[i] = pi;
    if (ema_mode == 1) ema[i] = pi;
    else if (ema_mode == 2) ema[i] = ema[i] * ema_beta + (1.f - ema_beta) * pi;
  }
}

__global__ void ema_kernel(float* __restrict__ ema, const float* __restrict__ p, long long n, float beta, int mode) {
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    ema[i] = mode == 1 ? p[i] : ema[i] * beta + (1.f - beta) * p[i];
}

}  // namespace

extern "C" int cd_ema_update(float* ema, const float* p, int64_t n, float beta, int mode, void* stream) {
  int blocks = cd_cdiv(n, 256 * 4); if (blocks > cd_num_sms() * 16) blocks = cd_num_sms() * 16; if (blocks < 1) blocks = 1;
  ema_kernel<<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(ema, p, n, beta, mode);
  CD_LAUNCH_CHECK();
  return 0;
}

static size_t blur_smem(int S, int planes) { return sizeof(float) * (size_t(S) * S + size_t(planes) * S * (S + 4) + 32); }

// grid of the strip kernels: one CTA per (plane, strip), strips of a plane adjacent
static int strip_grid(int B, int C, int S, unsigned* grid) {
  const long long n = static_cast<long long>(B) * C * cd_cdiv(S, kStripR);
  CD_REQUIRE(n >= 1 && n < (1ll << 31), "blur strip kernels: %lld CTAs out of range", n);
  *grid = static_cast<unsigned>(n);
  return 0;
}

template <int NQ, bool kAdj, bool kAxpy = false>
static int blur_apply_strips(const float* x, float* out, const float* ops, const int64_t* t, int t_scalar, int B, int C, int S,
                             int T, int collapse_last, int quantize, cudaStream_t stream, const float* g = nullptr, float w = 0.f) {
  unsigned grid = 0;
  if (strip_grid(B, C, S, &grid)) return -1;
  const size_t smem = strip_smem<NQ>(S);
  static size_t attr = 0;
  if (smem > attr) { CD_CUDA(cudaFuncSetAttribute(blur_apply_strip_kernel<NQ, kAdj, kAxpy>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); attr = smem; }
  blur_apply_strip_kernel<NQ, kAdj, kAxpy><<<grid, kStripThreads, smem, stream>>>(x, out, ops, reinterpret_cast<const long long*>(t),
                                                                                 t_scalar, C, S, T, collapse_last, quantize, g, w);
  CD_LAUNCH_CHECK();
  return 0;
}

template <int NQ, bool kAxpy = false>
static int blur_step_down_strips(const float* xt, const float* xhat, float* out, const float* ops, int t_hi, int t_lo, int B, int C,
                                 int S, int T, int collapse_last, cudaStream_t stream, const float* g = nullptr, float w = 0.f) {
  unsigned grid = 0;
  if (strip_grid(B, C, S, &grid)) return -1;
  const size_t smem = strip_smem<NQ>(S);
  static size_t attr = 0;
  if (smem > attr) { CD_CUDA(cudaFuncSetAttribute(blur_step_down_strip_kernel<NQ, kAxpy>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); attr = smem; }
  blur_step_down_strip_kernel<NQ, kAxpy><<<grid, kStripThreads, smem, stream>>>(xt, xhat, out, ops, t_hi, t_lo, S, T, collapse_last, g, w);
  CD_LAUNCH_CHECK();
  return 0;
}

// S <= 128: one CTA per plane (blur_apply_kernel / blur_step_down_kernel); 128 < S <= 512: one CTA per row strip.
// kEpi: see blur_apply_kernel; kEpiGuide is one-CTA only (cd_blur_guide_grad runs two passes above 128).
template <bool kAdj, int kEpi = kEpiNone>
static int blur_apply(const char* name, const float* x, float* out, const float* ops, const int64_t* t, int t_scalar, int B, int C,
                      int S, int T, int collapse_last, int quantize, cudaStream_t stream, const float* g = nullptr, float w = 0.f) {
  CD_REQUIRE(S % 4 == 0 && S >= 4 && S <= 512, "%s: image size %d unsupported (need S%%4==0, 4<=S<=512)", name, S);
  if (S > 128) {
    if constexpr (kEpi == kEpiGuide) {
      CD_FAIL("%s: the one-pass guidance gradient needs S <= 128", name);
    } else {
      constexpr bool kAxpy = kEpi == kEpiAxpy;
      if (S <= 256) return blur_apply_strips<2, kAdj, kAxpy>(x, out, ops, t, t_scalar, B, C, S, T, collapse_last, quantize, stream, g, w);
      if (S <= 384) return blur_apply_strips<3, kAdj, kAxpy>(x, out, ops, t, t_scalar, B, C, S, T, collapse_last, quantize, stream, g, w);
      return blur_apply_strips<4, kAdj, kAxpy>(x, out, ops, t, t_scalar, B, C, S, T, collapse_last, quantize, stream, g, w);
    }
  }
  const size_t smem = blur_smem(S, 2);
  static size_t attr = 0;
  if (smem > attr) { CD_CUDA(cudaFuncSetAttribute(blur_apply_kernel<kAdj, kEpi>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); attr = smem; }
  dim3 grid(C, B);
  blur_apply_kernel<kAdj, kEpi><<<grid, 256, smem, stream>>>(x, out, ops, reinterpret_cast<const long long*>(t), t_scalar, S, T,
                                                             collapse_last, quantize, g, w);
  CD_LAUNCH_CHECK();
  return 0;
}

extern "C" int cd_blur_apply(const float* x, float* out, const float* ops, const int64_t* t, int t_scalar,
                             int B, int C, int S, int T, int collapse_last, int quantize, void* stream) {
  return blur_apply<false>("cd_blur_apply", x, out, ops, t, t_scalar, B, C, S, T, collapse_last, quantize,
                           static_cast<cudaStream_t>(stream));
}

// the gradient of cd_blur_apply (without its quantize): out = A^T g A per plane, collapse adjoint first at T-1
extern "C" int cd_blur_apply_adjoint(const float* g, float* out, const float* ops, const int64_t* t, int t_scalar,
                                     int B, int C, int S, int T, int collapse_last, void* stream) {
  return blur_apply<true>("cd_blur_apply_adjoint", g, out, ops, t, t_scalar, B, C, S, T, collapse_last, 0,
                          static_cast<cudaStream_t>(stream));
}

template <bool kAxpy>
static int blur_step_down(const char* name, const float* xt, const float* xhat, float* out, const float* ops, int t_hi, int t_lo,
                          int B, int C, int S, int T, int collapse_last, cudaStream_t st, const float* g, float w) {
  CD_REQUIRE(S % 4 == 0 && S >= 4 && S <= 512, "%s: image size %d unsupported (need S%%4==0, 4<=S<=512)", name, S);
  if (S > 128) {
    if (S <= 256) return blur_step_down_strips<2, kAxpy>(xt, xhat, out, ops, t_hi, t_lo, B, C, S, T, collapse_last, st, g, w);
    if (S <= 384) return blur_step_down_strips<3, kAxpy>(xt, xhat, out, ops, t_hi, t_lo, B, C, S, T, collapse_last, st, g, w);
    return blur_step_down_strips<4, kAxpy>(xt, xhat, out, ops, t_hi, t_lo, B, C, S, T, collapse_last, st, g, w);
  }
  const size_t smem = blur_smem(S, 2);
  static size_t attr = 0;
  if (smem > attr) { CD_CUDA(cudaFuncSetAttribute(blur_step_down_kernel<kAxpy>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); attr = smem; }
  dim3 grid(C, B);
  blur_step_down_kernel<kAxpy><<<grid, 256, smem, st>>>(xt, xhat, out, ops, t_hi, t_lo, S, T, collapse_last, g, w);
  CD_LAUNCH_CHECK();
  return 0;
}

extern "C" int cd_blur_step_down(const float* xt, const float* xhat, float* out, const float* ops,
                                 int t_hi, int t_lo, int B, int C, int S, int T, int collapse_last, void* stream) {
  return blur_step_down<false>("cd_blur_step_down", xt, xhat, out, ops, t_hi, t_lo, B, C, S, T, collapse_last,
                               static_cast<cudaStream_t>(stream), nullptr, 0.f);
}

// ---- guided restoration (GaussianDiffusion.restore) ----------------------------------------------------------------------
// the guidance gradient D^T (D x0 - y) of D = A_idx (.) A_idx^T: one pass up to 128² (the residual never leaves shared memory),
// two above (the apply kernel with a "- y" epilogue into `work`, then the adjoint kernel)
extern "C" int cd_blur_guide_grad(const float* x0, const float* y, float* out, float* work, const float* ops, int idx,
                                  int B, int C, int S, int T, void* stream) {
  CD_REQUIRE(x0 && y && out && ops && idx < T && B >= 1 && C >= 1, "cd_blur_guide_grad: bad arguments");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (S <= 128)
    return blur_apply<false, kEpiGuide>("cd_blur_guide_grad", x0, out, ops, nullptr, idx, B, C, S, T, 0, 0, st, y, 1.f);
  CD_REQUIRE(work && work != out, "cd_blur_guide_grad: S = %d > 128 needs a workspace of B*C*S*S floats apart from out", S);
  if (blur_apply<false, kEpiAxpy>("cd_blur_guide_grad", x0, work, ops, nullptr, idx, B, C, S, T, 0, 0, st, y, 1.f)) return -1;
  return blur_apply<true>("cd_blur_guide_grad", work, out, ops, nullptr, idx, B, C, S, T, 0, 0, st);
}

// the guided update: xt == NULL -> `default`, out = D(xhat, t_lo) - w g; else `x0_step_down`, out = xt - D(xhat, t_hi) +
// D(xhat, t_lo) - w g.  g == NULL runs the unguided kernels themselves (their bits).
extern "C" int cd_blur_guided_step(const float* xt, const float* xhat, const float* g, float weight, float* out, const float* ops,
                                   int t_hi, int t_lo, int B, int C, int S, int T, void* stream) {
  CD_REQUIRE(xhat && out && ops && t_hi < T && t_lo < T, "cd_blur_guided_step: bad arguments");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (!xt) {
    if (!g) return blur_apply<false>("cd_blur_guided_step", xhat, out, ops, nullptr, t_lo, B, C, S, T, 0, 0, st);
    return blur_apply<false, kEpiAxpy>("cd_blur_guided_step", xhat, out, ops, nullptr, t_lo, B, C, S, T, 0, 0, st, g, weight);
  }
  if (!g) return blur_step_down<false>("cd_blur_guided_step", xt, xhat, out, ops, t_hi, t_lo, B, C, S, T, 0, st, nullptr, 0.f);
  return blur_step_down<true>("cd_blur_guided_step", xt, xhat, out, ops, t_hi, t_lo, B, C, S, T, 0, st, g, weight);
}

extern "C" int cd_loss_fwd_bwd(const float* x0, const float* xhat, int64_t n, int mode, float grad_scale,
                               float* loss, float* dxhat, void* stream) {
  CD_REQUIRE(mode == 0 || mode == 1, "cd_loss_fwd_bwd: mode must be 0 (l1) or 1 (l2)");
  int blocks = cd_cdiv(n, 256 * 4); if (blocks > cd_num_sms() * 8) blocks = cd_num_sms() * 8; if (blocks < 1) blocks = 1;
  loss_kernel<<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(x0, xhat, n, mode, 1.0f / static_cast<float>(n), grad_scale, loss, dxhat);
  CD_LAUNCH_CHECK();
  return 0;
}

extern "C" int cd_adam_ema_step(float* p, const float* g, float* m, float* v, float* ema, int64_t n,
                                float lr, float beta1, float beta2, float eps, int step,
                                int ema_mode, float ema_beta, float grad_scale, void* stream) {
  CD_REQUIRE(step >= 1, "cd_adam_ema_step: step counts from 1");
  // bias corrections in double on the host like torch.optim.Adam (1 - beta2^step loses ~5e-5 relative in fp32 at small steps)
  const float bc1 = static_cast<float>(1.0 - pow(static_cast<double>(beta1), static_cast<double>(step)));
  const float bc2s = static_cast<float>(sqrt(1.0 - pow(static_cast<double>(beta2), static_cast<double>(step))));
  int blocks = cd_cdiv(n, 256 * 4); if (blocks > cd_num_sms() * 16) blocks = cd_num_sms() * 16; if (blocks < 1) blocks = 1;
  adam_ema_kernel<<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(p, g, m, v, ema, n, lr, beta1, beta2, eps, bc1, bc2s,
                                                                       ema_mode, ema_beta, grad_scale);
  CD_LAUNCH_CHECK();
  return 0;
}

// -------------------------------------------------------------------------------------------------------------
// Gaussian-noise ("hot") baseline of denoising-diffusion-pytorch (DN = denoising-diffusion-pytorch/
// denoising_diffusion_pytorch/denoising_diffusion_pytorch.py): q_sample = per-sample lerp with the cosine-schedule
// coefficients (DN:517-522) and the ddim / x0_step_down reverse step (DN:383-434), one elementwise kernel each,
// same operation order as the reference.
// -------------------------------------------------------------------------------------------------------------
namespace {
__global__ void noise_lerp_kernel(const float* __restrict__ x1, const float* __restrict__ x2, const long long* __restrict__ t,
                                  int t_scalar, const float* __restrict__ sa, const float* __restrict__ sb, long long per_sample,
                                  long long n, float* __restrict__ out) {
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int tt = t ? static_cast<int>(t[i / per_sample]) : t_scalar;
    out[i] = sa[tt] * x1[i] + sb[tt] * x2[i];
  }
}
// mode 0: ddim (x2 estimated from x_t), mode 1: x0_step_down (x2 = the fixed initial noise)
__global__ void noise_step_kernel(const float* __restrict__ img, const float* __restrict__ x1, const float* __restrict__ noise,
                                  int mode, int t, const float* __restrict__ sa, const float* __restrict__ sb, long long n,
                                  float* __restrict__ out) {
  const float a1 = sa[t - 1], b1 = sb[t - 1];
  const float a2 = t - 1 != 0 ? sa[t - 2] : 0.f, b2 = t - 1 != 0 ? sb[t - 2] : 0.f;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float xv = x1[i], im = img[i];
    const float x2 = mode == 0 ? (im - a1 * xv) / b1 : noise[i];
    const float xt_bar = a1 * xv + b1 * x2;
    const float xt_sub1 = (t - 1 != 0) ? a2 * xv + b2 * x2 : xv;
    out[i] = im - xt_bar + xt_sub1;
  }
}
}  // namespace

extern "C" int cd_noise_lerp(const float* x1, const float* x2, const int64_t* t, int t_scalar, const float* sqrt_ac,
                             const float* sqrt_1mac, int64_t per_sample, int64_t n, float* out, void* stream) {
  int blocks = cd_cdiv(n, 256 * 4); if (blocks > cd_num_sms() * 8) blocks = cd_num_sms() * 8; if (blocks < 1) blocks = 1;
  noise_lerp_kernel<<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(x1, x2, reinterpret_cast<const long long*>(t), t_scalar,
                                                                         sqrt_ac, sqrt_1mac, per_sample, n, out);
  CD_LAUNCH_CHECK();
  return 0;
}

extern "C" int cd_noise_step(const float* img, const float* x1_bar, const float* noise, int mode, int t, const float* sqrt_ac,
                             const float* sqrt_1mac, int64_t n, float* out, void* stream) {
  CD_REQUIRE(t >= 1 && (mode == 0 || (mode == 1 && noise)), "cd_noise_step: bad arguments");
  int blocks = cd_cdiv(n, 256 * 4); if (blocks > cd_num_sms() * 8) blocks = cd_num_sms() * 8; if (blocks < 1) blocks = 1;
  noise_step_kernel<<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(img, x1_bar, noise, mode, t, sqrt_ac, sqrt_1mac, n, out);
  CD_LAUNCH_CHECK();
  return 0;
}

// -------------------------------------------------------------------------------------------------------------
// Strided reverse steps (cd_noise_step_to, cd_fade_step_to): the update of cd_noise_step / cd_fade_step from level t to any
// level s < t, x_s = img - D(x1, t) + D(x1, s), with D(x1, 0) = x1, in the same expressions as the one-step kernels.  s = t - 1
// launches the one-step kernel itself: the compiler may contract the same expressions into different FMAs in another kernel,
// and a K = T strided loop must be the one-step loop bit for bit.  kVec = 4: four consecutive elements per thread and
// iteration, with 16-byte loads and stores (every operand 16-byte aligned; for the fade tables also HW % 4 == 0, so that the
// four share one weight row); the n % 4 tail and misaligned operands take kVec = 1.
// -------------------------------------------------------------------------------------------------------------
namespace {
__device__ __forceinline__ float noise_step_to_elem(float im, float xv, float nz, int mode, int s, float a1, float b1, float a2,
                                                    float b2) {
  const float x2 = mode == 0 ? (im - a1 * xv) / b1 : nz;
  const float xt_bar = a1 * xv + b1 * x2;
  const float xs = (s != 0) ? a2 * xv + b2 * x2 : xv;
  return im - xt_bar + xs;
}
__device__ __forceinline__ float fade_step_to_elem(float im, float xv, float ev, float a1, float o1, bool to_clean, float a2, float o2) {
  const float xt_bar = a1 * xv + o1 * ev;
  float xs = xv;
  if (!to_clean) xs = a2 * xv + o2 * ev;
  return im - xt_bar + xs;
}
template <int kVec>
__global__ void noise_step_to_kernel(const float* __restrict__ img, const float* __restrict__ x1, const float* __restrict__ noise,
                                     int mode, int t, int s, const float* __restrict__ sa, const float* __restrict__ sb, long long n,
                                     float* __restrict__ out) {
  const float a1 = sa[t - 1], b1 = sb[t - 1];
  const float a2 = s != 0 ? sa[s - 1] : 0.f, b2 = s != 0 ? sb[s - 1] : 0.f;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  long long i0 = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (kVec == 4) {
    const long long n4 = n / 4;
    for (long long i = i0; i < n4; i += stride) {
      const float4 im = __ldg(reinterpret_cast<const float4*>(img) + i), xv = __ldg(reinterpret_cast<const float4*>(x1) + i);
      const float4 nz = mode == 0 ? make_float4(0.f, 0.f, 0.f, 0.f) : __ldg(reinterpret_cast<const float4*>(noise) + i);
      reinterpret_cast<float4*>(out)[i] = make_float4(noise_step_to_elem(im.x, xv.x, nz.x, mode, s, a1, b1, a2, b2),
                                                      noise_step_to_elem(im.y, xv.y, nz.y, mode, s, a1, b1, a2, b2),
                                                      noise_step_to_elem(im.z, xv.z, nz.z, mode, s, a1, b1, a2, b2),
                                                      noise_step_to_elem(im.w, xv.w, nz.w, mode, s, a1, b1, a2, b2));
    }
    i0 += n4 * 4;
  }
  for (long long i = i0; i < n; i += stride)
    out[i] = noise_step_to_elem(img[i], x1[i], mode == 0 ? 0.f : noise[i], mode, s, a1, b1, a2, b2);
}
template <int kVec>
__global__ void fade_step_to_kernel(const float* __restrict__ img, const float* __restrict__ x1, const float* __restrict__ x2,
                                    int t, int s, const float* __restrict__ al, const float* __restrict__ om, int HW, long long n,
                                    float* __restrict__ out) {
  const float* al1 = al + static_cast<long long>(t - 1) * HW;
  const float* om1 = om + static_cast<long long>(t - 1) * HW;
  const bool to_clean = s == 0;
  const float* al2 = to_clean ? al1 : al + static_cast<long long>(s - 1) * HW;   // not read when s == 0
  const float* om2 = to_clean ? om1 : om + static_cast<long long>(s - 1) * HW;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  long long i0 = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (kVec == 4) {
    const long long n4 = n / 4;
    for (long long i = i0; i < n4; i += stride) {
      const int p4 = static_cast<int>((i * 4) % HW) / 4;
      const float4 im = __ldg(reinterpret_cast<const float4*>(img) + i), xv = __ldg(reinterpret_cast<const float4*>(x1) + i);
      const float4 ev = __ldg(reinterpret_cast<const float4*>(x2) + i);
      const float4 a1 = __ldg(reinterpret_cast<const float4*>(al1) + p4), o1 = __ldg(reinterpret_cast<const float4*>(om1) + p4);
      float4 a2 = a1, o2 = o1;
      if (!to_clean) { a2 = __ldg(reinterpret_cast<const float4*>(al2) + p4); o2 = __ldg(reinterpret_cast<const float4*>(om2) + p4); }
      reinterpret_cast<float4*>(out)[i] = make_float4(fade_step_to_elem(im.x, xv.x, ev.x, a1.x, o1.x, to_clean, a2.x, o2.x),
                                                      fade_step_to_elem(im.y, xv.y, ev.y, a1.y, o1.y, to_clean, a2.y, o2.y),
                                                      fade_step_to_elem(im.z, xv.z, ev.z, a1.z, o1.z, to_clean, a2.z, o2.z),
                                                      fade_step_to_elem(im.w, xv.w, ev.w, a1.w, o1.w, to_clean, a2.w, o2.w));
    }
    i0 += n4 * 4;
  }
  for (long long i = i0; i < n; i += stride) {
    const int pix = static_cast<int>(i % HW);
    out[i] = fade_step_to_elem(img[i], x1[i], x2[i], al1[pix], om1[pix], to_clean, to_clean ? 0.f : al2[pix],
                               to_clean ? 0.f : om2[pix]);
  }
}
bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }
}  // namespace

extern "C" int cd_noise_step_to(const float* img, const float* x1_bar, const float* noise, int mode, int t, int s,
                                const float* sqrt_ac, const float* sqrt_1mac, int64_t n, float* out, void* stream) {
  CD_REQUIRE(0 <= s && s < t && (mode == 0 || (mode == 1 && noise)) && n >= 0, "cd_noise_step_to: bad arguments");
  if (n == 0) return 0;
  if (s == t - 1) return cd_noise_step(img, x1_bar, noise, mode, t, sqrt_ac, sqrt_1mac, n, out, stream);
  const bool vec = aligned16(img) && aligned16(x1_bar) && aligned16(out) && (mode == 0 || aligned16(noise));
  int blocks = cd_cdiv(vec ? n / 4 : n, 256); if (blocks > cd_num_sms() * 8) blocks = cd_num_sms() * 8; if (blocks < 1) blocks = 1;
  if (vec)
    noise_step_to_kernel<4><<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(img, x1_bar, noise, mode, t, s, sqrt_ac, sqrt_1mac, n, out);
  else
    noise_step_to_kernel<1><<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(img, x1_bar, noise, mode, t, s, sqrt_ac, sqrt_1mac, n, out);
  CD_LAUNCH_CHECK();
  return 0;
}

// -------------------------------------------------------------------------------------------------------------
// Fade-to-colour generation (defading-generation-diffusion-pytorch/defading_diffusion_pytorch/defading_diffusion_pytorch.py,
// "DFGEN"): the schedule is a per-PIXEL weight, alphas[t][y][x] = cumulative product of the fade kernels (DFGEN:320-344),
// q_sample = alphas[t_b] * x1 + one_minus_alphas[t_b] * x2 (DFGEN:543-548), reverse step = img - xt_bar + xt_sub1_bar with
// the fixed end image x2 (DFGEN:386-418).  Both weight tables are passed: in `reverse` mode the reference derives alphas from
// one_minus_alphas, not the other way round.
// -------------------------------------------------------------------------------------------------------------
namespace {
__global__ void fade_lerp_kernel(const float* __restrict__ x1, const float* __restrict__ x2, const long long* __restrict__ t,
                                 int t_scalar, const float* __restrict__ al, const float* __restrict__ om, int C, int HW,
                                 long long n, float* __restrict__ out) {
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int pix = static_cast<int>(i % HW);
    const int tt = t ? static_cast<int>(t[i / (static_cast<long long>(HW) * C)]) : t_scalar;
    const long long w = static_cast<long long>(tt) * HW + pix;
    out[i] = al[w] * x1[i] + om[w] * x2[i];
  }
}
__global__ void fade_step_kernel(const float* __restrict__ img, const float* __restrict__ x1, const float* __restrict__ x2,
                                 int t, const float* __restrict__ al, const float* __restrict__ om, int HW, long long n,
                                 float* __restrict__ out) {
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int pix = static_cast<int>(i % HW);
    const float xv = x1[i], ev = x2[i];
    const long long w1 = static_cast<long long>(t - 1) * HW + pix;
    const float xt_bar = al[w1] * xv + om[w1] * ev;
    float xt_sub1 = xv;
    if (t - 1 != 0) { const long long w2 = w1 - HW; xt_sub1 = al[w2] * xv + om[w2] * ev; }
    out[i] = img[i] - xt_bar + xt_sub1;
  }
}
}  // namespace

extern "C" int cd_fade_lerp(const float* x1, const float* x2, const int64_t* t, int t_scalar, const float* alphas,
                            const float* one_minus_alphas, int B, int C, int HW, float* out, void* stream) {
  const long long n = static_cast<long long>(B) * C * HW;
  int blocks = cd_cdiv(n, 256 * 4); if (blocks > cd_num_sms() * 8) blocks = cd_num_sms() * 8; if (blocks < 1) blocks = 1;
  fade_lerp_kernel<<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(x1, x2, reinterpret_cast<const long long*>(t), t_scalar,
                                                                        alphas, one_minus_alphas, C, HW, n, out);
  CD_LAUNCH_CHECK();
  return 0;
}

// -------------------------------------------------------------------------------------------------------------
// Gradient of the two lerps out = wa[w] x1 + wb[w] x2 (cd_noise_lerp, cd_fade_lerp): both input gradients from one read of g,
// w = t_b for per-sample scalars (per_pixel = 0) or t_b HW + pixel for per-pixel tables (per_pixel = 1).
// -------------------------------------------------------------------------------------------------------------
namespace {
__global__ void lerp2_adjoint_kernel(const float* __restrict__ g, const long long* __restrict__ t, int t_scalar,
                                     const float* __restrict__ wa, const float* __restrict__ wb, int C, long long HW, int per_pixel,
                                     long long n, float* __restrict__ ga, float* __restrict__ gb) {
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long tt = t ? t[i / (HW * C)] : t_scalar;
    const long long w = per_pixel ? tt * HW + i % HW : tt;
    const float gv = g[i];
    if (ga) ga[i] = wa[w] * gv;
    if (gb) gb[i] = wb[w] * gv;
  }
}
}  // namespace

extern "C" int cd_lerp2_adjoint(const float* g, const int64_t* t, int t_scalar, const float* wa, const float* wb, int B, int C,
                                int64_t HW, int per_pixel, float* ga, float* gb, void* stream) {
  CD_REQUIRE(g && wa && wb && (ga || gb) && B >= 0 && C >= 1 && HW >= 0 && (per_pixel == 0 || per_pixel == 1),
             "cd_lerp2_adjoint: bad arguments");
  const long long n = static_cast<long long>(B) * C * HW;
  if (n == 0) return 0;
  int blocks = cd_cdiv(n, 256 * 4); if (blocks > cd_num_sms() * 8) blocks = cd_num_sms() * 8; if (blocks < 1) blocks = 1;
  lerp2_adjoint_kernel<<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(g, reinterpret_cast<const long long*>(t), t_scalar, wa, wb,
                                                                            C, HW, per_pixel, n, ga, gb);
  CD_LAUNCH_CHECK();
  return 0;
}

extern "C" int cd_fade_step(const float* img, const float* x1_bar, const float* x2, int t, const float* alphas,
                            const float* one_minus_alphas, int B, int C, int HW, float* out, void* stream) {
  CD_REQUIRE(t >= 1 && x2, "cd_fade_step: bad arguments");
  const long long n = static_cast<long long>(B) * C * HW;
  int blocks = cd_cdiv(n, 256 * 4); if (blocks > cd_num_sms() * 8) blocks = cd_num_sms() * 8; if (blocks < 1) blocks = 1;
  fade_step_kernel<<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(img, x1_bar, x2, t, alphas, one_minus_alphas, HW, n, out);
  CD_LAUNCH_CHECK();
  return 0;
}

extern "C" int cd_fade_step_to(const float* img, const float* x1_bar, const float* x2, int t, int s, const float* alphas,
                               const float* one_minus_alphas, int B, int C, int HW, float* out, void* stream) {
  CD_REQUIRE(0 <= s && s < t && x2 && B >= 0 && C >= 1 && HW >= 1, "cd_fade_step_to: bad arguments");
  const long long n = static_cast<long long>(B) * C * HW;
  if (n == 0) return 0;
  if (s == t - 1) return cd_fade_step(img, x1_bar, x2, t, alphas, one_minus_alphas, B, C, HW, out, stream);
  const bool vec = HW % 4 == 0 && aligned16(img) && aligned16(x1_bar) && aligned16(x2) && aligned16(out) && aligned16(alphas) &&
                   aligned16(one_minus_alphas);
  int blocks = cd_cdiv(vec ? n / 4 : n, 256); if (blocks > cd_num_sms() * 8) blocks = cd_num_sms() * 8; if (blocks < 1) blocks = 1;
  if (vec)
    fade_step_to_kernel<4><<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(img, x1_bar, x2, t, s, alphas, one_minus_alphas, HW, n, out);
  else
    fade_step_to_kernel<1><<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(img, x1_bar, x2, t, s, alphas, one_minus_alphas, HW, n, out);
  CD_LAUNCH_CHECK();
  return 0;
}

// -------------------------------------------------------------------------------------------------------------
// Gaussian-mask fading (defading-diffusion-pytorch/defading_diffusion_pytorch/defading_diffusion_gaussian.py, "DFG"):
// D(x,t) = x * prod_{i<=t} K_i with K_i = (1 - g_i / max g_i)[1:,1:] (DFG:328-352).  masks: cumulative products
// [T][MS][MS] (MS = S, or 2S for the 'Random_*' routines where every sample uses its own S x S window at offset
// (rx[b], ry[b]), DFG:359-367, 499-507 -- integer indexing, bit-exact).  idx < 0 = identity.
// -------------------------------------------------------------------------------------------------------------
namespace {
__device__ __forceinline__ float mask_at(const float* __restrict__ masks, int idx, int MS, int y, int x) {
  return idx < 0 ? 1.f : masks[(static_cast<long long>(idx) * MS + y) * MS + x];
}
__device__ __forceinline__ float quantize8(float v) {            // DFG:380-384 / DB:954-958
  float q = (v + 1.f) * 0.5f;
  q = q * 255.f;
  q = static_cast<float>(static_cast<int>(q)) / 255.f;
  return q * 2.f - 1.f;
}
// kEpi (guided restoration; quantize is then 0): kEpiAxpy out = x m - w g (the guided `default` update); kEpiGuide out =
// m (x m - g), the guidance gradient with g = y
template <int kEpi = kEpiNone>
__global__ void mask_apply_kernel(const float* __restrict__ x, float* __restrict__ out, const float* __restrict__ masks,
                                  const long long* __restrict__ t, int t_scalar, const long long* __restrict__ rx,
                                  const long long* __restrict__ ry, int B, int C, int S, int MS, int quantize,
                                  const float* __restrict__ g, float w) {
  const long long n = static_cast<long long>(B) * C * S * S;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int xx = static_cast<int>(i % S), yy = static_cast<int>((i / S) % S);
    const int b = static_cast<int>(i / (static_cast<long long>(S) * S * C));
    const int idx = t ? static_cast<int>(t[b]) : t_scalar;
    const int oy = rx ? static_cast<int>(rx[b]) : 0, ox = ry ? static_cast<int>(ry[b]) : 0;   // reference: rows <- rand_x, cols <- rand_y
    const float m = mask_at(masks, idx, MS, yy + oy, xx + ox);
    float v = x[i] * m;
    if constexpr (kEpi == kEpiAxpy) v = v - w * g[i];
    if constexpr (kEpi == kEpiGuide) v = (v - g[i]) * m;
    if (quantize) v = quantize8(v);
    out[i] = v;
  }
}
template <bool kAxpy = false>
__global__ void mask_step_down_kernel(const float* __restrict__ xt, const float* __restrict__ xhat, float* __restrict__ out,
                                      const float* __restrict__ masks, int idx_hi, int idx_lo, const long long* __restrict__ rx,
                                      const long long* __restrict__ ry, int B, int C, int S, int MS, const float* __restrict__ g,
                                      float w) {
  const long long n = static_cast<long long>(B) * C * S * S;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int xx = static_cast<int>(i % S), yy = static_cast<int>((i / S) % S);
    const int b = static_cast<int>(i / (static_cast<long long>(S) * S * C));
    const int oy = rx ? static_cast<int>(rx[b]) : 0, ox = ry ? static_cast<int>(ry[b]) : 0;
    const float xv = xhat[i];
    const float hi = xv * mask_at(masks, idx_hi, MS, yy + oy, xx + ox);
    const float lo = xv * mask_at(masks, idx_lo, MS, yy + oy, xx + ox);
    float v = xt[i] - hi + lo;
    if constexpr (kAxpy) v = v - w * g[i];
    out[i] = v;
  }
}

template <int kEpi>
int mask_apply(const float* x, float* out, const float* masks, const int64_t* t, int t_scalar, const int64_t* rx, const int64_t* ry,
               int B, int C, int S, int MS, int quantize, cudaStream_t stream, const float* g, float w) {
  const long long n = static_cast<long long>(B) * C * S * S;
  int blocks = cd_cdiv(n, 256 * 4); if (blocks > cd_num_sms() * 8) blocks = cd_num_sms() * 8; if (blocks < 1) blocks = 1;
  mask_apply_kernel<kEpi><<<blocks, 256, 0, stream>>>(x, out, masks, reinterpret_cast<const long long*>(t), t_scalar,
      reinterpret_cast<const long long*>(rx), reinterpret_cast<const long long*>(ry), B, C, S, MS, quantize, g, w);
  CD_LAUNCH_CHECK();
  return 0;
}

template <bool kAxpy>
int mask_step_down(const float* xt, const float* xhat, float* out, const float* masks, int idx_hi, int idx_lo, const int64_t* rx,
                   const int64_t* ry, int B, int C, int S, int MS, cudaStream_t stream, const float* g, float w) {
  const long long n = static_cast<long long>(B) * C * S * S;
  int blocks = cd_cdiv(n, 256 * 4); if (blocks > cd_num_sms() * 8) blocks = cd_num_sms() * 8; if (blocks < 1) blocks = 1;
  mask_step_down_kernel<kAxpy><<<blocks, 256, 0, stream>>>(xt, xhat, out, masks, idx_hi, idx_lo,
      reinterpret_cast<const long long*>(rx), reinterpret_cast<const long long*>(ry), B, C, S, MS, g, w);
  CD_LAUNCH_CHECK();
  return 0;
}
}  // namespace

extern "C" int cd_mask_apply(const float* x, float* out, const float* masks, const int64_t* t, int t_scalar,
                             const int64_t* rx, const int64_t* ry, int B, int C, int S, int MS, int quantize, void* stream) {
  return mask_apply<kEpiNone>(x, out, masks, t, t_scalar, rx, ry, B, C, S, MS, quantize, static_cast<cudaStream_t>(stream), nullptr, 0.f);
}

extern "C" int cd_mask_step_down(const float* xt, const float* xhat, float* out, const float* masks, int idx_hi, int idx_lo,
                                 const int64_t* rx, const int64_t* ry, int B, int C, int S, int MS, void* stream) {
  return mask_step_down<false>(xt, xhat, out, masks, idx_hi, idx_lo, rx, ry, B, C, S, MS, static_cast<cudaStream_t>(stream), nullptr,
                               0.f);
}

// guided restoration: the guidance gradient m (m x0 - y) with m = the mask at idx in each sample's window, in one pass
extern "C" int cd_mask_guide_grad(const float* x0, const float* y, float* out, const float* masks, int idx, const int64_t* rx,
                                  const int64_t* ry, int B, int C, int S, int MS, void* stream) {
  CD_REQUIRE(x0 && y && out && masks && B >= 0 && C >= 1 && S >= 1 && MS >= S, "cd_mask_guide_grad: bad arguments");
  return mask_apply<kEpiGuide>(x0, out, masks, nullptr, idx, rx, ry, B, C, S, MS, 0, static_cast<cudaStream_t>(stream), y, 1.f);
}

// the guided update: xt == NULL -> `default`, out = xhat m_lo - w g; else out = xt - xhat m_hi + xhat m_lo - w g.  g == NULL runs
// the unguided kernels themselves (their bits).
extern "C" int cd_mask_guided_step(const float* xt, const float* xhat, const float* g, float weight, float* out, const float* masks,
                                   int idx_hi, int idx_lo, const int64_t* rx, const int64_t* ry, int B, int C, int S, int MS,
                                   void* stream) {
  CD_REQUIRE(xhat && out && masks && B >= 0 && C >= 1 && S >= 1 && MS >= S, "cd_mask_guided_step: bad arguments");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (!xt) {
    if (!g) return mask_apply<kEpiNone>(xhat, out, masks, nullptr, idx_lo, rx, ry, B, C, S, MS, 0, st, nullptr, 0.f);
    return mask_apply<kEpiAxpy>(xhat, out, masks, nullptr, idx_lo, rx, ry, B, C, S, MS, 0, st, g, weight);
  }
  if (!g) return mask_step_down<false>(xt, xhat, out, masks, idx_hi, idx_lo, rx, ry, B, C, S, MS, st, nullptr, 0.f);
  return mask_step_down<true>(xt, xhat, out, masks, idx_hi, idx_lo, rx, ry, B, C, S, MS, st, g, weight);
}

// -------------------------------------------------------------------------------------------------------------
// Decolorization / Snow forward processes of snowification/ (== decolor-diffusion/) diffusion/forward_process_impl.py
// ("FP") with the per-sample masked stepping of diffusion/diffusion.py ("SN", SN:195-245, 344-388):
//  * decolor: every step is a per-pixel C x C channel mix f I + (1-f)/C 11^T (FP:150-163); the cumulative mix after
//    steps 0..i is tabulated ([T][C][C]) so D(x, t_b) is one mat-vec per pixel with a PER-SAMPLE index (t_b = -1 =
//    untouched row, SN:349-355); the masked loops of sample_one_step collapse to per-sample indices t_b-1 / t_b-2.
//  * snow: D depends on the clean image only (FP:361-372): clip(bright_i(og) + snow_i + rot180(snow_i), 0, 1)*2-1.
// -------------------------------------------------------------------------------------------------------------
namespace {
// kEpi (guided restoration): kEpiAxpy = either mode's result - w g; kEpiGuide = the guidance gradient M^T (M xsrc - g) with
// M = mats[t_hi+hi_off] (mode 0 only; index < 0: xsrc - g)
template <int kEpi = kEpiNone>
__global__ void chanmix_kernel(const float* __restrict__ xt, const float* __restrict__ xsrc, float* __restrict__ out,
                               const float* __restrict__ mats, const long long* __restrict__ t_hi, const long long* __restrict__ t_lo,
                               int hi_off, int lo_off, int B, int C, long long HW, int mode, const float* __restrict__ g, float w) {
  // mode 0: out = M[t_hi+hi_off] xsrc ; mode 1: out = xt - M[t_hi+hi_off] xsrc + M[t_lo+lo_off] xsrc   (index < 0 = identity)
  const long long n = static_cast<long long>(B) * HW;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int b = static_cast<int>(i / HW);
    const long long p = i % HW;
    const int ih = static_cast<int>(t_hi[b]) + hi_off;
    const int il = mode ? static_cast<int>(t_lo[b]) + lo_off : -1;
    float v[8];
    for (int c = 0; c < C; ++c) v[c] = xsrc[(static_cast<long long>(b) * C + c) * HW + p];
    if constexpr (kEpi == kEpiGuide) {
      float r[8];
      for (int co = 0; co < C; ++co) {
        float hi = v[co];
        if (ih >= 0) { hi = 0.f; for (int c = 0; c < C; ++c) hi = fmaf(mats[(ih * C + co) * C + c], v[c], hi); }
        r[co] = hi - g[(static_cast<long long>(b) * C + co) * HW + p];
      }
      for (int c = 0; c < C; ++c) {
        float s = r[c];
        if (ih >= 0) { s = 0.f; for (int co = 0; co < C; ++co) s = fmaf(mats[(ih * C + co) * C + c], r[co], s); }
        out[(static_cast<long long>(b) * C + c) * HW + p] = s;
      }
    } else {
      for (int co = 0; co < C; ++co) {
        float hi = v[co], lo = v[co];
        if (ih >= 0) { hi = 0.f; for (int c = 0; c < C; ++c) hi = fmaf(mats[(ih * C + co) * C + c], v[c], hi); }
        if (il >= 0) { lo = 0.f; for (int c = 0; c < C; ++c) lo = fmaf(mats[(il * C + co) * C + c], v[c], lo); }
        const long long o = (static_cast<long long>(b) * C + co) * HW + p;
        float r = mode ? xt[o] - hi + lo : hi;
        if constexpr (kEpi == kEpiAxpy) r = r - w * g[o];
        out[o] = r;
      }
    }
  }
}
__global__ void snow_kernel(const float* __restrict__ xt, const float* __restrict__ og, float* __restrict__ out,
                            const float* __restrict__ snow, const float* __restrict__ br, const long long* __restrict__ t_hi,
                            const long long* __restrict__ t_lo, int hi_off, int lo_off, int B, int H, int W, int snow_batch,
                            int fix_brightness, int mode) {
  // snow: [T][snow_batch][3][H][W]; rot180 is an index flip.  3-channel RGB only (kornia rgb_to_grayscale weights).
  const long long HW = static_cast<long long>(H) * W, n = static_cast<long long>(B) * HW;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int b = static_cast<int>(i / HW);
    const long long p = i % HW, pr = HW - 1 - p;
    const int sb = snow_batch > 1 ? b : 0;
    float r[3], g3[3];
    for (int c = 0; c < 3; ++c) r[c] = (og[(static_cast<long long>(b) * 3 + c) * HW + p] + 1.f) / 2.f;
    const float gray = (0.299f * r[0] + 0.587f * r[1] + 0.114f * r[2]) * 1.5f + 0.5f;
    for (int c = 0; c < 3; ++c) g3[c] = fmaxf(r[c], gray);
    const int ih = static_cast<int>(t_hi[b]) + hi_off;
    const int il = mode ? static_cast<int>(t_lo[b]) + lo_off : -1;
    for (int c = 0; c < 3; ++c) {
      const long long o = (static_cast<long long>(b) * 3 + c) * HW + p;
      float res[2];
      const int idx[2] = {ih, il};
      for (int k = 0; k < 2; ++k) {
        if (idx[k] < 0) { res[k] = og[o]; continue; }
        const float bc = br[idx[k]];
        const float base = fix_brightness ? r[c] : bc * r[c] + (1.f - bc) * g3[c];
        const float* sl = snow + ((static_cast<long long>(idx[k]) * snow_batch + sb) * 3 + c) * HW;
        const float sn = fminf(fmaxf(base + sl[p] + sl[pr], 0.f), 1.f);
        res[k] = sn * 2.f - 1.f;
      }
      out[o] = mode ? xt[o] - res[0] + res[1] : res[0];
    }
  }
}
}  // namespace

namespace {
template <int kEpi>
int chanmix(const float* xt, const float* xsrc, float* out, const float* mats, const int64_t* t_hi, const int64_t* t_lo, int hi_off,
            int lo_off, int B, int C, int64_t HW, int mode, cudaStream_t stream, const float* g, float w) {
  const long long n = static_cast<long long>(B) * HW;
  int blocks = cd_cdiv(n, 256 * 2); if (blocks > cd_num_sms() * 8) blocks = cd_num_sms() * 8; if (blocks < 1) blocks = 1;
  chanmix_kernel<kEpi><<<blocks, 256, 0, stream>>>(xt, xsrc, out, mats, reinterpret_cast<const long long*>(t_hi),
      reinterpret_cast<const long long*>(t_lo), hi_off, lo_off, B, C, HW, mode, g, w);
  CD_LAUNCH_CHECK();
  return 0;
}
}  // namespace

extern "C" int cd_chanmix(const float* xt, const float* xsrc, float* out, const float* mats, const int64_t* t_hi,
                          const int64_t* t_lo, int hi_off, int lo_off, int B, int C, int64_t HW, int mode, void* stream) {
  CD_REQUIRE(C <= 8 && t_hi && (mode == 0 || (xt && t_lo)), "cd_chanmix: bad arguments");
  return chanmix<kEpiNone>(xt, xsrc, out, mats, t_hi, t_lo, hi_off, lo_off, B, C, HW, mode, static_cast<cudaStream_t>(stream), nullptr,
                           0.f);
}

// guided restoration: the guidance gradient M^T (M x0 - y) per pixel, M = mats[t[b] + off] (index < 0: x0 - y), in one pass
extern "C" int cd_chanmix_guide_grad(const float* x0, const float* y, float* out, const float* mats, const int64_t* t, int off,
                                     int B, int C, int64_t HW, void* stream) {
  CD_REQUIRE(x0 && y && out && mats && t && C >= 1 && C <= 8 && B >= 0 && HW >= 0, "cd_chanmix_guide_grad: bad arguments");
  return chanmix<kEpiGuide>(nullptr, x0, out, mats, t, nullptr, off, 0, B, C, HW, 0, static_cast<cudaStream_t>(stream), y, 1.f);
}

// the guided update: cd_chanmix's mode 0 / 1 result - w g.  g == NULL runs cd_chanmix itself (its bits).
extern "C" int cd_chanmix_guided(const float* xt, const float* xsrc, const float* g, float weight, float* out, const float* mats,
                                 const int64_t* t_hi, const int64_t* t_lo, int hi_off, int lo_off, int B, int C, int64_t HW, int mode,
                                 void* stream) {
  CD_REQUIRE(C <= 8 && t_hi && (mode == 0 || (mode == 1 && xt && t_lo)), "cd_chanmix_guided: bad arguments");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (!g) return chanmix<kEpiNone>(xt, xsrc, out, mats, t_hi, t_lo, hi_off, lo_off, B, C, HW, mode, st, nullptr, 0.f);
  return chanmix<kEpiAxpy>(xt, xsrc, out, mats, t_hi, t_lo, hi_off, lo_off, B, C, HW, mode, st, g, weight);
}

extern "C" int cd_snow(const float* xt, const float* og, float* out, const float* snow, const float* br_coef, const int64_t* t_hi,
                       const int64_t* t_lo, int hi_off, int lo_off, int B, int H, int W, int snow_batch, int fix_brightness,
                       int mode, void* stream) {
  CD_REQUIRE(t_hi && (mode == 0 || (xt && t_lo)), "cd_snow: bad arguments");
  const long long n = static_cast<long long>(B) * H * W;
  int blocks = cd_cdiv(n, 256 * 2); if (blocks > cd_num_sms() * 8) blocks = cd_num_sms() * 8; if (blocks < 1) blocks = 1;
  snow_kernel<<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(xt, og, out, snow, br_coef, reinterpret_cast<const long long*>(t_hi),
      reinterpret_cast<const long long*>(t_lo), hi_off, lo_off, B, H, W, snow_batch, fix_brightness, mode);
  CD_LAUNCH_CHECK();
  return 0;
}

// -------------------------------------------------------------------------------------------------------------
// Lab colour path of the decolorization package (`to_lab=True`): rgb2lab / lab2rgb of diffusion/utils.py:113-222 ("UT")
// and the decolorization step in Lab, rgb2lab(M_i lab2rgb(x)) (FP:189-195).  lab2rgb clamps fz and clips RGB to [0, 1]
// at every step, so the steps do not compose into one matrix: every thread keeps its pixel's three values in registers
// and runs the step chain 0..max(hi, lo), keeping the values after step hi and after step lo.
// The sRGB <-> linear RGB and linear RGB <-> XYZ stages are kornia's (rgb_to_linear_rgb, linear_rgb_to_rgb, rgb_to_xyz,
// xyz_to_rgb), which the reference imports without pinning a version; they are restated here from kornia's formulas, so
// parity is unpinned at those constants.  Full-precision powf: the thresholds below select branches.
// -------------------------------------------------------------------------------------------------------------
namespace {
__device__ __forceinline__ float srgb_to_linear(float x) {
  return x > 0.04045f ? powf((x + 0.055f) / 1.055f, 2.4f) : x / 12.92f;
}
__device__ __forceinline__ float linear_to_srgb(float x) {
  return x > 0.0031308f ? 1.055f * powf(fmaxf(x, 0.0031308f), 1.f / 2.4f) - 0.055f : 12.92f * x;
}
__device__ __forceinline__ float lab_f(float t) {          // UT:146-149
  return t > 0.008856f ? powf(fmaxf(t, 0.008856f), 1.f / 3.f) : 7.787f * t + 4.f / 29.f;
}
__device__ __forceinline__ float lab_finv(float f) {       // UT:198-200
  return f > 0.2068966f ? f * f * f : (f - 4.f / 29.f) / 7.787f;
}
// UT:113-163: RGB in [-1, 1] -> Lab (D65 white)
__device__ __forceinline__ void rgb_to_lab(float r, float g, float b, float& L, float& A, float& Bb) {
  r = srgb_to_linear((r + 1.f) * 0.5f); g = srgb_to_linear((g + 1.f) * 0.5f); b = srgb_to_linear((b + 1.f) * 0.5f);
  const float x = 0.412453f * r + 0.357580f * g + 0.180423f * b;
  const float y = 0.212671f * r + 0.715160f * g + 0.072169f * b;
  const float z = 0.019334f * r + 0.119193f * g + 0.950227f * b;
  const float fx = lab_f(x / 0.95047f), fy = lab_f(y), fz = lab_f(z / 1.08883f);
  L = 116.f * fy - 16.f;
  A = 500.f * (fx - fy);
  Bb = 200.f * (fy - fz);
}
// UT:166-222: Lab -> 2 rgb - 1 (rgb clipped to [0, 1] when `clip`)
__device__ __forceinline__ void lab_to_rgb(float L, float A, float Bb, bool clip, float& r, float& g, float& b) {
  const float fy = (L + 16.f) / 116.f;
  const float fx = A / 500.f + fy;
  const float fz = fmaxf(fy - Bb / 200.f, 0.f);
  const float x = lab_finv(fx) * 0.95047f, y = lab_finv(fy), z = lab_finv(fz) * 1.08883f;
  r = linear_to_srgb(3.2404813432005266f * x + -1.5371515162713185f * y + -0.4985363261688878f * z);
  g = linear_to_srgb(-0.9692549499965682f * x + 1.8759900014898907f * y + 0.0415559265582928f * z);
  b = linear_to_srgb(0.0556466391351772f * x + -0.2040413383665112f * y + 1.0572251624579105f * z);
  if (clip) { r = fminf(fmaxf(r, 0.f), 1.f); g = fminf(fmaxf(g, 0.f), 1.f); b = fminf(fmaxf(b, 0.f), 1.f); }
  r = 2.f * r - 1.f; g = 2.f * g - 1.f; b = 2.f * b - 1.f;
}

__global__ void lab_convert_kernel(const float* x, float* out, int B, long long HW, int to_lab, int clip) {
  // x and out may alias: every thread reads its pixel's three channels before writing them
  const long long n = static_cast<long long>(B) * HW;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long b = i / HW, p = i % HW;
    const long long o0 = b * 3 * HW + p, o1 = o0 + HW, o2 = o1 + HW;
    const float v0 = x[o0], v1 = x[o1], v2 = x[o2];
    float w0, w1, w2;
    if (to_lab) rgb_to_lab(v0, v1, v2, w0, w1, w2);
    else lab_to_rgb(v0, v1, v2, clip != 0, w0, w1, w2);
    out[o0] = w0; out[o1] = w1; out[o2] = w2;
  }
}

__global__ void chanmix_lab_kernel(const float* __restrict__ xt, const float* __restrict__ xsrc, float* __restrict__ out,
                                   const float* __restrict__ mats, const long long* __restrict__ t_hi,
                                   const long long* __restrict__ t_lo, int hi_off, int lo_off, int B, long long HW, int mode) {
  // mode 0: out = D(xsrc, t_hi+hi_off) ; mode 1: out = xt - D(xsrc, t_hi+hi_off) + D(xsrc, t_lo+lo_off)
  // D(v, k) = step k of ... step 0 of v, step i = rgb2lab(M_i lab2rgb(v)); index < 0 = v untouched
  const long long n = static_cast<long long>(B) * HW;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int b = static_cast<int>(i / HW);
    const long long p = i % HW;
    const long long o0 = static_cast<long long>(b) * 3 * HW + p, o1 = o0 + HW, o2 = o1 + HW;
    const int ih = static_cast<int>(t_hi[b]) + hi_off;
    const int il = mode ? static_cast<int>(t_lo[b]) + lo_off : -1;
    float c0 = xsrc[o0], c1 = xsrc[o1], c2 = xsrc[o2];
    float h0 = c0, h1 = c1, h2 = c2, l0 = c0, l1 = c1, l2 = c2;
    const int last = ih > il ? ih : il;
    for (int s = 0; s <= last; ++s) {
      float r, g, bl;
      lab_to_rgb(c0, c1, c2, true, r, g, bl);
      const float* M = mats + s * 9;
      const float m0 = fmaf(__ldg(M + 2), bl, fmaf(__ldg(M + 1), g, __ldg(M + 0) * r));
      const float m1 = fmaf(__ldg(M + 5), bl, fmaf(__ldg(M + 4), g, __ldg(M + 3) * r));
      const float m2 = fmaf(__ldg(M + 8), bl, fmaf(__ldg(M + 7), g, __ldg(M + 6) * r));
      rgb_to_lab(m0, m1, m2, c0, c1, c2);
      if (s == ih) { h0 = c0; h1 = c1; h2 = c2; }
      if (s == il) { l0 = c0; l1 = c1; l2 = c2; }
    }
    if (mode) {
      out[o0] = xt[o0] - h0 + l0; out[o1] = xt[o1] - h1 + l1; out[o2] = xt[o2] - h2 + l2;
    } else {
      out[o0] = h0; out[o1] = h1; out[o2] = h2;
    }
  }
}
}  // namespace

extern "C" int cd_lab_convert(const float* x, float* out, int B, int64_t HW, int to_lab, int clip, void* stream) {
  CD_REQUIRE(x && out && B >= 0 && HW >= 0, "cd_lab_convert: bad arguments");
  const long long n = static_cast<long long>(B) * HW;
  if (n == 0) return 0;
  int blocks = cd_cdiv(n, 256 * 2); if (blocks > cd_num_sms() * 8) blocks = cd_num_sms() * 8; if (blocks < 1) blocks = 1;
  lab_convert_kernel<<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(x, out, B, HW, to_lab, clip);
  CD_LAUNCH_CHECK();
  return 0;
}

extern "C" int cd_chanmix_lab(const float* xt, const float* xsrc, float* out, const float* step_mats, const int64_t* t_hi,
                              const int64_t* t_lo, int hi_off, int lo_off, int B, int64_t HW, int mode, void* stream) {
  CD_REQUIRE(xsrc && out && step_mats && t_hi && (mode == 0 || (mode == 1 && xt && t_lo)), "cd_chanmix_lab: bad arguments");
  const long long n = static_cast<long long>(B) * HW;
  if (n == 0) return 0;
  int blocks = cd_cdiv(n, 256 * 2); if (blocks > cd_num_sms() * 8) blocks = cd_num_sms() * 8; if (blocks < 1) blocks = 1;
  chanmix_lab_kernel<<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(xt, xsrc, out, step_mats, reinterpret_cast<const long long*>(t_hi),
      reinterpret_cast<const long long*>(t_lo), hi_off, lo_off, B, HW, mode);
  CD_LAUNCH_CHECK();
  return 0;
}
