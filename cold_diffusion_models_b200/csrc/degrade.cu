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
__global__ void __launch_bounds__(256)
blur_apply_kernel(const float* __restrict__ x, float* __restrict__ out, const float* __restrict__ ops,
                  const long long* __restrict__ t, int t_scalar, int S, int T, int collapse_last, int quantize) {
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
  if (idx >= 0) load_plane(As, S, ops + static_cast<long long>(idx) * S * S, S);
  __syncthreads();
  if (idx >= 0) plane_apply(As, Xs, Yt, Xs, S, ldp);
  float mean = 0.f;
  const bool collapse = collapse_last && idx == T - 1;
  if (collapse) {
    float s = 0.f;
    for (int i = threadIdx.x; i < S * S; i += blockDim.x) s += Xs[(i / S) * ldp + (i % S)];
    mean = block_sum(s, scratch) / (S * S);
  }
  const int per_row = S >> 2;
  for (int i = threadIdx.x; i < (S * S) >> 2; i += blockDim.x) {
    const int r = i / per_row, c = (i % per_row) * 4;
    float4 v = *reinterpret_cast<const float4*>(Xs + r * ldp + c);
    if (collapse) v = make_float4(mean, mean, mean, mean);
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
__global__ void __launch_bounds__(256)
blur_step_down_kernel(const float* __restrict__ xt, const float* __restrict__ xhat, float* __restrict__ out,
                      const float* __restrict__ ops, int t_hi, int t_lo, int S, int T, int collapse_last) {
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
    reinterpret_cast<float4*>(out + pl * S * S)[i] = o;
  }
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

extern "C" int cd_blur_apply(const float* x, float* out, const float* ops, const int64_t* t, int t_scalar,
                             int B, int C, int S, int T, int collapse_last, int quantize, void* stream) {
  CD_REQUIRE(S % 4 == 0 && S >= 4 && S <= 128, "cd_blur_apply: image size %d unsupported (need S%%4==0, S<=128)", S);
  const size_t smem = blur_smem(S, 2);
  static size_t attr = 0;
  if (smem > attr) { CD_CUDA(cudaFuncSetAttribute(blur_apply_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); attr = smem; }
  dim3 grid(C, B);
  blur_apply_kernel<<<grid, 256, smem, static_cast<cudaStream_t>(stream)>>>(x, out, ops, reinterpret_cast<const long long*>(t),
                                                                          t_scalar, S, T, collapse_last, quantize);
  CD_LAUNCH_CHECK();
  return 0;
}

extern "C" int cd_blur_step_down(const float* xt, const float* xhat, float* out, const float* ops,
                                 int t_hi, int t_lo, int B, int C, int S, int T, int collapse_last, void* stream) {
  CD_REQUIRE(S % 4 == 0 && S >= 4 && S <= 128, "cd_blur_step_down: image size %d unsupported", S);
  const size_t smem = blur_smem(S, 2);
  static size_t attr = 0;
  if (smem > attr) { CD_CUDA(cudaFuncSetAttribute(blur_step_down_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); attr = smem; }
  dim3 grid(C, B);
  blur_step_down_kernel<<<grid, 256, smem, static_cast<cudaStream_t>(stream)>>>(xt, xhat, out, ops, t_hi, t_lo, S, T, collapse_last);
  CD_LAUNCH_CHECK();
  return 0;
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

extern "C" int cd_fade_step(const float* img, const float* x1_bar, const float* x2, int t, const float* alphas,
                            const float* one_minus_alphas, int B, int C, int HW, float* out, void* stream) {
  CD_REQUIRE(t >= 1 && x2, "cd_fade_step: bad arguments");
  const long long n = static_cast<long long>(B) * C * HW;
  int blocks = cd_cdiv(n, 256 * 4); if (blocks > cd_num_sms() * 8) blocks = cd_num_sms() * 8; if (blocks < 1) blocks = 1;
  fade_step_kernel<<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(img, x1_bar, x2, t, alphas, one_minus_alphas, HW, n, out);
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
__global__ void mask_apply_kernel(const float* __restrict__ x, float* __restrict__ out, const float* __restrict__ masks,
                                  const long long* __restrict__ t, int t_scalar, const long long* __restrict__ rx,
                                  const long long* __restrict__ ry, int B, int C, int S, int MS, int quantize) {
  const long long n = static_cast<long long>(B) * C * S * S;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int xx = static_cast<int>(i % S), yy = static_cast<int>((i / S) % S);
    const int b = static_cast<int>(i / (static_cast<long long>(S) * S * C));
    const int idx = t ? static_cast<int>(t[b]) : t_scalar;
    const int oy = rx ? static_cast<int>(rx[b]) : 0, ox = ry ? static_cast<int>(ry[b]) : 0;   // reference: rows <- rand_x, cols <- rand_y
    float v = x[i] * mask_at(masks, idx, MS, yy + oy, xx + ox);
    if (quantize) v = quantize8(v);
    out[i] = v;
  }
}
__global__ void mask_step_down_kernel(const float* __restrict__ xt, const float* __restrict__ xhat, float* __restrict__ out,
                                      const float* __restrict__ masks, int idx_hi, int idx_lo, const long long* __restrict__ rx,
                                      const long long* __restrict__ ry, int B, int C, int S, int MS) {
  const long long n = static_cast<long long>(B) * C * S * S;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int xx = static_cast<int>(i % S), yy = static_cast<int>((i / S) % S);
    const int b = static_cast<int>(i / (static_cast<long long>(S) * S * C));
    const int oy = rx ? static_cast<int>(rx[b]) : 0, ox = ry ? static_cast<int>(ry[b]) : 0;
    const float xv = xhat[i];
    const float hi = xv * mask_at(masks, idx_hi, MS, yy + oy, xx + ox);
    const float lo = xv * mask_at(masks, idx_lo, MS, yy + oy, xx + ox);
    out[i] = xt[i] - hi + lo;
  }
}
}  // namespace

extern "C" int cd_mask_apply(const float* x, float* out, const float* masks, const int64_t* t, int t_scalar,
                             const int64_t* rx, const int64_t* ry, int B, int C, int S, int MS, int quantize, void* stream) {
  const long long n = static_cast<long long>(B) * C * S * S;
  int blocks = cd_cdiv(n, 256 * 4); if (blocks > cd_num_sms() * 8) blocks = cd_num_sms() * 8; if (blocks < 1) blocks = 1;
  mask_apply_kernel<<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(x, out, masks, reinterpret_cast<const long long*>(t), t_scalar,
      reinterpret_cast<const long long*>(rx), reinterpret_cast<const long long*>(ry), B, C, S, MS, quantize);
  CD_LAUNCH_CHECK();
  return 0;
}

extern "C" int cd_mask_step_down(const float* xt, const float* xhat, float* out, const float* masks, int idx_hi, int idx_lo,
                                 const int64_t* rx, const int64_t* ry, int B, int C, int S, int MS, void* stream) {
  const long long n = static_cast<long long>(B) * C * S * S;
  int blocks = cd_cdiv(n, 256 * 4); if (blocks > cd_num_sms() * 8) blocks = cd_num_sms() * 8; if (blocks < 1) blocks = 1;
  mask_step_down_kernel<<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(xt, xhat, out, masks, idx_hi, idx_lo,
      reinterpret_cast<const long long*>(rx), reinterpret_cast<const long long*>(ry), B, C, S, MS);
  CD_LAUNCH_CHECK();
  return 0;
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
__global__ void chanmix_kernel(const float* __restrict__ xt, const float* __restrict__ xsrc, float* __restrict__ out,
                               const float* __restrict__ mats, const long long* __restrict__ t_hi, const long long* __restrict__ t_lo,
                               int hi_off, int lo_off, int B, int C, long long HW, int mode) {
  // mode 0: out = M[t_hi+hi_off] xsrc ; mode 1: out = xt - M[t_hi+hi_off] xsrc + M[t_lo+lo_off] xsrc   (index < 0 = identity)
  const long long n = static_cast<long long>(B) * HW;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int b = static_cast<int>(i / HW);
    const long long p = i % HW;
    const int ih = static_cast<int>(t_hi[b]) + hi_off;
    const int il = mode ? static_cast<int>(t_lo[b]) + lo_off : -1;
    float v[8];
    for (int c = 0; c < C; ++c) v[c] = xsrc[(static_cast<long long>(b) * C + c) * HW + p];
    for (int co = 0; co < C; ++co) {
      float hi = v[co], lo = v[co];
      if (ih >= 0) { hi = 0.f; for (int c = 0; c < C; ++c) hi = fmaf(mats[(ih * C + co) * C + c], v[c], hi); }
      if (il >= 0) { lo = 0.f; for (int c = 0; c < C; ++c) lo = fmaf(mats[(il * C + co) * C + c], v[c], lo); }
      const long long o = (static_cast<long long>(b) * C + co) * HW + p;
      out[o] = mode ? xt[o] - hi + lo : hi;
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

extern "C" int cd_chanmix(const float* xt, const float* xsrc, float* out, const float* mats, const int64_t* t_hi,
                          const int64_t* t_lo, int hi_off, int lo_off, int B, int C, int64_t HW, int mode, void* stream) {
  CD_REQUIRE(C <= 8 && t_hi && (mode == 0 || (xt && t_lo)), "cd_chanmix: bad arguments");
  const long long n = static_cast<long long>(B) * HW;
  int blocks = cd_cdiv(n, 256 * 2); if (blocks > cd_num_sms() * 8) blocks = cd_num_sms() * 8; if (blocks < 1) blocks = 1;
  chanmix_kernel<<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(xt, xsrc, out, mats, reinterpret_cast<const long long*>(t_hi),
      reinterpret_cast<const long long*>(t_lo), hi_off, lo_off, B, C, HW, mode);
  CD_LAUNCH_CHECK();
  return 0;
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
