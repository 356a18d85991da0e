// LinearAttention backward, per-pixel part (see backward.cu for the formulas and the CUDA-core version it replaces):
//
//   P[n][d]  = exp(k[n][d] - kmax[d]) / ksum[d]
//   dv[n][e] = sum_d P[n][d] * dc[d][e]                         (dc = dctxn[b][h], 32 x 32 per head)
//   dk[n][d] = P[n][d] * (sum_e v[n][e] * dc[d][e] - rowdot[d])
//
// Two [pixels x 32] x [32 x 32] products per head: on the CUDA cores they cost 4 shared-memory wavefronts per 32 FMAs and run far
// below the HBM rate.  Here a warp owns 16 pixels of one head
// and issues them as warp-level mma.sync.m16n8k8 TF32 in the 3xTF32 split (both operands hi + lo, three MMAs: fp32-grade
// products -- the fp32 path of the engine keeps its 2e-6 gradient parity), accumulators in fp32.  k / v tiles of 32 pixels are double-buffered through shared memory with 16-byte
// LDGSTS; dv and dk leave as 8-byte stores that fill whole 32-byte sectors.  No atomics: deterministic.
#include "cd_common.cuh"

namespace {

constexpr int kP = 32;              // pixels per staged tile
constexpr int kLd = 132;            // padded tile row in floats: bank = 4 * pixel + channel -> conflict-free fragments
constexpr int kLc = 40;             // padded row of the staged 32 x 32 dc matrices: bank = 8 * row + col

__device__ __forceinline__ void cd_mma_m16n8k8_tf32(float* d, const float* a, const float* b) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(__float_as_uint(a[0])), "r"(__float_as_uint(a[1])), "r"(__float_as_uint(a[2])), "r"(__float_as_uint(a[3])),
                 "r"(__float_as_uint(b[0])), "r"(__float_as_uint(b[1])));
}

__global__ void __launch_bounds__(256)
attn_bwd_kv_mma_kernel(const float* __restrict__ qkv, int ld, int n, int ppb, const float* __restrict__ kmax,
                       const float* __restrict__ ksum, const float* __restrict__ dctxn, const float* __restrict__ rowdot,
                       float* __restrict__ dqkv, int dld) {
  extern __shared__ __align__(16) float sm[];
  float* dcs = sm;                              // [4][32][kLc]  dc[h][d][e] (fp32; split hi + lo at use)
  float* dct = dcs + 4 * 32 * kLc;              // [4][32][kLc]  dc[h][e][d] (transposed)
  float* kmx = dct + 4 * 32 * kLc;              // [128]
  float* kin = kmx + 128;                       // [128] 1 / ksum
  float* rdt = kin + 128;                       // [128] rowdot
  float* tiles = rdt + 128;                     // [2 stages][k | v][kP][kLd]
  const int b = blockIdx.y;
  const int p0 = blockIdx.x * ppb;
  int p1 = p0 + ppb; if (p1 > n) p1 = n;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const int h = warp & 3, r0 = (warp >> 2) * 16;          // this warp: head h, tile rows r0 .. r0 + 15
  const float* base = qkv + static_cast<long long>(b) * n * ld + 128;   // k at +0..127, v at +128..255 of every pixel row

  for (int i = tid; i < 4096; i += 256) {
    const float v = dctxn[static_cast<long long>(b) * 4096 + i];
    const int hh = i >> 10, d = (i >> 5) & 31, e = i & 31;
    dcs[(hh * 32 + d) * kLc + e] = v;
    dct[(hh * 32 + e) * kLc + d] = v;
  }
  if (tid < 128) {
    kmx[tid] = kmax[b * 128 + tid];
    kin[tid] = 1.f / ksum[b * 128 + tid];
    rdt[tid] = rowdot[b * 128 + tid];
  }

  auto issue = [&](int q0, int s) {
    float* kd = tiles + s * 2 * kP * kLd;
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

  int stage = 0;
  issue(p0, 0);
  for (int q0 = p0; q0 < p1; q0 += kP) {
    if (q0 + kP < p1) {
      issue(q0 + kP, stage ^ 1);
      asm volatile("cp.async.wait_group 1;" ::: "memory");
    } else {
      asm volatile("cp.async.wait_group 0;" ::: "memory");
    }
    __syncthreads();                                   // tile (and, the first time, dc / kmax / ksum / rowdot) staged
    const float* kd = tiles + stage * 2 * kP * kLd + r0 * kLd + h * 32;
    const float* vd = kd + kP * kLd;
    float dv[4][4], tt[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) { dv[i][j] = 0.f; tt[i][j] = 0.f; }
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      // A fragments (rows = pixels g / g + 8, columns = channels ks*8 + t / + 4) of P and of v, split hi + lo
      const int c0 = ks * 8 + t, c1 = c0 + 4;
      const float m0 = kmx[h * 32 + c0], m1 = kmx[h * 32 + c1], i0 = kin[h * 32 + c0], i1 = kin[h * 32 + c1];
      float pa[4], va[4], phi[4], plo[4], vhi[4], vlo[4];
      pa[0] = __expf(kd[g * kLd + c0] - m0) * i0;       pa[1] = __expf(kd[(g + 8) * kLd + c0] - m0) * i0;
      pa[2] = __expf(kd[g * kLd + c1] - m1) * i1;       pa[3] = __expf(kd[(g + 8) * kLd + c1] - m1) * i1;
      va[0] = vd[g * kLd + c0]; va[1] = vd[(g + 8) * kLd + c0]; va[2] = vd[g * kLd + c1]; va[3] = vd[(g + 8) * kLd + c1];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        phi[i] = cd_round_tf32(pa[i]); plo[i] = cd_round_tf32(pa[i] - phi[i]);
        vhi[i] = cd_round_tf32(va[i]); vlo[i] = cd_round_tf32(va[i] - vhi[i]);
      }
#pragma unroll
      for (int nt = 0; nt < 4; ++nt) {
        float b1[2], b2[2], b1h[2], b1l[2], b2h[2], b2l[2];
        b1[0] = dcs[(h * 32 + c0) * kLc + nt * 8 + g]; b1[1] = dcs[(h * 32 + c1) * kLc + nt * 8 + g];   // B[k = d][n = e] = dc[d][e]
        b2[0] = dct[(h * 32 + c0) * kLc + nt * 8 + g]; b2[1] = dct[(h * 32 + c1) * kLc + nt * 8 + g];   // B[k = e][n = d] = dc[d][e]
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          b1h[i] = cd_round_tf32(b1[i]); b1l[i] = cd_round_tf32(b1[i] - b1h[i]);
          b2h[i] = cd_round_tf32(b2[i]); b2l[i] = cd_round_tf32(b2[i] - b2h[i]);
        }
        cd_mma_m16n8k8_tf32(dv[nt], plo, b1h);       // 3xTF32: lo*hi + hi*lo + hi*hi = fp32-grade products
        cd_mma_m16n8k8_tf32(dv[nt], phi, b1l);
        cd_mma_m16n8k8_tf32(dv[nt], phi, b1h);
        cd_mma_m16n8k8_tf32(tt[nt], vlo, b2h);
        cd_mma_m16n8k8_tf32(tt[nt], vhi, b2l);
        cd_mma_m16n8k8_tf32(tt[nt], vhi, b2h);
      }
    }
    // accumulator layout: rows g / g + 8, columns nt*8 + 2t, + 1
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      const int row = r0 + g + half * 8;
      const int p = q0 + row;
      if (p < p1) {
        float* orow = dqkv + (static_cast<long long>(b) * n + p) * dld;
        const float* krow = tiles + stage * 2 * kP * kLd + row * kLd + h * 32;
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) {
          const int c = nt * 8 + 2 * t;
          const float2 kk = *reinterpret_cast<const float2*>(krow + c);
          const float pk0 = __expf(kk.x - kmx[h * 32 + c]) * kin[h * 32 + c];
          const float pk1 = __expf(kk.y - kmx[h * 32 + c + 1]) * kin[h * 32 + c + 1];
          float2 dk2, dv2;
          dk2.x = pk0 * (tt[nt][half * 2] - rdt[h * 32 + c]);
          dk2.y = pk1 * (tt[nt][half * 2 + 1] - rdt[h * 32 + c + 1]);
          dv2.x = dv[nt][half * 2]; dv2.y = dv[nt][half * 2 + 1];
          *reinterpret_cast<float2*>(orow + 128 + h * 32 + c) = dk2;
          *reinterpret_cast<float2*>(orow + 256 + h * 32 + c) = dv2;
        }
      }
    }
    __syncthreads();                                   // tile fully read before the next prefetch overwrites it
    stage ^= 1;
  }
}

}  // namespace

// returns 1 when the caller should use the CUDA-core kernel (ld % 4 != 0 or unaligned operands)
int cd_linattn_bwd_kv_mma(const float* qkv, int ld, int B, int n, const float* kmax, const float* ksum, const float* dctxn,
                          const float* rowdot, float* dqkv, int dld, cudaStream_t st) {
  if (ld % 4 != 0 || dld % 2 != 0 || (reinterpret_cast<uintptr_t>(qkv) & 15) != 0 || (reinterpret_cast<uintptr_t>(dqkv) & 7) != 0)
    return 1;
  const size_t smem = sizeof(float) * (2 * 4 * 32 * kLc + 3 * 128 + 2 * 2 * kP * kLd);
  static bool attr = false;
  if (!attr) { CD_CUDA(cudaFuncSetAttribute(attn_bwd_kv_mma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); attr = true; }
  // spans of ppb pixels (a multiple of 32): about one wave of resident blocks (2 per SM) over the batch; the 42 KB of per-image
  // operands are staged once per block, so spans are not made shorter than 4 tiles
  int per_img = 2 * cd_num_sms() / B; if (per_img < 1) per_img = 1;
  int ppb = cd_cdiv(cd_cdiv(n, per_img), kP) * kP;
  if (ppb < 4 * kP) ppb = 4 * kP;
  attn_bwd_kv_mma_kernel<<<dim3(cd_cdiv(n, ppb), B), 256, smem, st>>>(qkv, ld, n, ppb, kmax, ksum, dctxn, rowdot, dqkv, dld);
  CD_LAUNCH_CHECK();
  return 0;
}
