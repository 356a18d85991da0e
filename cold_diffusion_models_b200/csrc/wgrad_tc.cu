// Tensor-core weight gradient of the tap-list convolution (replaces cuDNN wgrad behind loss.backward() for the
// dense convolutions of the reference Unet, DB:149-154,173-174,105-109):
//
//   dW[tap][co][ci] += sum_{pixels p} dY[p][co] * X[p (+) tap][ci]
//
// as a GEMM whose K dimension is the PIXEL axis.  NHWC rows hold the channels contiguously, i.e. both operands are
// MN-major, which TF32 wgmma cannot read from shared memory.  Two kernels:
//  - wgrad_wgmma_kernel (every weight gradient of the Unet: 3x3, 1x1, the per-batch attention product, the 4x4 stride-2
//    downsample by input-parity class, the transposed-convolution parity problems and the Cin = 32 image edge) feeds wgmma with X
//    from registers and with dY transposed once per pixel chunk into a K-major tile (see its comment below);
//  - wgrad_tc_kernel, for the opt-in bias fusion, the forced modes 0 / 8 and problems the wgmma kernel does not take, below.
// wgrad_tc_kernel runs mma.sync.m16n8k8 (TF32, fp32 accumulate) with its fragments read from the swizzled TMA tiles.
// dY tiles ({32 co, CW px, R rows} TMA boxes) and
// X tiles land in SWIZZLE_128B shared memory.  One CTA owns (co tile, ci tile, tap group, pixel split) and keeps one
// register accumulator per tap of its group; with `halo` mode the dx = -1/0/+1 taps of a 3x3 kernel share ONE X tile
// that carries a one-pixel halo and are addressed by shifting the pixel row.  Partial sums of the pixel splits are
// combined with vector red.global.add.f32.
#include "tc_common.cuh"

namespace {

constexpr int kMmaWarps = 8;                      // 4 (co) x 2 (ci) warps, 32 co x BN/2 ci each
constexpr int kThreads = 32 * (kMmaWarps + 1);    // + warp 8: TMA producer
constexpr int kMaxTaps = 8;      // taps (accumulators) per CTA (mma.sync kernel: at most 4)
constexpr int kMaxGroups = 4;
constexpr int kMaxAccCols = 256; // taps x BN: register accumulators of one CTA (128 co rows)

struct WgParams {
  int B, Hg, Wg;
  int CW, R, KR;                  // pixel chunk: CW x R = KR K-rows of A per stage
  int chunks_x, chunks_y, total_chunks, chunks_per_split, splits;
  int Cout, Cin;
  int tiles_co, tiles_ci;
  int ngroups;
  int ntaps[kMaxGroups];
  int nloads[kMaxGroups];
  int tap_index[kMaxGroups][kMaxTaps];
  int tap_load[kMaxGroups][kMaxTaps];
  int tap_shift[kMaxGroups][kMaxTaps];    // pixel-row shift inside the (halo) X tile; wgmma kernel: (dy + 1) * (CW + 8) + dx + 1
  int load_dy[kMaxGroups][kMaxTaps], load_dx[kMaxGroups][kMaxTaps];
  int halo;                       // extra pixels per row in the X box (0 or 2)
  int sy, sx;                     // X coordinate = g*s + d
  int oys, oxs, oy0, ox0;         // dY coordinate = g*os + o0
  int per_batch, chunks_per_img, splits_per_img;   // per-batch weights: splits never cross images
  long long dw_batch_stride;
  float* dw;
  float* db;                      // BIAS kernels only: db[co] += sum over all pixels of dY (nullptr: not fused)
  // wgmma kernel: a CTA covers ci_tile input channels from ci0; group g loads wm_nbox[g] X boxes of 32 channels (ci0 + 32 j) per chunk; accumulator slot t of the
  // group is an m64 tile whose half h (warps 2h, 2h + 1: 32 rows) reads box wm_box[g][t][h] at pixel-row offset wm_shift[g][t][h]
  // and belongs to tap wm_tap[g][t][h] (-1: idle half)
  int wm_nbox[kMaxGroups], ci_tile;
  int wm_box[kMaxGroups][kMaxTaps][2], wm_shift[kMaxGroups][kMaxTaps][2], wm_tap[kMaxGroups][kMaxTaps][2];
};

// element (row, c) of a 32-channel SWIZZLE_128B tile whose base is 1024-byte aligned: 16-byte chunk index XOR row % 8
__device__ __forceinline__ float lds_sw(const uint8_t* base, int row, int c) {
  return cd_round_tf32(*reinterpret_cast<const float*>(base + row * 128 + ((((c >> 2) ^ row) & 7) << 4) + (c & 3) * 4));
}
__device__ __forceinline__ void mma_tf32_16x8x8(float (&d)[4], const float (&a)[4], const float (&b)[2]) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(__float_as_uint(a[0])), "r"(__float_as_uint(a[1])), "r"(__float_as_uint(a[2])), "r"(__float_as_uint(a[3])),
                 "r"(__float_as_uint(b[0])), "r"(__float_as_uint(b[1])));
}
__device__ __forceinline__ void red_add_v2(float* addr, float a, float b) {
  asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" :: "l"(addr), "f"(a), "f"(b) : "memory");
}

// BIAS = true (opt-in, cd_wgrad_tc_set_bias_fusion): the CTAs of the first ci tile and first tap group also accumulate the bias
// gradient db[co] = sum_pixels dY[p][co] from the dY fragments they load anyway, replacing the separate column-sum pass over dY.
template <int BN, int NT, bool BIAS>
__global__ void __launch_bounds__(kThreads, 1)
wgrad_tc_kernel(const __grid_constant__ CUtensorMap mapDY, const __grid_constant__ CUtensorMap mapX,
                const WgParams p, int stages, int a_bytes, int b_bytes, int b_tx_bytes) {
  constexpr int NCH = BN / 32;                    // ci chunks of the B operand
  constexpr int NJ = BN / 16;                     // 8-wide n tiles per warp
  static_assert(NT * BN <= kMaxAccCols, "accumulators of one CTA");
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + ((1024u - (raw_addr & 1023u)) & 1023u);
  const int g = blockIdx.z;
  const int nl = p.nloads[g];
  const int stage_bytes = a_bytes + nl * b_bytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + stages * stage_bytes);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + stages;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int i = 0; i < stages; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], kMmaWarps); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  const int tile = blockIdx.x;
  const int co0 = (tile % p.tiles_co) * 128, ci0 = (tile / p.tiles_co) * BN;
  const int split = blockIdx.y;
  int c_beg = split * p.chunks_per_split;
  int c_end = c_beg + p.chunks_per_split; if (c_end > p.total_chunks) c_end = p.total_chunks;
  long long dw_off = 0;
  if (p.per_batch) {
    const int n = split / p.splits_per_img, sp = split % p.splits_per_img;
    c_beg = n * p.chunks_per_img + sp * p.chunks_per_split;
    c_end = c_beg + p.chunks_per_split;
    if (c_end > (n + 1) * p.chunks_per_img) c_end = (n + 1) * p.chunks_per_img;
    dw_off = n * p.dw_batch_stride;
  }
  const int nchunks = c_end > c_beg ? c_end - c_beg : 0;

  if (warp == kMmaWarps) {
    // TMA producer: the whole warp walks the chunks and waits on the barriers, one elected lane issues
    for (int it = 0; it < nchunks; ++it) {
      const int c = c_beg + it;
      const int cx = c % p.chunks_x;
      const int cy = (c / p.chunks_x) % p.chunks_y;
      const int n = c / (p.chunks_x * p.chunks_y);
      const int gx0 = cx * p.CW, gy0 = cy * p.R;
      const uint32_t stage = it % stages, ph = (it / stages) & 1u;
      mbar_wait(&empty_bar[stage], ph ^ 1u);
      if (elect_one()) {
        mbar_expect_tx(&full_bar[stage], a_bytes + nl * b_tx_bytes);
        const uint32_t sa = smem_u32(smem + stage * stage_bytes);
#pragma unroll
        for (int ch = 0; ch < 4; ++ch)              // dY: 4 chunks of 32 out-channels
          tma_load_4d(sa + ch * (a_bytes / 4), &mapDY, &full_bar[stage], co0 + ch * 32, gx0 * p.oxs + p.ox0, gy0 * p.oys + p.oy0, n);
        for (int l = 0; l < nl; ++l) {
          const uint32_t sb = sa + a_bytes + l * b_bytes;
          const int xin = gx0 * p.sx + p.load_dx[g][l], yin = gy0 * p.sy + p.load_dy[g][l];
          for (int ch = 0; ch < NCH; ++ch)
            tma_load_4d(sb + ch * (b_bytes / NCH), &mapX, &full_bar[stage], ci0 + ch * 32, xin, yin, n);
        }
      }
      __syncwarp();
    }
    return;
  }

  // ---- MMA warps: warp (wm, wn) owns co rows [32 wm, 32 wm + 32) and ci columns [BN/2 wn, BN/2 wn + BN/2) of every tap
  const int wm = warp & 3, wn = warp >> 2;
  const int gq = lane >> 2, tq = lane & 3;
  const bool bias_cta = BIAS && p.db != nullptr && (tile / p.tiles_co) == 0 && g == 0 && wn == 0;
  int tap_load[NT], tap_shift[NT];
#pragma unroll
  for (int t = 0; t < NT; ++t) { tap_load[t] = p.tap_load[g][t]; tap_shift[t] = p.tap_shift[g][t]; }
  float acc[NT][2][NJ][4];
#pragma unroll
  for (int t = 0; t < NT; ++t)
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int j = 0; j < NJ; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) acc[t][i][j][e] = 0.f;
  float bsum[2][2] = {{0.f, 0.f}, {0.f, 0.f}};
  const int ksteps = p.KR / 8, cw_shift = __ffs(p.CW) - 1, rowlen = p.CW + p.halo;
  for (int it = 0; it < nchunks; ++it) {
    const uint32_t stage = it % stages, ph = (it / stages) & 1u;
    mbar_wait(&full_bar[stage], ph);
    const uint8_t* sA = smem + stage * stage_bytes + wm * (a_bytes / 4);      // this warp's 32 out-channels
    const uint8_t* sB = smem + stage * stage_bytes + a_bytes;
#pragma unroll 1
    for (int ks = 0; ks < ksteps; ++ks) {
      const int k0 = ks * 8 + tq, k1 = k0 + 4;          // pixels of this lane's A columns / B rows
      float a[2][4];
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        a[i][0] = lds_sw(sA, k0, i * 16 + gq);
        a[i][1] = lds_sw(sA, k0, i * 16 + gq + 8);
        a[i][2] = lds_sw(sA, k1, i * 16 + gq);
        a[i][3] = lds_sw(sA, k1, i * 16 + gq + 8);
        if (bias_cta) { bsum[i][0] += a[i][0] + a[i][2]; bsum[i][1] += a[i][1] + a[i][3]; }
      }
      const int r0 = (k0 >> cw_shift) * rowlen + (k0 & (p.CW - 1)), r1 = (k1 >> cw_shift) * rowlen + (k1 & (p.CW - 1));
#pragma unroll
      for (int t = 0; t < NT; ++t) {
        const uint8_t* sBt = sB + tap_load[t] * b_bytes;
#pragma unroll
        for (int j = 0; j < NJ; ++j) {
          const int cl = wn * (BN / 2) + j * 8 + gq;      // ci column (n) of this lane's B elements
          const uint8_t* sBc = sBt + (cl >> 5) * (b_bytes / NCH);
          const float b[2] = {lds_sw(sBc, r0 + tap_shift[t], cl & 31), lds_sw(sBc, r1 + tap_shift[t], cl & 31)};
          mma_tf32_16x8x8(acc[t][0][j], a[0], b);
          mma_tf32_16x8x8(acc[t][1][j], a[1], b);
        }
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty_bar[stage]);
  }
  if (nchunks == 0) return;
#pragma unroll
  for (int t = 0; t < NT; ++t) {
    if (t >= p.ntaps[g]) break;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int co = co0 + wm * 32 + i * 16 + gq + h * 8;
        if (co >= p.Cout) continue;
        float* wrow = p.dw + dw_off + (static_cast<long long>(p.tap_index[g][t]) * p.Cout + co) * p.Cin;
#pragma unroll
        for (int j = 0; j < NJ; ++j) {
          const int ci = ci0 + wn * (BN / 2) + j * 8 + tq * 2;
          if (ci < p.Cin) red_add_v2(wrow + ci, acc[t][i][j][2 * h], acc[t][i][j][2 * h + 1]);
        }
      }
    }
  }
  if (BIAS && bias_cta) {
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float v = bsum[i][h];
        v += __shfl_xor_sync(0xffffffffu, v, 1);
        v += __shfl_xor_sync(0xffffffffu, v, 2);
        const int co = co0 + wm * 32 + i * 16 + gq + h * 8;
        if (tq == 0 && co < p.Cout) atomicAdd(p.db + co, v);
      }
  }
}

// ---------------------------------------------------------------------------------------------
// wgmma kernel for stride-1 problems whose taps lie in [-1, 1]^2, Cin % 64 == 0 or Cin == 32, Cout % 64 == 0 (see wgrad_wgmma for
// how strided and parity problems are mapped onto it):
//
//   dW[tap][co][ci] += sum_q X[q + tap][ci] * dY[q][co]     M = 64 ci (A = X, registers), N = BN co (B = dY^T, shared memory)
//
// K runs over chunks of 64 pixels (CW x R) of one image.  Per chunk:
//  - the producer warp TMA-loads one X box {32 ci, CW + 8, R + 2, 1} at (x0 - 1, y0 - 1) per 32 input channels -- the halo of
//    every tap; a box row is CW + 8 pixels long so that a shift by whole rows keeps the 128-byte swizzle phase -- and the dY
//    boxes {32 co, CW, R, 1} (pixel-major, SWIZZLE_128B);
//  - the transposer warpgroup rewrites dY as a K-major SWIZZLE_128B tile (rows = co, 128 bytes = 32 pixels), rounded RN to TF32,
//    and hands it to the consumers through the async proxy;
//  - the consumer warpgroups split the accumulator slots of the CTA's group (ceil(n / 2) and the rest): a slot reads its A
//    fragment from an X box at a row offset (a register load is a free transpose), rounds it RN to TF32 and issues wgmma m64nBNk8
//    against the shared transposed dY tile.  A-fragment registers are double-buffered across k-steps (wgmma_wait<1>).
//    A slot is one tap of 64 ci (3x3, halves from the two 32-ci boxes), one 64-ci block of a 1x1 (up to wm_slots_1x1 blocks per
//    CTA, no halo: box {32 ci, CW, R}) or, at Cin = 32, two taps (one per 32-row half; the last half of an odd tap count idles).
// Inside each k8 step the eight pixels are ordered 0 2 4 6 1 3 5 7 in A and B alike: the four lanes of a quad then read pixel
// rows of four different swizzle phases, and the A loads are free of bank conflicts.
// Partial sums of the pixel splits are combined with red.global.add into the packed [tap][Cout][Cin] gradient.
// Warp roles (512 threads): warpgroup 0 = TMA producer (warp 0), warpgroup 1 = transposer, warpgroups 2-3 = consumers;
// setmaxnreg moves the registers of the first two to the consumers (ptxas, sm_90a: no spills and no serialized wgmma in any
// instantiation).
// CTA tile 64 ci x 128 co with two taps per consumer warpgroup (taps on grid z as {4, 4, 1}); Cout = 64: 64 ci x 64 co with four
// taps per warpgroup ({8, 1}).  3x3 shapes measured with tools/wgrad_shapes.py on an H100 80GB HBM3 at a 700 W power limit (1980 MHz, Unet
// config 3, batch 32): 160-220 TFLOP/s on the 3x3 shapes (133 at Cout = 64) against 46-91 for the mma.sync halo kernel; the 3x3
// weight gradients of one backward take 10.0 ms instead of 24.6 ms.
// ---------------------------------------------------------------------------------------------
constexpr int kWmThreads = 512;
constexpr int kWmKR = 64;                      // pixels per chunk
constexpr int kWmRegsLow = 40, kWmRegsHigh = 216;   // 128 x (40 + 40) + 256 x 216 <= 64 K registers

// HALO: the X box carries the halo of taps in [-1, 1]^2 ({32, CW + 8, R + 2}); otherwise (one tap at (0, 0)) it is the chunk itself
template <int CW, bool HALO> struct WmGeom {
  static constexpr int R = kWmKR / CW, RL = HALO ? CW + 8 : CW;
  static constexpr int kXBox = RL * (R + (HALO ? 2 : 0)) * 128;   // one 32-ci X box
  static_assert(kXBox % 1024 == 0, "X boxes keep 1024-byte alignment");
};
template <int BN> struct WmTiles {
  static constexpr int kRawBox = kWmKR * 128;              // one 32-co dY box as the TMA unit writes it
  static constexpr int kRawBytes = (BN / 32) * kRawBox;
  static constexpr int kBBytes = BN * kWmKR * 4;           // transposed dY: kWmKR / 32 atoms of BN rows x 128 bytes
};
// 1x1: up to this many 64-ci slots per CTA share one transposed dY tile (as many as keep two stages in shared memory)
constexpr int wm_slots_1x1(int BN) { return BN == 128 ? 3 : 4; }
// one pipeline stage: [raw dY boxes | transposed dY | X boxes]; a 3x3 CTA loads two halo boxes (64 ci; one at Cin = 32), a 1x1
// CTA up to 2 wm_slots_1x1 chunk boxes
template <int BN, int CW, bool HALO> struct WmStage {
  static constexpr int kXBytes = (HALO ? 2 : 2 * wm_slots_1x1(BN)) * WmGeom<CW, HALO>::kXBox;
  static constexpr int kBytes = WmTiles<BN>::kRawBytes + WmTiles<BN>::kBBytes + kXBytes;
  static_assert((224 * 1024) / kBytes >= 2, "two stages of the wgmma weight-gradient kernel fit shared memory");
};

template <int BN, int NTW, int CW, bool HALO>
__device__ __forceinline__ void wm_consume(const WgParams& p, const uint8_t* smem, int stages, int stage_bytes,
                                           uint64_t* afull, uint64_t* aempty, uint64_t* bfull, uint64_t* bempty, int nchunks, int g,
                                           int tbeg, int co0, int ci0) {
  using G = WmGeom<CW, HALO>;
  using T = WmTiles<BN>;
  const int lane = threadIdx.x & 31, w = (threadIdx.x & 127) >> 5, gq = lane >> 2, tq = lane & 3;
  // byte offsets inside a stage's X boxes of this thread's A elements: a[0] / a[1] = pixel 2 tq, ci c / c + 8; a[2] / a[3] =
  // pixel 2 tq + 1 (the k-step's first pixel row in box wm_box at row offset wm_shift)
  int off[NTW][2];
  const int c = 16 * (w & 1) + gq;
#pragma unroll
  for (int t = 0; t < NTW; ++t) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      // the box of half w >> 1 follows from the slot layout (see wm_plan): 3x3 boxes 0 / 1, 1x1 boxes 2 t / 2 t + 1, Cin = 32 box 0
      // with a shift per half; reading wm_box / wm_shift per half here costs the four-slot consumer registers it does not have (wm_plan keeps Cin = 32 to two slots per consumer)
      const int row = ((NTW <= 2 && p.Cin == 32) ? p.wm_shift[g][tbeg + t][w >> 1] : p.wm_shift[g][tbeg + t][0]) + 2 * tq + h;
      const int box = (NTW <= 2 && p.Cin == 32) ? 0 : (HALO ? 0 : 2 * (tbeg + t)) + (w >> 1);
      off[t][h] = box * G::kXBox + row * 128 + ((((c >> 2) ^ row) & 7) << 4) + (c & 3) * 4;
    }
  }
  float acc[NTW][BN / 2];
  uint32_t fr[2][NTW][4];
  // A fragments of k-step ks of the X tile at xs, rounded RN to TF32 (the first pixel of a k-step lies a multiple of 8 rows in)
  auto load_frags = [&](uint32_t (&f)[NTW][4], const uint8_t* xs, int ks) {
    const int kofs = (((ks * 8) / CW) * G::RL + (ks * 8) % CW) * 128;
#pragma unroll
    for (int t = 0; t < NTW; ++t)
#pragma unroll
      for (int e = 0; e < 4; ++e)        // ci + 8 (odd e): 16-byte chunk index + 2, as c >> 2 has bit 1 clear
        f[t][e] = __float_as_uint(cd_round_tf32(*reinterpret_cast<const float*>(xs + (off[t][e >> 1] ^ ((e & 1) * 32)) + kofs)));
  };
  if (nchunks == 0) return;
  mbar_wait(&afull[0], 0);
  load_frags(fr[0], smem + T::kRawBytes + T::kBBytes, 0);
  for (int it = 0; it < nchunks; ++it) {
    const uint32_t s = it % stages, ph = (it / stages) & 1u;
    mbar_wait(&bfull[s], ph);
    const uint8_t* xs = smem + s * stage_bytes + T::kRawBytes + T::kBBytes;
    const uint32_t bs = smem_u32(smem + s * stage_bytes + T::kRawBytes);
#pragma unroll
    for (int ks = 0; ks < kWmKR / 8; ++ks) {
      wgmma_fence();
      const uint64_t db = make_kmajor_sw128_desc(bs + (ks >> 2) * (BN * 128)) + uint64_t((ks & 3) * 2);
#pragma unroll
      for (int t = 0; t < NTW; ++t) wgmma_tf32_rs<BN>(acc[t], fr[ks & 1][t], db, (it | ks) != 0 ? 1u : 0u);
      wgmma_commit();
      // the next k-step's fragments load while these MMAs run (into the other buffer: the A registers of an MMA in flight
      // stay untouched); waiting for the MMAs before the next issue keeps ptxas from serializing the wgmmas
      if (ks + 1 < kWmKR / 8) {
        load_frags(fr[(ks + 1) & 1], xs, ks + 1);
      } else if (it + 1 < nchunks) {
        const uint32_t s1 = (it + 1) % stages, ph1 = ((it + 1) / stages) & 1u;
        mbar_wait(&afull[s1], ph1);
        load_frags(fr[0], smem + s1 * stage_bytes + T::kRawBytes + T::kBBytes, 0);
      }
      wgmma_wait<0>();
    }
    __syncwarp();                      // every MMA of the chunk has retired: its X boxes and transposed tile are free
    if (lane == 0) { mbar_arrive(&aempty[s]); mbar_arrive(&bempty[s]); }
  }
  // accumulator element (row, col) = (ci, co): rows 16 w + gq (+ 8), columns 8 j + 2 tq (+ 1); rows 32 h .. 32 h + 31 are the
  // 32 channels of box wm_box[..][h].  Per-batch weights: image n = split / splits_per_img writes its own slice.
  asm volatile("" ::: "memory");      // keeps the epilogue's parameter reads (and their registers) out of the main loop
  const long long dw_off = p.per_batch ? (blockIdx.y / p.splits_per_img) * p.dw_batch_stride : 0;
#pragma unroll
  for (int t = 0; t < NTW; ++t) {
    const int tap = p.wm_tap[g][tbeg + t][w >> 1];
    if (tap < 0) continue;
    float* wt = p.dw + dw_off + static_cast<long long>(tap) * p.Cout * p.Cin + ci0 + 32 * p.wm_box[g][tbeg + t][w >> 1] +
                16 * (w & 1) + gq;
#pragma unroll
    for (int j = 0; j < BN / 8; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int co = co0 + 8 * j + 2 * tq + (e & 1);
        if (co < p.Cout) atomicAdd(wt + static_cast<long long>(co) * p.Cin + (e >> 1) * 8, acc[t][4 * j + e]);
      }
  }
}

template <int BN, int NT, int CW, bool HALO>
__global__ void __launch_bounds__(kWmThreads, 1)
wgrad_wgmma_kernel(const __grid_constant__ CUtensorMap mapDY, const __grid_constant__ CUtensorMap mapX, const __grid_constant__ WgParams p,
                   int stages) {
  using G = WmGeom<CW, HALO>;
  using T = WmTiles<BN>;
  constexpr int kStage = WmStage<BN, CW, HALO>::kBytes;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + ((1024u - (raw_addr & 1023u)) & 1023u);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + stages * kStage);
  uint64_t* afull = bars;                       // X boxes landed (TMA)
  uint64_t* aempty = bars + stages;             // consumers done with the X boxes and the transposed tile
  uint64_t* rfull = bars + 2 * stages;          // dY boxes landed (TMA)
  uint64_t* rempty = bars + 3 * stages;         // transposer done with the dY boxes
  uint64_t* bfull = bars + 4 * stages;          // transposed tile written
  uint64_t* bempty = bars + 5 * stages;         // consumers done with the transposed tile
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = threadIdx.x >> 7;
  const int g = blockIdx.z, nt = p.ntaps[g];    // accumulator slots of the group: ceil(nt / 2) in consumer 0, the rest in 1
  const int ncons = nt > 1 ? 2 : 1;             // consumer warpgroups with slots
  if (threadIdx.x == 0) {
    for (int i = 0; i < stages; ++i) {
      mbar_init(&afull[i], 1); mbar_init(&aempty[i], 4 * ncons);
      mbar_init(&rfull[i], 1); mbar_init(&rempty[i], 4);
      mbar_init(&bfull[i], 4); mbar_init(&bempty[i], 4 * ncons);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  const int tile = blockIdx.x;
  const int co0 = (tile % p.tiles_co) * BN, ci0 = (tile / p.tiles_co) * p.ci_tile;
  int c_beg = blockIdx.y * p.chunks_per_split;
  int c_end = c_beg + p.chunks_per_split; if (c_end > p.total_chunks) c_end = p.total_chunks;
  if (p.per_batch) {                            // per-batch weights: splits never cross images
    const int n = blockIdx.y / p.splits_per_img, sp = blockIdx.y % p.splits_per_img;
    c_beg = n * p.chunks_per_img + sp * p.chunks_per_split;
    c_end = c_beg + p.chunks_per_split;
    if (c_end > (n + 1) * p.chunks_per_img) c_end = (n + 1) * p.chunks_per_img;
  }
  const int nchunks = c_end > c_beg ? c_end - c_beg : 0;

  if (wg == 0) {
    // ===================== TMA producer (warp 0; one elected lane issues) =====================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" :: "n"(kWmRegsLow));
    if (warp != 0) return;
    for (int it = 0; it < nchunks; ++it) {
      const int ch = c_beg + it;
      const int gx0 = (ch % p.chunks_x) * CW, gy0 = ((ch / p.chunks_x) % p.chunks_y) * G::R, n = ch / (p.chunks_x * p.chunks_y);
      const uint32_t s = it % stages, ph = (it / stages) & 1u;
      const uint32_t sx = smem_u32(smem + s * kStage);
      mbar_wait(&rempty[s], ph ^ 1u);
      if (elect_one()) {
        mbar_expect_tx(&rfull[s], T::kRawBytes);
#pragma unroll
        for (int b = 0; b < BN / 32; ++b)
          tma_load_4d(sx + b * T::kRawBox, &mapDY, &rfull[s], co0 + 32 * b, gx0, gy0, n);
      }
      __syncwarp();
      mbar_wait(&aempty[s], ph ^ 1u);
      if (elect_one()) {
        const int nb = p.wm_nbox[g], h = HALO ? 1 : 0;
        mbar_expect_tx(&afull[s], nb * G::kXBox);
        for (int b = 0; b < nb; ++b)
          tma_load_4d(sx + T::kRawBytes + T::kBBytes + b * G::kXBox, &mapX, &afull[s], ci0 + 32 * b, gx0 - h, gy0 - h, n);
      }
      __syncwarp();
    }
    return;
  }
  if (wg == 1) {
    // ===================== transposer: dY [pixel][32 co] boxes -> K-major [co][pixel] tile, RN-rounded to TF32 =====================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" :: "n"(kWmRegsLow));
    const int w4 = warp & 3;
    for (int it = 0; it < nchunks; ++it) {
      const uint32_t s = it % stages, ph = (it / stages) & 1u;
      mbar_wait(&rfull[s], ph);
      mbar_wait(&bempty[s], ph ^ 1u);
      const uint8_t* raw = smem + s * kStage;
      uint8_t* bt = smem + s * kStage + T::kRawBytes;
      // unit u = (co box b, K quad kq): lane = co; K positions 4 kq .. 4 kq + 3 hold pixels 8 (kq / 2) + (kq & 1) + 2 j
#pragma unroll 4
      for (int u = w4; u < (BN / 32) * (kWmKR / 4); u += 4) {
        const int b = u % (BN / 32), kq = u / (BN / 32);
        const int co = 32 * b + lane;
        const uint8_t* src = raw + b * T::kRawBox + (lane & 3) * 4;
        float v[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int px = 8 * (kq >> 1) + (kq & 1) + 2 * j;
          v[j] = cd_round_tf32(*reinterpret_cast<const float*>(src + px * 128 + ((((lane >> 2) ^ px) & 7) << 4)));
        }
        *reinterpret_cast<float4*>(bt + (kq >> 3) * (BN * 128) + co * 128 + (((kq ^ co) & 7) << 4)) = make_float4(v[0], v[1], v[2], v[3]);
      }
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");     // the consumers' wgmma reads through the async proxy
      __syncwarp();
      if (lane == 0) { mbar_arrive(&rempty[s]); mbar_arrive(&bfull[s]); }
    }
    return;
  }
  // ===================== consumers =====================
  const int half = (nt + 1) / 2;
  const int tbeg = (wg - 2) * half;
  const int ntw = wg == 2 ? half : nt - half;
  if (ntw <= 0) return;
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" :: "n"(kWmRegsHigh));
#define WM_CONSUME(n) wm_consume<BN, n, CW, HALO>(p, smem, stages, kStage, afull, aempty, bfull, bempty, nchunks, g, tbeg, co0, ci0)
  if constexpr (NT == 4 && HALO) {        // 1x1: at most two slots per consumer
    if (ntw == 4) WM_CONSUME(4);
    else if (ntw == 3) WM_CONSUME(3);
    else if (ntw == 2) WM_CONSUME(2);
    else WM_CONSUME(1);
  } else {
    if (ntw == 2) WM_CONSUME(2);
    else WM_CONSUME(1);
  }
#undef WM_CONSUME
}

int g_wg_mode = 1;      // 0: one X tile per tap (mma.sync); 8: mma.sync halo kernel; otherwise (default) the wgmma kernel where eligible

// largest dynamic shared memory a launch of either kernel requests: at most 224 KB of stages + 1024-byte alignment slack +
// barrier block
constexpr int kMaxSmem = 224 * 1024 + 1024 + 256;

template <int BN, int NT>
int launch_wg(bool bias, dim3 grid, size_t smem, cudaStream_t st, const CUtensorMap& mapDY, const CUtensorMap& mapX,
              const WgParams& p, int stages, int a_bytes, int b_bytes, int b_tx) {
  constexpr auto with_bias = wgrad_tc_kernel<BN, NT, true>, without = wgrad_tc_kernel<BN, NT, false>;
  CD_CUDA(bias ? smem_limit_once<with_bias>(kMaxSmem) : smem_limit_once<without>(kMaxSmem));
  auto kern = bias ? with_bias : without;
  kern<<<grid, kThreads, smem, st>>>(mapDY, mapX, p, stages, a_bytes, b_bytes, b_tx);
  CD_LAUNCH_CHECK();
  return 0;
}

}  // namespace

extern "C" int cd_wgrad_tc_set_mode(int mode) { g_wg_mode = mode; return 0; }

// opt-in: fold the bias gradient (column sums of dY) into the tensor-core weight gradient.  Off by default.
static int g_wg_bias_fusion = 0;
extern "C" int cd_wgrad_tc_set_bias_fusion(int enable) { g_wg_bias_fusion = enable; return 0; }

// K-split policy.  One CTA owns (Cout tile, Cin tile, tap group, pixel range); it runs alone on its SM (the stages fill the
// shared memory) and its red.add epilogue is not overlapped, so the launch costs waves x (chunks_per_split * t_chunk + t_over).
//   0: 2 waves rounded up (first version)   1 / 2: at most 1 / 2 full waves   3: minimise the modelled cost
static int g_split_policy = 3;
static int g_split_over_clk = 12000;     // fixed cost per CTA in SM clocks (prologue + first-load latency + red.add epilogue)
extern "C" int cd_wgrad_tc_set_split(int policy, int over_clk) { g_split_policy = policy; if (over_clk > 0) g_split_over_clk = over_clk; return 0; }

static int choose_splits(int tg, int total_chunks, int max_splits, double chunk_clk) {
  const int sms = cd_num_sms();
  if (max_splits < 1) max_splits = 1;
  int s;
  if (g_split_policy == 0) s = cd_cdiv(2 * sms, tg);
  else if (g_split_policy == 1) s = sms / tg;
  else if (g_split_policy == 2) s = 2 * sms / tg;
  else {
    double best = 1e30; s = 1;
    for (int c = 1; c <= max_splits && c * tg <= 4 * sms + tg; ++c) {
      const int cps = cd_cdiv(total_chunks, c);
      const int real = cd_cdiv(total_chunks, cps);
      const double cost = double(cd_cdiv(static_cast<long long>(tg) * real, sms)) * (cps * chunk_clk + g_split_over_clk);
      if (cost < best) { best = cost; s = c; }
    }
  }
  if (s > max_splits) s = max_splits;
  if (s < 1) s = 1;
  return s;
}

template <int BN, int NT, int CW, bool HALO>
static int launch_wm(dim3 grid, cudaStream_t st, const CUtensorMap& mapDY, const CUtensorMap& mapX, const WgParams& p) {
  constexpr int kStage = WmStage<BN, CW, HALO>::kBytes;
  int stages = (224 * 1024) / kStage; if (stages > 5) stages = 5;     // six barriers per stage in the 256-byte barrier block
  const size_t smem = size_t(stages) * kStage + 1024 + 256;
  constexpr auto kern = wgrad_wgmma_kernel<BN, NT, CW, HALO>;
  CD_CUDA(smem_limit_once<kern>(kMaxSmem));
  kern<<<grid, kWmThreads, smem, st>>>(mapDY, mapX, p, stages);
  CD_LAUNCH_CHECK();
  return 0;
}

// The stride-1 problem of one input-parity class: X pixel (ey + 2 (g + sy), ex + 2 (g + sx)) for the 4x4 stride-2 downsample,
// X pixel g + (sy, sx) otherwise.  Builds the accumulator slots and groups; returns 1 when they do not fit the kernel.
struct WmClass { int ey, ex, n, tap[16], sy[16], sx[16]; };

static int wm_plan(const CdConvDesc* d, const WmClass& k, int BN, int CW, WgParams& p, bool& halo) {
  const int Cin = d->s[0].C, NT = BN == 128 ? 2 : 4;
  halo = !(k.n == 1 && k.sy[0] == 0 && k.sx[0] == 0);
  p.tiles_co = d->Cout / BN;
  // slots: [half 0 | half 1] = (box, row shift, tap)
  int sb[16][2], ss[16][2], st[16][2], ns = 0, nbox = 2;
  auto shift = [&](int i) { return halo ? (k.sy[i] + 1) * (CW + 8) + k.sx[i] + 1 : 0; };
  if (Cin == 32) {              // image edge: one 32-ci box; the two halves of a slot take two taps
    if (halo && BN != 128) return 1;
    nbox = 1;
    for (int i = 0; i < k.n; i += 2, ++ns)
      for (int h = 0; h < 2; ++h) {
        const bool on = i + h < k.n;
        sb[ns][h] = 0; ss[ns][h] = on ? shift(i + h) : 0; st[ns][h] = on ? k.tap[i + h] : -1;
      }
  } else if (!halo) {
    // 1x1: the slots of a CTA are consecutive 64-ci blocks sharing one transposed dY tile: the most that divides Cin / 64
    ns = wm_slots_1x1(BN);
    while ((Cin / 64) % ns != 0) --ns;
    nbox = 2 * ns;
    for (int t = 0; t < ns; ++t)
      for (int h = 0; h < 2; ++h) { sb[t][h] = 2 * t + h; ss[t][h] = 0; st[t][h] = k.tap[0]; }
  } else {                      // one tap per slot, both halves from the two 32-ci boxes of the CTA's 64 ci
    for (int i = 0; i < k.n; ++i, ++ns)
      for (int h = 0; h < 2; ++h) { sb[ns][h] = h; ss[ns][h] = shift(i); st[ns][h] = k.tap[i]; }
  }
  p.ci_tile = Cin == 32 ? 32 : 32 * nbox;
  p.tiles_ci = Cin == 32 ? 1 : Cin / p.ci_tile;
  p.ngroups = cd_cdiv(ns, 2 * NT);           // tap groups on grid z (9 taps: {4, 4, 1} or {8, 1})
  if (p.ngroups > kMaxGroups) return 1;
  for (int g = 0; g < p.ngroups; ++g) {
    const int s0 = g * 2 * NT, n = ns - s0 < 2 * NT ? ns - s0 : 2 * NT;
    p.ntaps[g] = n;
    p.wm_nbox[g] = nbox;
    for (int t = 0; t < n; ++t)
      for (int h = 0; h < 2; ++h) { p.wm_box[g][t][h] = sb[s0 + t][h]; p.wm_shift[g][t][h] = ss[s0 + t][h]; p.wm_tap[g][t][h] = st[s0 + t][h]; }
  }
  return 0;
}

// wgmma kernel (see wgrad_wgmma_kernel); returns 1 when the problem is not eligible.  It takes stride-1 problems with taps in
// [-1, 1]^2 (3x3, 1x1, the four taps of a transposed-convolution parity class, whose dY is read at every second pixel) and the
// 4x4 stride-2 downsample, split into its four input-parity classes of four stride-1 taps each (one launch per class, X read at
// every second pixel).  Cin % 64 == 0 or Cin == 32 (image edge), Cout % 64 == 0, per-batch weights allowed.
static int wgrad_wgmma(const CdConvDesc* d, const float* dout, int dout_ld, float* dw, cudaStream_t st) {
  const CdConvSrc& c = d->s[0];
  if ((c.C % 64 != 0 && c.C != 32) || d->Cout % 64 != 0 || c.ntaps < 1) return 1;
  const bool dense_out = d->oys == 1 && d->oxs == 1 && d->oy0 == 0 && d->ox0 == 0 && d->Ho == d->Hg && d->Wo == d->Wg;
  const bool parity_out = d->oys == 2 && d->oxs == 2 && (d->oy0 & ~1) == 0 && (d->ox0 & ~1) == 0 && d->Ho == 2 * d->Hg &&
                          d->Wo == 2 * d->Wg;
  const bool s1 = d->sy == 1 && d->sx == 1 && c.H == d->Hg && c.W == d->Wg && (dense_out || parity_out);
  const bool s2 = d->sy == 2 && d->sx == 2 && c.H == 2 * d->Hg && c.W == 2 * d->Wg && dense_out;
  if (!s1 && !s2) return 1;
  const int CW = d->Wg >= 16 ? 16 : 8, R = kWmKR / CW;
  if (d->Hg < R) return 1;
  const int BN = d->Cout % 128 == 0 ? 128 : 64;
  WmClass cls[4];
  int ncls = 0;
  for (int e = 0; e < (s2 ? 4 : 1); ++e) {
    WmClass& k = cls[ncls];
    k.ey = e >> 1; k.ex = e & 1; k.n = 0;
    for (int t = 0; t < c.ntaps; ++t) {
      if (s2 && ((c.dy[t] & 1) != k.ey || (c.dx[t] & 1) != k.ex)) continue;
      const int sy = s2 ? (c.dy[t] - k.ey) / 2 : c.dy[t], sx = s2 ? (c.dx[t] - k.ex) / 2 : c.dx[t];
      if (sy < -1 || sy > 1 || sx < -1 || sx > 1) return 1;
      k.tap[k.n] = t; k.sy[k.n] = sy; k.sx[k.n] = sx; ++k.n;
    }
    if (k.n > 0) ++ncls;
  }
  // every class is checked before the first launch
  WgParams ps[4];
  bool halo[4];
  for (int i = 0; i < ncls; ++i) {
    ps[i] = WgParams{};
    if (wm_plan(d, cls[i], BN, CW, ps[i], halo[i])) return 1;
  }
  CUtensorMap mapDY;
  if (!encode_nhwc(&mapDY, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, dout, dout_ld, d->Cout, d->Wo, d->Ho, d->B, d->oxs, d->oys, d->ox0, d->oy0,
                   CW, R, 1, 1, 1, "wgmma dY"))
    return -1;
  for (int i = 0; i < ncls; ++i) {
    WgParams& p = ps[i];
    p.B = d->B; p.Hg = d->Hg; p.Wg = d->Wg; p.Cout = d->Cout; p.Cin = c.C;
    p.dw = dw;
    p.CW = CW; p.R = R; p.KR = kWmKR;
    p.chunks_x = d->Wg / CW; p.chunks_y = d->Hg / R;
    p.total_chunks = d->B * p.chunks_x * p.chunks_y;
    const int tiles = p.tiles_co * p.tiles_ci;
    // MMAs of one chunk: the group's slots x 8 k-steps of m64nBNk8, at the wgmma TF32 rate of 2048 FLOP/clk per SM shared by both
    // consumer warpgroups
    const double chunk_clk = double(p.ntaps[0]) * (kWmKR / 8) * (BN / 2);
    if (c.w_per_batch) {
      p.per_batch = 1;
      p.chunks_per_img = p.chunks_x * p.chunks_y;
      const int spi = choose_splits(tiles * p.ngroups * d->B, p.chunks_per_img, p.chunks_per_img, chunk_clk);
      p.chunks_per_split = cd_cdiv(p.chunks_per_img, spi);
      p.splits_per_img = cd_cdiv(p.chunks_per_img, p.chunks_per_split);
      p.splits = p.splits_per_img * d->B;
      p.dw_batch_stride = static_cast<long long>(c.ntaps) * d->Cout * c.C;
    } else {
      const int splits = choose_splits(tiles * p.ngroups, p.total_chunks, cd_cdiv(p.total_chunks, 8), chunk_clk);
      p.chunks_per_split = cd_cdiv(p.total_chunks, splits);
      p.splits = cd_cdiv(p.total_chunks, p.chunks_per_split);
    }
    CUtensorMap mapX;
    const int bw = halo[i] ? CW + 8 : CW, bh = halo[i] ? R + 2 : R;
    if (!encode_nhwc(&mapX, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, c.src, c.ld, c.C, c.W, c.H, d->B, d->sx, d->sy, cls[i].ex, cls[i].ey, bw, bh,
                     1, 1, 1, "wgmma X"))
      return -1;
    const dim3 grid(tiles, p.splits, p.ngroups);
#define WM_LAUNCH(bn, nt, cw) (halo[i] ? launch_wm<bn, nt, cw, true>(grid, st, mapDY, mapX, p) \
                                       : launch_wm<bn, nt, cw, false>(grid, st, mapDY, mapX, p))
    int rc;
    if (BN == 128) rc = CW == 16 ? WM_LAUNCH(128, 2, 16) : WM_LAUNCH(128, 2, 8);
    else rc = CW == 16 ? WM_LAUNCH(64, 4, 16) : WM_LAUNCH(64, 4, 8);
#undef WM_LAUNCH
    if (rc) return rc;
  }
  return 0;
}

// returns 1 if the problem is not tensor-core shaped (caller falls back to the SIMT kernel), 0 on success, <0 on error
int cd_conv_wgrad_tc(const CdConvDesc* d, const float* dout, int dout_ld, float* dw, float* db, int* bias_done, cudaStream_t st) {
  if (bias_done) *bias_done = 0;
  const CdConvSrc& c = d->s[0];
  if (c.C % 32 != 0 || d->Cout % 32 != 0 || c.ld % 4 != 0 || dout_ld % 4 != 0) return 1;
  if (!is_pow2(d->Wg) || d->Wg < 8 || !is_pow2(d->Hg)) return 1;
  if ((reinterpret_cast<uintptr_t>(c.src) & 15) || (reinterpret_cast<uintptr_t>(dout) & 15) || (reinterpret_cast<uintptr_t>(dw) & 15)) return 1;
  // wgmma kernel wherever eligible, unless a mma.sync kernel is forced (mode 0 / 8) or the bias gradient is to be fused
  if (g_wg_mode != 0 && g_wg_mode != 8 && !(g_wg_bias_fusion && db != nullptr)) {
    const int r = wgrad_wgmma(d, dout, dout_ld, dw, st);
    if (r <= 0) return r;
  }

  WgParams p{};
  p.B = d->B; p.Hg = d->Hg; p.Wg = d->Wg; p.Cout = d->Cout; p.Cin = c.C;
  p.sy = d->sy; p.sx = d->sx; p.oys = d->oys; p.oxs = d->oxs; p.oy0 = d->oy0; p.ox0 = d->ox0;
  p.dw = dw;
  int BN = c.C >= 128 ? 128 : 64;
  // ---- tap groups ----
  const bool is3x3 = (c.ntaps == 9 && d->sy == 1 && d->sx == 1);
  bool shape3 = is3x3;
  if (is3x3) for (int t = 0; t < 9; ++t) if (c.dy[t] != t / 3 - 1 || c.dx[t] != t % 3 - 1) shape3 = false;
  const bool halo = shape3 && g_wg_mode != 0;
  p.halo = halo ? 2 : 0;
  if (halo) {
    p.ngroups = 3;
    for (int gk = 0; gk < 3; ++gk) {
      p.ntaps[gk] = 3; p.nloads[gk] = 1; p.load_dy[gk][0] = gk - 1; p.load_dx[gk][0] = -1;
      for (int k = 0; k < 3; ++k) { p.tap_index[gk][k] = gk * 3 + k; p.tap_load[gk][k] = 0; p.tap_shift[gk][k] = k; }
    }
  } else {
    const int per = c.ntaps <= 4 ? c.ntaps : (c.ntaps == 9 ? 3 : 4);
    if (c.ntaps % per != 0 || c.ntaps / per > kMaxGroups) return 1;
    p.ngroups = c.ntaps / per;
    for (int gk = 0; gk < p.ngroups; ++gk) {
      p.ntaps[gk] = per; p.nloads[gk] = per;
      for (int k = 0; k < per; ++k) {
        const int t = gk * per + k;
        p.tap_index[gk][k] = t; p.tap_load[gk][k] = k; p.tap_shift[gk][k] = 0;
        p.load_dy[gk][k] = c.dy[t]; p.load_dx[gk][k] = c.dx[t];
      }
    }
  }
  const int max_taps = p.ntaps[0], max_loads = p.nloads[0];
  if (max_taps * BN > kMaxAccCols) BN = 64;                    // register accumulators: taps x BN <= 256 columns per CTA
  if (max_taps * BN > kMaxAccCols) return 1;
  // ---- pixel chunking: KR K-rows per stage ----
  int KR = (max_loads <= 1) ? 64 : 32;
  if (static_cast<long long>(d->Hg) * d->Wg < KR) KR = d->Hg * d->Wg;
  if (KR < 8) return 1;
  p.CW = d->Wg < KR ? d->Wg : KR;
  p.R = KR / p.CW;
  p.KR = KR;
  if (p.CW * d->sx > 256 || p.CW * d->oxs > 256) return 1;
  p.chunks_x = d->Wg / p.CW; p.chunks_y = d->Hg / p.R;
  p.total_chunks = d->B * p.chunks_x * p.chunks_y;
  p.tiles_co = cd_cdiv(d->Cout, 128); p.tiles_ci = cd_cdiv(c.C, BN);
  const int tiles = p.tiles_co * p.tiles_ci;
  // MMAs of one chunk: taps x KR/8 k-steps, 128 x BN x 8 each; modelled at 1024 TF32 FLOP/clk per SM for mma.sync (not measured)
  const double chunk_clk = double(max_taps) * (KR / 8) * (BN == 128 ? 256.0 : 128.0);
  int splits;
  if (c.w_per_batch) {
    const int cpi = p.chunks_x * p.chunks_y;
    const int spi0 = choose_splits(tiles * p.ngroups * d->B, cpi, cpi, chunk_clk);
    splits = spi0 * d->B;
  } else {
    splits = choose_splits(tiles * p.ngroups, p.total_chunks, cd_cdiv(p.total_chunks, 8), chunk_clk);
  }
  p.chunks_per_split = cd_cdiv(p.total_chunks, splits);
  p.splits = cd_cdiv(p.total_chunks, p.chunks_per_split);
  if (c.w_per_batch) {
    p.per_batch = 1;
    p.chunks_per_img = p.chunks_x * p.chunks_y;
    int spi = cd_cdiv(splits, d->B); if (spi < 1) spi = 1; if (spi > p.chunks_per_img) spi = p.chunks_per_img;
    p.chunks_per_split = cd_cdiv(p.chunks_per_img, spi);
    p.splits_per_img = cd_cdiv(p.chunks_per_img, p.chunks_per_split);
    p.splits = p.splits_per_img * d->B;
    p.dw_batch_stride = static_cast<long long>(c.ntaps) * d->Cout * c.C;
  }
  const int a_bytes = 4 * KR * 128;
  const int b_rows = p.R * (p.CW + p.halo);
  const int b_rows_pad = (b_rows + 7) / 8 * 8;                 // keep every chunk base 1024-byte aligned
  const int b_bytes = (BN / 32) * b_rows_pad * 128;
  const int b_tx = (BN / 32) * b_rows * 128;                   // bytes the TMA unit actually writes per X tile
  const int stage_bytes = a_bytes + max_loads * b_bytes;
  int stages = (224 * 1024) / stage_bytes; if (stages > 6) stages = 6;   // 3 x 68 KB halo stages fit the 227 KB carve-out
  if (stages < 2) return 1;
  // bias fusion: dense output grid, one weight set
  const bool fuse_bias = g_wg_bias_fusion && db != nullptr && !c.w_per_batch && d->oys == 1 && d->oxs == 1;
  p.db = fuse_bias ? db : nullptr;
  const size_t smem = size_t(stages) * stage_bytes + 1024 + 256;

  CUtensorMap mapDY, mapX;
  const CUtensorMapDataType dt = CU_TENSOR_MAP_DATA_TYPE_FLOAT32;   // operands are rounded to TF32 (RN) as they are read
  // boxes of the strided pixel grids, read with element strides
  if (!encode_nhwc(&mapDY, dt, dout, dout_ld, d->Cout, d->Wo, d->Ho, d->B, 1, 1, 0, 0, p.CW * d->oxs, p.R * d->oys, 1, d->oxs, d->oys,
                   "dY") ||
      !encode_nhwc(&mapX, dt, c.src, c.ld, c.C, c.W, c.H, d->B, 1, 1, 0, 0, (p.CW + p.halo) * d->sx, p.R * d->sy, 1, d->sx, d->sy, "X"))
    return -1;
  dim3 grid(tiles, p.splits, p.ngroups);
  int rc;
  if (BN == 128) rc = max_taps == 1 ? launch_wg<128, 1>(fuse_bias, grid, smem, st, mapDY, mapX, p, stages, a_bytes, b_bytes, b_tx)
                                    : launch_wg<128, 2>(fuse_bias, grid, smem, st, mapDY, mapX, p, stages, a_bytes, b_bytes, b_tx);
  else if (max_taps == 1) rc = launch_wg<64, 1>(fuse_bias, grid, smem, st, mapDY, mapX, p, stages, a_bytes, b_bytes, b_tx);
  else if (max_taps == 2) rc = launch_wg<64, 2>(fuse_bias, grid, smem, st, mapDY, mapX, p, stages, a_bytes, b_bytes, b_tx);
  else if (max_taps == 3) rc = launch_wg<64, 3>(fuse_bias, grid, smem, st, mapDY, mapX, p, stages, a_bytes, b_bytes, b_tx);
  else rc = launch_wg<64, 4>(fuse_bias, grid, smem, st, mapDY, mapX, p, stages, a_bytes, b_bytes, b_tx);
  if (rc == 0 && fuse_bias && bias_done) *bias_done = 1;
  return rc;
}
