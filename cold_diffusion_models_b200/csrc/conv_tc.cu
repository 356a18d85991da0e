// wgmma / TMA implicit-GEMM convolution for sm_90a (replaces the cuDNN calls behind nn.Conv2d /
// nn.ConvTranspose2d in the reference Unet: DB:105-109,149-154,173-174).
//
//   D[128 pixels x BN out-channels] (fp32, registers) += A[128 pixels x 32 ch] * B[BN x 32 ch]^T
//
// per (source, tap, 32-channel chunk).  A is an NHWC activation tile fetched by ONE 4-D TMA box
// {32 ch, TW, TH, TN} whose start coordinate carries the tap offset -- out-of-image pixels are
// zero-filled by the TMA unit, so padding costs nothing and no im2col buffer exists.  B is the
// packed weight slab [tap][Cout][Cin] (K-major), a 3-D TMA box {32, BN, 1}.  Both land in
// 128-byte-swizzled shared memory and feed wgmma (m64nBNk8 tf32) straight from descriptors.
//
// Warp roles (288 threads, persistent over output tiles, static round-robin schedule):
//   warpgroups 0-1: 64 GEMM rows each; wgmma mainloop, then the epilogue straight from the accumulator registers
//                   (+bias, (+residual), (GELU / x GELU'), (TF32 rounding))
//   warp 8        : TMA producer (one lane) -- full/empty mbarrier ring, STAGES deep
// The producer runs ahead into the next tile while the consumers finish the epilogue of this one.
#include "tc_common.cuh"
#include "conv_epilogue.cuh"

namespace {

constexpr int kTileM = 128;
constexpr int kChunkK = 32;                 // fp32 elements = 128 bytes = one swizzle row
constexpr int kABytes = kTileM * 128;       // 16 KiB per stage
constexpr int kThreads = 288;
constexpr int kConsumerWarps = 8;

struct TcParams {
  int B, Hg, Wg;
  int TW, TH, TN;
  int tiles_x, tiles_y, tiles_n, tiles_co, total_tiles;
  int sy, sx;
  int Cout;
  int nsrc;
  int ntaps[2];
  int kchunks[2];
  int wpb[2];
  int8_t dy[2][CD_MAX_TAPS];
  int8_t dx[2][CD_MAX_TAPS];
  float* out; int out_ld; int Ho, Wo; int oys, oxs, oy0, ox0;
  const float* bias;
  const float* resid; int resid_ld;
  int act; int round_tf32;
  float* out2; int out2_ld;
  const float* aux; int aux_ld;
};

// output pixel of GEMM row m of tile `tile` (-1: beyond the batch)
__device__ __forceinline__ long long tile_pixel(const TcParams& p, int tile, int m) {
  int mt = tile / p.tiles_co;
  const int tx = mt % p.tiles_x; mt /= p.tiles_x;
  const int ty = mt % p.tiles_y;
  const int tn = mt / p.tiles_y;
  const int gx = tx * p.TW + m % p.TW, gy = ty * p.TH + (m / p.TW) % p.TH, b = tn * p.TN + m / (p.TW * p.TH);
  if (b >= p.B) return -1;
  return (static_cast<long long>(b) * p.Ho + (gy * p.oys + p.oy0)) * p.Wo + (gx * p.oxs + p.ox0);
}

// two adjacent output channels (col, col + 1) of one pixel: acc + bias + resid -> out2 -> activation -> TF32 rounding -> out
__device__ __forceinline__ void epi_pair(const TcParams& p, long long pix, int col, float v0, float v1) {
  if (col + 1 < p.Cout) {
    float2 v = make_float2(v0, v1);
    if (p.bias) { const float2 b = __ldg(reinterpret_cast<const float2*>(p.bias + col)); v.x += b.x; v.y += b.y; }
    if (p.resid) { const float2 r = *reinterpret_cast<const float2*>(p.resid + pix * p.resid_ld + col); v.x += r.x; v.y += r.y; }
    if (p.out2) *reinterpret_cast<float2*>(p.out2 + pix * p.out2_ld + col) = v;
    if (p.act == CD_ACT_GELU) { v.x = cd_gelu(v.x); v.y = cd_gelu(v.y); }
    else if (p.act == CD_ACT_GELU_BWD) {
      const float2 a = *reinterpret_cast<const float2*>(p.aux + pix * p.aux_ld + col);
      v.x *= cd_gelu_grad(a.x); v.y *= cd_gelu_grad(a.y);
    }
    if (p.round_tf32) { v.x = cd_round_tf32(v.x); v.y = cd_round_tf32(v.y); }
    *reinterpret_cast<float2*>(p.out + pix * p.out_ld + col) = v;
  } else if (col < p.Cout) {
    float v = v0;
    if (p.bias) v += p.bias[col];
    if (p.resid) v += p.resid[pix * p.resid_ld + col];
    if (p.out2) p.out2[pix * p.out2_ld + col] = v;
    if (p.act == CD_ACT_GELU) v = cd_gelu(v);
    else if (p.act == CD_ACT_GELU_BWD) v *= cd_gelu_grad(p.aux[pix * p.aux_ld + col]);
    if (p.round_tf32) v = cd_round_tf32(v);
    p.out[pix * p.out_ld + col] = v;
  }
}

// STG: line-coalesced epilogue (conv_epilogue.cuh; opt-in, fewer mainloop stages): the warpgroup's 64 x 32 block of a column
//      chunk goes through shared memory so that a lane holds 32 consecutive channels of one pixel, as that epilogue expects
// F16: operand-format probe (cd_conv_fwd_f16_probe): sources and packed weights are FP16 arrays, one 128-byte swizzle row = 64 channels
// CTAS: co-resident CTAs per SM (2: half the stages each, so that one CTA's epilogue overlaps the other's mainloop)
// PAIR: SM-pair mode -- a cluster of two CTAs computes two neighbouring 128-pixel tiles of the same BN output channels; each CTA
//       fetches half of the weight tile and multicasts it into both, so every weight byte leaves L2 once per pair.  A stage may
//       only be refilled when the consumers of BOTH CTAs have released it (empty barriers count the warps of both).
template <int BN, int STAGES, bool STG = false, bool F16 = false, int CTAS = 1, bool PAIR = false>
__global__ void __launch_bounds__(kThreads, CTAS)
conv_tc_kernel(const __grid_constant__ CUtensorMap mapA0, const __grid_constant__ CUtensorMap mapA1,
               const __grid_constant__ CUtensorMap mapB0, const __grid_constant__ CUtensorMap mapB1,
               const TcParams p) {
  constexpr int kBBytes = BN * 128;
  constexpr int kStageBytes = kABytes + kBBytes;
  constexpr int kChunkElems = F16 ? 64 : kChunkK;   // elements per 128-byte row

  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  const uint32_t pad = (1024u - (raw_addr & 1023u)) & 1023u;
  uint8_t* smem = smem_raw + pad;                       // 1024-byte aligned (SWIZZLE_128B atoms)
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + STAGES * kStageBytes);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + STAGES;
  static_assert(2 * STAGES * 8 <= 256, "barrier block is 256 bytes");
  float* epi_stage = reinterpret_cast<float*>(smem + STAGES * kStageBytes + 256);     // STG: 2 x 64 x kEpiStageStride floats

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = threadIdx.x >> 7;

  if (threadIdx.x == 0) {
    for (int i = 0; i < STAGES; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], kConsumerWarps * (PAIR ? 2 : 1)); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if constexpr (PAIR) cluster_sync(); else __syncthreads();
  const uint32_t rank = PAIR ? cluster_ctarank() : 0;
  // work units: (M tile, co tile) -- or, in PAIR mode, (M tile pair, co tile) with this CTA taking M tile 2 * pair + rank
  const int unit0 = PAIR ? blockIdx.x / 2 : blockIdx.x, ustride = PAIR ? gridDim.x / 2 : gridDim.x;
  const int units = PAIR ? p.tiles_co * ((p.total_tiles / p.tiles_co + 1) / 2) : p.total_tiles;
  auto tile_of = [&](int u) { return PAIR ? ((u / p.tiles_co) * 2 + static_cast<int>(rank)) * p.tiles_co + u % p.tiles_co : u; };

  const int kiters = p.ntaps[0] * p.kchunks[0] + (p.nsrc > 1 ? p.ntaps[1] * p.kchunks[1] : 0);

  if (warp == kConsumerWarps) {
    // ===================== TMA producer: ONE elected thread runs the whole schedule =====================
    if (elect_one()) {
      uint32_t stage = 0, ph = 0;
      for (int u = unit0; u < units; u += ustride) {
        const int tile = tile_of(u);           // PAIR: may lie beyond the last M tile (zero-filled loads, no stores)
        const int co_t = tile % p.tiles_co;
        int mt = tile / p.tiles_co;
        const int tx = mt % p.tiles_x; mt /= p.tiles_x;
        const int ty = mt % p.tiles_y;
        const int tn = mt / p.tiles_y;
        const int x0 = tx * p.TW * p.sx, y0 = ty * p.TH * p.sy, n0 = tn * p.TN, co0 = co_t * BN;
        for (int s = 0; s < p.nsrc; ++s) {
          const CUtensorMap* mA = s ? &mapA1 : &mapA0;
          const CUtensorMap* mB = s ? &mapB1 : &mapB0;
          const int wbase = p.wpb[s] ? n0 * p.ntaps[s] : 0;
          for (int tap = 0; tap < p.ntaps[s]; ++tap) {
            const int xin = x0 + p.dx[s][tap], yin = y0 + p.dy[s][tap];
            for (int kc = 0; kc < p.kchunks[s]; ++kc) {
              mbar_wait(&empty_bar[stage], ph ^ 1u);
              mbar_expect_tx(&full_bar[stage], kStageBytes);
              const uint32_t sa = smem_u32(smem + stage * kStageBytes);
              tma_load_4d(sa, mA, &full_bar[stage], kc * kChunkElems, xin, yin, n0);
              if constexpr (PAIR)
                tma_load_3d_mc(sa + kABytes + rank * (kBBytes / 2), mB, &full_bar[stage], kc * kChunkElems, co0 + static_cast<int>(rank) * (BN / 2),
                               wbase + tap, static_cast<uint16_t>(3));
              else
                tma_load_3d(sa + kABytes, mB, &full_bar[stage], kc * kChunkElems, co0, wbase + tap);
              if (++stage == STAGES) { stage = 0; ph ^= 1u; }
            }
          }
        }
      }
    }
    __syncwarp();
  } else {
    // ===================== consumers: warpgroup cw owns GEMM rows [64 cw, 64 cw + 64) =====================
    const int cw = wg;
    const int tid = threadIdx.x & 127;
    const int rl = (tid >> 5) * 16 + (lane >> 2);        // local row of acc[4j], acc[4j + 1]; acc[4j + 2 / 3] are row rl + 8
    const int q2 = (lane & 3) * 2;                       // column pair inside each 8-column block
    float acc[BN / 2];
    uint32_t stage = 0, ph = 0;
    auto release = [&](uint32_t st) {
      __syncwarp();
      if (lane == 0) { mbar_arrive(&empty_bar[st]); if constexpr (PAIR) mbar_arrive_cluster(&empty_bar[st], rank ^ 1u); }
    };
    for (int u = unit0; u < units; u += ustride) {
      const int tile = tile_of(u);
      uint32_t prev = 0;
      for (int k = 0; k < kiters; ++k) {
        mbar_wait(&full_bar[stage], ph);
        wgmma_fence();
        const uint32_t sa = smem_u32(smem + stage * kStageBytes);
        const uint64_t da = make_kmajor_sw128_desc(sa + cw * (kABytes / 2));
        const uint64_t db = make_kmajor_sw128_desc(sa + kABytes);
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {          // 4 x 32 bytes per 128-byte row
          if constexpr (F16) wgmma_f16<BN>(acc, da + uint64_t(kk * 2), db + uint64_t(kk * 2), (k | kk) != 0 ? 1u : 0u);
          else wgmma_tf32<BN>(acc, da + uint64_t(kk * 2), db + uint64_t(kk * 2), (k | kk) != 0 ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait<1>();                          // the previous chunk's MMAs have retired: its slot can be refilled
        if (k > 0) release(prev);
        prev = stage;
        if (++stage == STAGES) { stage = 0; ph ^= 1u; }
      }
      wgmma_wait<0>();
      if (kiters > 0) release(prev);

      const int co0 = (tile % p.tiles_co) * BN;
      const long long pix0 = tile_pixel(p, tile, cw * 64 + rl);
      const long long pix1 = tile_pixel(p, tile, cw * 64 + rl + 8);
      if constexpr (STG) {
        float* st = epi_stage + cw * 64 * kEpiStageStride;
        const int bar_id = 1 + cw;
#pragma unroll
        for (int c = 0; c < BN; c += 32) {
          if (co0 + c + 32 <= p.Cout) {            // uniform: full 32-column chunk through shared memory
            asm volatile("bar.sync %0, 128;" :: "r"(bar_id) : "memory");
#pragma unroll
            for (int j = c / 8; j < c / 8 + 4; ++j) {
              *reinterpret_cast<float2*>(st + rl * kEpiStageStride + 8 * j - c + q2) = make_float2(acc[4 * j], acc[4 * j + 1]);
              *reinterpret_cast<float2*>(st + (rl + 8) * kEpiStageStride + 8 * j - c + q2) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
            }
            asm volatile("bar.sync %0, 128;" :: "r"(bar_id) : "memory");
            const int w4 = tid >> 5;
            if (w4 < 2) {                          // warps 0-1 of the warpgroup: lane = pixel row w4 * 32 + lane
              const int row = w4 * 32 + lane;
              uint32_t r[32];
#pragma unroll
              for (int e = 0; e < 32; ++e) r[e] = __float_as_uint(st[row * kEpiStageStride + e]);
              const long long pix = tile_pixel(p, tile, cw * 64 + row);
              cd_epilogue_staged32(r, st + w4 * 32 * kEpiStageStride, lane, pix < 0 ? 0 : pix, pix >= 0, co0 + c, p);
            }
          } else {
#pragma unroll
            for (int j = c / 8; j < c / 8 + 4; ++j) {
              if (pix0 >= 0) epi_pair(p, pix0, co0 + 8 * j + q2, acc[4 * j], acc[4 * j + 1]);
              if (pix1 >= 0) epi_pair(p, pix1, co0 + 8 * j + q2, acc[4 * j + 2], acc[4 * j + 3]);
            }
          }
        }
      } else {
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          if (pix0 >= 0) epi_pair(p, pix0, co0 + 8 * j + q2, acc[4 * j], acc[4 * j + 1]);
          if (pix1 >= 0) epi_pair(p, pix1, co0 + 8 * j + q2, acc[4 * j + 2], acc[4 * j + 3]);
        }
      }
    }
  }
  if constexpr (PAIR) cluster_sync();          // the peer may still multicast into / arrive on this CTA
}

// ---------------------------------------------------------------------------------------------
// Halo-tile kernel for stride-1 convolutions whose taps lie in [-1, 1]^2 (dense 3x3 forward / data gradient, fused [3x3 | 1x1]
// pairs): a CTA tile is 16 x TH output pixels of one image (TH = 8: 128 GEMM rows, one 64-row accumulator per consumer
// warpgroup; TH = 16: 256 rows, two accumulators per warpgroup that share every weight tile).  Per source and 32-channel chunk
// ONE TMA box fetches the (16 + 2) x (TH + 2) halo patch; every tap reads its shifted window of that patch into registers as the
// wgmma A operand (tf32, rounded to nearest), so activations leave L2 once per chunk instead of once per tap.  Weight tiles
// stream through their own STAGES-deep ring.  Grids need not be powers of two: pixels outside the grid are masked.
// ---------------------------------------------------------------------------------------------
constexpr int kHaloW = 16;

template <int BN, int MB, int STAGES, int CTAS = 1>
__global__ void __launch_bounds__(kThreads, CTAS)
conv_halo_kernel(const __grid_constant__ CUtensorMap mapA0, const __grid_constant__ CUtensorMap mapA1,
                 const __grid_constant__ CUtensorMap mapB0, const __grid_constant__ CUtensorMap mapB1, const TcParams p) {
  constexpr int TH = 8 * MB;
  constexpr int PW = kHaloW + 2, PH = TH + 2;
  constexpr int kPatchBytes = (PW * PH * 128 + 1023) / 1024 * 1024;
  constexpr int kBBytes = BN * 128;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + ((1024u - (raw_addr & 1023u)) & 1023u);
  uint8_t* patch = smem;                                   // 2 patch slots
  uint8_t* wtile = smem + 2 * kPatchBytes;                 // STAGES weight tiles
  uint64_t* bars = reinterpret_cast<uint64_t*>(wtile + STAGES * kBBytes);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + STAGES;
  uint64_t* pfull = bars + 2 * STAGES;
  uint64_t* pempty = bars + 2 * STAGES + 2;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = threadIdx.x >> 7;
  if (threadIdx.x == 0) {
    for (int i = 0; i < STAGES; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], kConsumerWarps); }
    for (int i = 0; i < 2; ++i) { mbar_init(&pfull[i], 1); mbar_init(&pempty[i], kConsumerWarps); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == kConsumerWarps) {
    if (elect_one()) {
      uint32_t stage = 0, ph = 0, pi = 0, pph = 0;
      for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
        const int co_t = tile % p.tiles_co;
        int mt = tile / p.tiles_co;
        const int tx = mt % p.tiles_x; mt /= p.tiles_x;
        const int ty = mt % p.tiles_y;
        const int n = mt / p.tiles_y;
        for (int s = 0; s < p.nsrc; ++s) {
          const CUtensorMap* mA = s ? &mapA1 : &mapA0;
          const CUtensorMap* mB = s ? &mapB1 : &mapB0;
          for (int kc = 0; kc < p.kchunks[s]; ++kc) {
            mbar_wait(&pempty[pi], pph ^ 1u);
            mbar_expect_tx(&pfull[pi], PW * PH * 128);
            tma_load_4d(smem_u32(patch + pi * kPatchBytes), mA, &pfull[pi], kc * kChunkK, tx * kHaloW - 1, ty * TH - 1, n);
            if (++pi == 2) { pi = 0; pph ^= 1u; }
            for (int tap = 0; tap < p.ntaps[s]; ++tap) {
              mbar_wait(&empty_bar[stage], ph ^ 1u);
              mbar_expect_tx(&full_bar[stage], kBBytes);
              tma_load_3d(smem_u32(wtile + stage * kBBytes), mB, &full_bar[stage], kc * kChunkK, co_t * BN, tap);
              if (++stage == STAGES) { stage = 0; ph ^= 1u; }
            }
          }
        }
      }
    }
    __syncwarp();
    return;
  }

  // consumers: warpgroup wg owns tile rows [64 MB wg, 64 MB (wg + 1)); row m = pixel (m % 16, m / 16) of the tile
  const int tid = threadIdx.x & 127;
  const int rl = (tid >> 5) * 16 + (lane >> 2);
  const int q2 = (lane & 3) * 2, t4 = lane & 3;
  int prow[MB][2];                                   // patch row of this lane's two A rows per block, tap (0, 0) of the window
#pragma unroll
  for (int mb = 0; mb < MB; ++mb)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int m = (wg * MB + mb) * 64 + rl + 8 * h;
      prow[mb][h] = (m / kHaloW + 1) * PW + (m % kHaloW) + 1;
    }
  float acc[MB][BN / 2];
  uint32_t stage = 0, ph = 0, pi = 0, pph = 0;
  for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
    bool first = true;
    for (int s = 0; s < p.nsrc; ++s) {
      for (int kc = 0; kc < p.kchunks[s]; ++kc) {
        mbar_wait(&pfull[pi], pph);
        const uint8_t* pt = patch + pi * kPatchBytes;
        for (int tap = 0; tap < p.ntaps[s]; ++tap) {
          const int shift = p.dy[s][tap] * PW + p.dx[s][tap];
          uint32_t a[MB][4][4];
#pragma unroll
          for (int mb = 0; mb < MB; ++mb)
#pragma unroll
            for (int kk = 0; kk < 4; ++kk)
#pragma unroll
              for (int e = 0; e < 4; ++e) {
                const int row = prow[mb][e & 1] + shift, c = kk * 8 + t4 + 4 * (e >> 1);
                a[mb][kk][e] = __float_as_uint(cd_round_tf32(
                    *reinterpret_cast<const float*>(pt + row * 128 + ((((c >> 2) ^ row) & 7) << 4) + (c & 3) * 4)));
              }
          mbar_wait(&full_bar[stage], ph);
          wgmma_fence();
          const uint64_t db = make_kmajor_sw128_desc(smem_u32(wtile + stage * kBBytes));
#pragma unroll
          for (int mb = 0; mb < MB; ++mb)
#pragma unroll
            for (int kk = 0; kk < 4; ++kk)
              wgmma_tf32_rs<BN>(acc[mb], a[mb][kk], db + uint64_t(kk * 2), (first && kk == 0) ? 0u : 1u);
          wgmma_commit();
          wgmma_wait<0>();                         // the A registers are reloaded for the next tap
          first = false;
          __syncwarp();
          if (lane == 0) mbar_arrive(&empty_bar[stage]);
          if (++stage == STAGES) { stage = 0; ph ^= 1u; }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&pempty[pi]);
        if (++pi == 2) { pi = 0; pph ^= 1u; }
      }
    }
    const int co_t = tile % p.tiles_co, co0 = co_t * BN;
    int mt = tile / p.tiles_co;
    const int tx = mt % p.tiles_x; mt /= p.tiles_x;
    const int ty = mt % p.tiles_y;
    const int n = mt / p.tiles_y;
#pragma unroll
    for (int mb = 0; mb < MB; ++mb)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int m = (wg * MB + mb) * 64 + rl + 8 * h;
        const int gx = tx * kHaloW + m % kHaloW, gy = ty * TH + m / kHaloW;
        if (gx >= p.Wg || gy >= p.Hg) continue;
        const long long pix = (static_cast<long long>(n) * p.Ho + (gy * p.oys + p.oy0)) * p.Wo + (gx * p.oxs + p.ox0);
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) epi_pair(p, pix, co0 + 8 * j + q2, acc[mb][4 * j + 2 * h], acc[mb][4 * j + 2 * h + 1]);
      }
  }
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------

int g_num_sms = 0;
int g_tf32_map_dtype = 1;   // 1: TFLOAT32 tensor maps; 0: FLOAT32 (diagnostic, cd_conv_tc_set_tf32_maps)


template <int BN, int STAGES, bool STG = false, bool F16 = false, int CTAS = 1, bool PAIR = false>
int launch(const CUtensorMap* maps, const TcParams& p, cudaStream_t st) {
  constexpr size_t smem = size_t(STAGES) * (kABytes + BN * 128) + 1024 + 256 + (STG ? sizeof(float) * 2 * 64 * kEpiStageStride : 0);
  static_assert(smem <= 232448, "dynamic shared memory of one CTA (227 KB)");
  static_assert(CTAS == 1 || 2 * (smem + 1024) <= 233472, "two CTAs per SM must fit the 228 KB of shared memory");
  auto kern = conv_tc_kernel<BN, STAGES, STG, F16, CTAS, PAIR>;
  static bool attr_done = false;
  if (!attr_done) {
    CD_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr_done = true;
  }
  if constexpr (PAIR) {
    const int units = p.tiles_co * ((p.total_tiles / p.tiles_co + 1) / 2), slots = g_num_sms / 2;
    cudaLaunchConfig_t cfg = {};
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = 2; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
    cfg.gridDim = dim3(2 * (units < slots ? units : slots)); cfg.blockDim = dim3(kThreads);
    cfg.dynamicSmemBytes = smem; cfg.stream = st; cfg.attrs = attr; cfg.numAttrs = 1;
    CD_CUDA(cudaLaunchKernelEx(&cfg, kern, maps[0], maps[1], maps[2], maps[3], p));
  } else {
    const int slots = g_num_sms * CTAS;
    const int grid = p.total_tiles < slots ? p.total_tiles : slots;
    kern<<<grid, kThreads, smem, st>>>(maps[0], maps[1], maps[2], maps[3], p);
  }
  CD_LAUNCH_CHECK();
  return 0;
}

template <int BN, int MB, int STAGES, int CTAS = 1>
int launch_halo(const CUtensorMap* maps, const TcParams& p, cudaStream_t st) {
  constexpr int kPatchBytes = ((kHaloW + 2) * (8 * MB + 2) * 128 + 1023) / 1024 * 1024;
  constexpr size_t smem = 2 * size_t(kPatchBytes) + size_t(STAGES) * BN * 128 + 1024 + 256;
  static_assert(smem <= 232448, "dynamic shared memory of one CTA (227 KB)");
  static_assert(CTAS == 1 || 2 * (smem + 1024) <= 233472, "two CTAs per SM must fit the 228 KB of shared memory");
  static bool attr_done = false;
  if (!attr_done) {
    CD_CUDA(cudaFuncSetAttribute(conv_halo_kernel<BN, MB, STAGES, CTAS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr_done = true;
  }
  const int slots = g_num_sms * CTAS;
  const int grid = p.total_tiles < slots ? p.total_tiles : slots;
  conv_halo_kernel<BN, MB, STAGES, CTAS><<<grid, kThreads, smem, st>>>(maps[0], maps[1], maps[2], maps[3], p);
  CD_LAUNCH_CHECK();
  return 0;
}

}  // namespace

extern "C" int cd_conv_tc_set_tf32_maps(int enable) { g_tf32_map_dtype = enable ? 1 : 0; return 0; }

// Defaults measured with tools/conv_shapes.py and bench.py on an H100 80GB HBM3 at a 400 W power limit (Unet config 3, batch 32):
// convolution forward time per training step 80 ms with the per-tap kernel at one CTA per SM, 74 ms with two CTAs per SM for the
// 64- and 128-wide N tiles (375 -> 387 images/s), 87 ms with the SM-pair kernel, 86 / 95 ms with the 16 x 8 / 16 x 16 halo-tile
// kernel.  So two CTAs per SM is on by default; the pair and halo variants are off.
static int g_use_2cta = 0;
extern "C" int cd_conv_tc_set_2cta(int mode) { g_use_2cta = mode; return 0; }   // 0 off, 1 where the cost model prefers it, 2 wherever eligible
// narrower pair tiles: bit mask of the N tiles below 256 (128 | 64) that go to the SM-pair kernel when the problem is eligible
static int g_2cta_bn = 0;
extern "C" int cd_conv_tc_set_2cta_bn(int mask) { g_2cta_bn = mask & (128 | 64); return 0; }
// halo-tile kernel for stride-1 convolutions with taps in [-1, 1]^2, bit mask: 1 = 16 x 8 pixel tiles wherever eligible,
// 2 = 16 x 16 tiles (two accumulators per weight tile) for Cout <= 128 on grids of at least 32 x 32, 4 (with 2) = 16 x 16 tiles
// for every eligible problem (tests); 0 = off (default)
static int g_use_halo = 0;
extern "C" int cd_conv_tc_set_halo(int enable) { g_use_halo = enable; return 0; }
// two CTAs per SM (half the stages each) for N <= 128: bit mask of N tiles (128 | 64)
static int g_ctas2 = 128 | 64;
extern "C" int cd_conv_tc_set_two_ctas(int mask) { g_ctas2 = mask & (128 | 64); return 0; }
// line-coalesced epilogue (conv_epilogue.cuh): 0 = off (default), 1 = for the short-K launches that are bound by their output
// stores (at most kStagedMaxKIters 32-channel K chunks per tile), 2 = for every launch (tests), 3 = up to kStagedMidKIters chunks
static int g_epi_staged = 0;
constexpr int kStagedMaxKIters = 16;
constexpr int kStagedMidKIters = 48;
extern "C" int cd_conv_tc_set_staged_epilogue(int mode) { g_epi_staged = mode; return 0; }

// Tile-shape choice: waves over the SMs x columns per tile / relative rate of that tile shape (a 64-row wgmma reads the whole
// B tile from shared memory for every 64 rows, so wide N tiles amortise the A reads best; an SM pair halves the weight traffic
// from L2).  The rates are a model, not a measurement.
static double tc_cost(long long m_tiles, int Cout, int BN, int sms, bool pair = false) {
  if (pair) {
    const long long tiles = ((m_tiles + 1) / 2) * (Cout / 256), slots = sms / 2;
    return double((tiles + slots - 1) / slots) * 256.0;
  }
  const long long tiles = m_tiles * ((Cout + BN - 1) / BN);
  const double rate = BN == 256 ? 0.92 : (BN == 128 ? 0.75 : 0.40);
  return double((tiles + sms - 1) / sms) * BN / rate;
}

static int conv_fwd_tc_impl(const CdConvDesc* d, cudaStream_t st, bool f16);
int cd_conv_fwd_tc(const CdConvDesc* d, cudaStream_t st) { return conv_fwd_tc_impl(d, st, false); }

// Operand-format probe (tools/conv_f16_probe.py; not used by the engine): the same convolution with FP16 sources and FP16 packed
// weights (src / w point to __half arrays, ld and the weight strides count elements), fp32 accumulate and the fp32 epilogue.
extern "C" int cd_conv_fwd_f16_probe(const CdConvDesc* d, void* stream) {
  CD_REQUIRE(d != nullptr && d->nsrc >= 1 && d->nsrc <= 2, "cd_conv_fwd_f16_probe: bad descriptor");
  return conv_fwd_tc_impl(d, static_cast<cudaStream_t>(stream), true);
}

static int conv_fwd_halo(const CdConvDesc* d, cudaStream_t st, int MB);

static int conv_fwd_tc_impl(const CdConvDesc* d, cudaStream_t st, bool f16) {
  if (!f16 && g_epi_staged == 0 && (g_use_halo & 2)) {
    const int r = conv_fwd_halo(d, st, 2);
    if (r <= 0) return r;                                     // 1 = not eligible
  }
  if (!f16 && g_epi_staged == 0 && (g_use_halo & 1)) {
    const int r = conv_fwd_halo(d, st, 1);
    if (r <= 0) return r;
  }
  const int chunk_elems = f16 ? 64 : kChunkK;
  const int esz = f16 ? 2 : 4;
  EncodeTiledFn enc = get_encode();
  CD_REQUIRE(enc != nullptr, "cuTensorMapEncodeTiled entry point unavailable");
  if (!g_num_sms) {
    int dev = 0; CD_CUDA(cudaGetDevice(&dev));
    CD_CUDA(cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev));
  }
  CD_REQUIRE(d->nsrc >= 1 && d->nsrc <= 2, "conv_tc: nsrc must be 1 or 2");
  TcParams p{};
  p.B = d->B; p.Hg = d->Hg; p.Wg = d->Wg; p.sy = d->sy; p.sx = d->sx; p.Cout = d->Cout; p.nsrc = d->nsrc;
  // tile geometry: 128 GEMM rows = TW x TH x TN pixels
  if (d->Wg >= 128) {
    CD_REQUIRE(d->Wg % 128 == 0, "conv_tc: Wg >= 128 must be a multiple of 128 (got %d)", d->Wg);
    p.TW = 128; p.TH = 1; p.TN = 1;
  } else {
    CD_REQUIRE(is_pow2(d->Wg), "conv_tc: Wg < 128 must be a power of two (got %d)", d->Wg);
    p.TW = d->Wg;
    int th = 128 / p.TW;
    if (th > d->Hg) th = d->Hg;
    CD_REQUIRE(is_pow2(th) && d->Hg % th == 0, "conv_tc: unsupported Hg %d for Wg %d", d->Hg, d->Wg);
    p.TH = th; p.TN = 128 / (p.TW * p.TH);
  }
  CD_REQUIRE(p.TW * d->sx <= 256 && p.TH * d->sy <= 256, "conv_tc: strided box too large");
  p.tiles_x = d->Wg / p.TW; p.tiles_y = d->Hg / p.TH; p.tiles_n = cd_cdiv(d->B, p.TN);
  int BN = (d->Cout % 256 == 0) ? 256 : (d->Cout > 64 ? 128 : 64);
  int kiters_host = 0;
  for (int s = 0; s < d->nsrc; ++s) kiters_host += d->s[s].ntaps * (d->s[s].C / chunk_elems);
  const bool staged = !f16 &&
                      ( g_epi_staged == 2 || (g_epi_staged == 1 && kiters_host <= kStagedMaxKIters) ||
                      (g_epi_staged == 3 && kiters_host <= kStagedMidKIters));
  bool pair = false;
  const long long mt = static_cast<long long>(p.tiles_x) * p.tiles_y * p.tiles_n;
  if (BN == 256) {
    // small spatial sizes (16^2, 32^2) give few M tiles: take the narrower N tile only when it saves whole waves
    double best = tc_cost(mt, d->Cout, 256, g_num_sms);
    if (tc_cost(mt, d->Cout, 128, g_num_sms) < best) { BN = 128; best = tc_cost(mt, d->Cout, 128, g_num_sms); }
    if (!f16 && !staged && g_use_2cta && mt >= 2 && (g_use_2cta == 2 || tc_cost(mt, d->Cout, 256, g_num_sms, true) < best)) {
      BN = 256; pair = true;
    }
  } else if (!f16 && !staged && g_use_2cta && (g_2cta_bn & BN) && d->Cout % BN == 0 && (g_use_2cta == 2 || mt >= 2 * g_num_sms)) {
    pair = true;                                              // narrow pair tile: only with at least one pair tile per SM pair
  }
  p.tiles_co = cd_cdiv(d->Cout, BN);
  p.total_tiles = p.tiles_x * p.tiles_y * p.tiles_n * p.tiles_co;
  p.out = d->out; p.out_ld = d->out_ld; p.Ho = d->Ho; p.Wo = d->Wo;
  p.oys = d->oys; p.oxs = d->oxs; p.oy0 = d->oy0; p.ox0 = d->ox0;
  p.bias = d->bias; p.resid = d->resid; p.resid_ld = d->resid_ld; p.act = d->act; p.round_tf32 = d->round_tf32;
  p.out2 = d->out2; p.out2_ld = d->out2_ld; p.aux = d->aux; p.aux_ld = d->aux_ld;
  CD_REQUIRE(d->act != CD_ACT_GELU_BWD || (d->aux && (reinterpret_cast<uintptr_t>(d->aux) & 15) == 0 && d->aux_ld % 4 == 0), "conv_tc: GELU_BWD needs an aligned aux");
  CD_REQUIRE((reinterpret_cast<uintptr_t>(d->out) & 15) == 0 && d->out_ld % 4 == 0, "conv_tc: out must be 16B aligned");
  CD_REQUIRE(!d->resid || ((reinterpret_cast<uintptr_t>(d->resid) & 15) == 0 && d->resid_ld % 4 == 0), "conv_tc: resid alignment");
  CD_REQUIRE(!d->out2 || ((reinterpret_cast<uintptr_t>(d->out2) & 15) == 0 && d->out2_ld % 4 == 0), "conv_tc: out2 alignment");
  CD_REQUIRE(!d->bias || (reinterpret_cast<uintptr_t>(d->bias) & 15) == 0, "conv_tc: bias alignment");

  CUtensorMap maps[4];
  const CUtensorMapDataType dt = f16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : (g_tf32_map_dtype ? CU_TENSOR_MAP_DATA_TYPE_TFLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32);
  for (int s = 0; s < 2; ++s) {
    const CdConvSrc& cs = d->s[s < d->nsrc ? s : 0];
    CD_REQUIRE(cs.C % chunk_elems == 0 && cs.C > 0, "conv_tc: source channels %d not a multiple of %d", cs.C, chunk_elems);
    CD_REQUIRE(cs.ntaps >= 1 && cs.ntaps <= CD_MAX_TAPS, "conv_tc: bad ntaps");
    CD_REQUIRE((reinterpret_cast<uintptr_t>(cs.src) & 15) == 0 && (cs.ld * esz) % 16 == 0, "conv_tc: src must be 16B aligned");
    CD_REQUIRE((reinterpret_cast<uintptr_t>(cs.w) & 15) == 0, "conv_tc: weights must be 16B aligned");
    CD_REQUIRE(!cs.w_per_batch || p.TN == 1, "conv_tc: per-batch weights need >=128 pixels per image");
    p.ntaps[s] = cs.ntaps; p.kchunks[s] = cs.C / chunk_elems; p.wpb[s] = cs.w_per_batch;
    for (int t = 0; t < cs.ntaps; ++t) { p.dy[s][t] = (int8_t)cs.dy[t]; p.dx[s][t] = (int8_t)cs.dx[t]; }
    {   // A: NHWC activations, dims {C, W, H, N}
      cuuint64_t dims[4] = {(cuuint64_t)cs.C, (cuuint64_t)cs.W, (cuuint64_t)cs.H, (cuuint64_t)d->B};
      cuuint64_t strides[3] = {(cuuint64_t)cs.ld * esz, (cuuint64_t)cs.ld * esz * cs.W, (cuuint64_t)cs.ld * esz * cs.W * cs.H};
      cuuint32_t box[4] = {(cuuint32_t)chunk_elems, (cuuint32_t)(p.TW * d->sx), (cuuint32_t)(p.TH * d->sy), (cuuint32_t)p.TN};
      cuuint32_t estr[4] = {1, (cuuint32_t)d->sx, (cuuint32_t)d->sy, 1};
      CUresult r = enc(&maps[s], dt, 4, const_cast<float*>(cs.src), dims, strides, box, estr,
                       CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                       CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
      CD_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(A%d) failed: %d", s, (int)r);
    }
    {   // B: packed weights, dims {Cin, Cout, ntaps * (per-batch ? B : 1)}
      const int BNl = BN;
      cuuint64_t dims[3] = {(cuuint64_t)cs.C, (cuuint64_t)d->Cout, (cuuint64_t)cs.ntaps * (cs.w_per_batch ? d->B : 1)};
      cuuint64_t strides[2] = {(cuuint64_t)cs.C * esz, (cuuint64_t)cs.C * esz * d->Cout};
      cuuint32_t box[3] = {(cuuint32_t)chunk_elems, (cuuint32_t)(pair ? BNl / 2 : BNl), 1};   // pair: each CTA fetches half
      cuuint32_t estr[3] = {1, 1, 1};
      CUresult r = enc(&maps[2 + s], dt, 3, const_cast<float*>(cs.w), dims, strides, box, estr,
                       CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                       CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
      CD_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(B%d) failed: %d", s, (int)r);
    }
  }
  if (f16) {
    if (BN == 256) return launch<256, 4, false, true>(maps, p, st);
    if (BN == 128) return launch<128, 6, false, true>(maps, p, st);
    return launch<64, 8, false, true>(maps, p, st);
  }
  if (staged) {          // 36 KB of epilogue staging: 3 / 4 / 6 mainloop stages instead of 4 / 6 / 8
    if (BN == 256) return launch<256, 3, true>(maps, p, st);
    if (BN == 128) return launch<128, 4, true>(maps, p, st);
    return launch<64, 6, true>(maps, p, st);
  }
  if (pair) {
    if (BN == 256) return launch<256, 4, false, false, 1, true>(maps, p, st);
    if (BN == 128) return launch<128, 6, false, false, 1, true>(maps, p, st);
    return launch<64, 8, false, false, 1, true>(maps, p, st);
  }
  if (BN == 256) return launch<256, 4>(maps, p, st);
  if (BN == 128) return (g_ctas2 & 128) ? launch<128, 3, false, false, 2>(maps, p, st) : launch<128, 6>(maps, p, st);
  return (g_ctas2 & 64) ? launch<64, 4, false, false, 2>(maps, p, st) : launch<64, 8>(maps, p, st);
}

// returns 1 when the problem is not eligible for the halo-tile kernel (MB = 1: 16 x 8 tiles, 2: 16 x 16 tiles)
static int conv_fwd_halo(const CdConvDesc* d, cudaStream_t st, int MB) {
  if (d->sy != 1 || d->sx != 1 || d->nsrc < 1 || d->nsrc > 2 || !g_tf32_map_dtype) return 1;
  for (int s = 0; s < d->nsrc; ++s) {
    const CdConvSrc& cs = d->s[s];
    if (cs.w_per_batch || cs.C % kChunkK != 0 || cs.C <= 0 || cs.ntaps < 1 || cs.ntaps > CD_MAX_TAPS) return 1;
    if (cs.W != d->Wg || cs.H != d->Hg) return 1;
    for (int t = 0; t < cs.ntaps; ++t) if (cs.dy[t] < -1 || cs.dy[t] > 1 || cs.dx[t] < -1 || cs.dx[t] > 1) return 1;
    if ((reinterpret_cast<uintptr_t>(cs.src) & 15) || (cs.ld * 4) % 16 || (reinterpret_cast<uintptr_t>(cs.w) & 15)) return 1;
  }
  if (MB == 2 && (d->Cout > 128 || (!(g_use_halo & 4) && (d->Hg < 32 || d->Wg < 32)))) return 1;
  if ((reinterpret_cast<uintptr_t>(d->out) & 15) || d->out_ld % 4) return 1;
  if (d->resid && ((reinterpret_cast<uintptr_t>(d->resid) & 15) || d->resid_ld % 4)) return 1;
  if (d->out2 && ((reinterpret_cast<uintptr_t>(d->out2) & 15) || d->out2_ld % 4)) return 1;
  if (d->bias && (reinterpret_cast<uintptr_t>(d->bias) & 15)) return 1;
  if (d->act == CD_ACT_GELU_BWD && (!d->aux || (reinterpret_cast<uintptr_t>(d->aux) & 15) || d->aux_ld % 4)) return 1;
  EncodeTiledFn enc = get_encode();
  CD_REQUIRE(enc != nullptr, "cuTensorMapEncodeTiled entry point unavailable");
  if (!g_num_sms) {
    int dev = 0; CD_CUDA(cudaGetDevice(&dev));
    CD_CUDA(cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev));
  }
  const int BN = (d->Cout % 256 == 0 && MB == 1) ? 256 : (d->Cout > 64 ? 128 : 64);
  const int TH = 8 * MB;
  TcParams p{};
  p.B = d->B; p.Hg = d->Hg; p.Wg = d->Wg; p.sy = 1; p.sx = 1; p.Cout = d->Cout; p.nsrc = d->nsrc;
  p.TW = kHaloW; p.TH = TH; p.TN = 1;
  p.tiles_x = cd_cdiv(d->Wg, kHaloW); p.tiles_y = cd_cdiv(d->Hg, TH); p.tiles_n = d->B;
  p.tiles_co = cd_cdiv(d->Cout, BN);
  p.total_tiles = p.tiles_x * p.tiles_y * p.tiles_n * p.tiles_co;
  p.out = d->out; p.out_ld = d->out_ld; p.Ho = d->Ho; p.Wo = d->Wo;
  p.oys = d->oys; p.oxs = d->oxs; p.oy0 = d->oy0; p.ox0 = d->ox0;
  p.bias = d->bias; p.resid = d->resid; p.resid_ld = d->resid_ld; p.act = d->act; p.round_tf32 = d->round_tf32;
  p.out2 = d->out2; p.out2_ld = d->out2_ld; p.aux = d->aux; p.aux_ld = d->aux_ld;
  CUtensorMap maps[4];
  for (int s = 0; s < 2; ++s) {
    const CdConvSrc& cs = d->s[s < d->nsrc ? s : 0];
    p.ntaps[s] = cs.ntaps; p.kchunks[s] = cs.C / kChunkK; p.wpb[s] = 0;
    for (int t = 0; t < cs.ntaps; ++t) { p.dy[s][t] = (int8_t)cs.dy[t]; p.dx[s][t] = (int8_t)cs.dx[t]; }
    {   // A: NHWC activations, one halo patch {32 ch, 18, TH + 2, 1} per chunk
      cuuint64_t dims[4] = {(cuuint64_t)cs.C, (cuuint64_t)cs.W, (cuuint64_t)cs.H, (cuuint64_t)d->B};
      cuuint64_t strides[3] = {(cuuint64_t)cs.ld * 4, (cuuint64_t)cs.ld * 4 * cs.W, (cuuint64_t)cs.ld * 4 * cs.W * cs.H};
      cuuint32_t box[4] = {(cuuint32_t)kChunkK, (cuuint32_t)(kHaloW + 2), (cuuint32_t)(TH + 2), 1};
      cuuint32_t estr[4] = {1, 1, 1, 1};
      CUresult r = enc(&maps[s], CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, const_cast<float*>(cs.src), dims, strides, box, estr,
                       CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                       CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
      CD_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(halo A%d) failed: %d", s, (int)r);
    }
    {   // B: packed weights [tap][Cout][Cin]
      cuuint64_t dims[3] = {(cuuint64_t)cs.C, (cuuint64_t)d->Cout, (cuuint64_t)cs.ntaps};
      cuuint64_t strides[2] = {(cuuint64_t)cs.C * 4, (cuuint64_t)cs.C * 4 * d->Cout};
      cuuint32_t box[3] = {(cuuint32_t)kChunkK, (cuuint32_t)BN, 1};
      cuuint32_t estr[3] = {1, 1, 1};
      CUresult r = enc(&maps[2 + s], CU_TENSOR_MAP_DATA_TYPE_TFLOAT32, 3, const_cast<float*>(cs.w), dims, strides, box, estr,
                       CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                       CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
      CD_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(halo B%d) failed: %d", s, (int)r);
    }
  }
  if (MB == 2) return BN == 128 ? launch_halo<128, 2, 4>(maps, p, st) : launch_halo<64, 2, 6>(maps, p, st);
  if (BN == 256) return launch_halo<256, 1, 4>(maps, p, st);
  if (BN == 128) return (g_ctas2 & 128) ? launch_halo<128, 1, 2, 2>(maps, p, st) : launch_halo<128, 1, 6>(maps, p, st);
  return (g_ctas2 & 64) ? launch_halo<64, 1, 3, 2>(maps, p, st) : launch_halo<64, 1, 8>(maps, p, st);
}
