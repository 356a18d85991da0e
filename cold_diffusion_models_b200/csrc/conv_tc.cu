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
  // shared-row kernel, per source: the dx of each box, the taps in column order (taps [boxend[b - 1], boxend[b]) read box b),
  // and each of those taps' byte offset inside its box
  int nbox[2];
  int8_t boxdx[2][3];
  int8_t boxend[2][3];
  int8_t taporder[2][CD_MAX_TAPS];
  int tapoff[2][CD_MAX_TAPS];
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
// Shared-row kernel for stride-1 convolutions whose taps lie in [-1, 1]^2 (dense 3x3 forward / data gradient, fused [3x3 | 1x1]
// pairs).  A CTA tile is 16 x 8 = 128 output pixels of one image by 64 or 128 output channels.  Per source and 32-channel
// chunk the producer fetches ONE 4-D TMA box {32 ch, 16, 8 + 2, 1} at (x0 + dx, y0 - 1) for each distinct tap column dx of
// that source (three for a 3x3 source, one for a 1x1 source).  Box row r = (y + 1) * 16 + x holds pixel (x0 + dx + x, y0 + y),
// so tap (dy, dx) reads the GEMM rows [64 w, 64 w + 64) of warpgroup w as the contiguous rows starting at (dy + 1) * 16 + 64 w
// of the dx box: a wgmma descriptor offset by a multiple of 1024 bytes (one SW128 atom), no registers involved.  Activations leave L2 once per (chunk, dx) instead
// of once per tap, and the TMA unit writes 160 pixel rows into shared memory per three taps instead of 3 x 128.
// The taps run grouped by column (p.taporder), so a box is released as soon as the taps of its column have retired: boxes
// stream through an ABOXES-deep ring, weight tiles through their own STAGES-deep ring.  Grids need not be multiples of the tile:
// pixels outside the grid are zero-filled on load and masked in the epilogue.
// ---------------------------------------------------------------------------------------------
constexpr int kRowsTW = 16, kRowsTH = kTileM / kRowsTW;
constexpr int kRowsBoxBytes = kRowsTW * (kRowsTH + 2) * 128;     // 20 KB: one tap column of one chunk

// TMA producer of both shared-row kernels (one elected thread of the producer warp): per tile of kRowsTW x TH pixels, source and
// 32-channel chunk, one box {32 ch, kRowsTW, TH + 2, 1} per tap column into the ABOXES-deep box ring, each followed by the weight
// tiles of that column's taps into the STAGES-deep weight ring
template <int BN, int TH, int ABOXES, int STAGES>
__device__ __forceinline__ void rows_producer(const CUtensorMap& mapA0, const CUtensorMap& mapA1, const CUtensorMap& mapB0,
                                              const CUtensorMap& mapB1, const TcParams& p, uint8_t* abox, uint8_t* wtile,
                                              uint64_t* afull, uint64_t* aempty, uint64_t* full_bar, uint64_t* empty_bar) {
  constexpr int kBBytes = BN * 128;
  constexpr int kBoxBytes = kRowsTW * (TH + 2) * 128;
  if (elect_one()) {
    uint32_t stage = 0, ph = 0, ai = 0, aph = 0;
    for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
      const int co0 = (tile % p.tiles_co) * BN;
      int mt = tile / p.tiles_co;
      const int x0 = (mt % p.tiles_x) * kRowsTW; mt /= p.tiles_x;
      const int y0 = (mt % p.tiles_y) * TH;
      const int n = mt / p.tiles_y;
      for (int s = 0; s < p.nsrc; ++s) {
        const CUtensorMap* mA = s ? &mapA1 : &mapA0;
        const CUtensorMap* mB = s ? &mapB1 : &mapB0;
        for (int kc = 0; kc < p.kchunks[s]; ++kc) {
          for (int b = 0, i = 0; b < p.nbox[s]; ++b) {
            mbar_wait(&aempty[ai], aph ^ 1u);
            mbar_expect_tx(&afull[ai], kBoxBytes);
            tma_load_4d(smem_u32(abox + ai * kBoxBytes), mA, &afull[ai], kc * kChunkK, x0 + p.boxdx[s][b], y0 - 1, n);
            if (++ai == ABOXES) { ai = 0; aph ^= 1u; }
            for (; i < p.boxend[s][b]; ++i) {
              mbar_wait(&empty_bar[stage], ph ^ 1u);
              mbar_expect_tx(&full_bar[stage], kBBytes);
              tma_load_3d(smem_u32(wtile + stage * kBBytes), mB, &full_bar[stage], kc * kChunkK, co0, p.taporder[s][i]);
              if (++stage == STAGES) { stage = 0; ph ^= 1u; }
            }
          }
        }
      }
    }
  }
  __syncwarp();
}

template <int BN, int ABOXES, int STAGES, int CTAS>
__global__ void __launch_bounds__(kThreads, CTAS)
conv_rows_kernel(const __grid_constant__ CUtensorMap mapA0, const __grid_constant__ CUtensorMap mapA1,
                 const __grid_constant__ CUtensorMap mapB0, const __grid_constant__ CUtensorMap mapB1, const __grid_constant__ TcParams p) {
  constexpr int kBBytes = BN * 128;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + ((1024u - (raw_addr & 1023u)) & 1023u);
  uint8_t* abox = smem;                                    // ABOXES activation boxes
  uint8_t* wtile = smem + ABOXES * kRowsBoxBytes;          // STAGES weight tiles
  uint64_t* bars = reinterpret_cast<uint64_t*>(wtile + STAGES * kBBytes);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + STAGES;
  uint64_t* afull = bars + 2 * STAGES;
  uint64_t* aempty = bars + 2 * STAGES + ABOXES;
  static_assert(2 * (STAGES + ABOXES) * 8 <= 256, "barrier block is 256 bytes");
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = threadIdx.x >> 7;
  if (threadIdx.x == 0) {
    for (int i = 0; i < STAGES; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], kConsumerWarps); }
    for (int i = 0; i < ABOXES; ++i) { mbar_init(&afull[i], 1); mbar_init(&aempty[i], kConsumerWarps); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == kConsumerWarps) {
    rows_producer<BN, kRowsTH, ABOXES, STAGES>(mapA0, mapA1, mapB0, mapB1, p, abox, wtile, afull, aempty, full_bar, empty_bar);
    return;
  }

  // ===================== consumers: warpgroup wg owns GEMM rows [64 wg, 64 wg + 64); row m = pixel (m % 16, m / 16) =====================
  const int tid = threadIdx.x & 127;
  const int rl = (tid >> 5) * 16 + (lane >> 2);
  const int q2 = (lane & 3) * 2;
  auto release = [&](uint64_t* bar) { __syncwarp(); if (lane == 0) mbar_arrive(bar); };
  float acc[BN / 2];
  uint32_t stage = 0, ph = 0, ai = 0, aph = 0;
  for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
    int k = 0;
    uint32_t prev = 0, prev_a = 0;
    for (int s = 0; s < p.nsrc; ++s) {
      for (int kc = 0; kc < p.kchunks[s]; ++kc) {
        for (int b = 0, i = 0; b < p.nbox[s]; ++b) {
          mbar_wait(&afull[ai], aph);
          const uint32_t abase = smem_u32(abox + ai * kRowsBoxBytes) + wg * (kABytes / 2);
          for (const int i0 = i; i < p.boxend[s][b]; ++i, ++k) {
            mbar_wait(&full_bar[stage], ph);
            wgmma_fence();
            const uint64_t da = make_kmajor_sw128_desc(abase + p.tapoff[s][i]);
            const uint64_t db = make_kmajor_sw128_desc(smem_u32(wtile + stage * kBBytes));
#pragma unroll
            for (int kk = 0; kk < 4; ++kk)
              wgmma_tf32<BN>(acc, da + uint64_t(kk * 2), db + uint64_t(kk * 2), (k | kk) != 0 ? 1u : 0u);
            wgmma_commit();
            wgmma_wait<1>();                         // the previous tap's MMAs have retired
            if (k > 0) release(&empty_bar[prev]);
            if (k > 0 && i == i0) release(&aempty[prev_a]);   // ... and with them every tap of the previous box
            prev = stage;
            if (++stage == STAGES) { stage = 0; ph ^= 1u; }
          }
          prev_a = ai;
          if (++ai == ABOXES) { ai = 0; aph ^= 1u; }
        }
      }
    }
    wgmma_wait<0>();
    if (k > 0) { release(&empty_bar[prev]); release(&aempty[prev_a]); }

    const int co0 = (tile % p.tiles_co) * BN;
    int mt = tile / p.tiles_co;
    const int x0 = (mt % p.tiles_x) * kRowsTW; mt /= p.tiles_x;
    const int y0 = (mt % p.tiles_y) * kRowsTH;
    const int n = mt / p.tiles_y;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int m = wg * 64 + rl + 8 * h;
      const int gx = x0 + m % kRowsTW, gy = y0 + m / kRowsTW;
      if (gx >= p.Wg || gy >= p.Hg) continue;
      const long long pix = (static_cast<long long>(n) * p.Ho + (gy * p.oys + p.oy0)) * p.Wo + (gx * p.oxs + p.ox0);
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) epi_pair(p, pix, co0 + 8 * j + q2, acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
    }
  }
}

// ---------------------------------------------------------------------------------------------
// Shared-row kernel with 16 x 16 pixel tiles: the problems, boxes and mainloop order of conv_rows_kernel, but a CTA tile is 256
// output pixels of one image by BN output channels at one CTA per SM, so every weight tile serves twice as many pixels.  Warpgroup
// w owns pixel rows 8 w .. 8 w + 7 (GEMM rows [128 w, 128 w + 128)) and issues two m64nBNk8 wgmmas per k step, one per 64-row
// half h.  Both warpgroups read the same weight tile and the same box {32 ch, 16, 16 + 2, 1}; tap (dy, dx) of half h of warpgroup
// w starts at byte (dy + 1) * 2 KB + w * 16 KB + h * 8 KB of its column's box, a whole number of SW128 atoms.  Every output
// element goes through the same wgmma sequence as in conv_rows_kernel, so the two kernels agree bit for bit.
// Epilogue: per 32-channel slice each warpgroup writes out (and out2) of its 128 pixels into SWIZZLE_128B staging slices, and one
// of its threads stores them with TMA tensor stores (the maps' bounds clip ragged tiles and Cout).  The consumers go on into the
// next tile's mainloop while the stores drain -- the overlap that the 16 x 8 kernel gets from two CTAs per SM.
// The epilogue operands come from shared memory: two otherwise idle producer warps, one per consumer warpgroup, copy the tile's
// bias values there and TMA-load the warpgroup's resid or aux pixels of each slice, in two halves of 64 pixels, into its out2
// staging slice.  A tile's first slice is loaded during its mainloop, each later half as soon as the previous slice's half has been
// used, so the epilogue no longer waits on dependent DRAM round trips.  (No engine launch with an operand writes out2; one that
// does overwrites the operand in place with out2 and frees the halves only once that store has read them.)
// ---------------------------------------------------------------------------------------------
constexpr int kR256TH = 16;
constexpr int kR256BoxBytes = kRowsTW * (kR256TH + 2) * 128;     // 36 KB: one tap column of one chunk
constexpr int kR256Slice = 128 * 128;                            // staging: 128 pixels x 32 fp32 channels = 16 KB
// warpgroup 0 = producer (warp 0 issues the TMA loads), warpgroups 1-2 = consumers.  Two 64 x BN accumulators per consumer thread
// do not fit the 168 registers of 384 threads, so setmaxnreg moves registers from the producer to the consumers.
constexpr int kR256Threads = 384;
constexpr int kR256RegsLow = 40, kR256RegsHigh = 232;          // 128 x 40 + 256 x 232 <= 64 K registers

// Epilogue barriers of one consumer warpgroup: the two operand halves (full, empty) and the bias values (full, empty)
constexpr int kOpFull = 0, kOpEmpty = 2, kBiasFull = 4, kBiasEmpty = 5, kEpiBars = 6;

// the one epilogue operand of a 16 x 16 launch (resid or GELU' aux; a launch with both is not eligible), nullptr without one
__host__ __device__ __forceinline__ const float* rows256_operand(const TcParams& p) {
  return p.resid ? p.resid : (p.act == CD_ACT_GELU_BWD ? p.aux : nullptr);
}

// Epilogue producer of consumer warpgroup cw (one warp of the producer warpgroup), tile by tile as the consumers walk them: the N
// tile's BN bias values into sbias (zeros from Cout on), then per 32-channel slice the warpgroup's two halves of 4 x 16 operand
// pixels, each into its half of the so2 slice.  The map's bounds zero-fill pixels outside the grid and channels from Cout on.
template <int BN>
__device__ __forceinline__ void rows256_epilogue_producer(const CUtensorMap& mapE, const TcParams& p, int cw, uint8_t* so2,
                                                          float* sbias, uint64_t* eb) {
  const int lane = threadIdx.x & 31;
  const bool opnd = rows256_operand(p) != nullptr;
  uint32_t bph = 0, oph = 0;                               // oph: parity bit of each half
  for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
    const int co0 = (tile % p.tiles_co) * BN;
    int mt = tile / p.tiles_co;
    const int x0 = (mt % p.tiles_x) * kRowsTW; mt /= p.tiles_x;
    const int yw = (mt % p.tiles_y) * kR256TH + 8 * cw;
    const int n = mt / p.tiles_y;
    if (yw >= p.Hg) continue;                              // the consumers skip this tile's epilogue too
    if (p.bias) {
      mbar_wait(&eb[kBiasEmpty], bph ^ 1u);
      for (int i = lane; i < BN; i += 32) sbias[i] = co0 + i < p.Cout ? p.bias[co0 + i] : 0.f;
      mbar_arrive(&eb[kBiasFull]);                         // one arrival per lane
      bph ^= 1u;
    }
    if (opnd && lane == 0) {
      for (int c = 0; c < BN / 32 && co0 + 32 * c < p.Cout; ++c)
        for (int h = 0; h < 2; ++h) {
          mbar_wait(&eb[kOpEmpty + h], ((oph >> h) & 1u) ^ 1u);
          mbar_expect_tx(&eb[kOpFull + h], kR256Slice / 2);
          tma_load_4d(smem_u32(so2 + h * (kR256Slice / 2)), &mapE, &eb[kOpFull + h], co0 + 32 * c, x0, yw + 4 * h, n);
          oph ^= 1u << h;
        }
    }
    __syncwarp();
  }
}

template <int BN, int ABOXES, int STAGES>
__global__ void __launch_bounds__(kR256Threads, 1)
conv_rows256_kernel(const __grid_constant__ CUtensorMap mapA0, const __grid_constant__ CUtensorMap mapA1,
                    const __grid_constant__ CUtensorMap mapB0, const __grid_constant__ CUtensorMap mapB1,
                    const __grid_constant__ CUtensorMap mapO, const __grid_constant__ CUtensorMap mapO2,
                    const __grid_constant__ CUtensorMap mapE, const __grid_constant__ TcParams p) {
  constexpr int kBBytes = BN * 128;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + ((1024u - (raw_addr & 1023u)) & 1023u);
  uint8_t* abox = smem;                                    // ABOXES activation boxes
  uint8_t* wtile = smem + ABOXES * kR256BoxBytes;          // STAGES weight tiles
  uint8_t* stg = wtile + STAGES * kBBytes;                 // per warpgroup: out slice, out2 (or operand) slice
  uint64_t* bars = reinterpret_cast<uint64_t*>(stg + 4 * kR256Slice);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + STAGES;
  uint64_t* afull = bars + 2 * STAGES;
  uint64_t* aempty = bars + 2 * STAGES + ABOXES;
  uint64_t* ebars = bars + 2 * (STAGES + ABOXES);          // kEpiBars per consumer warpgroup
  float* sbias = reinterpret_cast<float*>(bars + 32);      // after the 256-byte barrier block: BN bias values per warpgroup
  static_assert(2 * (STAGES + ABOXES) * 8 + 2 * kEpiBars * 8 <= 256, "barrier block is 256 bytes");
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = threadIdx.x >> 7;
  if (threadIdx.x == 0) {
    for (int i = 0; i < STAGES; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], kConsumerWarps); }
    for (int i = 0; i < ABOXES; ++i) { mbar_init(&afull[i], 1); mbar_init(&aempty[i], kConsumerWarps); }
    for (int w = 0; w < 2; ++w) {
      uint64_t* eb = ebars + w * kEpiBars;
      for (int h = 0; h < 2; ++h) { mbar_init(&eb[kOpFull + h], 1); mbar_init(&eb[kOpEmpty + h], kConsumerWarps / 2); }
      mbar_init(&eb[kBiasFull], 32);
      mbar_init(&eb[kBiasEmpty], kConsumerWarps / 2);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (wg == 0) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" :: "n"(kR256RegsLow));
    if (warp == 0)
      rows_producer<BN, kR256TH, ABOXES, STAGES>(mapA0, mapA1, mapB0, mapB1, p, abox, wtile, afull, aempty, full_bar, empty_bar);
    else if (warp <= 2 && (p.bias || rows256_operand(p)))
      rows256_epilogue_producer<BN>(mapE, p, warp - 1, stg + (warp - 1) * 2 * kR256Slice + kR256Slice, sbias + (warp - 1) * BN,
                                    ebars + (warp - 1) * kEpiBars);
    return;
  }
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" :: "n"(kR256RegsHigh));

  // ===================== consumers: warpgroup 1 + cw owns GEMM rows [128 cw, 128 cw + 128); row m = pixel (m % 16, m / 16) =====================
  const int cw = wg - 1;
  const int tid = threadIdx.x & 127;
  const int rl = (tid >> 5) * 16 + (lane >> 2);
  const int q2 = (lane & 3) * 2;
  const bool storer = tid == 0;                            // issues (and waits for) the warpgroup's bulk stores
  uint8_t* so = stg + cw * 2 * kR256Slice;
  uint8_t* so2 = so + kR256Slice;
  uint64_t* eb = ebars + cw * kEpiBars;
  const float* sb = sbias + cw * BN;
  const bool opnd = rows256_operand(p) != nullptr;
  auto release = [&](uint64_t* bar) { __syncwarp(); if (lane == 0) mbar_arrive(bar); };
  auto wg_sync = [&]() { asm volatile("bar.sync %0, 128;" :: "r"(1 + cw) : "memory"); };
  float acc[2][BN / 2];
  uint32_t stage = 0, ph = 0, ai = 0, aph = 0;
  uint32_t bph = 0, oph = 0;                               // parities of the bias barrier and of each operand half
  bool held = false;                                       // the operand halves hold the last slice's out2 until its store has read them
  for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
    int k = 0;
    uint32_t prev = 0, prev_a = 0;
    for (int s = 0; s < p.nsrc; ++s) {
      for (int kc = 0; kc < p.kchunks[s]; ++kc) {
        for (int b = 0, i = 0; b < p.nbox[s]; ++b) {
          mbar_wait(&afull[ai], aph);
          const uint32_t abase = smem_u32(abox + ai * kR256BoxBytes) + cw * kABytes;
          for (const int i0 = i; i < p.boxend[s][b]; ++i, ++k) {
            mbar_wait(&full_bar[stage], ph);
            wgmma_fence();
            const uint64_t da0 = make_kmajor_sw128_desc(abase + p.tapoff[s][i]);
            const uint64_t da1 = make_kmajor_sw128_desc(abase + p.tapoff[s][i] + kABytes / 2);
            const uint64_t db = make_kmajor_sw128_desc(smem_u32(wtile + stage * kBBytes));
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) {
              wgmma_tf32<BN>(acc[0], da0 + uint64_t(kk * 2), db + uint64_t(kk * 2), (k | kk) != 0 ? 1u : 0u);
              wgmma_tf32<BN>(acc[1], da1 + uint64_t(kk * 2), db + uint64_t(kk * 2), (k | kk) != 0 ? 1u : 0u);
            }
            wgmma_commit();
            wgmma_wait<1>();                         // the previous tap's MMAs have retired
            if (k > 0) release(&empty_bar[prev]);
            if (k > 0 && i == i0) release(&aempty[prev_a]);   // ... and with them every tap of the previous box
            prev = stage;
            if (++stage == STAGES) { stage = 0; ph ^= 1u; }
          }
          prev_a = ai;
          if (++ai == ABOXES) { ai = 0; aph ^= 1u; }
        }
      }
    }
    wgmma_wait<0>();
    if (k > 0) { release(&empty_bar[prev]); release(&aempty[prev_a]); }

    const int co0 = (tile % p.tiles_co) * BN;
    int mt = tile / p.tiles_co;
    const int x0 = (mt % p.tiles_x) * kRowsTW; mt /= p.tiles_x;
    const int yw = (mt % p.tiles_y) * kR256TH + 8 * cw;    // first pixel row of this warpgroup
    const int n = mt / p.tiles_y;
    if (yw >= p.Hg) continue;                              // ragged grid: no pixel of this warpgroup lies inside
    // local row r = 64 h + rl + 8 e (e: acc[4 j + 2 e], acc[4 j + 2 e + 1]) is pixel (x0 + r % 16, yw + r / 16); pixels outside
    // the grid and channels from Cout on are zero in the staged operands and clipped by the stores
    if (p.bias) { mbar_wait(&eb[kBiasFull], bph); bph ^= 1u; }
#pragma unroll
    for (int c = 0; c < BN / 32; ++c) {
      if (co0 + 32 * c >= p.Cout) break;
      if (storer) bulk_wait_read<0>();                     // the previous stores have read the staging slices
      wg_sync();
      if (held) { release(&eb[kOpEmpty]); release(&eb[kOpEmpty + 1]); held = false; }
      // epi_pair's arithmetic, one step at a time over the 8 column pairs of each half h of the slice: the branches on the epilogue
      // operands stay outside the element loops, so the 8 independent chains overlap
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        // SWIZZLE_128B staging: the 16-byte chunk (8 jj + q2) / 4 of local row rr lands at chunk ^ (rr % 8)
        auto soff = [&](int e, int jj) {
          const int rr = 64 * h + rl + 8 * e;
          return rr * 128 + ((((8 * jj + q2) >> 2) ^ (rr & 7)) << 4) + (q2 & 3) * 4;
        };
        // the operand (resid or aux) of this half, staged in so2 at the offsets out2 would take: read it before out2 overwrites it
        float2 o[2][4];
        if (opnd) {
          mbar_wait(&eb[kOpFull + h], (oph >> h) & 1u);
          oph ^= 1u << h;
#pragma unroll
          for (int e = 0; e < 2; ++e)
#pragma unroll
            for (int jj = 0; jj < 4; ++jj) o[e][jj] = *reinterpret_cast<const float2*>(so2 + soff(e, jj));
        }
        float2 v[2][4];
#pragma unroll
        for (int e = 0; e < 2; ++e)
#pragma unroll
          for (int jj = 0; jj < 4; ++jj) v[e][jj] = make_float2(acc[h][16 * c + 4 * jj + 2 * e], acc[h][16 * c + 4 * jj + 2 * e + 1]);
        if (p.bias) {
#pragma unroll
          for (int jj = 0; jj < 4; ++jj) {
            const float2 b = *reinterpret_cast<const float2*>(sb + 32 * c + 8 * jj + q2);
#pragma unroll
            for (int e = 0; e < 2; ++e) { v[e][jj].x += b.x; v[e][jj].y += b.y; }
          }
        }
        if (p.resid) {
#pragma unroll
          for (int e = 0; e < 2; ++e)
#pragma unroll
            for (int jj = 0; jj < 4; ++jj) { v[e][jj].x += o[e][jj].x; v[e][jj].y += o[e][jj].y; }
        }
        if (p.out2) {
#pragma unroll
          for (int e = 0; e < 2; ++e)
#pragma unroll
            for (int jj = 0; jj < 4; ++jj) *reinterpret_cast<float2*>(so2 + soff(e, jj)) = v[e][jj];
        }
        if (p.act == CD_ACT_GELU) {
#pragma unroll
          for (int e = 0; e < 2; ++e)
#pragma unroll
            for (int jj = 0; jj < 4; ++jj) { v[e][jj].x = cd_gelu(v[e][jj].x); v[e][jj].y = cd_gelu(v[e][jj].y); }
        } else if (p.act == CD_ACT_GELU_BWD) {
#pragma unroll
          for (int e = 0; e < 2; ++e)
#pragma unroll
            for (int jj = 0; jj < 4; ++jj) { v[e][jj].x *= cd_gelu_grad(o[e][jj].x); v[e][jj].y *= cd_gelu_grad(o[e][jj].y); }
        }
        if (p.round_tf32) {
#pragma unroll
          for (int e = 0; e < 2; ++e)
#pragma unroll
            for (int jj = 0; jj < 4; ++jj) { v[e][jj].x = cd_round_tf32(v[e][jj].x); v[e][jj].y = cd_round_tf32(v[e][jj].y); }
        }
#pragma unroll
        for (int e = 0; e < 2; ++e)
#pragma unroll
          for (int jj = 0; jj < 4; ++jj) *reinterpret_cast<float2*>(so + soff(e, jj)) = v[e][jj];
        // The half may be refilled once every warp's reads of it have completed.  An arrive does not wait for shared-memory loads
        // still in flight, so it comes after the stores above, which consume every loaded value.
        if (opnd && !p.out2) release(&eb[kOpEmpty + h]);
      }
      fence_proxy_async();                                 // the staging writes precede the bulk stores' reads
      wg_sync();
      if (storer) {
        tma_store_4d(&mapO, smem_u32(so), co0 + 32 * c, x0, yw, n);
        if (p.out2) tma_store_4d(&mapO2, smem_u32(so2), co0 + 32 * c, x0, yw, n);
        bulk_commit();
      }
      held = opnd && p.out2;
    }
    if (p.bias) release(&eb[kBiasEmpty]);
  }
  if (storer) bulk_wait<0>();
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------

int g_tf32_map_dtype = 1;   // 1: TFLOAT32 tensor maps; 0: FLOAT32 (diagnostic, cd_conv_tc_set_tf32_maps)

// Persistent launch of either kernel: at most CTAS CTAs per SM walk the tiles round-robin (PAIR: clusters of two CTAs over the
// (M tile pair, co tile) units, one cluster per SM pair)
template <auto Kernel, size_t kSmem, int CTAS, bool PAIR = false>
int launch_persistent(const CUtensorMap* maps, const TcParams& p, cudaStream_t st) {
  static_assert(kSmem <= 232448, "dynamic shared memory of one CTA (227 KB)");
  static_assert(CTAS == 1 || 2 * (kSmem + 1024) <= 233472, "two CTAs per SM must fit the 228 KB of shared memory");
  CD_CUDA(smem_limit_once<Kernel>(kSmem));
  if constexpr (PAIR) {
    const int units = p.tiles_co * ((p.total_tiles / p.tiles_co + 1) / 2), slots = cd_num_sms() / 2;
    cudaLaunchConfig_t cfg = {};
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = 2; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
    cfg.gridDim = dim3(2 * (units < slots ? units : slots)); cfg.blockDim = dim3(kThreads);
    cfg.dynamicSmemBytes = kSmem; cfg.stream = st; cfg.attrs = attr; cfg.numAttrs = 1;
    CD_CUDA(cudaLaunchKernelEx(&cfg, Kernel, maps[0], maps[1], maps[2], maps[3], p));
  } else {
    const int slots = cd_num_sms() * CTAS;
    const int grid = p.total_tiles < slots ? p.total_tiles : slots;
    Kernel<<<grid, kThreads, kSmem, st>>>(maps[0], maps[1], maps[2], maps[3], p);
  }
  CD_LAUNCH_CHECK();
  return 0;
}

template <int BN, int STAGES, bool STG = false, bool F16 = false, int CTAS = 1, bool PAIR = false>
int launch(const CUtensorMap* maps, const TcParams& p, cudaStream_t st) {
  constexpr size_t smem = size_t(STAGES) * (kABytes + BN * 128) + 1024 + 256 + (STG ? sizeof(float) * 2 * 64 * kEpiStageStride : 0);
  return launch_persistent<conv_tc_kernel<BN, STAGES, STG, F16, CTAS, PAIR>, smem, CTAS, PAIR>(maps, p, st);
}

template <int BN, int ABOXES, int STAGES, int CTAS = 1>
int launch_rows(const CUtensorMap* maps, const TcParams& p, cudaStream_t st) {
  constexpr size_t smem = size_t(ABOXES) * kRowsBoxBytes + size_t(STAGES) * BN * 128 + 1024 + 256;
  return launch_persistent<conv_rows_kernel<BN, ABOXES, STAGES, CTAS>, smem, CTAS>(maps, p, st);
}

// maps: A0, A1, B0, B1, out, out2, epilogue operand (one CTA per SM)
template <int BN, int ABOXES, int STAGES>
int launch_rows256(const CUtensorMap* maps, const TcParams& p, cudaStream_t st) {
  constexpr size_t smem = size_t(ABOXES) * kR256BoxBytes + size_t(STAGES) * BN * 128 + 4 * kR256Slice + 256 + 2 * BN * 4 + 1024;
  static_assert(smem <= 232448, "dynamic shared memory of one CTA (227 KB)");
  constexpr auto kernel = conv_rows256_kernel<BN, ABOXES, STAGES>;
  CD_CUDA(smem_limit_once<kernel>(smem));
  const int sms = cd_num_sms();
  const int grid = p.total_tiles < sms ? p.total_tiles : sms;
  kernel<<<grid, kR256Threads, smem, st>>>(maps[0], maps[1], maps[2], maps[3], maps[4], maps[5], maps[6], p);
  CD_LAUNCH_CHECK();
  return 0;
}

// Operand conditions of both kernels: nsrc, 16-byte aligned operands, source channels in whole chunks of chunk_elems and a tap
// count the descriptor can hold.  With `report` the first failed condition becomes the library's last error.
bool operands_ok(const CdConvDesc* d, int chunk_elems, int esz, bool report) {
#define TC_CHECK(cond, ...) do { if (!(cond)) { if (report) cd_set_error(__VA_ARGS__); return false; } } while (0)
  TC_CHECK(d->nsrc >= 1 && d->nsrc <= 2, "conv_tc: nsrc must be 1 or 2");
  TC_CHECK(d->act != CD_ACT_GELU_BWD || (d->aux && (reinterpret_cast<uintptr_t>(d->aux) & 15) == 0 && d->aux_ld % 4 == 0), "conv_tc: GELU_BWD needs an aligned aux");
  TC_CHECK((reinterpret_cast<uintptr_t>(d->out) & 15) == 0 && d->out_ld % 4 == 0, "conv_tc: out must be 16B aligned");
  TC_CHECK(!d->resid || ((reinterpret_cast<uintptr_t>(d->resid) & 15) == 0 && d->resid_ld % 4 == 0), "conv_tc: resid alignment");
  TC_CHECK(!d->out2 || ((reinterpret_cast<uintptr_t>(d->out2) & 15) == 0 && d->out2_ld % 4 == 0), "conv_tc: out2 alignment");
  TC_CHECK(!d->bias || (reinterpret_cast<uintptr_t>(d->bias) & 15) == 0, "conv_tc: bias alignment");
  for (int s = 0; s < d->nsrc; ++s) {
    const CdConvSrc& cs = d->s[s];
    TC_CHECK(cs.C % chunk_elems == 0 && cs.C > 0, "conv_tc: source channels %d not a multiple of %d", cs.C, chunk_elems);
    TC_CHECK(cs.ntaps >= 1 && cs.ntaps <= CD_MAX_TAPS, "conv_tc: bad ntaps");
    TC_CHECK((reinterpret_cast<uintptr_t>(cs.src) & 15) == 0 && (cs.ld * esz) % 16 == 0, "conv_tc: src must be 16B aligned");
    TC_CHECK((reinterpret_cast<uintptr_t>(cs.w) & 15) == 0, "conv_tc: weights must be 16B aligned");
  }
#undef TC_CHECK
  return true;
}

// the TcParams fields both kernels take from the descriptor as they are: grid, strides, taps, output and epilogue operands
// (a single source fills the second slot with the first)
TcParams desc_params(const CdConvDesc* d, int chunk_elems) {
  TcParams p{};
  p.B = d->B; p.Hg = d->Hg; p.Wg = d->Wg; p.sy = d->sy; p.sx = d->sx; p.Cout = d->Cout; p.nsrc = d->nsrc;
  for (int s = 0; s < 2; ++s) {
    const CdConvSrc& cs = d->s[s < d->nsrc ? s : 0];
    p.ntaps[s] = cs.ntaps; p.kchunks[s] = cs.C / chunk_elems; p.wpb[s] = cs.w_per_batch;
    for (int t = 0; t < cs.ntaps; ++t) { p.dy[s][t] = (int8_t)cs.dy[t]; p.dx[s][t] = (int8_t)cs.dx[t]; }
  }
  p.out = d->out; p.out_ld = d->out_ld; p.Ho = d->Ho; p.Wo = d->Wo;
  p.oys = d->oys; p.oxs = d->oxs; p.oy0 = d->oy0; p.ox0 = d->ox0;
  p.bias = d->bias; p.resid = d->resid; p.resid_ld = d->resid_ld; p.act = d->act; p.round_tf32 = d->round_tf32;
  p.out2 = d->out2; p.out2_ld = d->out2_ld; p.aux = d->aux; p.aux_ld = d->aux_ld;
  return p;
}

}  // namespace

extern "C" int cd_conv_tc_set_tf32_maps(int enable) { g_tf32_map_dtype = enable ? 1 : 0; return 0; }

// Defaults measured with tools/conv_shapes.py and bench.py on an H100 80GB HBM3 at a 400 W power limit (Unet config 3, batch 32).
// Per-tap kernel: 80 ms of convolution forward + data-gradient time per training step at one CTA per SM, 74 ms with two CTAs per
// SM for the 64- and 128-wide N tiles (375 -> 387 images/s); the SM-pair kernel took 87 ms.  The shared-row kernel cuts the
// modelled L2 -> SM bytes of the 3x3 layers 1.2-1.6x; what gains most, though, is that its 128-wide N tiles fit two CTAs per SM
// for the layers with Cout >= 256 too (a CTA's epilogue then overlaps the other's mainloop): 20-48 % faster on those layers
// than the per-tap kernel's 256-wide tiles, 0-10 % on the narrower ones.  16 x 16 pixel tiles (conv_rows256_kernel, one CTA per SM) are faster still wherever they fill most of a wave (see conv_fwd_rows).
// A single wave of tiles (16^2, Cout = 256) stays per-tap, and two CTAs per SM are used only with more than one wave of tiles.
static int g_use_2cta = 0;
extern "C" int cd_conv_tc_set_2cta(int mode) { g_use_2cta = mode; return 0; }   // 0 off, 1 where the cost model prefers it, 2 wherever eligible
// narrower pair tiles: bit mask of the N tiles below 256 (128 | 64) that go to the SM-pair kernel when the problem is eligible
static int g_2cta_bn = 0;
extern "C" int cd_conv_tc_set_2cta_bn(int mask) { g_2cta_bn = mask & (128 | 64); return 0; }
// kernel for stride-1 convolutions with taps in [-1, 1]^2: 0 = shape-based choice between the shared-row kernels and the per-tap
// kernel (default), 1, 2 or 6 = shared-row kernel with 16 x 8 tiles wherever eligible, 4 = shared-row kernel with 16 x 16 tiles
// wherever eligible, 8 = per-tap kernel everywhere
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

static int conv_fwd_rows(const CdConvDesc* d, cudaStream_t st, int mode);

static int conv_fwd_tc_impl(const CdConvDesc* d, cudaStream_t st, bool f16) {
  if (!f16 && g_epi_staged == 0) {
    // shared-row kernels: chosen by shape (0; the SM-pair switch keeps the per-tap family) or wherever eligible (1, 2, 4, 6)
    if ((g_use_halo == 0 && !g_use_2cta) || g_use_halo == 1 || g_use_halo == 2 || g_use_halo == 4 || g_use_halo == 6) {
      const int r = conv_fwd_rows(d, st, g_use_halo);
      if (r <= 0) return r;                                   // 1 = not eligible
    }
  }
  const CUtensorMapDataType dt = f16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : (g_tf32_map_dtype ? CU_TENSOR_MAP_DATA_TYPE_TFLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32);
  const int esz = map_elem_bytes(dt), chunk_elems = 128 / esz;
  if (!operands_ok(d, chunk_elems, esz, true)) return -1;
  TcParams p = desc_params(d, chunk_elems);
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
  const int sms = cd_num_sms();
  if (BN == 256) {
    // small spatial sizes (16^2, 32^2) give few M tiles: take the narrower N tile only when it saves whole waves
    double best = tc_cost(mt, d->Cout, 256, sms);
    if (tc_cost(mt, d->Cout, 128, sms) < best) { BN = 128; best = tc_cost(mt, d->Cout, 128, sms); }
    if (!f16 && !staged && g_use_2cta && mt >= 2 && (g_use_2cta == 2 || tc_cost(mt, d->Cout, 256, sms, true) < best)) {
      BN = 256; pair = true;
    }
  } else if (!f16 && !staged && g_use_2cta && (g_2cta_bn & BN) && d->Cout % BN == 0 && (g_use_2cta == 2 || mt >= 2 * sms)) {
    pair = true;                                              // narrow pair tile: only with at least one pair tile per SM pair
  }
  p.tiles_co = cd_cdiv(d->Cout, BN);
  p.total_tiles = p.tiles_x * p.tiles_y * p.tiles_n * p.tiles_co;

  CUtensorMap maps[4];
  for (int s = 0; s < 2; ++s) {
    const CdConvSrc& cs = d->s[s < d->nsrc ? s : 0];
    CD_REQUIRE(!cs.w_per_batch || p.TN == 1, "conv_tc: per-batch weights need >=128 pixels per image");
    // B: per-batch weight sets follow one another along the tap axis; in SM-pair mode each CTA fetches half of the tile
    if (!encode_nhwc(&maps[s], dt, cs.src, cs.ld, cs.C, cs.W, cs.H, d->B, 1, 1, 0, 0, p.TW * d->sx, p.TH * d->sy, p.TN, d->sx, d->sy,
                     s ? "A1" : "A0") ||
        !encode_weights(&maps[2 + s], dt, cs.w, cs.C, d->Cout, cs.ntaps * (cs.w_per_batch ? d->B : 1), pair ? BN / 2 : BN,
                        s ? "B1" : "B0"))
      return -1;
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
  // two CTAs per SM only with more than one wave of tiles: a single wave would pair CTAs on some SMs and leave others idle
  const int ctas2 = p.total_tiles > sms ? g_ctas2 : 0;
  if (BN == 256) return launch<256, 4>(maps, p, st);
  if (BN == 128) return (ctas2 & 128) ? launch<128, 3, false, false, 2>(maps, p, st) : launch<128, 6>(maps, p, st);
  return (ctas2 & 64) ? launch<64, 4, false, false, 2>(maps, p, st) : launch<64, 8>(maps, p, st);
}

// returns 1 when the problem is not eligible for the shared-row kernel -- it needs stride 1, taps in [-1, 1]^2 and a first source
// whose tap columns hold three taps each on average (dense 3x3; 1x1 and transposed-convolution parity tap lists stay per-tap) --
// or, in mode 0 (shape-based choice), when the per-tap kernel is the faster one for this shape (see the measurement above
// g_use_2cta).  Mode 4 takes the 16 x 16 tiles wherever they are eligible, modes 1, 2 and 6 the 16 x 8 tiles.
static int conv_fwd_rows(const CdConvDesc* d, cudaStream_t st, int mode) {
  const bool by_shape = mode == 0;
  if (d->sy != 1 || d->sx != 1 || !operands_ok(d, kChunkK, 4, false)) return 1;
  for (int s = 0; s < d->nsrc; ++s) {
    const CdConvSrc& cs = d->s[s];
    if (cs.w_per_batch || cs.W != d->Wg || cs.H != d->Hg) return 1;
    for (int t = 0; t < cs.ntaps; ++t) if (cs.dy[t] < -1 || cs.dy[t] > 1 || cs.dx[t] < -1 || cs.dx[t] > 1) return 1;
  }
  TcParams p = desc_params(d, kChunkK);
  p.TW = kRowsTW; p.TH = kRowsTH; p.TN = 1;
  p.tiles_x = cd_cdiv(d->Wg, kRowsTW); p.tiles_y = cd_cdiv(d->Hg, kRowsTH); p.tiles_n = d->B;
  // N tiles of at most 128 columns: two CTAs per SM fit (three boxes and three / six weight tiles each), so one CTA's epilogue
  // overlaps the other's mainloop.  For the layers with Cout >= 256 this beats the 256-wide tile at one CTA per SM by 20-45 %,
  // although every activation box is then fetched once per 128 output channels.
  const int BN = d->Cout > 64 ? 128 : 64;
  p.tiles_co = cd_cdiv(d->Cout, BN);
  p.total_tiles = p.tiles_x * p.tiles_y * p.tiles_n * p.tiles_co;
  // by shape: when the tiles fill more than one wave (a single wave, e.g. the 16^2 layers with Cout = 256, runs faster on the
  // per-tap kernel)
  const int sms = cd_num_sms();
  if (by_shape && p.total_tiles <= sms) return 1;
  // 16 x 16 tiles: the output is stored by TMA through a map over the grid itself (no output pixel map), so the grid must be the
  // output.  By shape with at least three quarters of a wave of 256-pixel tiles: measured with tools/conv_shapes.py on an H100 80GB
  // HBM3 at a 700 W power limit (1980 MHz, Unet config 3, batch 32), the 16 x 16 kernel is 4-54 % faster than the 16 x 8 kernel at
  // two CTAs per SM on every 3x3 forward and data-gradient layer with 128 or more such tiles (e.g. 393 against 804 us for 128^2,
  // Cout = 128, K = 576; 993 against 1154 us for its data gradient) but for one (+5 %, 16^2 data gradient, Cout = 512, K = 2304),
  // and 17-36 % slower with 64 tiles (16^2, Cout = 256), which stay on the per-tap kernel anyway.  The 3x3 forward + data-gradient
  // convolutions of one micro-batch take 23.5 ms instead of 27.2 ms.
  const int tiles256 = p.tiles_x * cd_cdiv(d->Hg, kR256TH) * p.tiles_n * p.tiles_co;
  // The 16 x 16 kernel stages at most one epilogue operand per slice, so a launch with both resid and aux takes the 16 x 8 tiles.
  // Its TMA output stores clip the channel dimension only in 16-byte units: with Cout % 4 != 0 they write zeros into the output
  // row up to the next multiple of 4 channels (the Model's 3-channel conv_out, or the live columns of a neighbouring slice), so
  // such a launch takes the 16 x 8 tiles, whose epilogue stores element by element.
  const bool rows256 = (mode == 4 || (by_shape && 4 * tiles256 >= 3 * sms)) && d->oys == 1 && d->oxs == 1 && d->oy0 == 0 &&
                       d->ox0 == 0 && d->Ho == d->Hg && d->Wo == d->Wg && !(d->resid && d->act == CD_ACT_GELU_BWD) &&
                       d->Cout % 4 == 0;
  if (rows256) { p.TH = kR256TH; p.tiles_y = cd_cdiv(d->Hg, kR256TH); p.total_tiles = tiles256; }
  const CUtensorMapDataType dt = g_tf32_map_dtype ? CU_TENSOR_MAP_DATA_TYPE_TFLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
  CUtensorMap maps[7] = {};
  for (int s = 0; s < 2; ++s) {
    const CdConvSrc& cs = d->s[s < d->nsrc ? s : 0];
    int i = 0;
    for (int dx = -1; dx <= 1; ++dx) {                       // taps grouped by column: one box per column present
      const int i0 = i;
      for (int t = 0; t < cs.ntaps; ++t)
        if (cs.dx[t] == dx) { p.taporder[s][i] = (int8_t)t; p.tapoff[s][i] = (cs.dy[t] + 1) * kRowsTW * 128; ++i; }
      if (i > i0) { p.boxdx[s][p.nbox[s]] = (int8_t)dx; p.boxend[s][p.nbox[s]] = (int8_t)i; ++p.nbox[s]; }
    }
    if (s == 0 && cs.ntaps < 3 * p.nbox[0]) return 1;
    // A: one box {32 ch, 16, TH + 2, 1} per chunk and tap column
    if (!encode_nhwc(&maps[s], dt, cs.src, cs.ld, cs.C, cs.W, cs.H, d->B, 1, 1, 0, 0, kRowsTW, p.TH + 2, 1, 1, 1,
                     s ? "rows A1" : "rows A0") ||
        !encode_weights(&maps[2 + s], dt, cs.w, cs.C, d->Cout, cs.ntaps, BN, s ? "rows B1" : "rows B0"))
      return -1;
  }
  if (rows256) {
    // out / out2: one warpgroup's box {32 ch, 16, 8, 1} per store, fp32 bits as computed
    const float* o2 = d->out2 ? d->out2 : d->out;
    const int o2ld = d->out2 ? d->out2_ld : d->out_ld;
    if (!encode_nhwc(&maps[4], CU_TENSOR_MAP_DATA_TYPE_FLOAT32, d->out, d->out_ld, d->Cout, d->Wg, d->Hg, d->B, 1, 1, 0, 0, kRowsTW,
                     kR256TH / 2, 1, 1, 1, "rows out") ||
        !encode_nhwc(&maps[5], CU_TENSOR_MAP_DATA_TYPE_FLOAT32, o2, o2ld, d->Cout, d->Wg, d->Hg, d->B, 1, 1, 0, 0, kRowsTW,
                     kR256TH / 2, 1, 1, 1, "rows out2"))
      return -1;
    // resid / aux: half a warpgroup's slice {32 ch, 16, 4, 1} per load, fp32 bits as stored (operands_ok: 16-byte aligned base
    // and pixel stride)
    const float* opnd = rows256_operand(p);
    const int opnd_ld = d->resid ? d->resid_ld : d->aux_ld;
    if (opnd && !encode_nhwc(&maps[6], CU_TENSOR_MAP_DATA_TYPE_FLOAT32, opnd, opnd_ld, d->Cout, d->Wg, d->Hg, d->B, 1, 1, 0, 0,
                             kRowsTW, kR256TH / 4, 1, 1, 1, "rows operand"))
      return -1;
    // three boxes (108 KB), 48 KB of weight tiles, 64 KB of staging slices and the bias values
    if (BN == 128) return launch_rows256<128, 3, 3>(maps, p, st);
    return launch_rows256<64, 3, 6>(maps, p, st);
  }
  // one CTA per SM: six boxes (120 KB) and 64 KB of weight tiles; two CTAs per SM: three boxes and 48 KB of weight tiles each
  const int ctas2 = p.total_tiles > sms ? g_ctas2 : 0;
  if (BN == 128) return (ctas2 & 128) ? launch_rows<128, 3, 3, 2>(maps, p, st) : launch_rows<128, 6, 4>(maps, p, st);
  return (ctas2 & 64) ? launch_rows<64, 3, 6, 2>(maps, p, st) : launch_rows<64, 6, 8>(maps, p, st);
}
