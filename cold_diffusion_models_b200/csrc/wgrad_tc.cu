// Tensor-core weight gradient of the tap-list convolution (replaces cuDNN wgrad behind loss.backward() for the
// dense convolutions of the reference Unet, DB:149-154,173-174,105-109):
//
//   dW[tap][co][ci] += sum_{pixels p} dY[p][co] * X[p (+) tap][ci]
//
// as a GEMM whose K dimension is the PIXEL axis.  NHWC rows hold the channels contiguously, i.e. both operands are
// MN-major, which TF32 wgmma cannot read from shared memory; the MMAs are therefore mma.sync.m16n8k8 (TF32, fp32
// accumulate) with their fragments read from the swizzled TMA tiles.  dY tiles ({32 co, CW px, R rows} TMA boxes) and
// X tiles land in SWIZZLE_128B shared memory.  One CTA owns (co tile, ci tile, tap group, pixel split) and keeps one
// register accumulator per tap of its group; with `halo` mode the dx = -1/0/+1 taps of a 3x3 kernel share ONE X tile
// that carries a one-pixel halo and are addressed by shifting the pixel row.  Partial sums of the pixel splits are
// combined with vector red.global.add.f32.
#include "tc_common.cuh"

namespace {

constexpr int kMmaWarps = 8;                      // 4 (co) x 2 (ci) warps, 32 co x BN/2 ci each
constexpr int kThreads = 32 * (kMmaWarps + 1);    // + warp 8: TMA producer
constexpr int kMaxTaps = 4;      // taps (accumulators) per CTA
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
  int tap_shift[kMaxGroups][kMaxTaps];    // pixel-row shift inside the (halo) X tile
  int load_dy[kMaxGroups][kMaxTaps], load_dx[kMaxGroups][kMaxTaps];
  int halo;                       // extra pixels per row in the X box (0 or 2)
  int sy, sx;                     // X coordinate = g*s + d
  int oys, oxs, oy0, ox0;         // dY coordinate = g*os + o0
  int per_batch, chunks_per_img, splits_per_img;   // per-batch weights: splits never cross images
  long long dw_batch_stride;
  float* dw;
  float* db;                      // BIAS kernels only: db[co] += sum over all pixels of dY (nullptr: not fused)
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


int g_wg_mode = 1;      // 0: one X tile per tap; otherwise (default) the dx taps of a 3x3 kernel share one halo tile
int g_sms = 0;

template <int BN, int NT>
int launch_wg(bool bias, dim3 grid, size_t smem, cudaStream_t st, const CUtensorMap& mapDY, const CUtensorMap& mapX,
              const WgParams& p, int stages, int a_bytes, int b_bytes, int b_tx) {
  if (bias) {
    CD_CUDA(cudaFuncSetAttribute(wgrad_tc_kernel<BN, NT, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    wgrad_tc_kernel<BN, NT, true><<<grid, kThreads, smem, st>>>(mapDY, mapX, p, stages, a_bytes, b_bytes, b_tx);
  } else {
    CD_CUDA(cudaFuncSetAttribute(wgrad_tc_kernel<BN, NT, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    wgrad_tc_kernel<BN, NT, false><<<grid, kThreads, smem, st>>>(mapDY, mapX, p, stages, a_bytes, b_bytes, b_tx);
  }
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

static int choose_splits(int tg, int total_chunks, int max_splits, int sms, double chunk_clk) {
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

// returns 1 if the problem is not tensor-core shaped (caller falls back to the SIMT kernel), 0 on success, <0 on error
int cd_conv_wgrad_tc(const CdConvDesc* d, const float* dout, int dout_ld, float* dw, float* db, int* bias_done, cudaStream_t st) {
  if (bias_done) *bias_done = 0;
  const CdConvSrc& c = d->s[0];
  if (c.C % 32 != 0 || d->Cout % 32 != 0 || c.ld % 4 != 0 || dout_ld % 4 != 0) return 1;
  if (!is_pow2(d->Wg) || d->Wg < 8 || !is_pow2(d->Hg)) return 1;
  if ((reinterpret_cast<uintptr_t>(c.src) & 15) || (reinterpret_cast<uintptr_t>(dout) & 15) || (reinterpret_cast<uintptr_t>(dw) & 15)) return 1;
  EncodeTiledFn enc = get_encode();
  CD_REQUIRE(enc != nullptr, "cuTensorMapEncodeTiled entry point unavailable");
  if (!g_sms) { int dev = 0; CD_CUDA(cudaGetDevice(&dev)); CD_CUDA(cudaDeviceGetAttribute(&g_sms, cudaDevAttrMultiProcessorCount, dev)); }

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
    const int spi0 = choose_splits(tiles * p.ngroups * d->B, cpi, cpi, g_sms, chunk_clk);
    splits = spi0 * d->B;
  } else {
    splits = choose_splits(tiles * p.ngroups, p.total_chunks, cd_cdiv(p.total_chunks, 8), g_sms, chunk_clk);
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
  {
    cuuint64_t dims[4] = {(cuuint64_t)d->Cout, (cuuint64_t)d->Wo, (cuuint64_t)d->Ho, (cuuint64_t)d->B};
    cuuint64_t strides[3] = {(cuuint64_t)dout_ld * 4, (cuuint64_t)dout_ld * 4 * d->Wo, (cuuint64_t)dout_ld * 4 * d->Wo * d->Ho};
    cuuint32_t box[4] = {32, (cuuint32_t)(p.CW * d->oxs), (cuuint32_t)(p.R * d->oys), 1};
    cuuint32_t estr[4] = {1, (cuuint32_t)d->oxs, (cuuint32_t)d->oys, 1};
    CUresult r = enc(&mapDY, dt, 4, const_cast<float*>(dout), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    CD_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(dY) failed: %d", (int)r);
  }
  {
    cuuint64_t dims[4] = {(cuuint64_t)c.C, (cuuint64_t)c.W, (cuuint64_t)c.H, (cuuint64_t)d->B};
    cuuint64_t strides[3] = {(cuuint64_t)c.ld * 4, (cuuint64_t)c.ld * 4 * c.W, (cuuint64_t)c.ld * 4 * c.W * c.H};
    cuuint32_t box[4] = {32, (cuuint32_t)((p.CW + p.halo) * d->sx), (cuuint32_t)(p.R * d->sy), 1};
    cuuint32_t estr[4] = {1, (cuuint32_t)d->sx, (cuuint32_t)d->sy, 1};
    CUresult r = enc(&mapX, dt, 4, const_cast<float*>(c.src), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    CD_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(X) failed: %d", (int)r);
  }
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
