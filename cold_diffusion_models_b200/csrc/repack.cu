// Batched weight repacks: every convolution weight of the network (reference layout OIHW / IOHW -> packed [tap][N][K]) and
// every packed weight gradient (-> reference layout, accumulating) in ONE launch each.  The single-weight entry points
// (cd_pack_weight / cd_unpack_wgrad, conv_simt.cu) cost one launch per weight: 64 + 98 latency-bound launches per optimizer
// step for ~0.9 GB of traffic.
// Here a block finds its job by a binary search over the ascending block0 column of a device-resident job table and
// then does exactly what the single-weight kernels do for one tile.
#include "cd_common.cuh"

namespace {

constexpr int kTileRows = 256;
constexpr int kMaxKHW = 16;

struct JobRef { int j; int lb; };     // job index and block index inside the job

__device__ __forceinline__ JobRef find_job(const CdRepackJob* __restrict__ jobs, int njobs) {
  int lo = 0, hi = njobs - 1;
  const int bx = static_cast<int>(blockIdx.x);
  while (lo < hi) {                                  // last job with block0 <= bx
    const int mid = (lo + hi + 1) >> 1;
    if (jobs[mid].block0 <= bx) lo = mid; else hi = mid - 1;
  }
  JobRef r; r.j = lo; r.lb = bx - jobs[lo].block0;
  return r;
}

// Conv2d (O,I,KH,KW) <-> packed [tap][O][I] through a shared-memory tile of 256 (o,i) rows x KH*KW taps: both sides coalesced
__global__ void __launch_bounds__(256)
pack_weight_batched_kernel(const CdRepackJob* __restrict__ jobs, int njobs) {
  __shared__ float tile[kTileRows * (kMaxKHW + 1)];
  __shared__ int tapk[CD_MAX_TAPS];
  const JobRef jr = find_job(jobs, njobs);
  const CdRepackJob& jb = jobs[jr.j];
  if (jr.lb >= jb.nblocks) return;
  const int O = jb.O, I = jb.I, KH = jb.KH, KW = jb.KW, ntaps = jb.ntaps, mode = jb.mode, tr = jb.transposed_conv;
  const int round_tf32 = jb.round_tf32;
  const float* __restrict__ w = jb.src;
  float* __restrict__ packed = jb.dst;
  const int KHW = KH * KW;
  if (!tr && mode == 0 && KHW <= kMaxKHW) {
    if (threadIdx.x < ntaps) tapk[threadIdx.x] = jb.ky[threadIdx.x] * KW + jb.kx[threadIdx.x];
    const int stride = KHW | 1;
    const long long rows = static_cast<long long>(O) * I;
    const long long r0 = static_cast<long long>(jr.lb) * kTileRows;
    if (r0 >= rows) return;
    const int nrows = static_cast<int>(rows - r0 < kTileRows ? rows - r0 : kTileRows);
    const float* src = w + r0 * KHW;
    for (int idx = threadIdx.x; idx < nrows * KHW; idx += 256) {
      const int rr = idx / KHW, k = idx - rr * KHW;
      tile[rr * stride + k] = src[idx];
    }
    __syncthreads();
    const long long r = r0 + threadIdx.x;
    if (r < rows)
      for (int t = 0; t < ntaps; ++t) {
        float v = tile[threadIdx.x * stride + tapk[t]];
        if (round_tf32) v = cd_round_tf32(v);
        packed[static_cast<long long>(t) * rows + r] = v;
      }
    return;
  }
  // element-wise: forward operand packed[t][o][i], data-gradient operand packed[t][i][o]; ConvTranspose2d stores (I,O,KH,KW)
  const int N = mode == 0 ? O : I, K = mode == 0 ? I : O;
  const long long total = static_cast<long long>(ntaps) * N * K;
  for (long long idx = static_cast<long long>(jr.lb) * 256 + threadIdx.x; idx < total; idx += static_cast<long long>(jb.nblocks) * 256) {
    const int k = static_cast<int>(idx % K);
    const int n = static_cast<int>((idx / K) % N);
    const int t = static_cast<int>(idx / (static_cast<long long>(K) * N));
    const int o = mode == 0 ? n : k, i = mode == 0 ? k : n;
    const int ky = jb.ky[t], kx = jb.kx[t];
    const long long s = tr ? ((static_cast<long long>(i) * O + o) * KH + ky) * KW + kx
                           : ((static_cast<long long>(o) * I + i) * KH + ky) * KW + kx;
    float v = w[s];
    if (round_tf32) v = cd_round_tf32(v);
    packed[idx] = v;
  }
}

__global__ void __launch_bounds__(256)
unpack_wgrad_batched_kernel(const CdRepackJob* __restrict__ jobs, int njobs, int accumulate, int clear_src) {
  __shared__ float tile[kTileRows * (kMaxKHW + 1)];
  __shared__ int tapk[CD_MAX_TAPS];
  __shared__ int covered[kMaxKHW];
  const JobRef jr = find_job(jobs, njobs);
  const CdRepackJob& jb = jobs[jr.j];
  if (jr.lb >= jb.nblocks) return;
  const int O = jb.O, I = jb.I, KH = jb.KH, KW = jb.KW, ntaps = jb.ntaps, tr = jb.transposed_conv;
  float* __restrict__ packed = const_cast<float*>(jb.src);
  float* __restrict__ wg = jb.dst;
  const int KHW = KH * KW;
  if (!tr && KHW <= kMaxKHW) {
    const long long rows = static_cast<long long>(O) * I;
    const long long r0 = static_cast<long long>(jr.lb) * kTileRows;
    if (r0 >= rows) return;
    if (threadIdx.x < KHW) covered[threadIdx.x] = 0;
    if (threadIdx.x < ntaps) tapk[threadIdx.x] = jb.ky[threadIdx.x] * KW + jb.kx[threadIdx.x];
    __syncthreads();
    if (threadIdx.x < ntaps) covered[tapk[threadIdx.x]] = 1;
    const int stride = KHW | 1;
    const long long r = r0 + threadIdx.x;
    for (int t = 0; t < ntaps; ++t) {
      float v = 0.f;
      if (r < rows) {
        const long long s = static_cast<long long>(t) * rows + r;
        v = packed[s];
        if (clear_src) packed[s] = 0.f;
      }
      tile[threadIdx.x * stride + tapk[t]] = v;
    }
    __syncthreads();
    const int nrows = static_cast<int>(rows - r0 < kTileRows ? rows - r0 : kTileRows);
    float* dst = wg + r0 * KHW;
    for (int idx = threadIdx.x; idx < nrows * KHW; idx += 256) {
      const int rr = idx / KHW, k = idx - rr * KHW;
      if (covered[k]) {
        const float v = tile[rr * stride + k];
        dst[idx] = accumulate ? dst[idx] + v : v;
      }
    }
    return;
  }
  const long long total = static_cast<long long>(ntaps) * O * I;
  for (long long idx = static_cast<long long>(jr.lb) * 256 + threadIdx.x; idx < total; idx += static_cast<long long>(jb.nblocks) * 256) {
    const int i = static_cast<int>(idx % I);
    const int o = static_cast<int>((idx / I) % O);
    const int t = static_cast<int>(idx / (static_cast<long long>(I) * O));
    const int ky = jb.ky[t], kx = jb.kx[t];
    const long long d = tr ? ((static_cast<long long>(i) * O + o) * KH + ky) * KW + kx
                           : ((static_cast<long long>(o) * I + i) * KH + ky) * KW + kx;
    const float v = packed[idx];
    if (clear_src) packed[idx] = 0.f;
    wg[d] = accumulate ? wg[d] + v : v;
  }
}

// data-gradient operands straight from PACKED forward operands (the engine keeps dense conv weights packed [tap][O][I] as the
// master copy): dst[t][i][o] = src[tap_t][o][i] with tap_t = ky[t] * KW + kx[t].  One 32x32 transpose tile
// per block through shared memory (both sides coalesced); job.nblocks = ntaps * ceil(O/32) * ceil(I/32).
__global__ void __launch_bounds__(256)
transpose_taps_batched_kernel(const CdRepackJob* __restrict__ jobs, int njobs) {
  __shared__ float tile[32][33];
  const JobRef jr = find_job(jobs, njobs);
  const CdRepackJob& jb = jobs[jr.j];
  if (jr.lb >= jb.nblocks) return;
  const int O = jb.O, I = jb.I;
  const int to = (O + 31) >> 5, ti = (I + 31) >> 5;
  const int t = jr.lb / (to * ti), rem = jr.lb - t * (to * ti);
  const int o0 = (rem / ti) * 32, i0 = (rem % ti) * 32;
  const float* __restrict__ src = jb.src + static_cast<long long>(jb.ky[t] * jb.KW + jb.kx[t]) * O * I;
  float* __restrict__ dst = jb.dst + static_cast<long long>(t) * O * I;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
#pragma unroll
  for (int r = ty; r < 32; r += 8) {
    const int o = o0 + r, i = i0 + tx;
    tile[r][tx] = (o < O && i < I) ? src[static_cast<long long>(o) * I + i] : 0.f;
  }
  __syncthreads();
#pragma unroll
  for (int r = ty; r < 32; r += 8) {
    const int i = i0 + r, o = o0 + tx;
    if (i < I && o < O) dst[static_cast<long long>(i) * O + o] = tile[tx][r];
  }
}

}  // namespace

extern "C" int cd_transpose_taps_batched(const CdRepackJob* jobs, int njobs, int total_blocks, void* stream) {
  CD_REQUIRE(jobs != nullptr && njobs >= 1 && total_blocks >= 1, "cd_transpose_taps_batched: empty job table");
  transpose_taps_batched_kernel<<<total_blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(jobs, njobs);
  CD_LAUNCH_CHECK();
  return 0;
}

extern "C" int cd_pack_weight_batched(const CdRepackJob* jobs, int njobs, int total_blocks, void* stream) {
  CD_REQUIRE(jobs != nullptr && njobs >= 1 && total_blocks >= 1, "cd_pack_weight_batched: empty job table");
  pack_weight_batched_kernel<<<total_blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(jobs, njobs);
  CD_LAUNCH_CHECK();
  return 0;
}

extern "C" int cd_unpack_wgrad_batched(const CdRepackJob* jobs, int njobs, int total_blocks, int accumulate, int clear_src,
                                       void* stream) {
  CD_REQUIRE(jobs != nullptr && njobs >= 1 && total_blocks >= 1, "cd_unpack_wgrad_batched: empty job table");
  unpack_wgrad_batched_kernel<<<total_blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(jobs, njobs, accumulate, clear_src);
  CD_LAUNCH_CHECK();
  return 0;
}
