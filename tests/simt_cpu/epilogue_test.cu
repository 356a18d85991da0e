// TEST INFRASTRUCTURE (never part of libcolddiff): drives cd_epilogue_staged32 of csrc/conv_epilogue.cuh the way conv_tc_kernel
// does after staging a warpgroup's accumulator chunk in shared memory -- warp w owns accumulator rows [32 w, 32 w + 32) of a
// 128 x BN tile, a lane holds the 32 columns of one chunk of ITS row, pixels map to arbitrary output rows.
#include "cd_common.cuh"
#include "conv_epilogue.cuh"

struct EpiTestParams {
  float* out; int out_ld;
  const float* bias;
  const float* resid; int resid_ld;
  int act; int round_tf32;
  float* out2; int out2_ld;
  const float* aux; int aux_ld;
};

__global__ void epilogue_test_kernel(const float* acc, int BN, const long long* pix, const int* valid, EpiTestParams p) {
  __shared__ __align__(16) float stage[4 * kEpiStageFloats];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m = warp * 32 + lane;
  for (int c = 0; c < BN; c += 32) {
    uint32_t r[32];
    for (int j = 0; j < 32; ++j) r[j] = __float_as_uint(acc[m * BN + c + j]);
    cd_epilogue_staged32(r, stage + warp * kEpiStageFloats, lane, pix[m], valid[m] != 0, c, p);
  }
}

extern "C" int cd_test_epilogue_staged(const float* acc, int BN, const long long* pix, const int* valid, float* out, int out_ld,
                                       const float* bias, const float* resid, int resid_ld, int act, int round_tf32, float* out2,
                                       int out2_ld, const float* aux, int aux_ld) {
  EpiTestParams p{out, out_ld, bias, resid, resid_ld, act, round_tf32, out2, out2_ld, aux, aux_ld};
  epilogue_test_kernel<<<1, 128, 0, 0>>>(acc, BN, pix, valid, p);
  CD_LAUNCH_CHECK();
  return 0;
}
