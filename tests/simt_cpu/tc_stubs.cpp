// TEST INFRASTRUCTURE: the tensor-core (wgmma / TMA) translation units cannot execute on the CPU.  In the all-SIMT CPU build
// of the library their internal entry points defer to the fp32 CUDA-core kernels of conv_simt.cu (the library's own fallback for
// shapes that are not tensor-core shaped), and their tuning switches are accepted and ignored.
#include "shim/cuda_runtime.h"
#include "colddiff.h"

extern "C" int cd_conv_fwd(const CdConvDesc* d, int impl, void* stream);
int cd_conv_fwd_tc(const CdConvDesc* d, cudaStream_t st) { return cd_conv_fwd(d, CD_CONV_SIMT, st); }
int cd_conv_wgrad_tc(const CdConvDesc*, const float*, int, float*, float*, int* bias_done, cudaStream_t) { *bias_done = 0; return 1; }
extern "C" int cd_conv_tc_set_tf32_maps(int) { return 0; }
extern "C" int cd_conv_tc_set_2cta(int) { return 0; }
extern "C" int cd_conv_tc_set_2cta_bn(int) { return 0; }
extern "C" int cd_conv_tc_set_halo(int) { return 0; }
extern "C" int cd_conv_tc_set_two_ctas(int) { return 0; }
extern "C" int cd_wgrad_tc_set_mode(int) { return 0; }
extern "C" int cd_wgrad_tc_set_bias_fusion(int) { return 0; }
extern "C" int cd_wgrad_tc_set_split(int, int) { return 0; }
int cd_dwconv7_fwd_tma(const float*, int, int, int, int, int, const float*, const float*, const float*, int, float*, int, int, const float*, int,
                       cudaStream_t) { return 1; }
int cd_dwconv7_wgrad_tma(const float*, int, const float*, int, int, int, int, int, float*, cudaStream_t) { return 1; }
extern "C" int cd_dwconv7_set_tma(int) { return 0; }
