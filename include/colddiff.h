/*
 * colddiff.h -- C ABI of libcolddiff.so: the H100 (sm_90a) engine behind the Cold-Diffusion
 * hot path (GaussianDiffusion.p_losses training step + x0_step_down / ddim sampling around the
 * UNet restoration operator R(x,t) and the degradation operators D(x,t)).
 *
 * The upstream reference (arpitbansal297/Cold-Diffusion-Models) is pure Python/PyTorch and has NO
 * FFI / plugin interface of its own.  The boundary callers depend on is the
 * Python class surface of each *_diffusion_pytorch package; cold_diffusion_models_b200/ mirrors
 * that surface and calls the entry points below through ctypes.  Every entry point cites the
 * reference code it replaces (DB = deblurring-diffusion-pytorch/deblurring_diffusion_pytorch/
 * deblurring_diffusion_pytorch.py).
 *
 * Conventions
 *   - plain pointers and sizes only; all pointers are DEVICE pointers unless named host_*;
 *   - the library never synchronises, and allocates device memory only for the split-plane GroupNorm
 *     partials (a per-(device, stream) cached buffer, see cd_groupnorm_fwd): otherwise the caller passes
 *     outputs/workspaces (torch caching allocator) and a cudaStream_t (as void*);
 *   - return value: 0 = ok, <0 = error (text via cd_last_error); no exceptions cross the ABI;
 *   - activations inside the engine are NHWC fp32 ("pixel rows" of `ld` floats, channel slice
 *     selected by offsetting the base pointer); reference-facing images are NCHW fp32;
 *   - no global mutable state except a per-process cache of the driver entry point used to
 *     encode TMA descriptors.
 */
#ifndef COLDDIFF_H_
#define COLDDIFF_H_

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CD_ABI_VERSION 1
#define CD_MAX_TAPS 16

int cd_version(void);
/* copies the calling thread's last error text; returns its length */
int cd_last_error(char* buf, size_t n);

/* ------------------------------------------------------------------------------------------
 * Dense convolution as an implicit GEMM over a "tap list" (replaces nn.Conv2d 3x3 / 1x1 /
 * 4x4 stride 2 and nn.ConvTranspose2d 4x4 stride 2 in Unet: DB:105-109,149-154,173-174,253;
 * also their data-gradients, which are the same contraction with transposed/flipped weights).
 *
 *   out[b, gy*oys+oy0, gx*oxs+ox0, co] = act( bias[co] + resid[...] +
 *        sum_{s<nsrc} sum_{t<ntaps[s]} sum_{ci<C[s]}
 *            src[s][b, gy*sy+dy[s][t], gx*sx+dx[s][t], ci] * w[s][(b*wb) , t, co, ci] )
 *   for (gy,gx) in the Hg x Wg GEMM pixel grid; reads outside the source image are zero.
 *
 * impl: CD_CONV_TC = wgmma/TMA tensor-core kernel (tf32, fp32 accumulate in registers;
 *       needs C[s] % 32 == 0 and 16-byte aligned rows), CD_CONV_SIMT = fp32 CUDA-core kernel
 *       (any shape; used for 3-channel image edges and as the on-device cross-check).
 * ------------------------------------------------------------------------------------------ */
enum { CD_CONV_SIMT = 0, CD_CONV_TC = 1 };
enum { CD_ACT_NONE = 0, CD_ACT_GELU = 1, CD_ACT_GELU_BWD = 2 /* out = acc * gelu'(aux) : dgrad through GELU */ };

typedef struct {
  const float* src;       /* NHWC base of the channel slice                         */
  int32_t ld;             /* floats between consecutive pixels                      */
  int32_t C;              /* channels contracted from this source                   */
  int32_t H, W;           /* source image size                                      */
  int32_t ntaps;
  int32_t dy[CD_MAX_TAPS], dx[CD_MAX_TAPS];
  const float* w;         /* packed weights [wb? B:1][ntaps][Cout][C], C contiguous */
  int32_t w_per_batch;    /* 1: a separate weight set per batch element             */
} CdConvSrc;

typedef struct {
  int32_t B, Hg, Wg;      /* GEMM pixel grid                                        */
  int32_t sy, sx;         /* source stride                                          */
  int32_t Cout;
  int32_t nsrc;
  CdConvSrc s[2];
  float* out; int32_t out_ld; int32_t Ho, Wo;
  int32_t oys, oxs, oy0, ox0;
  const float* bias;      /* [Cout] or NULL                                         */
  const float* resid; int32_t resid_ld; /* same pixel mapping as out, or NULL       */
  int32_t act;
  int32_t round_tf32;     /* round outputs to TF32 (RN) so the next TC conv sees RN operands */
  float* out2; int32_t out2_ld; /* optional second output: the pre-activation (for backward) */
  const float* aux; int32_t aux_ld; /* CD_ACT_GELU_BWD: saved pre-activation, same pixel mapping as out */
} CdConvDesc;

int cd_conv_fwd(const CdConvDesc* d, int impl, void* stream);

/* weight-gradient of the same contraction (single source, single weight set):
 *   dw[t, co, ci] (+)= sum_{b,gy,gx} dout[b, gy*oys+oy0, gx*oxs+ox0, co] * src[b, gy*sy+dy[t], gx*sx+dx[t], ci]
 * dw is the packed [ntaps][Cout][C] layout; accumulate!=0 adds into dw (else dw must be zeroed by
 * the caller; the kernel uses atomics across pixel splits). db (optional) += sum dout.           */
int cd_conv_wgrad(const CdConvDesc* d, const float* dout, int dout_ld, float* dw, float* db,
                  int impl, void* stream);
/* with d->s[0].w_per_batch = 1 the gradient is kept per batch element: dw[b][t][co][ci] (used for the
 * per-batch effective weights of LinearAttention). */

/* repack reference-layout weights: OIHW (transposed_conv=0) or IOHW (nn.ConvTranspose2d,
 * transposed_conv=1) -> packed [tap][N][K].  mode 0: forward operand (N=out ch, K=in ch);
 * mode 1: data-gradient operand (N=in ch, K=out ch). Tap order is given by (ky,kx) lists.     */
int cd_pack_weight(const float* w, int O, int I, int KH, int KW, int transposed_conv, int mode,
                   const int32_t* host_ky, const int32_t* host_kx, int ntaps, int round_tf32,
                   float* packed, void* stream);
/* inverse for gradients: packed [tap][O][I] -> OIHW / IOHW (accumulating) */
int cd_unpack_wgrad(const float* packed, int O, int I, int KH, int KW, int transposed_conv,
                    const int32_t* host_ky, const int32_t* host_kx, int ntaps, float* w_grad, int accumulate,
                    void* stream);

/* The same two repacks for MANY weights in one launch (one optimizer step repacks ~64 convolution weights and
 * unpacks ~98 packed weight gradients: as single launches they are launch/latency-bound).
 * `jobs` is a DEVICE array of njobs descriptors (built once by the caller; pointers are stable across steps);
 * blocks [block0, block0 + nblocks) of the 256-thread grid of total_blocks work on job j, block0 ascending with j.
 * nblocks is the caller's choice (any value >= 1 is correct for transposed_conv / mode 1 / KH*KW > 16 jobs, which
 * stride over the elements; the other jobs need nblocks == ceil(O*I / 256): one 256-row tile per block).
 * cd_unpack_wgrad_batched with clear_src != 0 also zeroes the packed gradient after reading it, which leaves the
 * accumulation buffers of cd_conv_wgrad ready for the next backward pass without ~98 fill launches.          */
typedef struct {
  const float* src;       /* pack: reference-layout weight;  unpack: packed gradient [tap][O][I]               */
  float* dst;             /* pack: packed operand;           unpack: reference-layout gradient                 */
  int32_t O, I, KH, KW;
  int32_t transposed_conv, mode, ntaps, round_tf32;     /* mode / round_tf32: pack only                       */
  int32_t ky[CD_MAX_TAPS], kx[CD_MAX_TAPS];
  int32_t block0, nblocks;
} CdRepackJob;
int cd_pack_weight_batched(const CdRepackJob* jobs, int njobs, int total_blocks, void* stream);
int cd_unpack_wgrad_batched(const CdRepackJob* jobs, int njobs, int total_blocks, int accumulate, int clear_src,
                            void* stream);
/* data-gradient operands of ALL dense convolutions in one launch, from forward operands that are already packed [KH*KW][O][I]
 * (the engine's master layout of dense conv weights): dst[t][i][o] = src[ky[t]*KW + kx[t]][o][i]; a job covers
 * nblocks = ntaps * ceil(O/32) * ceil(I/32) transpose tiles (mode / transposed_conv / round_tf32 are ignored) */
int cd_transpose_taps_batched(const CdRepackJob* jobs, int njobs, int total_blocks, void* stream);

/* ------------------------------------------------------------------------------------------
 * ConvNeXt block front half (DB:145, 140-143/159-162, 111-121/148):
 *   h = dwconv7x7(x) + b_dw + cond[b,:] ;  y = LayerNorm_c(h) * g + beta   (g==NULL: y = h)
 * x,y NHWC.  stats (optional, [B*H*W][2] = mean, rstd) and hpre (optional, h) are saved for the
 * backward pass.
 * ------------------------------------------------------------------------------------------ */
int cd_dwconv7_ln_fwd(const float* x, int x_ld, int B, int H, int W, int C,
                      const float* w_dw /*[C][49]*/, const float* b_dw /*[C]*/,
                      const float* cond /*[B][cond_ld] or NULL*/, int cond_ld,
                      const float* g, const float* beta /*[C] or NULL: no norm*/,
                      float eps, float* y, int y_ld, float* stats, float* hpre, int hpre_ld,
                      int round_tf32, int flip /*1: rotate the 7x7 kernel by 180 deg (data-gradient)*/,
                      const float* addend, int addend_ld /*optional NHWC tensor added to h*/, void* stream);

/* depthwise 7x7 + bias + cond (+addend) without the norm, shared-memory tiled (the production path for C >= 32; the
 * LayerNorm then runs as cd_layernorm_fwd on its output, which training keeps anyway as `hpre`).  flip=1: data-gradient. */
int cd_dwconv7_fwd(const float* x, int x_ld, int B, int H, int W, int C, const float* w_dw, const float* b_dw,
                   const float* cond, int cond_ld, float* out, int out_ld, int flip, const float* addend,
                   int addend_ld, void* stream);
/* diagnostic switch: 1 (default) = persistent double-buffered depthwise kernel where eligible, 0 = one tile per block */
int cd_dwconv7_set_pipe(int enable);
/* diagnostic switch: 1 (default) = the persistent depthwise kernels stage their tiles with TMA (one bulk tensor copy per tile,
 * border zero fill by the tensor map: dwconv_tma.cu), 0 = with 16-byte LDGSTS (elementwise.cu) */
int cd_dwconv7_set_tma(int enable);
/* channel LayerNorm alone (PreNorm in front of LinearAttention, DB:123-131; also the ConvNextBlock norm) */
int cd_layernorm_fwd(const float* x, int x_ld, int64_t npix, int C, const float* g, const float* beta,
                     float eps, float* y, int y_ld, float* stats, int round_tf32, void* stream);

/* time embedding (DB:91-103, 209-216) + every block's GELU->Linear conditioning (DB:140-143):
 *   temb = W2 gelu(W1 sinemb(t) + b1) + b2 ; cond_all[b, :] = Wc gelu(temb[b]) + bc
 * Wc/bc are the row-concatenation of all blocks' mlp.1 weights ([sumC][dim]).               */
int cd_time_mlp_fwd(const int64_t* t, int B, int dim, const float* w1, const float* b1,
                    const float* w2, const float* b2, const float* wc, const float* bc, int sumC,
                    float* sinemb /*[B][dim]*/, float* hid_pre /*[B][4dim]*/, float* temb /*[B][dim]*/,
                    float* cond_all /*[B][sumC]*/, void* stream);

/* LinearAttention core (DB:176-187) on qkv NHWC [B][n][ld] (q|k|v at channel 0|128|256, 4 heads x 32):
 *   kmax[b,h,d]   = max_n k[b,h,d,n]
 *   ctx[b,h,d,e]  = sum_n exp(k[b,h,d,n] - kmax[b,h,d]) * v[b,h,e,n]      (un-normalised)
 *   ksum[b,h,d]   = sum_n exp(k[b,h,d,n] - kmax[b,h,d])
 *   weff[b, co, h*32+d] = scale * sum_e w_out[co, h*32+e] * ctx[b,h,d,e] / ksum[b,h,d]
 * so that to_out(einsum(context, q*scale)) == conv1x1(q, weff[b]) -- a per-batch-weight tap-list
 * convolution (cd_conv_fwd with w_per_batch=1).  kmax/ksum ([B][128]) are kept for backward. */
int cd_linattn_weff(const float* ctx, const float* ksum, const float* w_out /*[dim][128]*/, int B, int dim,
                    float scale, int round_tf32, float* weff /*[B][dim][128]*/, void* stream);
/* kmax / ksum / ctx as above, DETERMINISTIC (bit-identical run to run) and in one pass over k and v
 * (csrc/linattn_ctx.cu): blocks walk spans of `ppb` pixels with a running max (flash-attention recurrence), the per-head E^T V
 * products run as 3xTF32 mma.sync, each block writes one partial (ctx[4][32][32] | m[128] | s[128] = 4352 floats) to `ws`
 * ([B][nblk][4352] floats, caller-allocated) and a second kernel merges the partials of an image in block order.
 * The caller picks ppb (a multiple of 32; about one wave of blocks at 3 blocks per SM over the batch) and nblk = ceil(n / ppb). */
int cd_linattn_context_det(const float* qkv, int ld, int B, int n, int nblk, int ppb, float* ws, float* kmax, float* ksum,
                           float* ctx /*[B][4][32][32]*/, void* stream);

/* final 1x1 conv to image channels + optional residual, NHWC -> reference NCHW (DB:253,279-282) */
int cd_conv1x1_to_nchw(const float* x, int ld, int B, int H, int W, int C, const float* w /*[Co][C]*/,
                       const float* b, int Co, const float* resid_nchw, float* out_nchw, void* stream);
/* reference NCHW image -> NHWC with zero-padded pixel stride ld (>= C) */
int cd_nchw_to_nhwc(const float* x, int B, int C, int H, int W, float* out, int ld, void* stream);
/* out[c] += sum_rows x[row*ld + c]  (bias / LayerNorm-beta gradients) */
int cd_colsum(const float* x, int ld, int64_t rows, int C, float* out, void* stream);
/* kernel switch of the tensor-core wgrad: 0 = mma.sync kernel with one X tile per tap; 8 = mma.sync kernel whose dx taps of a 3x3
 * kernel share one halo tile; any other value (default 1) = the wgmma kernel for stride-1 problems with taps in [-1, 1]^2, one weight
 * set, Cin % 64 == 0 and Cout % 64 == 0 (and no bias fusion), the mma.sync halo kernel for the rest */
int cd_wgrad_tc_set_mode(int mode);
/* K-split policy of the tensor-core wgrad: 0 = two waves rounded up, 1 / 2 = at most one / two full waves of CTAs,
 * 3 (default) = minimise waves x (chunks_per_split x t_chunk + over_clk); over_clk > 0 sets the per-CTA fixed cost (SM clocks) */
int cd_wgrad_tc_set_split(int policy, int over_clk);
/* opt-in (default 0): fold the bias gradient (column sums of dY) into the tensor-core weight gradient */
int cd_wgrad_tc_set_bias_fusion(int enable);
/* EXPERIMENTAL operand-format probe, not used by the engine (tools/conv_f16_probe.py): cd_conv_fwd with impl = CD_CONV_TC on FP16
 * operands -- d->s[i].src and d->s[i].w point to __half arrays (ld and the packed-weight layout count elements, C % 64 == 0),
 * wgmma on FP16 operands with fp32 accumulation, fp32 epilogue and outputs as usual. */
int cd_conv_fwd_f16_probe(const CdConvDesc* d, void* stream);
/* opt-in (default 0): line-coalesced epilogue of the tensor-core convolution (csrc/conv_epilogue.cuh;
 * bit-identical results): 1 = for launches with at most 16 K chunks of 32 channels per tile (the store-bound 1x1 projections),
 * 2 = for every launch, 3 = at most 48 K chunks */
int cd_conv_tc_set_staged_epilogue(int mode);
/* diagnostic switch: 1 (default) = TFLOAT32 tensor maps, 0 = FLOAT32 tensor maps for the convolution operands */
int cd_conv_tc_set_tf32_maps(int enable);
/* SM-pair variant of the tap-list convolution: a cluster of two CTAs computes two neighbouring 128-pixel tiles of the same output
 * channels, each CTA fetching half of the weight tile and multicasting it to both.  0 = off (default), 1 = where the tile cost
 * model prefers it (256-wide N tiles), 2 = wherever the problem is eligible (tests) */
int cd_conv_tc_set_2cta(int mode);
/* N tiles below 256 that also go to the SM-pair kernel (bit mask: 128 | 64; default 0) */
int cd_conv_tc_set_2cta_bn(int mask);
/* kernel choice for stride-1 convolutions whose taps lie in [-1, 1]^2 (dense 3x3 forward / data gradient, fused [3x3 | 1x1]
 * pairs).  The shared-row kernel fetches one TW x (TH + 2) activation box per 32-channel chunk and tap column and feeds the three
 * row taps of that column from it; the per-tap kernel fetches one 128-pixel box per tap.  0 = shape-based choice (default),
 * 1, 2 or 6 = shared-row kernel with 16 x 8 pixel tiles wherever eligible, 4 = shared-row kernel with 16 x 16 pixel tiles (one
 * CTA per SM, output stored by TMA) wherever eligible and the output map is the identity, 8 = per-tap kernel everywhere.  With the SM-pair kernel on (cd_conv_tc_set_2cta), 0 keeps the per-tap family. */
int cd_conv_tc_set_halo(int enable);
/* two co-resident CTAs per SM (half the pipeline stages each) for the tensor-core convolution with N <= 128: one CTA's epilogue
 * overlaps the other's mainloop.  Bit mask of N tiles (128 | 64); default 192 (both), 0 = one CTA per SM */
int cd_conv_tc_set_two_ctas(int mask);

/* ------------------------------------------------------------------------------------------
 * Backward of the HBM-bound pieces (autograd of the reference modules restated as kernels).
 * ------------------------------------------------------------------------------------------ */
/* LayerNorm (DB:111-121): dh = dLN(dy) (+addend); dg, dbeta accumulated (+=).  dg = dbeta = NULL (both or neither): dh only,
 * the same bits, with no parameter reduction (frozen g and b) */
int cd_layernorm_bwd(const float* dy, int dy_ld, const float* h, int h_ld, const float* stats,
                     const float* g, int64_t npix, int C, const float* addend, int addend_ld,
                     float* dh, int dh_ld, float* dg, float* dbeta, void* stream);
/* depthwise 7x7 weight gradient: dw[c][49] += sum dh * shifted(x) */
int cd_dwconv7_wgrad(const float* dh, int dh_ld, const float* x, int x_ld, int B, int H, int W, int C,
                     float* dw, void* stream);
/* out[b*out_ld + c] += sum over the `rows` pixels of image b of x[.., c]  (time-conditioning gradient) */
int cd_colsum_batched(const float* x, int ld, int B, int64_t rows, int C, float* out, int out_ld, void* stream);
/* LinearAttention backward (see cd_linattn_context_det): per-batch small part and per-pixel k/v part */
int cd_linattn_bwd_small(const float* dweff, const float* ctx, const float* ksum, const float* w_out,
                         int B, int dim, float scale, float* dw_out, float* dctxn, float* rowdot, void* stream);
/* cd_linattn_bwd_kv runs its two [pixels x 32] x [32 x 32] products per head on warp-level tensor-core MMAs (csrc/linattn_bwd.cu:
 * 3xTF32: fp32-grade products); ld % 4 != 0 or a qkv that is not 16-byte aligned takes a CUDA-core kernel */
int cd_linattn_bwd_kv(const float* qkv, int ld, int B, int n, const float* kmax, const float* ksum,
                      const float* dctxn, const float* rowdot, float* dqkv, int dld, void* stream);
int cd_transpose_weff(const float* weff, int B, int dim, float* weff_t, void* stream);
int cd_conv1x1_to_nchw_bwd(const float* dout_nchw, const float* x, int ld, int B, int H, int W, int C,
                           const float* w, int Co, float* dx, int dx_ld, float* dw, float* db, void* stream);
/* tiny dense helpers (time-MLP backward): C (+)= op(A) op(B);  y = dy * gelu'(pre), act_out = gelu(pre) */
int cd_small_gemm(const float* A, int lda, int transA, const float* B, int ldb, int transB,
                  float* C, int ldc, int M, int N, int K, int accumulate, void* stream);
int cd_gelu_bwd(const float* dy, const float* pre, int64_t n, float* y, float* act_out, void* stream);
/* out = a + b on NHWC channel slices (sum of two gradient branches) */
int cd_add(const float* a, int a_ld, const float* b, int b_ld, float* out, int out_ld, int64_t npix, int C,
           void* stream);

/* ------------------------------------------------------------------------------------------
 * Degradation D(x,t) for the Gaussian-blur family (DB:348-389 kernels; DB:927-960 q_sample;
 * DB:436-451 Algorithm-2 update).  Every blur step is separable with circular or reflect
 * boundary handling, hence the cumulative degradation of a plane X is  A_t X A_t^T  with a
 * precomputed S x S operator per step (ops: [T][S][S], row-major, ops[t] = K_t ... K_0).
 *   cd_blur_apply     : out[b,c] = A_{t_b} x[b,c] A_{t_b}^T    (t_b < 0: copy)  -- q_sample / opt
 *   cd_blur_step_down : out = x_t - A_t xhat A_t^T + A_{t-1} xhat A_{t-1}^T    -- DB:451
 * Images are reference-layout NCHW planes.  collapse_last: `discrete` mean-collapse for the
 * last operator index (DB:938-940); quantize: 8-bit truncation (DB:954-958).
 * Image sizes: S % 4 == 0 and 4 <= S <= 512.  S <= 128 runs one CTA per plane; 128 < S <= 512
 * one CTA per 32-row strip, and there `out` must not alias `x` / `xhat` (other strips still
 * read the plane).  Other sizes return an error.
 * ------------------------------------------------------------------------------------------ */
int cd_blur_apply(const float* x, float* out, const float* ops, const int64_t* t, int t_scalar,
                  int B, int C, int S, int T, int collapse_last, int quantize, void* stream);
int cd_blur_step_down(const float* xt, const float* xhat, float* out, const float* ops,
                      int t_hi, int t_lo, int B, int C, int S, int T, int collapse_last, void* stream);
/* cd_blur_apply_adjoint: the gradient of cd_blur_apply (without its quantize) with respect to x: out[b,c] = A_{t_b}^T g[b,c] A_{t_b}
 * (t_b < 0: copy).  With collapse_last, planes at t_b = T-1 first become mean(g) everywhere (the adjoint of the mean-collapse).
 * Same operator table, shapes, size limits and aliasing rule as cd_blur_apply; A^T is formed in shared memory, not tabulated. */
int cd_blur_apply_adjoint(const float* g, float* out, const float* ops, const int64_t* t, int t_scalar,
                          int B, int C, int S, int T, int collapse_last, void* stream);

/* loss (DB:968-971): mode 0 = L1 mean, 1 = L2 mean; writes *loss (device) and dL/dxhat*scale */
int cd_loss_fwd_bwd(const float* x0, const float* xhat, int64_t n, int mode, float grad_scale,
                    float* loss /*device scalar, accumulated*/, float* dxhat, void* stream);

/* Adam (torch defaults, DB:1117) + EMA (DB:73-81) fused multi-tensor step on flat buffers */
int cd_adam_ema_step(float* p, const float* g, float* m, float* v, float* ema, int64_t n,
                     float lr, float beta1, float beta2, float eps, int step,
                     int ema_mode /*0 none,1 copy,2 lerp*/, float ema_beta, float grad_scale, void* stream);

/* Gaussian-noise baseline (denoising-diffusion-pytorch/denoising_diffusion_pytorch/denoising_diffusion_pytorch.py, "DN"):
 *   cd_noise_lerp : q_sample = sqrt_ac[t_b] x1 + sqrt_1mac[t_b] x2                                  (DN:517-522)
 *   cd_noise_step : one reverse step img - xt_bar + xt_sub1_bar; mode 0 'ddim' (x2 from x_t, DN:377-381, 392-412),
 *                   mode 1 'x0_step_down' (x2 = fixed noise, DN:414-432)                                              */
int cd_noise_lerp(const float* x1, const float* x2, const int64_t* t, int t_scalar, const float* sqrt_ac,
                  const float* sqrt_1mac, int64_t per_sample, int64_t n, float* out, void* stream);
int cd_noise_step(const float* img, const float* x1_bar, const float* noise, int mode, int t, const float* sqrt_ac,
                  const float* sqrt_1mac, int64_t n, float* out, void* stream);
/* cd_noise_step_to: the same reverse step from level t to any level s, 0 <= s < t (strided sampling, `sample(steps=K)`):
 * img - xt_bar + xs_bar with xt_bar from sqrt_ac / sqrt_1mac at t-1 and xs_bar at s-1; s = 0: xs_bar = x1_bar (the clean
 * estimate).  Both modes of cd_noise_step; s = t-1 runs cd_noise_step itself (its bits).                              */
int cd_noise_step_to(const float* img, const float* x1_bar, const float* noise, int mode, int t, int s, const float* sqrt_ac,
                     const float* sqrt_1mac, int64_t n, float* out, void* stream);
/* Fade-to-colour generation (defading-generation-diffusion-pytorch/defading_diffusion_pytorch/defading_diffusion_pytorch.py,
 * "DFGEN"): per-pixel schedule alphas / one_minus_alphas [T][HW] (DFGEN:320-344, 371-381).
 *   cd_fade_lerp : q_sample = alphas[t_b] * x1 + one_minus_alphas[t_b] * x2 (t: int64 [B], or NULL -> t_scalar)  (DFGEN:543-548)
 *   cd_fade_step : one reverse step img - xt_bar + xt_sub1_bar with the fixed end image x2            (DFGEN:386-418)     */
int cd_fade_lerp(const float* x1, const float* x2, const int64_t* t, int t_scalar, const float* alphas,
                 const float* one_minus_alphas, int B, int C, int HW, float* out, void* stream);
int cd_fade_step(const float* img, const float* x1_bar, const float* x2, int t, const float* alphas,
                 const float* one_minus_alphas, int B, int C, int HW, float* out, void* stream);
/* cd_fade_step_to: cd_fade_step from level t to any level s, 0 <= s < t: the tables are read at rows t-1 and s-1; s = 0 goes
 * to the clean estimate x1_bar.  s = t-1 runs cd_fade_step itself (its bits).                                             */
int cd_fade_step_to(const float* img, const float* x1_bar, const float* x2, int t, int s, const float* alphas,
                    const float* one_minus_alphas, int B, int C, int HW, float* out, void* stream);
/* cd_lerp2_adjoint: the gradients of out = wa[w] x1 + wb[w] x2 (cd_noise_lerp, cd_fade_lerp) from one pass over g [B][C][HW]:
 * ga = wa[w] g, gb = wb[w] g, with w = t_b (per_pixel = 0: per-sample scalars, cd_noise_lerp) or t_b * HW + pixel (per_pixel = 1:
 * [T][HW] tables, cd_fade_lerp).  t: int64 [B], or NULL -> t_scalar.  ga or gb may be NULL (that gradient is not written). */
int cd_lerp2_adjoint(const float* g, const int64_t* t, int t_scalar, const float* wa, const float* wb, int B, int C,
                     int64_t HW, int per_pixel, float* ga, float* gb, void* stream);
/* Gaussian-mask fading (defading-diffusion-pytorch/defading_diffusion_pytorch/defading_diffusion_gaussian.py, "DFG"):
 * masks = cumulative products of the fade kernels [T][MS][MS]; rx/ry (optional, int64 [B]) = per-sample window
 * offsets of the 'Random_*' routines (DFG:359-367); index -1 = identity.
 *   cd_mask_apply     : out = x * M[t_b] (+ 8-bit truncation when quantize)     -- q_sample / sample head (DFG:371-384, 495-533)
 *   cd_mask_step_down : out = x_t - xhat * M[idx_hi] + xhat * M[idx_lo]         -- DFG:410-420                      */
int cd_mask_apply(const float* x, float* out, const float* masks, const int64_t* t, int t_scalar,
                  const int64_t* rx, const int64_t* ry, int B, int C, int S, int MS, int quantize, void* stream);
int cd_mask_step_down(const float* xt, const float* xhat, float* out, const float* masks, int idx_hi, int idx_lo,
                      const int64_t* rx, const int64_t* ry, int B, int C, int S, int MS, void* stream);
/* Decolorization / Snow forward processes (snowification/diffusion/forward_process_impl.py "FP", diffusion.py "SN") with
 * PER-SAMPLE step indices (masked stepping, SN:195-245; t_b = -1 rows untouched, SN:349-355).  index = t[b] + off, < 0 = identity.
 *   mode 0: out = D(src, t_hi+hi_off)                       (q_sample SN:344-388 / degradation of the input SN:271-274)
 *   mode 1: out = xt - D(src, t_hi+hi_off) + D(src, t_lo+lo_off)   (x0_step_down, SN:226-238)
 * cd_chanmix: D = cumulative C x C channel mix mats[idx] (FP:150-163,189-195).  cd_snow: D(og, i) = clip(bright_i(og) + snow_i +
 * rot180(snow_i), 0, 1)*2-1 with snow [T][snow_batch][3][H][W] (FP:361-372).                                                   */
int cd_chanmix(const float* xt, const float* xsrc, float* out, const float* mats, const int64_t* t_hi,
               const int64_t* t_lo, int hi_off, int lo_off, int B, int C, int64_t HW, int mode, void* stream);
/* Guided restoration (`GaussianDiffusion.restore`): reconstruction guidance for the linear degradations D_s.
 * Guidance gradient in image space, ghat = D_s^T (D_s x0 - y), fp32 NCHW, one entry point per family:
 *   cd_blur_guide_grad    : D_s = A_idx (.) A_idx^T per plane (idx < 0: identity), the cd_blur_apply operator table.  S <= 128
 *                           runs one pass (the residual stays on chip); 128 < S <= 512 runs cd_blur_apply with a "- y" epilogue
 *                           into `work` (B*C*S*S floats, not `out`), then the adjoint.  Same size rule as cd_blur_apply.
 *   cd_mask_guide_grad    : m (m x0 - y), m = masks[idx] in each sample's window (rx / ry as cd_mask_apply), one pass.
 *   cd_chanmix_guide_grad : M^T (M x0 - y) per pixel, M = mats[t[b] + off] (index < 0: x0 - y), one pass.
 * Guided update: the reverse step with "- weight * g" in its epilogue.  xt == NULL (mask, blur) or mode 0 (chanmix): the `default`
 * update D(xhat, lo) - weight g; otherwise `x0_step_down`, xt - D(xhat, hi) + D(xhat, lo) - weight g.  Indices as in
 * cd_blur_apply / cd_blur_step_down, cd_mask_step_down and cd_chanmix.  g == NULL runs the unguided kernel itself, bit for bit. */
int cd_blur_guide_grad(const float* x0, const float* y, float* out, float* work, const float* ops, int idx,
                       int B, int C, int S, int T, void* stream);
int cd_blur_guided_step(const float* xt, const float* xhat, const float* g, float weight, float* out, const float* ops,
                        int t_hi, int t_lo, int B, int C, int S, int T, void* stream);
int cd_mask_guide_grad(const float* x0, const float* y, float* out, const float* masks, int idx, const int64_t* rx,
                       const int64_t* ry, int B, int C, int S, int MS, void* stream);
int cd_mask_guided_step(const float* xt, const float* xhat, const float* g, float weight, float* out, const float* masks,
                        int idx_hi, int idx_lo, const int64_t* rx, const int64_t* ry, int B, int C, int S, int MS, void* stream);
int cd_chanmix_guide_grad(const float* x0, const float* y, float* out, const float* mats, const int64_t* t, int off,
                          int B, int C, int64_t HW, void* stream);
int cd_chanmix_guided(const float* xt, const float* xsrc, const float* g, float weight, float* out, const float* mats,
                      const int64_t* t_hi, const int64_t* t_lo, int hi_off, int lo_off, int B, int C, int64_t HW, int mode,
                      void* stream);
int cd_snow(const float* xt, const float* og, float* out, const float* snow, const float* br_coef, const int64_t* t_hi,
            const int64_t* t_lo, int hi_off, int lo_off, int B, int H, int W, int snow_batch, int fix_brightness,
            int mode, void* stream);
/* Lab colour path of the decolorization package (to_lab=True; diffusion/utils.py:113-222 "UT", FP:189-218).  NCHW, 3 channels.
 * cd_lab_convert: to_lab = 1: rgb2lab (RGB in [-1, 1] -> L 0..100, a, b); to_lab = 0: lab2rgb(x, clip) -> 2 rgb - 1 (fz clamped
 *   at 0, rgb clipped to [0, 1] when `clip`).  out == x is allowed.
 * cd_chanmix_lab: the masked stepping of cd_chanmix (same t_hi / t_lo / offsets / modes) with D = the Lab step chain:
 *   D(v, k) = step_k(... step_0(v)), step_i(v) = rgb2lab(step_mats[i] lab2rgb(v, clip=True)), step_mats = the PER-STEP [T][3][3]
 *   table (not cumulative: the clamp and clip at every step make the chain nonlinear).  index < 0 = v untouched (no round trip).
 * sRGB / XYZ stages restate kornia's formulas (unpinned upstream).                                                            */
int cd_lab_convert(const float* x, float* out, int B, int64_t HW, int to_lab, int clip, void* stream);
int cd_chanmix_lab(const float* xt, const float* xsrc, float* out, const float* step_mats, const int64_t* t_hi,
                   const int64_t* t_lo, int hi_off, int lo_off, int B, int64_t HW, int mode, void* stream);
/* Snow-layer generation (FP:32-42 clipped_zoom + FP:252-355 generate_snow_layer), everything after the host's random draws:
 *   base[s]  = fp32( trim( zoom_order1( noise[s] : ch x ch fp64 -> m x m ) ) )  : H x H, scipy.ndimage.zoom arithmetic, bit-exact
 *   snow[t][s][0..2] = motion_blur_t( clip( base[s] < thres[t] ? 0 : base[s], 0, 1 ) )
 * noise [SB][ch][ch] (the centre crop FP:36-38), thres [T], taps [T][k] (1-D Gaussian, k odd), vertical [T][SB] (0: blur along x,
 * 1: along y with reversed taps = torch.rot90 of the horizontal kernel), base [SB][H][H] (workspace / output),
 * snow [T][SB][3][H][H] in the layout cd_snow reads.  Square images only (upstream crops with shape[0] on both axes). */
int cd_snow_layers(const double* noise, int SB, int ch, int m, int trim, int H, const float* thres, const float* taps,
                   int k, const unsigned char* vertical, int T, float* base, float* snow, void* stream);
/* ------------------------------------------------------------------------------------------
 * DDPM-style `Model` (deblurring-diffusion-pytorch/deblurring_diffusion_pytorch/Model2.py, "M2") forward pieces; the dense
 * convolutions (3x3, 1x1 q/k/v/proj/nin_shortcut, asymmetric-pad stride-2 Downsample, and the two batched matmuls of AttnBlock
 * as per-batch-weight 1x1 tap-list convolutions) run through cd_conv_fwd.
 * ------------------------------------------------------------------------------------------ */
/* GroupNorm(groups, eps) of (x + cond[b,c]) [* swish] on NHWC (M2:32-33, 114-123).  Statistics are Chan-merged (count,
 * mean, M2) triples and every sum within an image is added in a fixed order (cd_groupnorm_bwd too): accurate for inputs
 * with a large mean, and the same bits run to run (except dgamma / dbeta on planes of at most 128*128 pixels, to which the
 * images add atomically).  HW <= 128*128: one CTA per image.  Larger planes: a (pixel chunk x image) grid; its partials go to
 * a device buffer cached per (device, stream) that grows outside CUDA-graph capture only (a capture that would need it larger
 * fails: run the shape once before capturing).  Needs C % 4 == 0, C / 4 <= 512 and B <= 65535. */
int cd_groupnorm_fwd(const float* x, int x_ld, int B, int64_t HW, int C, int groups, const float* cond, int cond_ld,
                     const float* gamma, const float* beta, float eps, int swish, float* y, int y_ld, void* stream);
/* in-place softmax(scale * s) over the last dimension of [rows][n] (M2:172-175) */
int cd_softmax_rows(float* s, int ld, int64_t rows, int n, float scale, void* stream);
/* [B][R][C] -> [B][C][R] */
int cd_transpose_batched(const float* src, int ld, int B, int R, int C, float* dst, void* stream);
/* F.interpolate(scale_factor=2, mode='nearest') on NHWC (M2:47-48) */
int cd_upsample_nearest2x(const float* x, int x_ld, int B, int H, int W, int C, float* y, int y_ld, void* stream);
int cd_nhwc_to_nchw(const float* x, int ld, int B, int H, int W, int C, float* out, void* stream);
/* out = x (NHWC, row stride ld) + add (NCHW, the shape of out) in one pass; add = NULL is cd_nhwc_to_nchw (input gradient of the
 * networks, with the `x +` term of Unet(residual=True) as the addend) */
int cd_nhwc_to_nchw_add(const float* x, int ld, int B, int H, int W, int C, const float* add, float* out, void* stream);
/* get_timestep_embedding -> dense0 -> act -> dense1 (= temb) ; cond_all = Wc act(temb) + bc (all blocks' temb_proj) (M2:6-24,289-294,122).
 * temb ([B][tdim], optional output): when given, the dense layers run one block per sample and the sumC conditioning rows are
 * spread over the whole grid (2 launches); with temb == NULL everything runs in one block per sample (1 launch, slow for large sumC). */
int cd_time_mlp2_fwd(const int64_t* t, int B, int dim, int hid, int tdim, int act, const float* w1, const float* b1,
                     const float* w2, const float* b2, const float* wc, const float* bc, int sumC, float* temb,
                     float* cond_all, void* stream);
/* stand-alone EMA (DB:73-81): mode 1 copy, 2 lerp */
int cd_ema_update(float* ema, const float* p, int64_t n, float beta, int mode, void* stream);

/* ------------------------------------------------------------------------------------------
 * Training-mode pieces of the DDPM-style `Model` (Model2.py, "M2"); wired behind COLDDIFF_MODEL_TRAINING=1.
 *   cd_groupnorm_bwd         : backward of GroupNorm(32, eps 1e-6) [+ swish] (M2:32-33,116-125); x is the forward input, cond the
 *                              per-sample channel offset added before the norm (temb_proj row, M2:121); accumulates dgamma / dbeta,
 *                              writes dx and (optionally) dcond[b][c] = sum over pixels of dx.  dgamma = dbeta = NULL (both or
 *                              neither): no parameter reduction (frozen gamma and beta), dx and dcond unchanged
 *   cd_dropout               : y = x * keep / (1 - p) with a counter-based mask of (seed, element index) -- the same call with the
 *                              same seed on the gradient is the backward (M2:125; torch's RNG stream is not reproduced)
 *   cd_dropout_seed_dev      : cd_dropout with the seed read from device memory (*seed) when the kernel runs: the same mask
 *                              function, so the masks are bit-identical to cd_dropout's for the same seed value.  A captured
 *                              CUDA graph keeps the pointer, and a new seed staged there before each replay gives a new mask
 *   cd_softmax_bwd_rows      : ds <- s * (ds - sum_j ds*s) * scale for s = softmax(scale * logits) (M2:172-175)
 *   cd_upsample_nearest2x_bwd: sum of the four children (M2:47-48)
 *   cd_swish                 : act_out = swish(pre) and / or y = dy * swish'(pre) (M2:27-29)
 *   cd_timestep_embedding    : get_timestep_embedding (M2:6-24);  cd_linear_fwd: y = x W^T + b (M2:295-299, temb_proj M2:121)
 * ------------------------------------------------------------------------------------------ */
int cd_groupnorm_bwd(const float* x, int x_ld, int B, int64_t HW, int C, int groups, const float* cond, int cond_ld,
                     const float* gamma, const float* beta, float eps, int swish, const float* dy, int dy_ld,
                     float* dx, int dx_ld, float* dgamma, float* dbeta, float* dcond, int dcond_ld, void* stream);
int cd_dropout(const float* x, int x_ld, int64_t npix, int C, float p, uint64_t seed, float* y, int y_ld, void* stream);
int cd_dropout_seed_dev(const float* x, int x_ld, int64_t npix, int C, float p, const uint64_t* seed, float* y, int y_ld,
                        void* stream);
int cd_softmax_bwd_rows(const float* s, float* ds, int ld, int64_t rows, int n, float scale, void* stream);
int cd_upsample_nearest2x_bwd(const float* dy, int dy_ld, int B, int H, int W, int C, float* dx, int dx_ld, void* stream);
int cd_swish(const float* dy, const float* pre, int64_t n, float* y, float* act_out, void* stream);
int cd_timestep_embedding(const int64_t* t, int B, int dim, float* emb, void* stream);
int cd_linear_fwd(const float* x, int K, const float* w, const float* bias, int M, int N, float* y, void* stream);

/* Input pipeline (reference Dataset / Dataset_Aug1, DB:983-1026) with the decoded uint8 images resident in HBM ([N][Hs][Ws][3]):
 * out[b][c][y][x] = src[index[b]][oy[b]+y][ox[b] + (flip[b] ? S-1-x : x)][c] / 255 * 2 - 1   (RandomCrop / CenterCrop + flip + ToTensor*2-1).
 * Opt-in (Trainer(dataset='device...')). */
int cd_augment_u8(const uint8_t* src, int N, int Hs, int Ws, const int64_t* index, const int32_t* oy, const int32_t* ox,
                  const int32_t* flip, int B, int S, float* out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* COLDDIFF_H_ */
