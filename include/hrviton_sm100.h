/* hrviton_sm100.h — C-ABI of libhrviton_sm100.so (H100 / sm_90a only).
 *
 * The reference (sangyun884/HR-VITON) has no FFI layer: its seam is the Python module surface of
 * networks.py / network_generator.py, whose arithmetic is delegated to ATen/cuDNN ops.  Each entry
 * point below replaces the ATen op(s) the reference calls at the cited file:line; the Python drop-in
 * modules at the repo root (networks.py, network_generator.py) bind them through ctypes
 * (hr-viton_b200/capi.py).  See INTEGRATION.md for the reference-side binding.
 *
 * Conventions: every pointer is a DEVICE pointer owned by the caller; activations are NHWC
 * ("pixel-major") with a channel pitch; kernels are enqueued on the given stream and never allocate
 * or synchronise; every function returns 0 on success or a negative hrv_status, text via
 * hrv_last_error() (thread-local).  There is no CPU fallback.
 *
 * Storage flavours: every entry point below exists twice in the library — hrv_<op> keeps activations and packed weights in
 * bf16 (the training configuration), hrv_<op>_f16 (include/hrviton_sm100_f16.h, generated from this file) keeps them in IEEE
 * fp16: same signatures, same kernels compiled against the other 16-bit type, wgmma operand format f16 instead of bf16.
 * fp32 buffers (flows, logits, images, statistics, weight gradients) are identical in both.  Wherever a comment says "bf16" read
 * "the flavour's 16-bit storage type"; hrv_dtype code 0 denotes it.
 *
 * fp32 storage (the reference-precision inference mode): the forward entry points marked "fp32 storage" below also take activations
 * with dtype HRV_F32, in either flavour, and then run the same algorithm on fp32 NHWC tensors.  Every activation tensor of such a
 * call must be fp32 (mixed storage returns HRV_EINVAL).  hrv_conv2d_fwd on an fp32 input runs a 3xTF32 wgmma kernel over weights
 * packed by hrv_pack_conv_weight_tf32x2.  There is no fp32 backward pass.
 */
#ifndef HRVITON_SM100_H_
#define HRVITON_SM100_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* hrv_stream; /* cudaStream_t */

enum hrv_status { HRV_OK = 0, HRV_EINVAL = -1, HRV_ECUDA = -2, HRV_EUNSUPPORTED = -3 };
enum hrv_dtype {
  HRV_BF16 = 0, /* = the flavour's 16-bit type: bf16 in hrv_<op>, fp16 in hrv_<op>_f16 */
  HRV_F32 = 1   /* fp32: flows, logits, images, statistics; and activation storage of the fp32 inference mode */
};
enum hrv_act { HRV_ACT_NONE = 0, HRV_ACT_RELU = 1, HRV_ACT_LRELU02 = 2, HRV_ACT_TANH = 3 };
enum hrv_layout { HRV_NHWC = 0, HRV_NCHW = 1 };
enum hrv_epilogue { HRV_EPI_LINEAR = 0, HRV_EPI_SPADE = 1 };
enum hrv_res_mode { HRV_RES_ADD = 0, HRV_RES_GATE_RELU = 1, HRV_RES_GATE_LRELU = 2 };

/* NHWC view: element (n,y,x,c) lives at ptr + (((n*h + y)*w + x)*pitch + c) elements.
 * For tensors read through TMA (conv inputs): bf16, ptr 16-byte aligned, pitch % 8 == 0. */
typedef struct hrv_tensor {
  void* ptr;
  int32_t n, h, w, c;
  int32_t pitch;
  int32_t dtype; /* hrv_dtype */
} hrv_tensor;

/* One 2-D convolution as an implicit GEMM on wgmma tensor cores (bf16 in, fp32 accumulate in registers).
 * Replaces nn.Conv2d forward at networks.py:60-93,178-192 ; network_generator.py:97-99,132-135,184-201,
 * 263-272 and, with HRV_EPI_SPADE, the whole SPADENorm tail `normalized*(1+gamma)+beta` + LeakyReLU
 * (network_generator.py:115-121,170-171) fused into the gamma/beta convolution.
 *
 *   out[n,y,x,:] = epilogue( sum_{ky,kx,ci} in[n, y+ky-off_y, x+kx-off_x, ci] * W[:,ky,kx,ci] )
 *
 * (stride-1 taps; stride-2 convolutions are expressed on a space-to-depth input, see hrv_space_to_depth).
 * Out-of-range input pixels and channels read as zero (TMA OOB fill).
 *
 * wpack: bf16 [kh*kw][n_pad][cin_k], cin_k = ceil(in.c/bk)*bk, n_pad = ceil(n_gemm/bn)*bn, zero padded.
 *
 * LINEAR epilogue:  v = acc*scale[j] + shift[j] (+ res[n,y,x,j]);  out = act(v)            (j < cout)
 * SPADE  epilogue:  GEMM column 2c = gamma_c, 2c+1 = beta_c (n_gemm = 2*C);  xs = x0|x1 concat source,
 *                   v = ((xs + noise[n,y,x]*noise_scale[c]) - mean[n,c]) * rstd[n,c]
 *                       * (1 + acc[2c] + shift[2c]) + (acc[2c+1] + shift[2c+1]);  out[c] = act(v)
 *                   x0 may be half resolution (x0_shift=1: nearest x2 up-sampling folded into the index,
 *                   network_generator.py:203,226-242); x1 supplies channels [x0.c, x0.c+x1.c) (the torch.cat).
 *
 * One kernel (pixels as M, 64 or 128 output channels as N, K walked tap by tap in 64-channel blocks) runs every case; results are
 * bit-identical from launch to launch.
 *
 * fp32 storage: with in.dtype == HRV_F32 the call runs the 3xTF32 kernel (K walked in 32-channel blocks; every operand split into
 * hi = rna_tf32(v) and lo = rna_tf32(v - hi), products hi*hi + hi*lo + lo*hi summed in fp32: fp32-class accuracy).  wpack is then
 * the fp32 [2][kh*kw][n_pad][cin_k] operand of hrv_pack_conv_weight_tf32x2; out, res, x0 and x1 must be fp32 (HRV_EINVAL otherwise),
 * NHWC outputs with room in their pitch write the pad channels up to the next multiple of 8 as in 16-bit storage, and the training-only
 * gate res_modes and gamma_out are refused (HRV_EUNSUPPORTED).
 */
typedef struct hrv_conv_params {
  hrv_tensor in;
  const void* wpack;
  int32_t kh, kw, off_y, off_x;
  int32_t bk;     /* K chunk in elements: 64, 32 or 16 (=> TMA/UMMA swizzle 128B/64B/32B) */
  int32_t bn;     /* GEMM N tile: multiple of 16, 16..256 */
  int32_t n_gemm; /* GEMM N (cout, or 2*C for SPADE) */
  hrv_tensor out; /* n,h,w = output extent; dtype bf16|f32 */
  int32_t out_layout; /* hrv_layout; NCHW only with f32 */
  int32_t epi;    /* hrv_epilogue */
  int32_t act;    /* hrv_act */
  const float* scale; /* [n_gemm] or NULL (=1) */
  const float* shift; /* [n_gemm] or NULL (=0) */
  hrv_tensor res;     /* optional residual (ptr NULL = none), same n,h,w as out */
  hrv_tensor x0, x1;  /* SPADE sources (x1.ptr may be NULL) */
  int32_t x0_shift;
  const float* mean;  /* [N][C] */
  const float* rstd;  /* [N][C] */
  const float* noise; /* [N][H][W] or NULL */
  const float* noise_scale; /* [C] or NULL */
  hrv_tensor gamma_out; /* SPADE only, optional (ptr NULL = none): bf16 (n,h,w,C) receives gamma (incl. bias) for the backward pass */
  int32_t res_mode;     /* what `res` does in the LINEAR epilogue: 0 (HRV_RES_ADD) v += res;  1 (HRV_RES_GATE_RELU) out = act(v) * (res > 0);
                         * 2 (HRV_RES_GATE_LRELU) out = act(v) * (res > 0 ? 1 : 0.2).  The gate modes fuse the activation backward of the
                         * layer BELOW into the data-gradient convolution of the layer above (res = that layer's saved output), so that
                         * no separate dv = dy * act'(y) pass exists for ReLU chains such as Vgg19 (networks.py:201-231). */
} hrv_conv_params;

int hrv_conv2d_fwd(const hrv_conv_params* p, hrv_stream stream);

/* Per-(n,c) InstanceNorm statistics of  v = src(c) + noise[n,y,x]*noise_scale[c]  over the h*w pixels of
 * the (virtual) tensor  cat(up2^x0_shift(x0), x1)  — nn.InstanceNorm2d(affine=False) statistics
 * (network_generator.py:86,110; biased variance, eps inside the sqrt) without materialising the sum,
 * the up-sampling or the concatenation.  h,w = statistics extent.  workspace: hrv_instnorm_stats_workspace_bytes(...) bytes,
 * 8-byte aligned: every block writes its sums into its own slab, added in a fixed order (reproducible run to run); the first 2*N*C
 * doubles hold the raw sums {sum v, sum v^2}[N][C] afterwards.  Writes mean[N][C], rstd[N][C].  fp32 storage: x0/x1 may be fp32 (both). */
size_t hrv_instnorm_stats_workspace_bytes(const hrv_tensor* x0, const hrv_tensor* x1, int32_t h, int32_t w);
int hrv_instnorm_stats(const hrv_tensor* x0, int32_t x0_shift, const hrv_tensor* x1, int32_t h, int32_t w,
                       const float* noise, const float* noise_scale, float eps,
                       float* mean, float* rstd, void* workspace, size_t workspace_bytes, hrv_stream stream);

/* The same statistics for up to TWO norms that share the input but draw their own noise (norm_s and norm_0 of a SPADEResBlock,
 * network_generator.py:160-170), from ONE pass over the SOURCE tensors: x0 is read at its own (half) resolution, the noise enters
 * through the sums {sum nz, sum nz^2, sum x*nz} (see csrc/aux_kernels.cu).  noise1 / mean1 / rstd1 may be NULL (one norm).
 * workspace: hrv_instnorm_stats2_workspace_bytes(...) bytes (per-block slabs, added in a fixed order).  fp32 storage: x0/x1 may be
 * fp32 (both). */
size_t hrv_instnorm_stats2_workspace_bytes(const hrv_tensor* x0, const hrv_tensor* x1);
int hrv_instnorm_stats2(const hrv_tensor* x0, int32_t x0_shift, const hrv_tensor* x1, int32_t h, int32_t w, const float* noise0,
                        const float* noise_scale0, const float* noise1, const float* noise_scale1, float eps, float* mean0,
                        float* rstd0, float* mean1, float* rstd1, void* workspace, size_t workspace_bytes, hrv_stream stream);

/* y = act((x - mean[n,c]) * rstd[n,c]) elementwise on an NHWC bf16 tensor (InstanceNorm + LeakyReLU of the
 * discriminators, network_generator.py:269-270,427; networks.py:366-386). In place allowed.  fp32 storage: x and y fp32. */
int hrv_instnorm_apply(const hrv_tensor* x, const float* mean, const float* rstd, int32_t act,
                       const hrv_tensor* y, hrv_stream stream);

/* y = act(((x - mean[n,c]) * rstd[n,c]) * gamma[c] + beta[c] + res): train-mode BatchNorm2d (mean/rstd = batch statistics
 * replicated per image) + ReLU + residual of ResBlock (networks.py:188-198). gamma/beta/res optional. */
int hrv_norm_apply_affine(const hrv_tensor* x, const float* mean, const float* rstd, const float* gamma, const float* beta,
                          const hrv_tensor* res, int32_t act, const hrv_tensor* y, hrv_stream stream);

/* Backward of  h = act(xn*(1+gamma)+beta),  xn = InstanceNorm(cat(up2^x0_shift(x0), x1) + noise*noise_scale)
 * (network_generator.py:101-122,170-171), pass 1 of 2: per element dv = dh*act'(h), dgamma = dv*xn, dbeta = dv,
 * dxn = dv*(1+gamma); writes dgb (bf16 (n,h,w,2C), columns 2c = dgamma_c, 2c+1 = dbeta_c = dY of the gamma|beta GEMM; optional)
 * and dxn (bf16 (n,h,w,C)); writes sums[N][C][4] (fp64) = {sum dxn, sum dxn*xn, sum dgamma, sum dbeta}: per-block slabs in
 * `workspace` (hrv_norm_bwd_reduce_workspace_bytes(...) bytes, 8-byte aligned), added in a fixed order (reproducible run to run).
 * gamma == NULL means plain Instance/BatchNorm + activation: dxn = dv * chan_scale[c] (chan_scale = the BatchNorm affine weight,
 * NULL = 1). h is ignored when act == NONE. */
size_t hrv_norm_bwd_reduce_workspace_bytes(const hrv_tensor* x0, const hrv_tensor* x1, int32_t H, int32_t W);
int hrv_norm_bwd_reduce(const hrv_tensor* dh, const hrv_tensor* h, const hrv_tensor* gamma, const hrv_tensor* x0,
                        int32_t x0_shift, const hrv_tensor* x1, int32_t H, int32_t W, const float* noise,
                        const float* noise_scale, const float* mean, const float* rstd, const float* chan_scale, int32_t act,
                        const hrv_tensor* dgb, const hrv_tensor* dxn, double* sums, void* workspace, size_t workspace_bytes,
                        hrv_stream stream);

/* Pass 2: InstanceNorm backward dxs = rstd*(dxn - m1 - xn*m2) (m1 = sum dxn / HW, m2 = sum dxn*xn / HW, [N][C] fp32) for the
 * channel slice [c_off, c_off+src.c) of the virtual input; src = x0 (shift = x0_shift: the 2x2 children of every source pixel are
 * summed = backward of the nearest up-sampling) or x1 (shift 0). Writes dx (bf16, src extent) and
 * dns[c] = sum dxs*noise for c in [c_off, c_off+src.c) (fp64; may be NULL), from per-block slabs in `workspace`
 * (hrv_norm_bwd_apply_workspace_bytes(src) bytes, needed only with dns) added in a fixed order. */
size_t hrv_norm_bwd_apply_workspace_bytes(const hrv_tensor* src);
int hrv_norm_bwd_apply(const hrv_tensor* dxn, const hrv_tensor* src, int32_t shift, int32_t c_off, int32_t C, int32_t H,
                       int32_t W, const float* noise, const float* noise_scale, const float* mean, const float* rstd,
                       const float* m1, const float* m2, const hrv_tensor* dx, double* dns, void* workspace, size_t workspace_bytes,
                       hrv_stream stream);

/* Convolution weight gradient on wgmma: dw[co][ci][ky][kx] = sum_{n,y,x} dy[n,y,x,co] * x[n,y+ky-pad,x+kx-pad,ci]
 * (stride 1; x: (n,h,w,cin), dy: (n,h+2pad-kh+1, w+2pad-kw+1, cout), both bf16 NHWC; kw <= 4). dw is fp32 in the reference's
 * parameter layout (cout,cin,kh,kw) and is OVERWRITTEN.  The pixel (K) dimension is split over CTAs; each writes its partial tile
 * into its own slab of `workspace` and a second kernel adds the slabs in a fixed order: the result is bit-reproducible run to run.
 * workspace: hrv_conv2d_wgrad_workspace_bytes(...) bytes, 16-byte aligned (0 bytes when one CTA per output tile suffices).
 * The weight-gradient half of nn.Conv2d's backward for every convolution cited at hrv_conv2d_fwd. */
size_t hrv_conv2d_wgrad_workspace_bytes(const hrv_tensor* x, const hrv_tensor* dy, int32_t kh, int32_t kw);
int hrv_conv2d_wgrad(const hrv_tensor* x, const hrv_tensor* dy, int32_t kh, int32_t kw, int32_t pad, float* dw, void* workspace,
                     size_t workspace_bytes, hrv_stream stream);

/* dv = dy * act'(y) on NHWC bf16 (dv optional) and bias_sum[c] = sum over all pixels of dv (fp64 [roundup8(C)]; optional):
 * the activation backward + bias gradient of a conv epilogue act(conv + b) in one pass.  The blocks' sums land in per-block slabs of
 * `workspace` (hrv_act_bwd_bias_ordered_workspace_bytes(dy) bytes, needed only with bias_sum), added in a fixed order: reproducible. */
size_t hrv_act_bwd_bias_ordered_workspace_bytes(const hrv_tensor* dy);
int hrv_act_bwd_bias_ordered(const hrv_tensor* dy, const hrv_tensor* y, int32_t act, const hrv_tensor* dv, double* bias_sum,
                             void* workspace, size_t workspace_bytes, hrv_stream stream);
/* Legacy, non-reproducible form of hrv_act_bwd_bias_ordered that the package no longer calls: the block sums meet in bias_sum
 * (zeroed by the call) through fp64 atomics, so the last bits depend on block timing. */
int hrv_act_bwd_bias(const hrv_tensor* dy, const hrv_tensor* y, int32_t act, const hrv_tensor* dv, double* bias_sum,
                     hrv_stream stream);

/* fp32 NCHW -> bf16 NHWC with nearest resampling to (dst.h, dst.w): src index = min(floorf(dst * (in/out)), in-1), the scale
 * in/out and the product rounded to fp32 as F.interpolate(mode='nearest') computes them (network_generator.py:164,222; not the
 * exact floor(dst*in/out), which differs where the fp32 product falls just below an integer), and zero fill of dst channels >= C.
 * src: [n][c][src_h][src_w] fp32 contiguous.  fp32 storage: dst may be fp32 NHWC. */
int hrv_nchw_to_nhwc(const float* src, int32_t c, int32_t src_h, int32_t src_w, const hrv_tensor* dst, hrv_stream stream);

/* The condition discriminator's input for discriminator rejection (test_condition.py:106-120, get_norm_const.py:99-115) in one pass:
 *   dst[n,y,x,:] = [ input1 (c1) | input2 (c2) | third (k) ], zero fill of the pad channels of the last 8-channel group,
 *   third = softmax ? softmax_over_channels(composed) : composed,
 *   composed = seg with channel cm_channel multiplied by cm (mode 1, 'warp_grad') or by (cm > 0.5) (mode 2, 'detach'); mode 0: seg.
 * input1, input2, seg: fp32 [n][c][h][w] contiguous at dst's (n,h,w); cm: fp32 [n][1][h][w] (NULL with mode 0).  softmax = 0 copies
 * the third operand (the one-hot label of the real branch, get_norm_const.py:114).  The soft-max is fp32 with the maximum
 * subtracted, expf and a correctly rounded division; every output is rounded once to dst's type.  dst: bf16 NHWC view with
 * c = c1+c2+k, pitch % 8 == 0; fp32 storage: dst may be fp32 NHWC.  seg_out (optional): `composed` as fp32 [n][k][h][w]. */
int hrv_seg_softmax_cat(const float* input1, int32_t c1, const float* input2, int32_t c2, const float* seg, int32_t k,
                        const float* cm, int32_t cm_channel, int32_t mode, int32_t softmax, const hrv_tensor* dst,
                        float* seg_out, hrv_stream stream);

/* bf16|f32 NHWC view -> fp32 NCHW contiguous [n][c][h][w]. */
int hrv_nhwc_to_nchw(const hrv_tensor* src, float* dst, hrv_stream stream);

/* Space-to-depth by 2 with zero fill of odd edges: dst[n,Y,X,(py*2+px)*C8 + ci] = src[n,2Y+py,2X+px,ci], C8 = 8*ceil(src.c/8);
 * dst.h = ceil(src.h/2), dst.w = ceil(src.w/2), dst.c >= 4*C8 (every other channel zeroed; nothing past the view is read). Turns the
 * stride-2 convolutions (networks.py:185; network_generator.py:263-269; networks.py:360-372) into stride-1
 * 2x2 implicit GEMMs.  fp32 storage: src and dst fp32. */
int hrv_space_to_depth(const hrv_tensor* src, const hrv_tensor* dst, hrv_stream stream);

/* F.avg_pool2d(3, stride 2, pad 1, count_include_pad=False) on NHWC bf16 (network_generator.py:302,
 * networks.py:320). dst.h = (src.h-1)/2+1.  fp32 storage: src and dst fp32. */
int hrv_avgpool3s2(const hrv_tensor* src, const hrv_tensor* dst, hrv_stream stream);

/* dst = bilinear_up2(a) (+ b), align_corners=False (F.interpolate / nn.Upsample, networks.py:130,181).
 * a: (n,h,w,c) bf16; b (optional, ptr NULL = none) and dst: (n,2h,2w,c) bf16.  fp32 storage: a, b and dst fp32. */
int hrv_bilinear_up2_add(const hrv_tensor* a, const hrv_tensor* b, const hrv_tensor* dst, hrv_stream stream);

/* The appearance-flow warp (networks.py:133-135,147-152,161-168) in one kernel:
 *   flow_up = bilinear_up2(flow_lo)                      (fp32 [n][H][W][2], written to flow_up if non-NULL)
 *   g = flow_up / ((W/2-1)/2, (H/2-1)/2) + (lin_x[x], lin_y[y])      (correctly rounded fp32 division)
 *   ix = clamp(((g.x+1)*src.w-1)/2, 0, src.w-1)  (grid_sample, bilinear, border, align_corners=False)
 *   dst[n,y,x,:] = 4-tap lerp of src around (floor(ix), floor(iy))
 * flow_lo: fp32 [n][H/2][W/2][2]; lin_x/lin_y: torch.linspace(-1,1,W|H) tables; src: bf16|f32 NHWC (n,H,W,c);
 * dst: bf16|f32 NHWC view (n,H,W,c).  idx_out (optional): int32 [n][H][W][2] = (x0,y0) gather indices. */
int hrv_flow_warp(const float* flow_lo, const float* lin_x, const float* lin_y, const hrv_tensor* src,
                  const hrv_tensor* dst, float* flow_up, int32_t* idx_out, hrv_stream stream);

/* Backward of hrv_bilinear_up2_add w.r.t. `a`: da = adjoint of the x2 bilinear up-sampling applied to dout (bf16 NHWC;
 * the gradient w.r.t. `b` is dout itself). */
int hrv_bilinear_up2_bwd(const hrv_tensor* dout, const hrv_tensor* da, hrv_stream stream);

/* Backward of hrv_flow_warp (F.grid_sample backward with border padding, networks.py:135,152, fused with the flow chain),
 * reproducible bit for bit:
 *   dsrc32 [n][src.h][src.w][roundup8(c)] fp32, WRITTEN (may be NULL): d_dst * lerp weight gathered at every source pixel from the
 *          (destination pixel, tap) pairs that sample it, summed in ascending (destination pixel, tap) order without FMA contraction
 *          (one thread per destination pixel writes the taps, a stable radix sort by source pixel orders them, then a gather);
 *   dflow_up [n][H][W][2] fp32, caller-initialised (zeros, or the gradient arriving directly at the up-sampled flow):
 *            += analytic d/d(flow_up) of the sampled values, added per 8-channel group in ascending group order (zero where the
 *               coordinate was clamped; a coordinate exactly on the border, 0 or size-1, counts as clamped, as in torch's
 *               grid_sample backward);
 *   dflow_lo [n][H/2][W/2][2] fp32: written = adjoint of the x2 bilinear flow up-sampling applied to dflow_up (may be NULL).
 * workspace: hrv_flow_warp_bwd_ordered_workspace_bytes(src, ddst) bytes, 256-byte aligned (sort keys and values, weights, partials). */
size_t hrv_flow_warp_bwd_ordered_workspace_bytes(const hrv_tensor* src, const hrv_tensor* ddst);
int hrv_flow_warp_bwd_ordered(const float* flow_lo, const float* lin_x, const float* lin_y, const hrv_tensor* src, const hrv_tensor* ddst,
                              float* dsrc32, float* dflow_up, float* dflow_lo, void* workspace, size_t workspace_bytes, hrv_stream stream);
/* Legacy, non-reproducible form of hrv_flow_warp_bwd_ordered that the package no longer calls: dsrc32 is caller-zeroed and
 * receives d_dst * weight through fp32 atomics (+=), dflow_up likewise, so the last bits depend on thread timing. */
int hrv_flow_warp_bwd(const float* flow_lo, const float* lin_x, const float* lin_y, const hrv_tensor* src, const hrv_tensor* ddst,
                      float* dsrc32, float* dflow_up, float* dflow_lo, hrv_stream stream);

/* ---- training-step glue (SURVEY.md §8 rows N1/N2): pooling / re-layout backward passes and the parse-map post-processing ---- */

/* Backward of hrv_space_to_depth: dx[n,y,x,c] = d[n, y/2, x/2, ((y&1)*2+(x&1))*C8 + c], C8 = 8*ceil(dx.c/8). */
int hrv_space_to_depth_bwd(const hrv_tensor* d, const hrv_tensor* dx, hrv_stream stream);

/* nn.MaxPool2d(2, 2) of Vgg19 (networks.py:201-231) on NHWC bf16: y = (n, h/2, w/2, c) (floor mode). The backward routes dy to
 * the first maximum of each window (recomputed from x; no index tensor); relu_gate != 0 additionally multiplies by (x > 0), i.e. applies the
 * ReLU backward of the convolution that produced x (see hrv_conv_params.res_mode). */
int hrv_maxpool2_fwd(const hrv_tensor* x, const hrv_tensor* y, hrv_stream stream);
int hrv_maxpool2_bwd(const hrv_tensor* x, const hrv_tensor* dy, const hrv_tensor* dx, int32_t relu_gate, hrv_stream stream);

/* Backward of hrv_avgpool3s2 (count_include_pad=False): dx (n,h,w,c) from dy (n,(h-1)/2+1,(w-1)/2+1,c). */
int hrv_avgpool3s2_bwd(const hrv_tensor* dy, const hrv_tensor* dx, hrv_stream stream);

/* train_generator.py:247-273 in one kernel: bilinear resize of the (n,c,h,w) fp32 class scores to (H,W) (align_corners=False),
 * 15x15 Gaussian blur (sigma 3, zero padding; tgm.image.GaussianBlur), arg-max over classes (first maximum).
 * idx (optional): (n,H,W) int64 class ids.  onehot (optional): (n,groups,H,W) fp32, channel group_of[class] set to 1
 * (group_of: HOST array of c entries; the 13 -> 7 label regrouping).  overlap (optional): (n,1,H,W) fp32 = sum over the classes
 * whose bit is set in occl_mask of softmax_c(blurred scores) — the operand of remove_overlap under --occlusion
 * (train_generator.py:26-31,242-243), computed with an online softmax so the 13 blurred planes never reach HBM. */
int hrv_parse_blur_argmax(const float* seg, int32_t n, int32_t c, int32_t h, int32_t w, int32_t H, int32_t W,
                          const int32_t* group_of, int32_t groups, int64_t* idx, float* onehot, uint32_t occl_mask,
                          float* overlap, hrv_stream stream);

/* Input feeding (cp_dataset.py:150-172 ships a one-hot fp32 parse map; here the host ships one byte per pixel):
 * out (n,classes,h,w) fp32 with out[n,c,y,x] = (labels[n,y,x] == c). */
int hrv_onehot_u8(const uint8_t* labels, int32_t n, int32_t classes, int32_t h, int32_t w, float* out, hrv_stream stream);

/* tgm.image.GaussianBlur((ksize,ksize),(sigma,sigma)) on `planes` fp32 planes of h x w (train_generator.py:181,247;
 * test_generator.py:91,185): separable, zero padding ksize/2, taps exp(-d^2/(2 sigma^2)) normalised to sum 1; odd ksize <= 31. */
int hrv_gaussian_blur(const float* src, int32_t planes, int32_t h, int32_t w, int32_t ksize, float sigma, float* dst,
                      hrv_stream stream);

/* The hi-resolution cloth warp of the glue (train_generator.py:232-238, test_generator.py:170-176) in one kernel:
 *   flow = F.interpolate(flow_lo (n,hl,wl,2), size=(h,w), bilinear, align_corners=False)      (any scale)
 *   g = flow / (div_x, div_y) + (lin_x[x], lin_y[y])          (correctly rounded fp32 division; lin_* = torch.linspace(-1,1,w|h))
 *   dst[n,:,y,x] = grid_sample(src (n,c,hs,ws) fp32 NCHW, g, bilinear, border, align_corners=False)
 * grid_out (optional): (n,h,w,2) fp32 receives g.
 * mask_src (optional, (n,1,hs,ws)): the cloth mask, sampled with the same taps -> wm; overlap (optional, (n,1,h,w)):
 * wm -= overlap*wm (remove_overlap); mask_out (optional) receives wm; composite != 0: dst = sample*wm + (1 - wm)
 * (the white-background composite of train_generator.py:244 / test_generator.py:178). */
int hrv_flow_warp_nchw(const float* flow_lo, int32_t n, int32_t hl, int32_t wl, const float* lin_x, const float* lin_y,
                       const float* src, int32_t c, int32_t hs, int32_t ws, float* dst, int32_t h, int32_t w, float div_x,
                       float div_y, float* grid_out, const float* mask_src, const float* overlap, float* mask_out,
                       int32_t composite, hrv_stream stream);

/* Backward of hrv_flow_warp_nchw w.r.t. flow_lo only (the cloth and its mask are data; overlap / composite have no backward here:
 * apply remove_overlap and the composite outside, as differentiable ops).  d_dst (n,c,h,w) and d_mask (n,1,h,w) are the incoming
 * gradients of the warped cloth and mask (either may be NULL, not both).  Writes d_flow_lo (n,hl,wl,2) fp32: the analytic
 * grid_sample(border) coordinate gradient per hi-res pixel (channels then mask, in that order; none where the coordinate was clamped
 * or exactly on the border), times 1/div, then the adjoint of the any-factor bilinear resize (align_corners=False) as a row-then-column
 * gather in ascending order: reproducible bit for bit.  workspace: hrv_flow_warp_nchw_bwd_workspace_bytes(n, h, w, wl) bytes, 8-byte aligned. */
size_t hrv_flow_warp_nchw_bwd_workspace_bytes(int32_t n, int32_t h, int32_t w, int32_t wl);
int hrv_flow_warp_nchw_bwd(const float* flow_lo, int32_t n, int32_t hl, int32_t wl, const float* lin_x, const float* lin_y,
                           const float* src, int32_t c, int32_t hs, int32_t ws, const float* d_dst, int32_t h, int32_t w,
                           float div_x, float div_y, const float* mask_src, const float* d_mask, float* d_flow_lo,
                           void* workspace, size_t workspace_bytes, hrv_stream stream);

/* im2col for tiny-Cin convolutions: dst[n,y,x, (ky*kw+kx)*src.c + ci] = src[n, y+ky-pad, x+kx-pad, ci], zero outside the image
 * and in channels >= kh*kw*src.c.  Lets SPADE's 3x3 mlp_shared convolution over the 7-channel label map
 * (network_generator.py:182-184) run as a single K=64 GEMM block (hrv_conv2d_fwd with kh=kw=1) and its weight gradient as a 1x1.
 * fp32 storage: src and dst fp32. */
int hrv_im2col(const hrv_tensor* src, const hrv_tensor* dst, int32_t kh, int32_t kw, int32_t pad, hrv_stream stream);

/* L1 feature loss (VGGLoss, networks.py:244-251): *sum = sum |a - b| over the views (fp64; every block writes its partial into
 * `workspace`, hrv_l1_sum_workspace_bytes(a) bytes, added in a fixed order: reproducible); da = sign(a - b) * (*gscale)
 * (times (a > 0) when relu_gate != 0: the ReLU backward of the producer of a, fused). */
size_t hrv_l1_sum_workspace_bytes(const hrv_tensor* a);
int hrv_l1_sum(const hrv_tensor* a, const hrv_tensor* b, double* sum, void* workspace, size_t workspace_bytes, hrv_stream stream);
int hrv_l1_bwd(const hrv_tensor* a, const hrv_tensor* b, const float* gscale, const hrv_tensor* da, int32_t relu_gate, hrv_stream stream);

/* Dynamic loss scaling (the reference's apex-O1 --fp16 runs, train_generator.py:161-169,317-321,355-359): one in-place pass over
 * fp32 gradient tensors after the backward of a loss multiplied by a scale S.  For every element g of every segment:
 *   g = g * (*inv_scale)                         (inv_scale: device scalar, read at run time so a graph replay sees the current 1/S)
 *   *found_inf = 1.0f   if g was inf or NaN      (otherwise *found_inf is left as is: the caller zeroes it before the call)
 * segments: DEVICE array of num_segments {ptr, n} entries (n fp32 elements at ptr, 4-byte aligned; n may be 0).  Aligned 16-byte
 * accesses, scalar head and tail.  No workspace; no atomics: every writer of found_inf stores the same value, so the result does not
 * depend on timing.  With S a power of two the product is exact unless it falls below fp32's normal range. */
typedef struct hrv_grad_segment {
  float* ptr;
  int64_t n;
} hrv_grad_segment;
int hrv_grad_unscale_check(const hrv_grad_segment* segments, int32_t num_segments, const float* inv_scale, float* found_inf,
                           hrv_stream stream);

/* Synchronised train-mode BatchNorm2d across data-parallel ranks (the reference's sync_batchnorm.SynchronizedBatchNorm2d): each
 * rank reduces its shard with the kernels above, the caller all-reduces (sum) one fp64 wire buffer per layer and direction, and a
 * finalize kernel turns the global sums into the per-image tables the apply kernels read.  No atomics: reproducible run to run.
 *
 * Combine: wire[2c + k] = sum over images i = 0..n-1, added in index order, of sums[(i*c_count + c)*stride + k] (k = 0, 1), and
 * wire[2*c_count] = count (the elements behind the sums: n*h*w).  sums = the {sum x, sum x^2}[n][C] hrv_instnorm_stats leaves at the
 * start of its workspace (stride 2), or the {sum dxn, sum dxn*xn, ...}[n][C][4] of hrv_norm_bwd_reduce (stride 4).  The wire holds
 * 2*c_count + 1 doubles; since the count is summed with the sums, ranks with unequal shards are still normalised by the global count. */
int hrv_syncbn_combine(const double* sums, int32_t n, int32_t c_count, int32_t stride, double count, double* wire, hrv_stream stream);

/* Forward finalize of the all-reduced wire (2*c + 1 doubles): mean = S1/count and biased var = S2/count - mean^2 (>= 0) in fp64,
 * rounded to fp32; rstd = rsqrtf(var + eps) in fp32 (the arithmetic of the per-rank BatchNorm path).  Writes mean[n][c], rstd[n][c] (fp32, the same row for every image: the layout of
 * hrv_norm_apply_affine).  running_mean / running_var (fp32 [c_run], both or neither) are updated in place for channels < c_run
 * as torch's BatchNorm2d does: r = r*(1-momentum) + x*momentum, the variance with the unbiased factor count/(count-1). */
int hrv_syncbn_fwd_finalize(const double* wire, int32_t n, int32_t c, int32_t c_run, float eps, double momentum, float* mean,
                            float* rstd, float* running_mean, float* running_var, hrv_stream stream);

/* Backward finalize of the all-reduced wire of the backward sums: m1[n][c] = S1/count, m2[n][c] = S2/count (fp32), the inputs of
 * hrv_norm_bwd_apply for BatchNorm statistics over every rank's pixels. */
int hrv_syncbn_bwd_finalize(const double* wire, int32_t n, int32_t c, float* m1, float* m2, hrv_stream stream);

/* fp32 parameter (cout,cin,kh,kw) -> bf16 GEMM operand [kh*kw][n_pad][cin_k] of hrv_conv2d_fwd, zero padded, in one pass.
 * w1 (optional): second parameter of identical shape whose rows are interleaved with w0's (row 2c = w0[c], 2c+1 = w1[c]: the
 * SPADE gamma|beta GEMM).  transpose_flip != 0 packs the operand of the data-gradient convolution instead (rows = input channels,
 * K = output channels, taps mirrored).  inv_scale (optional, device scalar) multiplies every element (1/sigma of spectral norm). */
int hrv_pack_conv_weight(const float* w0, const float* w1, int32_t cout, int32_t cin, int32_t kh, int32_t kw,
                         int32_t transpose_flip, const float* inv_scale, void* dst, int32_t n_pad, int32_t cin_k, hrv_stream stream);

/* The weight operand of hrv_conv2d_fwd on fp32 storage, same arguments and element mapping as hrv_pack_conv_weight: dst is fp32
 * [2][kh*kw][n_pad][cin_k], plane 0 = hi = rna_tf32(v), plane 1 = lo = rna_tf32(v - hi) (rna = round to nearest, ties away). */
int hrv_pack_conv_weight_tf32x2(const float* w0, const float* w1, int32_t cout, int32_t cin, int32_t kh, int32_t kw,
                                int32_t transpose_flip, const float* inv_scale, void* dst, int32_t n_pad, int32_t cin_k,
                                hrv_stream stream);

/* Library / device introspection. */
const char* hrv_last_error(void);
int hrv_version(void);
int hrv_device_sm_count(void);

#ifdef __cplusplus
}
#endif

/* The evaluation metrics (LPIPS, SSIM): fp32 / fp64 only, one flavour, declared in their own header. */
#include "hrviton_sm100_metrics.h"

#endif /* HRVITON_SM100_H_ */
