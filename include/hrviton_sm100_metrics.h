/* hrviton_sm100_metrics.h — evaluation-metric entry points of libhrviton_sm100.so (H100 / sm_90a only), included by hrviton_sm100.h.
 *
 * They replace the ATen / scipy code behind the reference's quality measurements: LPIPS (eval_models, AlexNet with the v0.1 linear
 * heads; train_generator.py:480-584, evaluate.py:41,72) and skimage's Gaussian SSIM (evaluate.py:67).  Same conventions as
 * hrviton_sm100.h (device pointers owned by the caller, enqueued on `stream`, 0 or a negative hrv_status, text via hrv_last_error()),
 * but unlike the entry points there these have ONE flavour: they compute in fp32 and fp64 only, whatever the activation storage of
 * the rest of the library, so there is no _f16 twin.  The AlexNet convolutions themselves run on hrv_conv2d_fwd in fp32 storage
 * (3xTF32), conv1 as a 1x1 GEMM over the operand hrv_lpips_input writes.  No floating-point atomics: results are reproducible.
 */
#ifndef HRVITON_SM100_METRICS_H_
#define HRVITON_SM100_METRICS_H_

#include "hrviton_sm100.h"

#ifdef __cplusplus
extern "C" {
#endif

/* LPIPS ScalingLayer + conv1 operand (eval_models/networks_basic.py:94-101, AlexNet features[0]: 11x11, stride 4, pad 2).
 * x: fp32 NCHW [n_img][3][h][w] (the two inputs of a comparison stacked: the N first images against the N last), h, w >= 7.
 * dst: fp32 NHWC (n_img, ho, wo, c = 363), ho = (h - 7)/4 + 1, wo = (w - 7)/4 + 1, pitch % 8 == 0, 16-byte aligned:
 *   dst[i,oy,ox,(ky*11+kx)*3+ci] = (x[i,ci,4oy-2+ky,4ox-2+kx] - shift[ci]) / scale[ci]   (fp32, correctly rounded division)
 * and 0 where the tap falls outside the image (the padding applies to the scaled input) and in the pad channels [363, pitch).
 * shift, scale: fp32 [3] (the ScalingLayer buffers). */
int hrv_lpips_input(const float* x, int32_t n_img, int32_t h, int32_t w, const float* shift, const float* scale, const hrv_tensor* dst,
                    hrv_stream stream);

/* nn.MaxPool2d(3, 2) of AlexNet (floor mode, no padding) on fp32 NHWC: y = (n, (h-3)/2+1, (w-3)/2+1, c).  torch's comparison (NaN
 * propagates, ties keep the first value): bit-exact. */
int hrv_maxpool3s2(const hrv_tensor* x, const hrv_tensor* y, hrv_stream stream);

/* One LPIPS layer (eval_models/__init__.py normalize_tensor, networks_basic.py:70-78): feat is fp32 NHWC holding 2N images, image i
 * compared with image i + N.  Per pixel  d = sum_c lin_w[c] * (f0_c - f1_c)^2,  f = x / (sqrt(sum_c x_c^2) + 1e-10), computed in fp64;
 * out[i] (fp32 [N]) = the mean of d over the pixels (spatial_average), rounded once. */
int hrv_lpips_dist(const hrv_tensor* feat, const float* lin_w, float* out, hrv_stream stream);

/* Mean SSIM per image of two (n,h,w) grayscale stacks, as skimage.metrics.structural_similarity(im1, im2, data_range=data_range,
 * gaussian_weights=True, use_sample_covariance=False) computes it (sigma 1.5, truncate 3.5: an 11-tap Gaussian; K1 0.01, K2 0.03), in
 * fp64: the five Gaussian moment maps, the SSIM map, its mean over the outputs 5 pixels or more from every border.  Only those outputs
 * are computed and their windows lie inside the image, so the filter's border mode plays no part.  h, w >= 11 (HRV_EINVAL otherwise,
 * as skimage refuses a window larger than the image).  dtype: HRV_SSIM_U8 (uint8 pixels) or HRV_SSIM_F32 (fp32 pixels, e.g. uint8
 * values).  out: fp64 [n].  workspace: hrv_ssim_workspace_bytes(n, h, w) bytes, 8-byte aligned (per-block sums, added in a fixed order). */
enum hrv_ssim_dtype { HRV_SSIM_U8 = 0, HRV_SSIM_F32 = 1 };
size_t hrv_ssim_workspace_bytes(int32_t n, int32_t h, int32_t w);
int hrv_ssim(const void* im1, const void* im2, int32_t dtype, int32_t n, int32_t h, int32_t w, double data_range, double* out,
             void* workspace, size_t workspace_bytes, hrv_stream stream);

#ifdef __cplusplus
}
#endif
#endif /* HRVITON_SM100_METRICS_H_ */
