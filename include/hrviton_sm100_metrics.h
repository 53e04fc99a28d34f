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

/* ---- Inception-v3 (Inception Score, FID, KID; evaluate.py:43,75-76,96-106).  The convolutions run on hrv_conv2d_fwd in fp32 storage
 * (3xTF32) with BatchNorm as the epilogue's scale / shift, stride-2 ones on hrv_space_to_depth, the max pools on hrv_maxpool3s2. */

/* F.interpolate(x, (dst.h, dst.w), mode='bilinear', align_corners=False, antialias=False), bit-identical to torch's kernel, from fp32
 * NCHW x [n][c][h][w] to fp32 NHWC dst (n, oh, ow, c), pitch >= round_up(c, 8); channels [c, round_up(c, 8)) are written as zeros.
 * unit_range != 0 maps every input value v to 2v - 1 before the interpolation (images in [0, 1] to the network's [-1, 1]). */
int hrv_resize_bilinear_nhwc(const float* x, int32_t n, int32_t c, int32_t h, int32_t w, int32_t unit_range, const hrv_tensor* dst,
                             hrv_stream stream);

/* ---- pytorch-fid's FID Inception (fid_inception_v3): torchvision's Inception3(num_classes=1008, aux_logits=False) whose pool
 * branches are F.avg_pool2d(3, 1, 1, count_include_pad=False) (Mixed_5b-5d, 6b-6e, 7b) and F.max_pool2d(3, 1, 1) (Mixed_7c). */

/* pytorch-fid's input: F.interpolate(v, (dst.h, dst.w), mode='bilinear', align_corners=False), then 2v - 1 (after the blend), written
 * as fp32 NHWC dst (n, oh, ow, c), pitch >= round_up(c, 8), channels [c, round_up(c, 8)) zero; bit-identical to those torch calls.
 * src HRV_FID_SRC_F32_NCHW: x is fp32 NCHW [n][c][h][w], v = x (images in [0, 1]).  src HRV_FID_SRC_U8_NHWC: x is uint8 NHWC
 * [n][h][w][c] (interleaved, as PIL decodes RGB), v = u8 / 255 correctly rounded in fp32, as TF.to_tensor computes it. */
enum hrv_fid_src { HRV_FID_SRC_F32_NCHW = 0, HRV_FID_SRC_U8_NHWC = 1 };
int hrv_resize_bilinear_fid(const void* x, int32_t src, int32_t n, int32_t c, int32_t h, int32_t w, const hrv_tensor* dst, hrv_stream stream);

/* A 3x3, stride-1, padding-1 pool of fp32 NHWC x into fp32 NHWC y of the same extent (y may be a channel slice of a wider buffer).
 * mode HRV_POOL3X3_AVG_EXCL_PAD: F.avg_pool2d(count_include_pad=False), the in-image taps summed in raster order in fp32 and divided
 * once by their count; mode HRV_POOL3X3_MAX: F.max_pool2d (NaN propagates, ties keep the first value).  Both bit-identical to torch's
 * CUDA kernels.  16-byte accesses when c, both pitches and both pointers allow them. */
enum hrv_pool3x3_mode { HRV_POOL3X3_AVG_EXCL_PAD = 0, HRV_POOL3X3_MAX = 1 };
int hrv_pool3x3s1(const hrv_tensor* x, int32_t mode, const hrv_tensor* y, hrv_stream stream);

/* Global average pool: y (n, 1, 1, c) fp32 = the mean of x (n, h, w, c) fp32 over its h*w pixels, summed in fp64 in raster order and
 * rounded once. */
int hrv_global_avgpool(const hrv_tensor* x, const hrv_tensor* y, hrv_stream stream);

/* C = A B^T in fp64:  c[i*ldc + j] (+)= sum_{k'<k} A(i,k') B(j,k'),  A(i,k') = a[i*sam + k'*sak] (i < m),  B(j,k') = b[j*sbn + k'*sbk]
 * (j < n), elements fp32 (HRV_GRAM_F32) or fp64 (HRV_GRAM_F64); accumulate != 0 adds the product to c instead of overwriting it.
 * Every product is summed in increasing k' by one thread; a long K over few output tiles is split into ranges whose partial results
 * land in workspace slabs that a second kernel adds in range order.  The split depends on (m, n, k) only: the result is the same on
 * every run and every device.  Accesses are coalesced when one of each operand's strides is 1.
 * workspace: hrv_gram_f64_workspace_bytes(m, n, k) bytes, 8-byte aligned (0: none needed). */
enum hrv_gram_dtype { HRV_GRAM_F32 = 0, HRV_GRAM_F64 = 1 };
size_t hrv_gram_f64_workspace_bytes(int32_t m, int32_t n, int32_t k);
int hrv_gram_f64(const void* a, int64_t sam, int64_t sak, const void* b, int64_t sbn, int64_t sbk, int32_t dtype, int32_t m, int32_t n, int32_t k,
                 double* c, int64_t ldc, int32_t accumulate, void* workspace, size_t workspace_bytes, hrv_stream stream);

/* The three sums of KID's unbiased MMD^2 for each of `subsets` subsets, over the cubic polynomial kernel k(g) = (g*gamma + 1)^3 of the
 * precomputed fp64 Gram matrices gxx [na][na] = X X^T, gyy [nb][nb] = Y Y^T and gxy [na][nb] = X Y^T.  ix, iy: int32 [subsets][m]
 * feature indices (distinct within a subset).  out: fp64 [subsets][3] = { sum_{i!=j} k(gxx[ix_i][ix_j]), sum_{i!=j} k(gyy[iy_i][iy_j]),
 * sum_{i,j} k(gxy[ix_i][iy_j]) }, each in a fixed order.  2 <= m <= min(na, nb). */
int hrv_kid_sums(const double* gxx, const double* gyy, const double* gxy, int32_t na, int32_t nb, const int32_t* ix, const int32_t* iy,
                 int32_t subsets, int32_t m, double gamma, double* out, hrv_stream stream);

#ifdef __cplusplus
}
#endif
#endif /* HRVITON_SM100_METRICS_H_ */
