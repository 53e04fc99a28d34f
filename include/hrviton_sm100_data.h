/* hrviton_sm100_data.h — input-pipeline entry points of libhrviton_sm100.so (H100 / sm_90a only): the device half of the VITON-HD
 * loader (hrviton_b200.data), which turns the uint8 planes its CPU workers decode into the fp32 tensors cp_dataset.py /
 * cp_dataset_test.py produce, bit for bit.
 *
 * Same conventions as hrviton_sm100.h (device pointers owned by the caller, enqueued on `stream`, 0 or a negative hrv_status, text via
 * hrv_last_error()).  Inputs are uint8 and outputs fp32 whatever the activation storage of the rest of the library, so there is ONE
 * flavour of each (no _f16 twin).  Integer arithmetic only, except the normalisation in hrv_viton_assemble, which is IEEE fp32.
 */
#ifndef HRVITON_SM100_DATA_H_
#define HRVITON_SM100_DATA_H_

#include "hrviton_sm100.h"

#ifdef __cplusplus
extern "C" {
#endif

/* One pass of Pillow's separable bilinear resample (Image.resize(..., BILINEAR), which transforms.Resize(interpolation=2) runs on a
 * PIL image), over `planes` uint8 NHWC images (planes, h, w, c), c = 1 or 3.  axis 0 resamples x into dst (planes, h, out_len, c),
 * axis 1 resamples y into dst (planes, out_len, w, c).  bounds: int32 [out_len][2] = {first source index, tap count <= ksize},
 * coeffs: int32 [out_len][ksize], the normalised weights in 22-bit fixed point (the host builds both as Pillow's precompute_coeffs
 * and normalize_coeffs_8bpc do).  dst = clip8((2^21 + sum_k src * coeff) >> 22).  Pillow runs the x pass first, then the y pass on
 * the uint8 result. */
int hrv_pil_resample_pass(const uint8_t* src, int32_t planes, int32_t h, int32_t w, int32_t c, int32_t axis, const int32_t* bounds,
                          const int32_t* coeffs, int32_t ksize, int32_t out_len, uint8_t* dst, hrv_stream stream);

/* Pillow's nearest resize of `planes` one-channel uint8 images (planes, h, w) into dst (planes, oh, ow):
 * dst[p,y,x] = lut ? lut[src[p, ys[y], xs[x]]] : src[p, ys[y], xs[x]].  ys: int32 [oh], xs: int32 [ow] (source indices, built on the
 * host by Pillow's accumulating stepping); lut: uint8 [256] or NULL (the label regrouping of cp_dataset.py:150-172). */
int hrv_pil_nearest(const uint8_t* src, int32_t planes, int32_t h, int32_t w, const int32_t* ys, int32_t oh, const int32_t* xs, int32_t ow,
                    const uint8_t* lut, uint8_t* dst, hrv_stream stream);

/* cp_dataset.get_agnostic's composite at source resolution: image (n, h, w, 3) uint8, parse (n, h, w) uint8 labels 0-19, bits
 * (n, h, w) uint8 with bit 0 = covered by the grey torso / neck / arm shapes, bit 1 / bit 2 = covered by the black shapes of the
 * arm masks of labels 14 / 15.  dst (n, h, w, 3) = (bit0 && !R) ? 128 : image, with the restored set
 * R = (!bit1 && parse == 14) || (!bit2 && parse == 15) || parse in {4, 13} || parse in {9, 12, 16, 17, 18, 19}. */
int hrv_agnostic_composite(const uint8_t* image, const uint8_t* parse, const uint8_t* bits, int32_t n, int32_t h, int32_t w, uint8_t* dst,
                           hrv_stream stream);

/* The ImageDraw shapes of the reference's agnostic masks, rasterised pixel for pixel as Pillow 12.2 draws them (csrc/draw_kernels.cu
 * states the rules).  keypoints: (n, 25, 2) fp64 OpenPose keypoints as read from the JSON, a keypoint (0, 0) being absent; every
 * coordinate finite and within +-4096 (the Python layer checks this).  workspace: device memory of hrv_draw_workspace_bytes(n, h)
 * bytes that no other launch uses until this one has finished.
 *
 * hrv_agnostic_bits: cp_dataset.get_agnostic's shapes as the bit plane of hrviton_b200.data.agnostic_bits, bits (n, h, w) uint8:
 * bit 0 = a grey torso / neck / arm shape, bits 1 / 2 = the label-14 / label-15 arm masks.  get_agnostic draws the arm masks on a
 * 768 x 1024 canvas whatever the image size, so the result is the reference's only for h = 1024, w = 768.
 *
 * hrv_parse_agnostic: get_parse_agnostic.get_im_parse_agnostic(labels, keypoints, w, h) on a batch: labels (n, h, w) uint8,
 * out (n, h, w) uint8 = 0 where the pixel is labelled 5, 6, 7 or 10, or labelled 14 / 15 and covered by that label's arm mask
 * (r = 10: lines of width 100, joint ellipses of radius 150, the hand's of radius 40), else the label. */
size_t hrv_draw_workspace_bytes(int32_t n, int32_t h);
int hrv_agnostic_bits(const double* keypoints, int32_t n, int32_t h, int32_t w, uint8_t* bits, void* workspace, size_t workspace_bytes,
                      hrv_stream stream);
int hrv_parse_agnostic(const double* keypoints, const uint8_t* labels, int32_t n, int32_t h, int32_t w, uint8_t* out, void* workspace,
                       size_t workspace_bytes, hrv_stream stream);

/* Fine-size uint8 planes of one batch (NULL: absent).  RGB planes are (n, h, w, 3); cloth[s] / cloth_mask[s] hold the paired (s = 0)
 * and unpaired (s = 1) cloth; parse holds the regrouped label ids 0-12, (n, h, w). */
typedef struct hrv_viton_planes {
  const uint8_t* image;
  const uint8_t* cloth[2];
  const uint8_t* cloth_mask[2];
  const uint8_t* pose;
  const uint8_t* densepose;
  const uint8_t* agnostic;
  const uint8_t* parse;
} hrv_viton_planes;

/* fp32 NCHW outputs of one batch (NULL: not written): image, cloth, pose, densepose, agnostic (n, 3, h, w) = (u / 255 - 0.5) / 0.5 as
 * ToTensor + Normalize compute it (fp32 divide, subtract, divide); cloth_mask (n, 1, h, w) = (u >= 128); pcm (n, 1, h, w) =
 * (parse == 3); parse_cloth (n, 3, h, w) = image * pcm + (1 - pcm); parse_onehot (n, 1, h, w) = parse. */
typedef struct hrv_viton_outputs {
  float* image;
  float* cloth[2];
  float* cloth_mask[2];
  float* pose;
  float* densepose;
  float* agnostic;
  float* pcm;
  float* parse_cloth;
  float* parse_onehot;
} hrv_viton_outputs;

/* Every output of one batch in one launch (one thread per pixel).  An output needs its plane (image for parse_cloth, parse for pcm,
 * parse_cloth and parse_onehot): HRV_EINVAL otherwise. */
int hrv_viton_assemble(const hrv_viton_planes* src, const hrv_viton_outputs* dst, int32_t n, int32_t h, int32_t w, hrv_stream stream);

#ifdef __cplusplus
}
#endif
#endif /* HRVITON_SM100_DATA_H_ */
