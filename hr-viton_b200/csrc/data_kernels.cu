// data_kernels.cu — the device half of the VITON-HD loader (include/hrviton_sm100_data.h, hrviton_b200/data.py): Pillow's bilinear
// and nearest resizes restated in integers, get_agnostic's composite, and the batch assembly from fine-size uint8 planes to the fp32
// tensors of cp_dataset.py.  uint8 in, fp32 out whatever the activation storage, so this translation unit is compiled once.  Every
// result is bit-identical to the reference's CPU path: the resizes use the host's fixed-point tables and integer sums only, and the
// normalisation is written with correctly rounded intrinsics so that no multiply-add is contracted.
#include "hrv_host.h"
#include "../../include/hrviton_sm100_data.h"

namespace hrv_data {
using hrv_host::set_error;

int launched(const char* what) {
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? HRV_OK : set_error(HRV_ECUDA, "%s: %s", what, cudaGetErrorString(e));
}
unsigned nblocks(long long total, int threads) { return (unsigned)((total + threads - 1) / threads); }

constexpr int kPrecisionBits = 22;  // Pillow's PRECISION_BITS for 8-bit images: 32 - 8 - 2

__device__ __forceinline__ unsigned char clip8(int ss) {
  const int v = ss >> kPrecisionBits;
  return (unsigned char)(v < 0 ? 0 : v > 255 ? 255 : v);
}

// ------------------------------------------------------------------------------------------------ Pillow bilinear, one pass
// thread = one output pixel (all C channels, so the tap table is read once).  AXIS 0: x pass, taps along a row; AXIS 1: y pass, taps
// down a column (a warp reads 32 consecutive pixels of each source row).  Integer sums in Pillow's order (tap 0 first).
template <int C, int AXIS>
__global__ void __launch_bounds__(256) pil_resample_kernel(const unsigned char* __restrict__ src, int h, int w, const int* __restrict__ bounds,
                                                           const int* __restrict__ coeffs, int ksize, int oh, int ow,
                                                           unsigned char* __restrict__ dst, long long total) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int x = (int)(idx % ow);
  const long long py = idx / ow;
  const int y = (int)(py % oh);
  const long long p = py / oh;
  const int o = AXIS == 0 ? x : y;
  const int first = __ldg(bounds + 2 * o), count = __ldg(bounds + 2 * o + 1);
  const int* k = coeffs + (long long)o * ksize;
  int ss[C];
#pragma unroll
  for (int ch = 0; ch < C; ++ch) ss[ch] = 1 << (kPrecisionBits - 1);
  // source pixel of tap t: AXIS 0 (p, y, first + t), AXIS 1 (p, first + t, x)
  const long long base = AXIS == 0 ? ((p * h + y) * w + first) * C : ((p * h + first) * w + x) * C;
  const long long step = AXIS == 0 ? C : (long long)w * C;
  for (int t = 0; t < count; ++t) {
    const int kt = __ldg(k + t);
    const unsigned char* s = src + base + t * step;
#pragma unroll
    for (int ch = 0; ch < C; ++ch) ss[ch] += (int)__ldg(s + ch) * kt;
  }
  unsigned char* d = dst + idx * C;
#pragma unroll
  for (int ch = 0; ch < C; ++ch) d[ch] = clip8(ss[ch]);
}

// ------------------------------------------------------------------------------------------------ Pillow nearest (+ label lookup)
__global__ void __launch_bounds__(256) pil_nearest_kernel(const unsigned char* __restrict__ src, int h, int w, const int* __restrict__ ys,
                                                          int oh, const int* __restrict__ xs, int ow, const unsigned char* __restrict__ lut,
                                                          unsigned char* __restrict__ dst, long long total) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int x = (int)(idx % ow);
  const long long py = idx / ow;
  const int y = (int)(py % oh);
  const long long p = py / oh;
  const unsigned char v = __ldg(src + (p * h + __ldg(ys + y)) * w + __ldg(xs + x));
  dst[idx] = lut ? __ldg(lut + v) : v;
}

// ------------------------------------------------------------------------------------------------ get_agnostic composite
// The grey shapes are drawn over the image, then the image is pasted back through four 0/255 masks (the two arm masks, head, lower
// body): a pixel ends grey exactly when a grey shape covers it and no paste restores it.
__global__ void __launch_bounds__(256) agnostic_composite_kernel(const unsigned char* __restrict__ image, const unsigned char* __restrict__ parse,
                                                                 const unsigned char* __restrict__ bits, unsigned char* __restrict__ dst,
                                                                 long long npix) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= npix) return;
  const int b = __ldg(bits + p), l = __ldg(parse + p);
  const bool restore = (!(b & 2) && l == 14) || (!(b & 4) && l == 15) || l == 4 || l == 13 || l == 9 || l == 12 || (l >= 16 && l <= 19);
  const bool grey = (b & 1) && !restore;
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) dst[p * 3 + ch] = grey ? (unsigned char)128 : __ldg(image + p * 3 + ch);
}

// ------------------------------------------------------------------------------------------------ batch assembly
// ToTensor (u8 -> fp32, divide by 255) then Normalize(0.5, 0.5) (subtract, divide), each correctly rounded.
__device__ __forceinline__ float normalise(unsigned char u) { return __fdiv_rn(__fsub_rn(__fdiv_rn((float)u, 255.f), 0.5f), 0.5f); }

__device__ __forceinline__ void rgb_out(const unsigned char* __restrict__ s, float* __restrict__ d, long long b, long long p, long long hw) {
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) d[(b * 3 + ch) * hw + p] = normalise(__ldg(s + (b * hw + p) * 3 + ch));
}

// thread = one pixel (b, p) of the batch, writing every requested output at that pixel: each plane's stores are coalesced.
__global__ void __launch_bounds__(256) viton_assemble_kernel(const hrv_viton_planes src, const hrv_viton_outputs dst, long long hw,
                                                             long long npix) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= npix) return;
  const long long b = i / hw, p = i - b * hw;
  if (dst.image) rgb_out(src.image, dst.image, b, p, hw);
  if (dst.pose) rgb_out(src.pose, dst.pose, b, p, hw);
  if (dst.densepose) rgb_out(src.densepose, dst.densepose, b, p, hw);
  if (dst.agnostic) rgb_out(src.agnostic, dst.agnostic, b, p, hw);
#pragma unroll
  for (int s = 0; s < 2; ++s) {
    if (dst.cloth[s]) rgb_out(src.cloth[s], dst.cloth[s], b, p, hw);
    if (dst.cloth_mask[s]) dst.cloth_mask[s][i] = __ldg(src.cloth_mask[s] + i) >= 128 ? 1.f : 0.f;
  }
  if (dst.pcm || dst.parse_cloth || dst.parse_onehot) {
    const int g = __ldg(src.parse + i);
    const float pcm = g == 3 ? 1.f : 0.f;
    if (dst.pcm) dst.pcm[i] = pcm;
    if (dst.parse_onehot) dst.parse_onehot[i] = (float)g;
    if (dst.parse_cloth) {
#pragma unroll
      for (int ch = 0; ch < 3; ++ch) {
        const float im = normalise(__ldg(src.image + i * 3 + ch));
        dst.parse_cloth[(b * 3 + ch) * hw + p] = __fadd_rn(__fmul_rn(im, pcm), __fsub_rn(1.f, pcm));
      }
    }
  }
}

}  // namespace hrv_data

using namespace hrv_data;

extern "C" int hrv_pil_resample_pass(const uint8_t* src, int32_t planes, int32_t h, int32_t w, int32_t c, int32_t axis, const int32_t* bounds,
                                     const int32_t* coeffs, int32_t ksize, int32_t out_len, uint8_t* dst, hrv_stream stream) {
  if (!src || !dst || !bounds || !coeffs || planes < 1 || h < 1 || w < 1 || (c != 1 && c != 3) || (axis != 0 && axis != 1) || ksize < 1 ||
      out_len < 1)
    return set_error(HRV_EINVAL, "pil_resample_pass: bad arguments");
  const int oh = axis == 1 ? out_len : h, ow = axis == 0 ? out_len : w;
  const long long total = (long long)planes * oh * ow;
  cudaStream_t st = (cudaStream_t)stream;
  const unsigned g = nblocks(total, 256);
  if (c == 3) {
    if (axis == 0) pil_resample_kernel<3, 0><<<g, 256, 0, st>>>(src, h, w, bounds, coeffs, ksize, oh, ow, dst, total);
    else pil_resample_kernel<3, 1><<<g, 256, 0, st>>>(src, h, w, bounds, coeffs, ksize, oh, ow, dst, total);
  } else {
    if (axis == 0) pil_resample_kernel<1, 0><<<g, 256, 0, st>>>(src, h, w, bounds, coeffs, ksize, oh, ow, dst, total);
    else pil_resample_kernel<1, 1><<<g, 256, 0, st>>>(src, h, w, bounds, coeffs, ksize, oh, ow, dst, total);
  }
  return launched("pil_resample_pass");
}

extern "C" int hrv_pil_nearest(const uint8_t* src, int32_t planes, int32_t h, int32_t w, const int32_t* ys, int32_t oh, const int32_t* xs,
                               int32_t ow, const uint8_t* lut, uint8_t* dst, hrv_stream stream) {
  if (!src || !dst || !ys || !xs || planes < 1 || h < 1 || w < 1 || oh < 1 || ow < 1) return set_error(HRV_EINVAL, "pil_nearest: bad arguments");
  const long long total = (long long)planes * oh * ow;
  pil_nearest_kernel<<<nblocks(total, 256), 256, 0, (cudaStream_t)stream>>>(src, h, w, ys, oh, xs, ow, lut, dst, total);
  return launched("pil_nearest");
}

extern "C" int hrv_agnostic_composite(const uint8_t* image, const uint8_t* parse, const uint8_t* bits, int32_t n, int32_t h, int32_t w,
                                      uint8_t* dst, hrv_stream stream) {
  if (!image || !parse || !bits || !dst || n < 1 || h < 1 || w < 1) return set_error(HRV_EINVAL, "agnostic_composite: bad arguments");
  const long long npix = (long long)n * h * w;
  agnostic_composite_kernel<<<nblocks(npix, 256), 256, 0, (cudaStream_t)stream>>>(image, parse, bits, dst, npix);
  return launched("agnostic_composite");
}

extern "C" int hrv_viton_assemble(const hrv_viton_planes* src, const hrv_viton_outputs* dst, int32_t n, int32_t h, int32_t w, hrv_stream stream) {
  if (!src || !dst || n < 1 || h < 1 || w < 1) return set_error(HRV_EINVAL, "viton_assemble: bad arguments");
  bool ok = (!dst->image || src->image) && (!dst->pose || src->pose) && (!dst->densepose || src->densepose) &&
            (!dst->agnostic || src->agnostic) && (!(dst->pcm || dst->parse_cloth || dst->parse_onehot) || src->parse) &&
            (!dst->parse_cloth || src->image);
  for (int s = 0; s < 2; ++s) ok = ok && (!dst->cloth[s] || src->cloth[s]) && (!dst->cloth_mask[s] || src->cloth_mask[s]);
  if (!ok) return set_error(HRV_EINVAL, "viton_assemble: an output without its source plane");
  const long long hw = (long long)h * w, npix = hw * n;
  viton_assemble_kernel<<<nblocks(npix, 256), 256, 0, (cudaStream_t)stream>>>(*src, *dst, hw, npix);
  return launched("viton_assemble");
}
