// hrv_bilinear.cuh — torch's upsample_bilinear2d (align_corners=False, explicit output size, accscalar_t = float) as device functions:
// the source index, the clamped taps, the lambdas and the blend are torch's own expressions in the same order, with the fma
// contraction its kernel is compiled with spelled out, so every caller is bit-identical to F.interpolate(mode='bilinear') on CUDA.
#pragma once

namespace hrv_bilinear {

// area_pixel_compute_source_index: max(scale * (d + 0.5) - 0.5, 0), contracted as in torch's kernel.  scale = (float)in / out.
__device__ __forceinline__ float bilinear_src(float scale, int d) {
  const float s = __fmaf_rn(scale, __fadd_rn((float)d, 0.5f), -0.5f);
  return s < 0.f ? 0.f : s;
}

// The two taps of output index d along an axis of n input samples: i1 = i0 + 1, or i0 at the last sample; lambdas l0 + l1 = 1.
struct Taps {
  int i0, i1;
  float l0, l1;
};
__device__ __forceinline__ Taps bilinear_taps(float scale, int d, int n) {
  const float r = bilinear_src(scale, d);
  Taps t;
  t.i0 = (int)r;
  t.i1 = t.i0 + ((t.i0 < n - 1) ? 1 : 0);
  t.l1 = r - t.i0;
  t.l0 = 1.f - t.l1;
  return t;
}

// h0lambda * (w0lambda * v00 + w1lambda * v01) + h1lambda * (w0lambda * v10 + w1lambda * v11); left to the compiler, the contraction
// could differ between callers.
__device__ __forceinline__ float bilinear_blend(const Taps& ty, const Taps& tx, float v00, float v01, float v10, float v11) {
  const float top = __fmaf_rn(tx.l0, v00, __fmul_rn(tx.l1, v01));
  const float bottom = __fmaf_rn(tx.l0, v10, __fmul_rn(tx.l1, v11));
  return __fmaf_rn(ty.l0, top, __fmul_rn(ty.l1, bottom));
}

}  // namespace hrv_bilinear
