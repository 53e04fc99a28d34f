// hrv_host.h — host-side helpers shared by the translation units of libhrviton_sm100.so.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#ifdef HRV_F16
#include "hrv_f16_rename.h"  // the fp16-storage flavour of every entry point: hrv_xxx -> hrv_xxx_f16 (same signatures)
#endif
#include "../../include/hrviton_sm100.h"

// Helpers defined once (capi.cu) and shared by both storage flavours of the kernel translation units.  The kernel TUs are
// compiled twice: as namespace hrv (bf16 storage) and, with -DHRV_F16 -Dhrv=hrv_f16, as namespace hrv_f16 (IEEE fp16 storage).
namespace hrv_host {
// Records a thread-local error string (printf-style) and returns `code`.
int set_error(int code, const char* fmt, ...);
int sm_count();
// cuTensorMapEncodeTiled through cudaGetDriverEntryPoint (no link-time dependency on libcuda).
int encode_tensor_map(CUtensorMap* map, int rank, void* base, const cuuint64_t* dims, const cuuint64_t* strides_bytes,
                      const cuuint32_t* box, const cuuint32_t* elem_strides, CUtensorMapSwizzle swizzle,
                      CUtensorMapDataType type = CU_TENSOR_MAP_DATA_TYPE_BFLOAT16);
// 4-D SWIZZLE_128B map {c, w, h, n} of the NHWC tensor `t` (bf16 / fp16 or fp32 by t.dtype) with box {box_c, box_w, box_h, box_n}.
int encode_nhwc_map(CUtensorMap* map, const hrv_tensor& t, int box_c, int box_w, int box_h, int box_n);
// hrv_conv2d_fwd on fp32 storage (conv_f32.cu, compiled once): both flavours of hrv_conv2d_fwd hand an fp32 input to it.
int conv2d_fwd_tf32x3(const hrv_conv_params* p, hrv_stream stream);

// Pixel-tile geometry shared by the convolution kernels.
inline int log2i(int v) {
  int l = 0;
  while ((1 << l) < v) ++l;
  return l;
}
// Pick the power-of-two tile extent p <= cap for a dimension of size `dim`: least padding, ties -> larger.
inline int pick_pow2(int dim, int cap) {
  int best = 1;
  double best_waste = 1e30;
  for (int p = 1; p <= cap; p <<= 1) {
    const int tiles = (dim + p - 1) / p;
    const double waste = (double)tiles * p / dim;
    if (waste <= best_waste + 0.031) {
      if (waste < best_waste) best_waste = waste;
      best = p;
    }
  }
  return best;
}

// Launches `kKernel` with `smem` bytes of dynamic shared memory; the first call raises the kernel's limit to `smem_max`.
template <auto kKernel, typename Args>
int launch_dyn_smem(const char* name, int grid, int threads, size_t smem, uint32_t smem_max, cudaStream_t st, const Args& args) {
  static bool raised = false;
  if (!raised) {
    cudaError_t e = cudaFuncSetAttribute(kKernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_max);
    if (e != cudaSuccess) return set_error(HRV_ECUDA, "cudaFuncSetAttribute(%s): %s", name, cudaGetErrorString(e));
    raised = true;
  }
  kKernel<<<grid, threads, smem, st>>>(args);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(HRV_ECUDA, "%s launch: %s", name, cudaGetErrorString(e));
  return HRV_OK;
}
}  // namespace hrv_host
namespace hrv {
using namespace hrv_host;
// out[o * out_stride + j] = sum over r < rows of slab[(o * rows + r) * cols + j] (fp64), in a fixed order that does not depend on
// timing: the finishing pass of the per-block slabs that replace cross-block atomics (csrc/norm_bwd.cu).
int slab_sum(const double* slab, int outer, int rows, int cols, double* out, int out_stride, cudaStream_t st, const char* what);
}
