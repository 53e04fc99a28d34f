// capi.cu — error handling, device introspection and the TMA descriptor encoder of libhrviton_sm100.so.
#include <stdarg.h>
#include <stdio.h>

#include "hrv_host.h"

namespace hrv_host {

static thread_local char g_err[512] = "";

int set_error(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

int sm_count() {
  static int cached = 0;
  if (cached) return cached;
  int dev = 0, n = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 132;
  if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) return 132;
  cached = n;
  return n;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

int encode_tensor_map(CUtensorMap* map, int rank, void* base, const cuuint64_t* dims, const cuuint64_t* strides_bytes,
                      const cuuint32_t* box, const cuuint32_t* elem_strides, CUtensorMapSwizzle swizzle, CUtensorMapDataType type) {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* sym = nullptr;
    cudaDriverEntryPointQueryResult q;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &sym, cudaEnableDefault, &q);
    if (e != cudaSuccess || q != cudaDriverEntryPointSuccess || !sym)
      return set_error(HRV_ECUDA, "cuTensorMapEncodeTiled entry point unavailable (%s)", cudaGetErrorString(e));
    fn = (EncodeTiledFn)sym;
  }
  CUresult r = fn(map, type, (cuuint32_t)rank, base, dims, strides_bytes, box, elem_strides,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return set_error(HRV_ECUDA, "cuTensorMapEncodeTiled failed: CUresult %d (rank %d dims %llu,%llu box %u,%u)", (int)r, rank,
                     (unsigned long long)dims[0], (unsigned long long)dims[1], box[0], box[1]);
  return HRV_OK;
}

int encode_nhwc_map(CUtensorMap* map, const hrv_tensor& t, int box_c, int box_w, int box_h, int box_n, CUtensorMapSwizzle swizzle) {
  const bool f32 = t.dtype == HRV_F32;
  const cuuint64_t elem = f32 ? 4 : 2;
  const cuuint64_t dims[4] = {(cuuint64_t)t.c, (cuuint64_t)t.w, (cuuint64_t)t.h, (cuuint64_t)t.n};
  const cuuint64_t strides[3] = {(cuuint64_t)t.pitch * elem, (cuuint64_t)t.w * t.pitch * elem, (cuuint64_t)t.h * t.w * t.pitch * elem};
  const cuuint32_t box[4] = {(cuuint32_t)box_c, (cuuint32_t)box_w, (cuuint32_t)box_h, (cuuint32_t)box_n};
  const cuuint32_t es[4] = {1, 1, 1, 1};
  return encode_tensor_map(map, 4, t.ptr, dims, strides, box, es, swizzle,
                           f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16);
}

}  // namespace hrv_host

extern "C" const char* hrv_last_error(void) { return hrv_host::g_err; }
extern "C" int hrv_version(void) { return 200; }
extern "C" int hrv_device_sm_count(void) { return hrv_host::sm_count(); }
