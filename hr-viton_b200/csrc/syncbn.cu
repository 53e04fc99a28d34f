// syncbn.cu — the per-layer exchange of synchronised train-mode BatchNorm (sync_batchnorm.SynchronizedBatchNorm2d).
//
// Every rank reduces its own shard with the existing statistics kernels (forward: hrv_instnorm_stats leaves per-image
// {sum x, sum x^2}; backward: hrv_norm_bwd_reduce leaves per-image {sum dxn, sum dxn*xn}).  Per layer and direction:
//   combine   : the local per-image fp64 sums -> one wire buffer [C][2] + element count (images added in index order)
//   all-reduce: sum of the wire buffers over the ranks (the caller's collective)
//   finalize  : forward  -> mean / rstd [N][C8] for hrv_norm_apply_affine and the running-statistics update
//               backward -> m1 / m2 [N][C] for hrv_norm_bwd_apply
// The count travels with the sums, so ranks holding shards of different sizes still get the global statistics.  One thread per
// channel, plain loads and stores: no atomics, the result depends on the inputs only.
#include "hrv_host.h"

namespace hrv {

__global__ void syncbn_combine_kernel(const double* __restrict__ sums, int n, int C, int stride, double count, double* __restrict__ wire) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < C) {
    double s0 = 0.0, s1 = 0.0;
    for (int i = 0; i < n; ++i) {
      const double* p = sums + ((long long)i * C + c) * stride;
      s0 += p[0];
      s1 += p[1];
    }
    wire[2 * c] = s0;
    wire[2 * c + 1] = s1;
  }
  if (c == 0) wire[2 * C] = count;
}

// The arithmetic of the per-rank path (hrviton_b200.autograd_tocg.BatchNormActFn) on the global sums: mean and biased variance in
// fp64, rounded to fp32, rstd = rsqrtf(var + eps) in fp32 as torch.rsqrt computes it; running statistics updated in fp32 with
// separately rounded products, as the torch ops mul_(1 - m).add_(x * m) do.  So N ranks compute the bits one process computes on
// the concatenated batch, unless the differently associated fp64 sums round to a different fp32 value.
__global__ void syncbn_fwd_finalize_kernel(const double* __restrict__ wire, int n, int C, int c_run, float eps, double momentum,
                                           float* __restrict__ mean_nc, float* __restrict__ rstd_nc, float* __restrict__ running_mean,
                                           float* __restrict__ running_var) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const double cnt = wire[2 * C];
  const double mean = wire[2 * c] / cnt;
  double var = wire[2 * c + 1] / cnt - mean * mean;
  if (var < 0.0) var = 0.0;
  const float mean32 = (float)mean, var32 = (float)var;
  const float rstd32 = rsqrtf(__fadd_rn(var32, eps));
  for (int i = 0; i < n; ++i) {
    mean_nc[(long long)i * C + c] = mean32;
    rstd_nc[(long long)i * C + c] = rstd32;
  }
  if (running_mean && c < c_run) {
    const float keep = (float)(1.0 - momentum), m = (float)momentum;
    const float unbias = (float)(cnt / (cnt - 1.0 > 1.0 ? cnt - 1.0 : 1.0));
    running_mean[c] = __fadd_rn(__fmul_rn(running_mean[c], keep), __fmul_rn(mean32, m));
    running_var[c] = __fadd_rn(__fmul_rn(running_var[c], keep), __fmul_rn(__fmul_rn(var32, unbias), m));
  }
}

__global__ void syncbn_bwd_finalize_kernel(const double* __restrict__ wire, int n, int C, float* __restrict__ m1, float* __restrict__ m2) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const double cnt = wire[2 * C];
  const float a = (float)(wire[2 * c] / cnt), b = (float)(wire[2 * c + 1] / cnt);
  for (int i = 0; i < n; ++i) {
    m1[(long long)i * C + c] = a;
    m2[(long long)i * C + c] = b;
  }
}

static int syncbn_launched(const char* what) {
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? HRV_OK : set_error(HRV_ECUDA, "%s launch: %s", what, cudaGetErrorString(e));
}
static unsigned syncbn_blocks(int C) { return (unsigned)((C + 127) / 128); }

}  // namespace hrv

using namespace hrv;

extern "C" int hrv_syncbn_combine(const double* sums, int32_t n, int32_t c, int32_t stride, double count, double* wire, hrv_stream stream) {
  if (!sums || !wire) return set_error(HRV_EINVAL, "syncbn_combine: null pointer");
  if (n < 1 || c < 1 || stride < 2) return set_error(HRV_EINVAL, "syncbn_combine: bad extent (n %d, c %d, stride %d)", n, c, stride);
  if (!(count > 0.0)) return set_error(HRV_EINVAL, "syncbn_combine: element count must be positive");
  syncbn_combine_kernel<<<syncbn_blocks(c), 128, 0, (cudaStream_t)stream>>>(sums, n, c, stride, count, wire);
  return syncbn_launched("syncbn_combine");
}

extern "C" int hrv_syncbn_fwd_finalize(const double* wire, int32_t n, int32_t c, int32_t c_run, float eps, double momentum, float* mean,
                                       float* rstd, float* running_mean, float* running_var, hrv_stream stream) {
  if (!wire || !mean || !rstd) return set_error(HRV_EINVAL, "syncbn_fwd_finalize: null pointer");
  if (n < 1 || c < 1 || c_run < 0 || c_run > c) return set_error(HRV_EINVAL, "syncbn_fwd_finalize: bad extent (n %d, c %d, c_run %d)", n, c, c_run);
  if (!running_mean != !running_var) return set_error(HRV_EINVAL, "syncbn_fwd_finalize: running_mean and running_var go together");
  syncbn_fwd_finalize_kernel<<<syncbn_blocks(c), 128, 0, (cudaStream_t)stream>>>(wire, n, c, c_run, eps, momentum, mean, rstd, running_mean,
                                                                                  running_var);
  return syncbn_launched("syncbn_fwd_finalize");
}

extern "C" int hrv_syncbn_bwd_finalize(const double* wire, int32_t n, int32_t c, float* m1, float* m2, hrv_stream stream) {
  if (!wire || !m1 || !m2) return set_error(HRV_EINVAL, "syncbn_bwd_finalize: null pointer");
  if (n < 1 || c < 1) return set_error(HRV_EINVAL, "syncbn_bwd_finalize: bad extent (n %d, c %d)", n, c);
  syncbn_bwd_finalize_kernel<<<syncbn_blocks(c), 128, 0, (cudaStream_t)stream>>>(wire, n, c, m1, m2);
  return syncbn_launched("syncbn_bwd_finalize");
}
