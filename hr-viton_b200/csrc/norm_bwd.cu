// norm_bwd.cu — fused backward of the SPADE modulation + InstanceNorm (and of plain InstanceNorm+activation).
//
// Forward (network_generator.py:101-122,170-171):  xn = (xs + noise*ns - mean) * rstd ;  v = xn*(1+gamma) + beta ; h = act(v)
// Backward, two HBM-bound passes (NHWC bf16, 8 channels per thread, fp32 math, fp64 per-block sums written to per-block slabs and
// added in a fixed order by a finishing kernel, so every sum is reproducible run to run):
//   pass 1 (reduce):  dv = dh*act'(h);  dgamma = dv*xn;  dbeta = dv;  dxn = dv*(1+gamma)
//                     writes d(gamma|beta) interleaved (the dY of the gamma/beta GEMM) and dxn; accumulates per (n,c):
//                     S1 = sum dxn, S2 = sum dxn*xn, Sg = sum dgamma, Sb = sum dbeta
//   pass 2 (apply):   dxs = rstd * (dxn - S1/HW - xn * S2/HW)   (InstanceNorm backward, biased variance)
//                     dx0 = sum over the 2x2 children when x0 was nearest-up-sampled, dx1 = dxs[:, C0:];
//                     accumulates d(noise_scale)[c] = sum dxs*noise
// The virtual tensor xs = cat(up2^shift(x0), x1) is never materialised, exactly as in the forward kernels.
#include "hrv_host.h"
#include "hrv_ptx.cuh"

namespace hrv {

struct NView {
  const void* ptr;
  int n, h, w, c, pitch;
};
static NView mkview(const hrv_tensor* t) {
  NView v;
  if (t && t->ptr) { v.ptr = t->ptr; v.n = t->n; v.h = t->h; v.w = t->w; v.c = t->c; v.pitch = t->pitch; }
  else { v.ptr = nullptr; v.n = v.h = v.w = v.c = v.pitch = 0; }
  return v;
}

__device__ __forceinline__ void un8(const uint4& u, float (&f)[8]) {
  f[0] = bf16_lo(u.x); f[1] = bf16_hi(u.x); f[2] = bf16_lo(u.y); f[3] = bf16_hi(u.y);
  f[4] = bf16_lo(u.z); f[5] = bf16_hi(u.z); f[6] = bf16_lo(u.w); f[7] = bf16_hi(u.w);
}
__device__ __forceinline__ uint4 pk8(const float (&f)[8]) {
  uint4 o;
  o.x = pack_bf16(f[0], f[1]); o.y = pack_bf16(f[2], f[3]); o.z = pack_bf16(f[4], f[5]); o.w = pack_bf16(f[6], f[7]);
  return o;
}
__device__ __forceinline__ uint4 ld16(const void* p) { return __ldg(reinterpret_cast<const uint4*>(p)); }
__device__ __forceinline__ float act_grad(float dy, float y, int act) {
  switch (act) {
    case 1: return y > 0.f ? dy : 0.f;
    case 2: return y > 0.f ? dy : 0.2f * dy;
    case 3: return dy * (1.f - y * y);
    default: return dy;
  }
}

struct BwdArgs {
  NView dh, h, gamma, x0, x1, dgb, dxn;
  int x0_shift, H, W, G, PL, chunk, act;
  const float* noise;
  const float* ns;
  const float* mean;
  const float* rstd;
  const float* chan_scale;  // optional per-channel affine weight (BatchNorm): dxn = dv * chan_scale[c]
  double* slab;  // [N][gridDim.x][C][4]
};

// grid (chunks, N); thread = (pixel lane, channel group)
__global__ void __launch_bounds__(256) spade_bwd_reduce_kernel(BwdArgs a) {
  extern __shared__ float shf[];  // [PL][C][4]
  const int n = blockIdx.y;
  const int C = a.G * 8;
  const int g = threadIdx.x % a.G;
  const int pl = threadIdx.x / a.G;
  if (pl < a.PL) {
    const int c0 = g * 8;
    const long long HW = (long long)a.H * a.W;
    const long long p_begin = (long long)blockIdx.x * a.chunk;
    long long p_end = p_begin + a.chunk;
    if (p_end > HW) p_end = HW;
    float s1[8], s2[8], sg[8], sb[8], nsv[8], mu[8], rs[8], cs[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      s1[i] = s2[i] = sg[i] = sb[i] = 0.f;
      cs[i] = a.chan_scale ? __ldg(a.chan_scale + c0 + i) : 1.f;
      nsv[i] = a.ns ? __ldg(a.ns + c0 + i) : 0.f;
      mu[i] = __ldg(a.mean + (long long)n * C + c0 + i);
      rs[i] = __ldg(a.rstd + (long long)n * C + c0 + i);
    }
    const bool from0 = c0 < a.x0.c;
    const int W0 = a.W >> a.x0_shift, H0 = a.H >> a.x0_shift;
    for (long long p = p_begin + pl; p < p_end; p += a.PL) {
      const long long pix = (long long)n * HW + p;
      const int y = (int)(p / a.W), x = (int)(p - (long long)y * a.W);
      const __nv_bfloat16* xs = from0
          ? reinterpret_cast<const __nv_bfloat16*>(a.x0.ptr) + (((long long)n * H0 + (y >> a.x0_shift)) * W0 + (x >> a.x0_shift)) * a.x0.pitch + c0
          : reinterpret_cast<const __nv_bfloat16*>(a.x1.ptr) + pix * a.x1.pitch + (c0 - a.x0.c);
      float fx[8], fdh[8], fh[8], fg[8];
      un8(ld16(xs), fx);
      un8(ld16(reinterpret_cast<const __nv_bfloat16*>(a.dh.ptr) + pix * a.dh.pitch + c0), fdh);
      if (a.act != 0) un8(ld16(reinterpret_cast<const __nv_bfloat16*>(a.h.ptr) + pix * a.h.pitch + c0), fh);
      if (a.gamma.ptr) un8(ld16(reinterpret_cast<const __nv_bfloat16*>(a.gamma.ptr) + pix * a.gamma.pitch + c0), fg);
      const float nz = a.noise ? __ldg(a.noise + pix) : 0.f;
      float dgm[8], dbt[8], dxn[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float xn = (fmaf(nz, nsv[i], fx[i]) - mu[i]) * rs[i];
        const float dv = a.act != 0 ? act_grad(fdh[i], fh[i], a.act) : fdh[i];
        dgm[i] = dv * xn;
        dbt[i] = dv;
        dxn[i] = a.gamma.ptr ? dv * (1.f + fg[i]) : dv * cs[i];
        s1[i] += dxn[i];
        s2[i] = fmaf(dxn[i], xn, s2[i]);
        sg[i] += dgm[i];
        sb[i] += dbt[i];
      }
      *reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(const_cast<void*>(a.dxn.ptr)) + pix * a.dxn.pitch + c0) = pk8(dxn);
      if (a.dgb.ptr) {
        float lo[8] = {dgm[0], dbt[0], dgm[1], dbt[1], dgm[2], dbt[2], dgm[3], dbt[3]};
        float hi[8] = {dgm[4], dbt[4], dgm[5], dbt[5], dgm[6], dbt[6], dgm[7], dbt[7]};
        uint4* o = reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(const_cast<void*>(a.dgb.ptr)) + pix * a.dgb.pitch + 2 * c0);
        o[0] = pk8(lo);
        o[1] = pk8(hi);
      }
    }
    float* dst = shf + ((long long)pl * C + c0) * 4;
#pragma unroll
    for (int i = 0; i < 8; ++i) { dst[4 * i] = s1[i]; dst[4 * i + 1] = s2[i]; dst[4 * i + 2] = sg[i]; dst[4 * i + 3] = sb[i]; }
  }
  __syncthreads();
  for (int j = threadIdx.x; j < C * 4; j += blockDim.x) {
    double t = 0.0;
    for (int l = 0; l < a.PL; ++l) t += (double)shf[(long long)l * C * 4 + j];
    a.slab[((long long)n * gridDim.x + blockIdx.x) * C * 4 + j] = t;
  }
}

struct ApplyArgs {
  NView dxn, src, dx;      // src = x0 or x1 (the tensor whose gradient this launch produces), dx at src resolution
  int shift, H, W, G, PL, chunk, c_off, C;  // H,W = statistics (hi-res) extent; c_off = channel offset of src inside xs
  const float* noise;
  const float* ns;
  const float* mean;
  const float* rstd;
  const float* m1;   // [N][C] = S1/HW
  const float* m2;   // [N][C] = S2/HW
  double* dns_slab;  // [N][gridDim.x][Gs*8] per-block sums of dxs*noise (may be null)
};

// grid (chunks over src pixels, N); thread = (pixel lane, channel group of src)
template <int KIDS>  // 2: src is the half-resolution tensor behind a virtual nearest x2 (each src pixel gathers its 2x2 children); 1: same resolution
__global__ void __launch_bounds__(256) spade_bwd_apply_kernel(ApplyArgs a) {
  extern __shared__ float shf[];  // [PL][Gs*8]
  const int n = blockIdx.y;
  const int Cs = a.G * 8;
  const int g = threadIdx.x % a.G;
  const int pl = threadIdx.x / a.G;
  const int Hs = a.H >> a.shift, Ws = a.W >> a.shift;
  if (pl < a.PL) {
    const int cs = g * 8, c0 = a.c_off + cs;
    const long long HWs = (long long)Hs * Ws;
    const long long p_begin = (long long)blockIdx.x * a.chunk;
    long long p_end = p_begin + a.chunk;
    if (p_end > HWs) p_end = HWs;
    float nsv[8], mu[8], rs[8], k1[8], k2[8], dn[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      nsv[i] = a.ns ? __ldg(a.ns + c0 + i) : 0.f;
      mu[i] = __ldg(a.mean + (long long)n * a.C + c0 + i);
      rs[i] = __ldg(a.rstd + (long long)n * a.C + c0 + i);
      k1[i] = __ldg(a.m1 + (long long)n * a.C + c0 + i);
      k2[i] = __ldg(a.m2 + (long long)n * a.C + c0 + i);
      dn[i] = 0.f;
    }
    constexpr int NK = KIDS * KIDS;
    for (long long p = p_begin + pl; p < p_end; p += a.PL) {
      const int ys = (int)(p / Ws), xs_ = (int)(p - (long long)ys * Ws);
      // issue every load of this pixel (src + its children + their noise) before the arithmetic
      const uint4 vx = ld16(reinterpret_cast<const __nv_bfloat16*>(a.src.ptr) + ((long long)n * HWs + p) * a.src.pitch + cs);
      uint4 vd[NK];
      float nz[NK];
#pragma unroll
      for (int k = 0; k < NK; ++k) {
        const long long pix = ((long long)n * a.H + (ys * KIDS + k / KIDS)) * a.W + (xs_ * KIDS + k % KIDS);
        vd[k] = ld16(reinterpret_cast<const __nv_bfloat16*>(a.dxn.ptr) + pix * a.dxn.pitch + c0);
        nz[k] = a.noise ? __ldg(a.noise + pix) : 0.f;
      }
      float fx[8], o[8];
      un8(vx, fx);
#pragma unroll
      for (int i = 0; i < 8; ++i) o[i] = 0.f;
#pragma unroll
      for (int k = 0; k < NK; ++k) {
        float fd[8];
        un8(vd[k], fd);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float xn = (fmaf(nz[k], nsv[i], fx[i]) - mu[i]) * rs[i];
          const float dxs = rs[i] * (fd[i] - k1[i] - xn * k2[i]);
          o[i] += dxs;
          dn[i] = fmaf(dxs, nz[k], dn[i]);
        }
      }
      *reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(const_cast<void*>(a.dx.ptr)) + ((long long)n * HWs + p) * a.dx.pitch + cs) = pk8(o);
    }
    float* dst = shf + (long long)pl * Cs + cs;
#pragma unroll
    for (int i = 0; i < 8; ++i) dst[i] = dn[i];
  }
  __syncthreads();
  if (a.dns_slab) {
    for (int j = threadIdx.x; j < Cs; j += blockDim.x) {
      double t = 0.0;
      for (int l = 0; l < a.PL; ++l) t += (double)shf[(long long)l * Cs + j];
      a.dns_slab[((long long)n * gridDim.x + blockIdx.x) * Cs + j] = t;
    }
  }
}

// Finishing pass of the slabs: out[o * out_stride + j] = sum over slab rows r = 0..rows-1 of slab[(o * rows + r) * cols + j].
// block = 32 columns x 32 row groups, grid = (column chunks, o): thread (j, g) adds rows g, g+32, g+64, ... in that order (coalesced
// across j), then a fixed shared-memory tree combines the 32 groups.  The order is the same on every launch, and no thread walks
// the up to ~1000 slabs of a small-image reduction serially.
__global__ void __launch_bounds__(1024) slab_sum_kernel(const double* __restrict__ slab, int rows, int cols, double* __restrict__ out, int out_stride) {
  __shared__ double part[32][33];
  const int j = blockIdx.x * 32 + threadIdx.x, g = threadIdx.y, o = blockIdx.y;
  double t = 0.0;
  if (j < cols) {
    const double* p = slab + (long long)o * rows * cols + j;
#pragma unroll 4
    for (int r = g; r < rows; r += 32) t += p[(long long)r * cols];
  }
  part[g][threadIdx.x] = t;
  __syncthreads();
  for (int s = 16; s > 0; s >>= 1) {
    if (g < s) part[g][threadIdx.x] += part[g + s][threadIdx.x];
    __syncthreads();
  }
  if (g == 0 && j < cols) out[(long long)o * out_stride + j] = part[0][threadIdx.x];
}
int slab_sum(const double* slab, int outer, int rows, int cols, double* out, int out_stride, cudaStream_t st, const char* what) {
  slab_sum_kernel<<<dim3((unsigned)((cols + 31) / 32), (unsigned)outer), dim3(32, 32), 0, st>>>(slab, rows, cols, out, out_stride);
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? HRV_OK : set_error(HRV_ECUDA, "%s launch: %s", what, cudaGetErrorString(e));
}

static int chk(const hrv_tensor* t, const char* what, bool optional = false) {
  if (!t || !t->ptr) return optional ? 0 : set_error(HRV_EINVAL, "%s: null tensor", what);
  if (t->dtype != HRV_BF16) return set_error(HRV_EINVAL, "%s: must be bf16", what);
  if (((uintptr_t)t->ptr & 15) || (t->pitch % 8)) return set_error(HRV_EINVAL, "%s: needs 16-byte alignment and pitch %% 8 == 0", what);
  return 0;
}
static void plan(long long HW, int N, int G, int& PL, int& chunk, unsigned& gx) {
  PL = 256 / G;
  long long target = (long long)sm_count() * 8 / (N > 0 ? N : 1);
  if (target < 1) target = 1;
  long long ch = (HW + target - 1) / target;
  const long long min_chunk = (long long)PL * 8;
  if (ch < min_chunk) ch = min_chunk;
  chunk = (int)ch;
  gx = (unsigned)((HW + ch - 1) / ch);
}

}  // namespace hrv

using namespace hrv;

extern "C" size_t hrv_norm_bwd_reduce_workspace_bytes(const hrv_tensor* x0, const hrv_tensor* x1, int32_t H, int32_t W) {
  if (!x0) return 0;
  const int C = x0->c + ((x1 && x1->ptr) ? x1->c : 0), G = (C + 7) / 8;
  int PL, chunk;
  unsigned gx;
  plan((long long)H * W, x0->n, G > 0 ? G : 1, PL, chunk, gx);
  return (size_t)x0->n * gx * G * 8 * 4 * sizeof(double);
}

extern "C" int hrv_norm_bwd_reduce(const hrv_tensor* dh, const hrv_tensor* h, const hrv_tensor* gamma, const hrv_tensor* x0,
                                   int32_t x0_shift, const hrv_tensor* x1, int32_t H, int32_t W, const float* noise,
                                   const float* noise_scale, const float* mean, const float* rstd, const float* chan_scale, int32_t act,
                                   const hrv_tensor* dgb, const hrv_tensor* dxn, double* sums, void* workspace, size_t workspace_bytes,
                                   hrv_stream stream) {
  int rc;
  if ((rc = chk(dh, "norm_bwd dh")) || (rc = chk(x0, "norm_bwd x0")) || (rc = chk(dxn, "norm_bwd dxn")) || (rc = chk(h, "norm_bwd h", act == 0)) ||
      (rc = chk(gamma, "norm_bwd gamma", true)) || (rc = chk(x1, "norm_bwd x1", true)) || (rc = chk(dgb, "norm_bwd dgb", true)))
    return rc;
  const bool has1 = x1 && x1->ptr;
  const int C = x0->c + (has1 ? x1->c : 0);
  if ((x0->c % 8) || (C % 8) || C / 8 > 256) return set_error(HRV_EINVAL, "norm_bwd: channels must be multiples of 8 (<= 2048)");
  if ((x0->h << x0_shift) != H || (x0->w << x0_shift) != W) return set_error(HRV_EINVAL, "norm_bwd: x0 extent mismatch");
  if (!mean || !rstd || !sums) return set_error(HRV_EINVAL, "norm_bwd: mean/rstd/sums required");
  const int N = x0->n;
  BwdArgs a;
  a.dh = mkview(dh); a.h = mkview(h); a.gamma = mkview(gamma); a.x0 = mkview(x0); a.x1 = mkview(has1 ? x1 : nullptr); a.dgb = mkview(dgb); a.dxn = mkview(dxn);
  a.x0_shift = x0_shift; a.H = H; a.W = W; a.G = C / 8; a.act = act;
  a.noise = noise; a.ns = noise_scale; a.mean = mean; a.rstd = rstd; a.chan_scale = chan_scale; a.slab = (double*)workspace;
  unsigned gx;
  plan((long long)H * W, N, a.G, a.PL, a.chunk, gx);
  const size_t need = hrv_norm_bwd_reduce_workspace_bytes(x0, x1, H, W);
  if (!workspace || workspace_bytes < need) return set_error(HRV_EINVAL, "norm_bwd_reduce: workspace too small (%zu < %zu)", workspace_bytes, need);
  cudaStream_t st = (cudaStream_t)stream;
  spade_bwd_reduce_kernel<<<dim3(gx, N), 256, (size_t)a.PL * C * 4 * sizeof(float), st>>>(a);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(HRV_ECUDA, "norm_bwd_reduce launch: %s", cudaGetErrorString(e));
  return slab_sum(a.slab, N, (int)gx, C * 4, sums, C * 4, st, "norm_bwd_reduce sum");
}

extern "C" size_t hrv_norm_bwd_apply_workspace_bytes(const hrv_tensor* src) {
  if (!src) return 0;
  const int G = (src->c + 7) / 8;
  int PL, chunk;
  unsigned gx;
  plan((long long)src->h * src->w, src->n, G > 0 ? G : 1, PL, chunk, gx);
  return (size_t)src->n * gx * G * 8 * sizeof(double);
}

extern "C" int hrv_norm_bwd_apply(const hrv_tensor* dxn, const hrv_tensor* src, int32_t shift, int32_t c_off, int32_t C, int32_t H,
                                  int32_t W, const float* noise, const float* noise_scale, const float* mean, const float* rstd,
                                  const float* m1, const float* m2, const hrv_tensor* dx, double* dns, void* workspace,
                                  size_t workspace_bytes, hrv_stream stream) {
  int rc;
  if ((rc = chk(dxn, "norm_bwd_apply dxn")) || (rc = chk(src, "norm_bwd_apply src")) || (rc = chk(dx, "norm_bwd_apply dx"))) return rc;
  if ((src->c % 8) || (c_off % 8) || c_off + src->c > C) return set_error(HRV_EINVAL, "norm_bwd_apply: bad channel slice");
  if ((src->h << shift) != H || (src->w << shift) != W || dx->h != src->h || dx->w != src->w)
    return set_error(HRV_EINVAL, "norm_bwd_apply: extent mismatch");
  ApplyArgs a;
  a.dxn = mkview(dxn); a.src = mkview(src); a.dx = mkview(dx);
  a.shift = shift; a.H = H; a.W = W; a.G = src->c / 8; a.c_off = c_off; a.C = C;
  a.noise = noise; a.ns = noise_scale; a.mean = mean; a.rstd = rstd; a.m1 = m1; a.m2 = m2; a.dns_slab = dns ? (double*)workspace : nullptr;
  unsigned gx;
  plan((long long)src->h * src->w, src->n, a.G, a.PL, a.chunk, gx);
  if (dns) {
    const size_t need = hrv_norm_bwd_apply_workspace_bytes(src);
    if (!workspace || workspace_bytes < need) return set_error(HRV_EINVAL, "norm_bwd_apply: workspace too small (%zu < %zu)", workspace_bytes, need);
  }
  cudaStream_t st = (cudaStream_t)stream;
  if (a.shift)
    spade_bwd_apply_kernel<2><<<dim3(gx, src->n), 256, (size_t)a.PL * a.G * 8 * sizeof(float), st>>>(a);
  else
    spade_bwd_apply_kernel<1><<<dim3(gx, src->n), 256, (size_t)a.PL * a.G * 8 * sizeof(float), st>>>(a);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(HRV_ECUDA, "norm_bwd_apply launch: %s", cudaGetErrorString(e));
  // one slab row per (n, block): every image's blocks and all images meet in one fixed-order sum
  return dns ? slab_sum(a.dns_slab, 1, src->n * (int)gx, a.G * 8, dns + c_off, 0, st, "norm_bwd_apply sum") : HRV_OK;
}

// ------------------------------------------------------------------------------------------------ activation backward + bias gradient
namespace hrv {
// dv = dy * act'(y) (bf16, NHWC) and bias_grad[c] = sum over all pixels of dv — one pass instead of where() + float() + sum().
// kSlab = false: the block sums meet in bsum through fp64 atomics (hrv_act_bwd_bias, order-dependent); kSlab = true: every block
// writes its sums to row blockIdx.x of the slab bsum[gridDim.x][C], added in a fixed order afterwards (hrv_act_bwd_bias_ordered).
template <bool kSlab>
__global__ void __launch_bounds__(256, 1) act_bwd_bias_kernel(NView dy, NView y, NView dv, int act, int G, int PL, int chunk,
                                                          long long npix, double* __restrict__ bsum) {
  extern __shared__ float shf[];  // [PL][C]
  const int C = G * 8;
  const int g = threadIdx.x % G;
  const int pl = threadIdx.x / G;
  if (pl < PL) {
    const int c0 = g * 8;
    const long long p_begin = (long long)blockIdx.x * chunk;
    long long p_end = p_begin + chunk;
    if (p_end > npix) p_end = npix;
    float s[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    const __nv_bfloat16* dyp = reinterpret_cast<const __nv_bfloat16*>(dy.ptr) + c0;
    const __nv_bfloat16* yp = reinterpret_cast<const __nv_bfloat16*>(y.ptr) + c0;
    __nv_bfloat16* dvp = reinterpret_cast<__nv_bfloat16*>(const_cast<void*>(dv.ptr)) + c0;
    constexpr int U = 4;  // pixels per thread per iteration: 2*U independent 16-byte loads in flight (HBM latency hiding)
    long long p = p_begin + pl;
    for (; p + (long long)(U - 1) * PL < p_end; p += (long long)U * PL) {
      uint4 vd[U], vy[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        vd[u] = ld16(dyp + (p + (long long)u * PL) * dy.pitch);
        vy[u] = act != 0 ? ld16(yp + (p + (long long)u * PL) * y.pitch) : make_uint4(0, 0, 0, 0);
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        float fd[8], fy[8], o[8];
        un8(vd[u], fd);
        un8(vy[u], fy);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          o[i] = act != 0 ? act_grad(fd[i], fy[i], act) : fd[i];
          s[i] += o[i];
        }
        if (dv.ptr) *reinterpret_cast<uint4*>(dvp + (p + (long long)u * PL) * dv.pitch) = pk8(o);
      }
    }
    for (; p < p_end; p += PL) {
      float fd[8], fy[8], o[8];
      un8(ld16(dyp + p * dy.pitch), fd);
      if (act != 0) un8(ld16(yp + p * y.pitch), fy);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        o[i] = act != 0 ? act_grad(fd[i], fy[i], act) : fd[i];
        s[i] += o[i];
      }
      if (dv.ptr) *reinterpret_cast<uint4*>(dvp + p * dv.pitch) = pk8(o);
    }
    float* dst = shf + (long long)pl * C + c0;
#pragma unroll
    for (int i = 0; i < 8; ++i) dst[i] = s[i];
  }
  __syncthreads();
  if (bsum) {
    for (int j = threadIdx.x; j < C; j += blockDim.x) {
      double t = 0.0;
      for (int l = 0; l < PL; ++l) t += (double)shf[(long long)l * C + j];
      if constexpr (kSlab) bsum[(long long)blockIdx.x * C + j] = t;
      else atomicAdd(&bsum[j], t);
    }
  }
}
}  // namespace hrv

extern "C" int hrv_act_bwd_bias(const hrv_tensor* dy, const hrv_tensor* y, int32_t act, const hrv_tensor* dv, double* bias_sum,
                                hrv_stream stream) {
  int rc;
  if ((rc = chk(dy, "act_bwd dy")) || (rc = chk(y, "act_bwd y", act == 0)) || (rc = chk(dv, "act_bwd dv", true))) return rc;
  const int G = (dy->c + 7) / 8;
  if (G > 256) return set_error(HRV_EUNSUPPORTED, "act_bwd: more than 2048 channels");
  const long long npix = (long long)dy->n * dy->h * dy->w;
  int PL, chunk;
  unsigned gx;
  plan(npix, 1, G, PL, chunk, gx);
  cudaStream_t st = (cudaStream_t)stream;
  if (bias_sum) cudaMemsetAsync(bias_sum, 0, (size_t)G * 8 * sizeof(double), st);
  act_bwd_bias_kernel<false><<<gx, 256, (size_t)PL * G * 8 * sizeof(float), st>>>(mkview(dy), mkview(y), mkview(dv), act, G, PL, chunk, npix, bias_sum);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(HRV_ECUDA, "act_bwd_bias launch: %s", cudaGetErrorString(e));
  return HRV_OK;
}

extern "C" size_t hrv_act_bwd_bias_ordered_workspace_bytes(const hrv_tensor* dy) {
  if (!dy) return 0;
  const int G = (dy->c + 7) / 8;
  int PL, chunk;
  unsigned gx;
  plan((long long)dy->n * dy->h * dy->w, 1, G > 0 ? G : 1, PL, chunk, gx);
  return (size_t)gx * G * 8 * sizeof(double);
}

extern "C" int hrv_act_bwd_bias_ordered(const hrv_tensor* dy, const hrv_tensor* y, int32_t act, const hrv_tensor* dv, double* bias_sum,
                                        void* workspace, size_t workspace_bytes, hrv_stream stream) {
  int rc;
  if ((rc = chk(dy, "act_bwd dy")) || (rc = chk(y, "act_bwd y", act == 0)) || (rc = chk(dv, "act_bwd dv", true))) return rc;
  const int G = (dy->c + 7) / 8;
  if (G > 256) return set_error(HRV_EUNSUPPORTED, "act_bwd: more than 2048 channels");
  const long long npix = (long long)dy->n * dy->h * dy->w;
  int PL, chunk;
  unsigned gx;
  plan(npix, 1, G, PL, chunk, gx);
  if (bias_sum) {
    const size_t need = hrv_act_bwd_bias_ordered_workspace_bytes(dy);
    if (!workspace || workspace_bytes < need) return set_error(HRV_EINVAL, "act_bwd_bias_ordered: workspace too small (%zu < %zu)", workspace_bytes, need);
  }
  cudaStream_t st = (cudaStream_t)stream;
  double* slab = bias_sum ? (double*)workspace : nullptr;
  act_bwd_bias_kernel<true><<<gx, 256, (size_t)PL * G * 8 * sizeof(float), st>>>(mkview(dy), mkview(y), mkview(dv), act, G, PL, chunk, npix, slab);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(HRV_ECUDA, "act_bwd_bias_ordered launch: %s", cudaGetErrorString(e));
  return bias_sum ? slab_sum(slab, 1, (int)gx, G * 8, bias_sum, 0, st, "act_bwd_bias_ordered sum") : HRV_OK;
}
