// aux_kernels.cu — the HBM-bound kernels of the hot path (NHWC bf16, 16-byte vector accesses, 8 channels/thread):
// InstanceNorm statistics (with the SPADE noise, virtual up-sampling and concat), InstanceNorm apply, layout
// converters with nearest resampling, space-to-depth, 3x3/s2 average pool, bilinear x2 (+add), and the fused
// appearance-flow warp.  Citations: see include/hrviton_sm100.h.
#include <cub/device/device_radix_sort.cuh>

#include "hrv_host.h"
#include "hrv_ptx.cuh"

namespace hrv {

struct View {
  const void* ptr;
  int n, h, w, c, pitch, dtype;
};
static View mk(const hrv_tensor* t) {
  View v;
  if (t) { v.ptr = t->ptr; v.n = t->n; v.h = t->h; v.w = t->w; v.c = t->c; v.pitch = t->pitch; v.dtype = t->dtype; }
  else { memset(&v, 0, sizeof(v)); }
  return v;
}

__device__ __forceinline__ void unpack8(const uint4& u, float (&f)[8]) {
  f[0] = bf16_lo(u.x); f[1] = bf16_hi(u.x); f[2] = bf16_lo(u.y); f[3] = bf16_hi(u.y);
  f[4] = bf16_lo(u.z); f[5] = bf16_hi(u.z); f[6] = bf16_lo(u.w); f[7] = bf16_hi(u.w);
}
__device__ __forceinline__ uint4 pack8(const float (&f)[8]) {
  uint4 o;
  o.x = pack_bf16(f[0], f[1]); o.y = pack_bf16(f[2], f[3]); o.z = pack_bf16(f[4], f[5]); o.w = pack_bf16(f[6], f[7]);
  return o;
}
__device__ __forceinline__ uint4 ldg16(const void* p) { return __ldg(reinterpret_cast<const uint4*>(p)); }

// 8 consecutive channels of one pixel in the storage type T: one 16-byte vector of the flavour's 16-bit type, or two of fp32 (the
// fp32 reference-precision storage).  The kernels below are templates on T; the 16-bit instantiations are the original code.
template <typename T> struct Vec8 { uint4 u; };
template <> struct Vec8<float> { float4 a, b; };
__device__ __forceinline__ Vec8<__nv_bfloat16> ldv8(const __nv_bfloat16* p) { return Vec8<__nv_bfloat16>{ldg16(p)}; }
__device__ __forceinline__ Vec8<float> ldv8(const float* p) {
  return Vec8<float>{__ldg(reinterpret_cast<const float4*>(p)), __ldg(reinterpret_cast<const float4*>(p) + 1)};
}
__device__ __forceinline__ void unpack8(const Vec8<__nv_bfloat16>& v, float (&f)[8]) { unpack8(v.u, f); }
__device__ __forceinline__ void unpack8(const Vec8<float>& v, float (&f)[8]) {
  f[0] = v.a.x; f[1] = v.a.y; f[2] = v.a.z; f[3] = v.a.w; f[4] = v.b.x; f[5] = v.b.y; f[6] = v.b.z; f[7] = v.b.w;
}
__device__ __forceinline__ void stv8(__nv_bfloat16* p, const Vec8<__nv_bfloat16>& v) { *reinterpret_cast<uint4*>(p) = v.u; }
__device__ __forceinline__ void stv8(float* p, const Vec8<float>& v) {
  reinterpret_cast<float4*>(p)[0] = v.a;
  reinterpret_cast<float4*>(p)[1] = v.b;
}
__device__ __forceinline__ void st8(__nv_bfloat16* p, const float (&f)[8]) { *reinterpret_cast<uint4*>(p) = pack8(f); }
__device__ __forceinline__ void st8(float* p, const float (&f)[8]) {
  reinterpret_cast<float4*>(p)[0] = make_float4(f[0], f[1], f[2], f[3]);
  reinterpret_cast<float4*>(p)[1] = make_float4(f[4], f[5], f[6], f[7]);
}
// The first k < 8 elements of a group (a view's last channels), the rest zero: nothing past the view is read.
__device__ __forceinline__ Vec8<__nv_bfloat16> ldv8_head(const __nv_bfloat16* p, int k) {
  const unsigned short* q = reinterpret_cast<const unsigned short*>(p);
  uint32_t w[4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
    w[i] = (2 * i < k ? (uint32_t)__ldg(q + 2 * i) : 0u) | ((2 * i + 1 < k ? (uint32_t)__ldg(q + 2 * i + 1) : 0u) << 16);
  return Vec8<__nv_bfloat16>{make_uint4(w[0], w[1], w[2], w[3])};
}
__device__ __forceinline__ Vec8<float> ldv8_head(const float* p, int k) {
  float f[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) f[i] = i < k ? __ldg(p + i) : 0.f;
  return Vec8<float>{make_float4(f[0], f[1], f[2], f[3]), make_float4(f[4], f[5], f[6], f[7])};
}
template <typename T> __device__ __forceinline__ Vec8<T> zero8();
template <> __device__ __forceinline__ Vec8<__nv_bfloat16> zero8<__nv_bfloat16>() { return Vec8<__nv_bfloat16>{make_uint4(0, 0, 0, 0)}; }
template <> __device__ __forceinline__ Vec8<float> zero8<float>() { return Vec8<float>{make_float4(0.f, 0.f, 0.f, 0.f), make_float4(0.f, 0.f, 0.f, 0.f)}; }

// ------------------------------------------------------------------------------------------------ IN statistics
// grid (chunks, N); thread = (pixel lane pl, channel group g of 8).  Each thread accumulates fp32 partial sums over its
// pixels (4 independent 16-byte loads in flight), partials meet in shared memory (one slot per thread, no atomics),
// then every block writes its fp64 per-channel sums into its own slab [n][blockIdx.x][C][2]; slab_sum adds the slabs in a fixed
// order, so the statistics do not depend on which block finishes first.
template <typename T>
struct StatsSrc {
  const T* p0;
  const T* p1;
  const float* noise;
  long long pitch0, pitch1;
  int W, W0, sh, from0;
};
template <typename T>
__device__ __forceinline__ void stats_load(const StatsSrc<T>& S, long long p, Vec8<T>& v, float& nz) {
  const int y = (int)(p / S.W), x = (int)(p - (long long)y * S.W);
  const T* src = S.from0 ? S.p0 + ((long long)(y >> S.sh) * S.W0 + (x >> S.sh)) * S.pitch0 : S.p1 + p * S.pitch1;
  v = ldv8(src);
  nz = S.noise ? __ldg(S.noise + p) : 0.f;
}
template <typename T>
__global__ void __launch_bounds__(256) instnorm_stats_kernel(View x0, int x0_shift, View x1, int H, int W, int G, int PL,
                                                            int chunk, const float* __restrict__ noise,
                                                            const float* __restrict__ ns, double* __restrict__ slab) {
  extern __shared__ float shf[];  // [PL][C][2]
  const int n = blockIdx.y;
  const int C = G * 8;
  const int g = threadIdx.x % G;
  const int pl = threadIdx.x / G;
  if (pl < PL) {
    const int c0 = g * 8;
    const long long HW = (long long)H * W;
    const long long p_begin = (long long)blockIdx.x * chunk;
    long long p_end = p_begin + chunk;
    if (p_end > HW) p_end = HW;
    float s[8], q[8], nsv[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) { s[i] = 0.f; q[i] = 0.f; nsv[i] = ns ? __ldg(ns + c0 + i) : 0.f; }
    StatsSrc<T> S;
    S.from0 = c0 < x0.c;
    S.sh = x0_shift; S.W = W; S.W0 = W >> x0_shift;
    S.pitch0 = x0.pitch; S.pitch1 = x1.pitch;
    S.p0 = reinterpret_cast<const T*>(x0.ptr) + (long long)n * (H >> x0_shift) * S.W0 * x0.pitch + c0;
    S.p1 = reinterpret_cast<const T*>(x1.ptr) + (long long)n * HW * x1.pitch + (c0 - x0.c);
    S.noise = noise ? noise + (long long)n * HW : nullptr;
    long long p = p_begin + pl;
    for (; p + 3LL * PL < p_end; p += 4LL * PL) {
      Vec8<T> v[4];
      float nz[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) stats_load(S, p + (long long)u * PL, v[u], nz[u]);
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        float f[8];
        unpack8(v[u], f);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float t = fmaf(nz[u], nsv[i], f[i]);
          s[i] += t;
          q[i] = fmaf(t, t, q[i]);
        }
      }
    }
    for (; p < p_end; p += PL) {
      Vec8<T> v;
      float nz, f[8];
      stats_load(S, p, v, nz);
      unpack8(v, f);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float t = fmaf(nz, nsv[i], f[i]);
        s[i] += t;
        q[i] = fmaf(t, t, q[i]);
      }
    }
    float* dst = shf + ((long long)pl * C + c0) * 2;
#pragma unroll
    for (int i = 0; i < 8; ++i) { dst[2 * i] = s[i]; dst[2 * i + 1] = q[i]; }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    double S1 = 0.0, S2 = 0.0;
    for (int l = 0; l < PL; ++l) {
      S1 += (double)shf[((long long)l * C + c) * 2];
      S2 += (double)shf[((long long)l * C + c) * 2 + 1];
    }
    double* o = slab + (((long long)n * gridDim.x + blockIdx.x) * C + c) * 2;
    o[0] = S1;
    o[1] = S2;
  }
}

// ------------------------------------------------------------------------------------------------ IN statistics, fused form
// Statistics of up to TWO SPADE norms that share one input (norm_s and norm_0 of a block both normalise x = cat(up2(x0), x1), each with
// its own noise draw and noise scale, network_generator.py:101-113,160-170) from ONE pass over the SOURCE tensors:
//   sum_P (x_c[P] + nz_j[P] ns_jc)   = S1_c + ns_jc * NZ1_j               S1_c = sum x_c,   NZ1_j = sum nz_j
//   sum_P (x_c[P] + nz_j[P] ns_jc)^2 = S2_c + 2 ns_jc X_jc + ns_jc^2 NZ2_j   S2_c = sum x_c^2, X_jc = sum x_c nz_j, NZ2_j = sum nz_j^2
// x0 is read at ITS OWN resolution: with x0_shift = 1 every source pixel stands for its 2x2 children, so S1/S2 count it four times and
// X_jc pairs it with the sum of the children's noise — 4x fewer bytes than walking the virtual up-sampled tensor, and the second
// norm costs no second pass.  One launch per segment: segment 0 covers x0, segment 1 covers x1.  Every block writes its sums into
// its own slab, added in a fixed order by slab_sum: slab [N][gridDim.x][Cs][4] doubles {S1, S2, X_0, X_1} -> acc [N][C][4];
// nzslab [N][gridDim.x][4] doubles {NZ1_0, NZ2_0, NZ1_1, NZ2_1} (segment 0 only) -> nzacc [N][4].
template <typename T>
__global__ void __launch_bounds__(256) instnorm_stats2_kernel(View xs, int shift, int W_full, int G, int PL, int chunk,
                                                             const float* __restrict__ nz0, const float* __restrict__ nz1,
                                                             double* __restrict__ slab, double* __restrict__ nzslab, int do_noise_sums) {
  extern __shared__ float shf[];  // [PL][G*8][4]
  __shared__ float nzred[8][4];
  const int n = blockIdx.y;
  const int g = threadIdx.x % G, pl = threadIdx.x / G;
  const int Cs = G * 8;
  const long long HWs = (long long)xs.h * xs.w;           // source pixels
  const long long HWf = HWs << (2 * shift);               // full-resolution pixels
  float s[8], q[8], x0a[8], x1a[8], nsum[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int i = 0; i < 8; ++i) { s[i] = 0.f; q[i] = 0.f; x0a[i] = 0.f; x1a[i] = 0.f; }
  if (pl < PL) {
    const long long p_begin = (long long)blockIdx.x * chunk;
    long long p_end = p_begin + chunk;
    if (p_end > HWs) p_end = HWs;
    const T* base = reinterpret_cast<const T*>(xs.ptr) + (long long)n * HWs * xs.pitch + g * 8;
    const float* n0 = nz0 ? nz0 + (long long)n * HWf : nullptr;
    const float* n1 = nz1 ? nz1 + (long long)n * HWf : nullptr;
    for (long long p = p_begin + pl; p < p_end; p += PL) {
      const Vec8<T> v = ldv8(base + p * xs.pitch);
      float a0 = 0.f, a1 = 0.f, b0 = 0.f, b1 = 0.f;  // noise sum / sum of squares over the pixel's footprint, per norm
      if (shift) {
        const int y = (int)(p / xs.w), x = (int)(p - (long long)y * xs.w);
        const long long f = (long long)(2 * y) * W_full + 2 * x;
        if (n0) {
          const float2 t = __ldg(reinterpret_cast<const float2*>(n0 + f)), u = __ldg(reinterpret_cast<const float2*>(n0 + f + W_full));
          a0 = (t.x + t.y) + (u.x + u.y);
          b0 = fmaf(t.x, t.x, fmaf(t.y, t.y, fmaf(u.x, u.x, u.y * u.y)));
        }
        if (n1) {
          const float2 t = __ldg(reinterpret_cast<const float2*>(n1 + f)), u = __ldg(reinterpret_cast<const float2*>(n1 + f + W_full));
          a1 = (t.x + t.y) + (u.x + u.y);
          b1 = fmaf(t.x, t.x, fmaf(t.y, t.y, fmaf(u.x, u.x, u.y * u.y)));
        }
      } else {
        if (n0) { a0 = __ldg(n0 + p); b0 = a0 * a0; }
        if (n1) { a1 = __ldg(n1 + p); b1 = a1 * a1; }
      }
      float f8[8];
      unpack8(v, f8);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        s[i] += f8[i];
        q[i] = fmaf(f8[i], f8[i], q[i]);
        x0a[i] = fmaf(f8[i], a0, x0a[i]);
        x1a[i] = fmaf(f8[i], a1, x1a[i]);
      }
      if (g == 0) { nsum[0] += a0; nsum[1] += b0; nsum[2] += a1; nsum[3] += b1; }
    }
    float* dst = shf + ((long long)pl * Cs + g * 8) * 4;
#pragma unroll
    for (int i = 0; i < 8; ++i) { dst[4 * i] = s[i]; dst[4 * i + 1] = q[i]; dst[4 * i + 2] = x0a[i]; dst[4 * i + 3] = x1a[i]; }
  }
  __syncthreads();
  const double mult = (double)(1 << (2 * shift));  // every source pixel stands for 4^shift full-resolution pixels
  for (int c = threadIdx.x; c < Cs; c += blockDim.x) {
    double t[4] = {0.0, 0.0, 0.0, 0.0};
    for (int l = 0; l < PL; ++l) {
      const float* e = shf + ((long long)l * Cs + c) * 4;
      t[0] += (double)e[0]; t[1] += (double)e[1]; t[2] += (double)e[2]; t[3] += (double)e[3];
    }
    reinterpret_cast<double4*>(slab)[(size_t)(n * gridDim.x + blockIdx.x) * Cs + c] = make_double4(t[0] * mult, t[1] * mult, t[2], t[3]);
  }
  if (do_noise_sums) {  // NZ1/NZ2 of both norms: only the g == 0 threads hold contributions; warp reduce, then one slab entry per block
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      float v = nsum[k];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      if ((threadIdx.x & 31) == 0) nzred[threadIdx.x >> 5][k] = v;
    }
    __syncthreads();
    if (threadIdx.x < 4) {
      double t = 0.0;
      for (int wv = 0; wv < 8; ++wv) t += (double)nzred[wv][threadIdx.x];
      nzslab[(size_t)(n * gridDim.x + blockIdx.x) * 4 + threadIdx.x] = t;
    }
  }
}

__global__ void instnorm_finalize2_kernel(const double* __restrict__ acc, const double* __restrict__ nzacc, int N, int C, double inv_hw, float eps,
                                          const float* __restrict__ ns0, const float* __restrict__ ns1, float* __restrict__ mean0,
                                          float* __restrict__ rstd0, float* __restrict__ mean1, float* __restrict__ rstd1) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N * C) return;
  const int n = i / C, c = i - n * C;
  const double S1 = acc[4 * (long long)i], S2 = acc[4 * (long long)i + 1];
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    float* mean = j ? mean1 : mean0;
    float* rstd = j ? rstd1 : rstd0;
    if (!mean) continue;
    const float* nsp = j ? ns1 : ns0;
    const double ns = nsp ? (double)nsp[c] : 0.0;
    const double X = acc[4 * (long long)i + 2 + j], NZ1 = nzacc[n * 4 + 2 * j], NZ2 = nzacc[n * 4 + 2 * j + 1];
    const double m = (S1 + ns * NZ1) * inv_hw;
    double var = (S2 + 2.0 * ns * X + ns * ns * NZ2) * inv_hw - m * m;
    if (var < 0.0) var = 0.0;
    mean[i] = (float)m;
    rstd[i] = (float)(1.0 / sqrt(var + (double)eps));
  }
}

__global__ void instnorm_finalize_kernel(const double* __restrict__ acc, int NC, double inv_hw, float eps,
                                         float* __restrict__ mean, float* __restrict__ rstd) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= NC) return;
  const double m = acc[2 * i] * inv_hw;
  double var = acc[2 * i + 1] * inv_hw - m * m;
  if (var < 0.0) var = 0.0;
  mean[i] = (float)m;
  rstd[i] = (float)(1.0 / sqrt(var + (double)eps));
}

template <typename T>
__global__ void instnorm_apply_kernel(View x, const float* __restrict__ mean, const float* __restrict__ rstd,
                                      const float* __restrict__ gamma, const float* __restrict__ beta, View res, int act, View y,
                                      long long total, int G) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int g = (int)(idx % G);
  const long long pix = idx / G;
  const int n = (int)(pix / ((long long)x.h * x.w));
  float f[8], r[8];
  unpack8(ldv8(reinterpret_cast<const T*>(x.ptr) + pix * x.pitch + g * 8), f);
  if (res.ptr) unpack8(ldv8(reinterpret_cast<const T*>(res.ptr) + pix * res.pitch + g * 8), r);
  const float* mp = mean + (long long)n * x.c + g * 8;
  const float* rp = rstd + (long long)n * x.c + g * 8;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int c = g * 8 + i;
    if (c < x.c) {
      float v = (f[i] - __ldg(mp + i)) * __ldg(rp + i);
      if (gamma) v = fmaf(v, __ldg(gamma + c), beta ? __ldg(beta + c) : 0.f);
      if (res.ptr) v += r[i];
      f[i] = apply_act(v, act);
    } else {
      f[i] = 0.f;
    }
  }
  st8(reinterpret_cast<T*>(const_cast<void*>(y.ptr)) + pix * y.pitch + g * 8, f);
}

// ------------------------------------------------------------------------------------------------ layout converters
// thread = (dst pixel, 8-channel group); src fp32 NCHW with nearest resampling.
template <typename T>
__global__ void nchw_to_nhwc_kernel(const float* __restrict__ src, int C, int SH, int SW, View dst, int G, long long total) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int g = (int)(idx % G);
  const long long pix = idx / G;
  const int x = (int)(pix % dst.w);
  const int y = (int)((pix / dst.w) % dst.h);
  const int n = (int)(pix / ((long long)dst.w * dst.h));
  // F.interpolate(mode='nearest'): src = min(floor(dst * (in / out)), in - 1) with the scale and the product rounded to fp32, as torch
  // computes it.  The exact integer floor(dst * in / out) picks the next pixel where the fp32 product falls just below an integer.
  const int sy = min((int)floorf(__fmul_rn((float)y, __fdiv_rn((float)SH, (float)dst.h))), SH - 1);
  const int sx = min((int)floorf(__fmul_rn((float)x, __fdiv_rn((float)SW, (float)dst.w))), SW - 1);
  float f[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int c = g * 8 + i;
    f[i] = c < C ? __ldg(src + (((long long)n * C + c) * SH + sy) * SW + sx) : 0.f;
  }
  st8(reinterpret_cast<T*>(const_cast<void*>(dst.ptr)) + pix * dst.pitch + g * 8, f);
}

// The condition discriminator's input [input1 | input2 | third] built in one pass from three fp32 NCHW tensors (test_condition.py:
// 106-120, get_norm_const.py:99-115).  thread = one pixel: it needs all K scores of the pixel for the soft-max, reads every plane
// coalesced, and writes the pixel's G 8-channel groups.  `third` is seg with channel cm_channel multiplied by cm (mode 1) or by
// (cm > 0.5) (mode 2), then its channel soft-max (softmax = 1: maximum subtracted, expf, true division) or itself (softmax = 0).
// The scores are re-read from L1 for the maximum, the sum and the write rather than held in K registers.
struct SegCatSrc {
  const float* in1;
  const float* in2;
  const float* seg;
  const float* cm;
  int c1, c2, K, cm_channel, mode, softmax;
};
// The per-pixel decisions that seg_softmax_cat_kernel and seg_iou_kernel share, so that both compose and soft-max alike.
// seg_cm_factor: the composition factor of the pixel (mode 0: 1, mode 1: cm, mode 2: cm > 0.5).  seg_score: the composed score of
// channel k (seg_px points at channel 0 of the pixel, planes hw apart; cm_channel < 0: none is composed).  SegSoftmax: the channel
// maximum and the sum of expf(score - maximum) in channel order, so that p_k = seg_prob(score_k) = expf(score_k - mx) / sum.
__device__ __forceinline__ float seg_cm_factor(const float* cm, long long pix, int mode) {
  if (mode == 0) return 1.f;
  const float m = __ldg(cm + pix);
  return mode == 2 ? (m > 0.5f ? 1.f : 0.f) : m;
}
__device__ __forceinline__ float seg_score(const float* seg_px, long long hw, int k, int cm_channel, float m) {
  const float s = __ldg(seg_px + (long long)k * hw);
  return k == cm_channel ? __fmul_rn(s, m) : s;
}
struct SegSoftmax {
  float mx, sum;
  __device__ __forceinline__ SegSoftmax(const float* seg_px, long long hw, int K, int cm_channel, float m) : mx(-INFINITY), sum(0.f) {
    for (int k = 0; k < K; ++k) mx = fmaxf(mx, seg_score(seg_px, hw, k, cm_channel, m));
    for (int k = 0; k < K; ++k) sum += expf(seg_score(seg_px, hw, k, cm_channel, m) - mx);
  }
  __device__ __forceinline__ float prob(float s) const { return __fdiv_rn(expf(s - mx), sum); }
};
__device__ __forceinline__ float seg_cat_score(const SegCatSrc& S, const float* seg_px, long long hw, int k, float m) {
  return seg_score(seg_px, hw, k, S.cm_channel, m);
}
template <typename T>
__global__ void seg_softmax_cat_kernel(SegCatSrc S, View dst, float* __restrict__ seg_out, int G, long long npix) {
  const long long pix = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= npix) return;
  const long long hw = (long long)dst.h * dst.w;
  const long long n = pix / hw, rem = pix - n * hw;
  const float* seg_px = S.seg + n * S.K * hw + rem;
  const float m = seg_cm_factor(S.cm, pix, S.mode);
  SegSoftmax sm = S.softmax ? SegSoftmax(seg_px, hw, S.K, S.cm_channel, m) : SegSoftmax(seg_px, hw, 0, S.cm_channel, m);
  if (seg_out)
    for (int k = 0; k < S.K; ++k) seg_out[n * S.K * hw + (long long)k * hw + rem] = seg_cat_score(S, seg_px, hw, k, m);
  const int c12 = S.c1 + S.c2;
  T* out = reinterpret_cast<T*>(const_cast<void*>(dst.ptr)) + pix * dst.pitch;
  for (int g = 0; g < G; ++g) {
    float f[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int c = g * 8 + i;
      if (c < S.c1) {
        f[i] = __ldg(S.in1 + (n * S.c1 + c) * hw + rem);
      } else if (c < c12) {
        f[i] = __ldg(S.in2 + (n * S.c2 + (c - S.c1)) * hw + rem);
      } else if (c < c12 + S.K) {
        const float s = seg_cat_score(S, seg_px, hw, c - c12, m);
        f[i] = S.softmax ? sm.prob(s) : s;
      } else {
        f[i] = 0.f;
      }
    }
    st8(out + g * 8, f);
  }
}

// The stage-1 validation IoU (train_condition.py:18-36 on F.softmax(fake_segmap * cloth_mask, 1), :314-356).  grid (blocks, N),
// thread = pixels of one sample, strided: the pixel's scores composed ('warp_grad': channel SEG_IOU_CM_CHANNEL times cm) and
// soft-maxed by the functions seg_softmax_cat_kernel uses, then per channel pred = p > 0.5, lab = (parse == 1).  Each warp adds its
// counts with integer reductions and writes (P, L, I) to its own slot of `partial`; no shared memory, no atomics.
constexpr int SEG_IOU_THREADS = 256, SEG_IOU_WARPS = SEG_IOU_THREADS / 32, SEG_IOU_MAX_BLOCKS = 64, SEG_IOU_CM_CHANNEL = 3;
__global__ void __launch_bounds__(SEG_IOU_THREADS) seg_iou_count_kernel(const float* __restrict__ seg, const float* __restrict__ cm,
                                                                        const float* __restrict__ parse, int K, long long hw,
                                                                        int4* __restrict__ partial) {
  const int n = blockIdx.y;
  const float* seg_n = seg + (long long)n * K * hw;
  const float* lab_n = parse + (long long)n * K * hw;
  int P = 0, L = 0, I = 0;
  for (long long rem = (long long)blockIdx.x * blockDim.x + threadIdx.x; rem < hw; rem += (long long)gridDim.x * blockDim.x) {
    const float m = seg_cm_factor(cm, (long long)n * hw + rem, 1);
    const SegSoftmax sm(seg_n + rem, hw, K, SEG_IOU_CM_CHANNEL, m);
    for (int k = 0; k < K; ++k) {
      const int pred = sm.prob(seg_score(seg_n + rem, hw, k, SEG_IOU_CM_CHANNEL, m)) > 0.5f;
      const int lab = __ldg(lab_n + (long long)k * hw + rem) == 1.f;
      P += pred;
      L += lab;
      I += pred & lab;
    }
  }
  P = __reduce_add_sync(0xffffffffu, P);
  L = __reduce_add_sync(0xffffffffu, L);
  I = __reduce_add_sync(0xffffffffu, I);
  if ((threadIdx.x & 31) == 0)
    partial[((long long)n * gridDim.x + blockIdx.x) * SEG_IOU_WARPS + (threadIdx.x >> 5)] = make_int4(P, L, I, 0);
}

// One warp: per sample (in order) the counts of its `parts` slots, then the reference's fp32 arithmetic.  iou_metric computes
// intersection = sum(y_pred[y_true == 1]) (int64 I), union = sum(y_pred) + sum(y_true) (int64 P promoted to fp32, plus the fp32 sum
// of the 0/1 labels, exactly L below 2^24), and iou += (intersection + 1e-7) / (union - intersection + 1e-7) / B from iou = 0, each
// operation rounded to fp32.  Restated:  iou = sum over n in order of ((f32(I) + 1e-7f) / ((f32(P) + f32(L)) - f32(I) + 1e-7f)) / f32(B).
__global__ void seg_iou_finish_kernel(const int4* __restrict__ partial, int parts, int N, float* __restrict__ iou) {
  const int lane = threadIdx.x;
  float acc = 0.f;
  for (int n = 0; n < N; ++n) {
    int P = 0, L = 0, I = 0;
    for (int i = lane; i < parts; i += 32) {
      const int4 v = partial[(long long)n * parts + i];
      P += v.x;
      L += v.y;
      I += v.z;
    }
    P = __reduce_add_sync(0xffffffffu, P);
    L = __reduce_add_sync(0xffffffffu, L);
    I = __reduce_add_sync(0xffffffffu, I);
    const float fi = __int2float_rn(I);
    const float uni = __fadd_rn(__int2float_rn(P), __int2float_rn(L));
    const float t = __fdiv_rn(__fdiv_rn(__fadd_rn(fi, 1e-7f), __fadd_rn(__fsub_rn(uni, fi), 1e-7f)), __int2float_rn(N));
    acc = __fadd_rn(acc, t);
  }
  if (lane == 0) *iou = acc;
}

// thread = (pixel); loops channels; writes are coalesced per plane.
__global__ void nhwc_to_nchw_kernel(View src, float* __restrict__ dst, long long npix) {
  const long long pix = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= npix) return;
  const long long hw = (long long)src.h * src.w;
  const int n = (int)(pix / hw);
  const long long rem = pix - (long long)n * hw;
  float* d = dst + (long long)n * src.c * hw + rem;
  if (src.dtype == 0) {
    const __nv_bfloat16* s = reinterpret_cast<const __nv_bfloat16*>(src.ptr) + pix * src.pitch;
    for (int c = 0; c < src.c; ++c) d[(long long)c * hw] = __bfloat162float(s[c]);
  } else {
    const float* s = reinterpret_cast<const float*>(src.ptr) + pix * src.pitch;
    for (int c = 0; c < src.c; ++c) d[(long long)c * hw] = s[c];
  }
}

// thread = (dst pixel, sub-pixel 0..3, 8-channel group of src)
template <typename T>
__global__ void space_to_depth_kernel(View src, View dst, int G, int Gd, long long total) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int gd = (int)(idx % Gd);  // dst channel group
  const long long pix = idx / Gd;
  const int X = (int)(pix % dst.w);
  const int Y = (int)((pix / dst.w) % dst.h);
  const int n = (int)(pix / ((long long)dst.w * dst.h));
  Vec8<T> v = zero8<T>();
  const int sub = gd / G, g = gd % G;
  if (sub < 4) {
    const int sy = 2 * Y + (sub >> 1), sx = 2 * X + (sub & 1);
    if (sy < src.h && sx < src.w) {
      const T* p = reinterpret_cast<const T*>(src.ptr) + (((long long)n * src.h + sy) * src.w + sx) * src.pitch + g * 8;
      // a partial last group copies the view's channels only: [c, c8) of each sub-image is zero, whatever lies past the view
      v = g * 8 + 8 <= src.c ? ldv8(p) : ldv8_head(p, src.c - g * 8);
    }
  }
  stv8(reinterpret_cast<T*>(const_cast<void*>(dst.ptr)) + pix * dst.pitch + gd * 8, v);
}

template <typename T>
__global__ void avgpool3s2_kernel(View src, View dst, int G, long long total) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int g = (int)(idx % G);
  const long long pix = idx / G;
  const int X = (int)(pix % dst.w);
  const int Y = (int)((pix / dst.w) % dst.h);
  const int n = (int)(pix / ((long long)dst.w * dst.h));
  float s[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  int cnt = 0;
  for (int dy = -1; dy <= 1; ++dy) {
    const int y = 2 * Y + dy;
    if (y < 0 || y >= src.h) continue;
    for (int dx = -1; dx <= 1; ++dx) {
      const int x = 2 * X + dx;
      if (x < 0 || x >= src.w) continue;
      float f[8];
      unpack8(ldv8(reinterpret_cast<const T*>(src.ptr) + (((long long)n * src.h + y) * src.w + x) * src.pitch + g * 8), f);
#pragma unroll
      for (int i = 0; i < 8; ++i) s[i] += f[i];
      ++cnt;
    }
  }
  const float inv = 1.f / (float)cnt;
#pragma unroll
  for (int i = 0; i < 8; ++i) s[i] *= inv;
  st8(reinterpret_cast<T*>(const_cast<void*>(dst.ptr)) + pix * dst.pitch + g * 8, s);
}

// F.interpolate(bilinear, x2, align_corners=False): s = max((d+0.5)/2-0.5, 0); i0=floor(s); i1=min(i0+1,n-1)
__device__ __forceinline__ void up2_taps(int d, int n, int& i0, int& i1, float& w0, float& w1) {
  float s = __fsub_rn(__fmul_rn(__fadd_rn((float)d, 0.5f), 0.5f), 0.5f);
  s = fmaxf(s, 0.f);
  const float fl = floorf(s);
  i0 = (int)fl;
  i1 = min(i0 + 1, n - 1);
  w1 = __fsub_rn(s, fl);
  w0 = __fsub_rn(1.f, w1);
}

template <typename T>
__global__ void bilinear_up2_add_kernel(View a, View b, View dst, int G, long long total) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int g = (int)(idx % G);
  const long long pix = idx / G;
  const int x = (int)(pix % dst.w);
  const int y = (int)((pix / dst.w) % dst.h);
  const int n = (int)(pix / ((long long)dst.w * dst.h));
  int x0, x1, y0, y1;
  float wx0, wx1, wy0, wy1;
  up2_taps(x, a.w, x0, x1, wx0, wx1);
  up2_taps(y, a.h, y0, y1, wy0, wy1);
  const T* ap = reinterpret_cast<const T*>(a.ptr) + (long long)n * a.h * a.w * a.pitch + g * 8;
  float f00[8], f01[8], f10[8], f11[8], o[8];
  unpack8(ldv8(ap + ((long long)y0 * a.w + x0) * a.pitch), f00);
  unpack8(ldv8(ap + ((long long)y0 * a.w + x1) * a.pitch), f01);
  unpack8(ldv8(ap + ((long long)y1 * a.w + x0) * a.pitch), f10);
  unpack8(ldv8(ap + ((long long)y1 * a.w + x1) * a.pitch), f11);
#pragma unroll
  for (int i = 0; i < 8; ++i) o[i] = wy0 * (wx0 * f00[i] + wx1 * f01[i]) + wy1 * (wx0 * f10[i] + wx1 * f11[i]);
  if (b.ptr) {
    float fb[8];
    unpack8(ldv8(reinterpret_cast<const T*>(b.ptr) + pix * b.pitch + g * 8), fb);
#pragma unroll
    for (int i = 0; i < 8; ++i) o[i] += fb[i];
  }
  st8(reinterpret_cast<T*>(const_cast<void*>(dst.ptr)) + pix * dst.pitch + g * 8, o);
}

// ------------------------------------------------------------------------------------------------ flow warp
// The sampling coordinates of destination pixel (x, y) of image n, shared by the forward and the ordered backward passes so they
// cannot drift apart.  The chain uses explicitly rounded fp32 operations (no FMA contraction) in the exact order of
// oracle/hrviton_oracle.py:np_flow_warp_coords so that the gather indices are bit-exact.
struct WarpTaps {
  float fx, fy;    // the up-sampled flow
  float ixr, iyr;  // source coordinates before the border clamp
  int x0, y0, x1, y1;
  float tx, ty, wx0, wx1, wy0, wy1;  // wx1 / wy1 are zero where the second tap falls outside the image
  bool vx, vy;     // the second tap lies inside the image
};
__device__ __forceinline__ WarpTaps warp_taps(const float* __restrict__ flow_lo, const float* __restrict__ lin_x, const float* __restrict__ lin_y,
                                              int n, int x, int y, int H, int W, int Hs, int Ws, float sx, float sy) {
  const int hl = H >> 1, wl = W >> 1;
  int xa, xb, ya, yb;
  float wxa, wxb, wya, wyb;
  up2_taps(x, wl, xa, xb, wxa, wxb);
  up2_taps(y, hl, ya, yb, wya, wyb);
  const float2* fl = reinterpret_cast<const float2*>(flow_lo) + (long long)n * hl * wl;
  const float2 f00 = __ldg(fl + (long long)ya * wl + xa), f01 = __ldg(fl + (long long)ya * wl + xb);
  const float2 f10 = __ldg(fl + (long long)yb * wl + xa), f11 = __ldg(fl + (long long)yb * wl + xb);
  // lerp along x inside each source row, then along y (torch's CPU kernel order)
  const float ux0 = __fadd_rn(__fmul_rn(f00.x, wxa), __fmul_rn(f01.x, wxb));
  const float ux1 = __fadd_rn(__fmul_rn(f10.x, wxa), __fmul_rn(f11.x, wxb));
  const float uy0 = __fadd_rn(__fmul_rn(f00.y, wxa), __fmul_rn(f01.y, wxb));
  const float uy1 = __fadd_rn(__fmul_rn(f10.y, wxa), __fmul_rn(f11.y, wxb));
  WarpTaps t;
  t.fx = __fadd_rn(__fmul_rn(ux0, wya), __fmul_rn(ux1, wyb));
  t.fy = __fadd_rn(__fmul_rn(uy0, wya), __fmul_rn(uy1, wyb));
  const float gx = __fadd_rn(__fdiv_rn(t.fx, sx), __ldg(lin_x + x));
  const float gy = __fadd_rn(__fdiv_rn(t.fy, sy), __ldg(lin_y + y));
  t.ixr = __fdiv_rn(__fsub_rn(__fmul_rn(__fadd_rn(gx, 1.f), (float)Ws), 1.f), 2.f);
  t.iyr = __fdiv_rn(__fsub_rn(__fmul_rn(__fadd_rn(gy, 1.f), (float)Hs), 1.f), 2.f);
  const float ix = fminf(fmaxf(t.ixr, 0.f), (float)(Ws - 1));
  const float iy = fminf(fmaxf(t.iyr, 0.f), (float)(Hs - 1));
  const float fx0 = floorf(ix), fy0 = floorf(iy);
  t.x0 = (int)fx0;
  t.y0 = (int)fy0;
  t.tx = __fsub_rn(ix, fx0);
  t.ty = __fsub_rn(iy, fy0);
  t.vx = t.x0 + 1 <= Ws - 1;
  t.vy = t.y0 + 1 <= Hs - 1;
  t.x1 = t.vx ? t.x0 + 1 : t.x0;
  t.y1 = t.vy ? t.y0 + 1 : t.y0;
  t.wx1 = t.vx ? t.tx : 0.f;
  t.wy1 = t.vy ? t.ty : 0.f;
  t.wx0 = __fsub_rn(1.f, t.tx);
  t.wy0 = __fsub_rn(1.f, t.ty);
  return t;
}

// thread = (dst pixel, 8-channel group).
__global__ void flow_warp_kernel(const float* __restrict__ flow_lo, const float* __restrict__ lin_x, const float* __restrict__ lin_y,
                                 View src, View dst, float* __restrict__ flow_up, int* __restrict__ idx_out, float sx, float sy,
                                 int G, long long total) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int g = (int)(idx % G);
  const long long pix = idx / G;
  const int W = dst.w, H = dst.h;
  const int x = (int)(pix % W);
  const int y = (int)((pix / W) % H);
  const int n = (int)(pix / ((long long)W * H));
  const WarpTaps t = warp_taps(flow_lo, lin_x, lin_y, n, x, y, H, W, src.h, src.w, sx, sy);
  const int x0 = t.x0, y0 = t.y0, x1 = t.x1, y1 = t.y1;
  if (g == 0) {
    if (flow_up) reinterpret_cast<float2*>(flow_up)[pix] = make_float2(t.fx, t.fy);
    if (idx_out) reinterpret_cast<int2*>(idx_out)[pix] = make_int2(x0, y0);
  }
  if (g * 8 >= ((src.c + 7) & ~7)) return;
  const float w00 = t.wy0 * t.wx0, w01 = t.wy0 * t.wx1, w10 = t.wy1 * t.wx0, w11 = t.wy1 * t.wx1;
  float o[8];
  const long long ib = (long long)n * src.h * src.w;
  if (src.dtype == 0) {
    const __nv_bfloat16* sp = reinterpret_cast<const __nv_bfloat16*>(src.ptr) + g * 8;
    float a[8], b[8], c[8], d[8];
    unpack8(ldg16(sp + (ib + (long long)y0 * src.w + x0) * src.pitch), a);
    unpack8(ldg16(sp + (ib + (long long)y0 * src.w + x1) * src.pitch), b);
    unpack8(ldg16(sp + (ib + (long long)y1 * src.w + x0) * src.pitch), c);
    unpack8(ldg16(sp + (ib + (long long)y1 * src.w + x1) * src.pitch), d);
#pragma unroll
    for (int i = 0; i < 8; ++i) o[i] = a[i] * w00 + b[i] * w01 + c[i] * w10 + d[i] * w11;
  } else {
    const float* sp = reinterpret_cast<const float*>(src.ptr) + g * 8;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      if (g * 8 + i < src.c) {
        o[i] = __ldg(sp + (ib + (long long)y0 * src.w + x0) * src.pitch + i) * w00 + __ldg(sp + (ib + (long long)y0 * src.w + x1) * src.pitch + i) * w01 +
               __ldg(sp + (ib + (long long)y1 * src.w + x0) * src.pitch + i) * w10 + __ldg(sp + (ib + (long long)y1 * src.w + x1) * src.pitch + i) * w11;
      } else {
        o[i] = 0.f;
      }
    }
  }
  if (dst.dtype == 0) {
    *reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(const_cast<void*>(dst.ptr)) + pix * dst.pitch + g * 8) = pack8(o);
  } else {
    float* dp = reinterpret_cast<float*>(const_cast<void*>(dst.ptr)) + pix * dst.pitch + g * 8;
#pragma unroll
    for (int i = 0; i < 8; ++i)
      if (g * 8 + i < dst.c) dp[i] = o[i];
  }
}

static int check_bf16_vec(const hrv_tensor* t, const char* what) {
  if (!t || !t->ptr) return set_error(HRV_EINVAL, "%s: null tensor", what);
  if (t->dtype != HRV_BF16) return set_error(HRV_EINVAL, "%s: must be bf16", what);
  if (((uintptr_t)t->ptr & 15) || (t->pitch % 8)) return set_error(HRV_EINVAL, "%s: needs 16-byte alignment and pitch %% 8 == 0", what);
  return 0;
}
// The entry points that also take fp32 storage: every tensor of one call shares the storage type `dt` of its first one.
static int storage_of(const hrv_tensor* t) { return (t && t->dtype == HRV_F32) ? HRV_F32 : HRV_BF16; }
static int check_vec(const hrv_tensor* t, const char* what, int dt) {
  if (dt == HRV_BF16) return check_bf16_vec(t, what);
  if (!t || !t->ptr) return set_error(HRV_EINVAL, "%s: null tensor", what);
  if (t->dtype != HRV_F32) return set_error(HRV_EINVAL, "%s: must be fp32 like the call's other tensors (one storage type per call)", what);
  if (((uintptr_t)t->ptr & 15) || (t->pitch % 8)) return set_error(HRV_EINVAL, "%s: needs 16-byte alignment and pitch %% 8 == 0", what);
  return 0;
}
// kernel<T><<<...>>>(args) with T = the flavour's 16-bit type or float, after the storage type dt.
#define HRV_LAUNCH_STORAGE(dt, kernel, grid, block, smem, st, ...)                           \
  do {                                                                                       \
    if ((dt) == HRV_F32) kernel<float><<<(grid), (block), (smem), (st)>>>(__VA_ARGS__);      \
    else kernel<__nv_bfloat16><<<(grid), (block), (smem), (st)>>>(__VA_ARGS__);              \
  } while (0)
static int launch_ok(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(HRV_ECUDA, "%s launch: %s", what, cudaGetErrorString(e));
  return HRV_OK;
}
static inline unsigned blocks_for(long long total, int bs) { return (unsigned)((total + bs - 1) / bs); }
static inline size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

// Grid of the statistics kernels: blocks per image over HW pixels, PL pixel lanes per block.  Depends on the shapes and the SM
// count only, so the per-block slabs, and the order they are added in, are fixed for a given device and shape.
static unsigned stats_blocks(long long HW, int N, int PL, long long& chunk) {
  long long target_blocks = (long long)sm_count() * 8 / (N > 0 ? N : 1);
  if (target_blocks < 1) target_blocks = 1;
  chunk = (HW + target_blocks - 1) / target_blocks;
  const long long min_chunk = (long long)PL * 16;
  if (chunk < min_chunk) chunk = min_chunk;
  return (unsigned)((HW + chunk - 1) / chunk);
}

}  // namespace hrv

using namespace hrv;

extern "C" size_t hrv_instnorm_stats_workspace_bytes(const hrv_tensor* x0, const hrv_tensor* x1, int32_t h, int32_t w) {
  if (!x0) return 0;
  const int C = x0->c + ((x1 && x1->ptr) ? x1->c : 0);
  const int N = x0->n, G = (C + 7) / 8, PL = G > 0 && G <= 256 ? 256 / G : 1;
  long long chunk;
  const unsigned gx = stats_blocks((long long)h * w, N, PL, chunk);
  return ((size_t)N * C * 2 + (size_t)N * gx * C * 2) * sizeof(double);
}

extern "C" int hrv_instnorm_stats(const hrv_tensor* x0, int32_t x0_shift, const hrv_tensor* x1, int32_t h, int32_t w,
                                  const float* noise, const float* noise_scale, float eps, float* mean, float* rstd,
                                  void* workspace, size_t workspace_bytes, hrv_stream stream) {
  const int dt = storage_of(x0);
  int rc = check_vec(x0, "instnorm_stats x0", dt);
  if (rc) return rc;
  const bool has1 = x1 && x1->ptr;
  if (has1 && (rc = check_vec(x1, "instnorm_stats x1", dt))) return rc;
  const int C = x0->c + (has1 ? x1->c : 0);
  if ((x0->c % 8) || (C % 8)) return set_error(HRV_EINVAL, "instnorm_stats: channel counts must be multiples of 8");
  if (C / 8 > 256) return set_error(HRV_EUNSUPPORTED, "instnorm_stats: more than 2048 channels");
  if ((x0->h << x0_shift) != h || (x0->w << x0_shift) != w) return set_error(HRV_EINVAL, "instnorm_stats: x0 extent mismatch");
  if (has1 && (x1->h != h || x1->w != w || x1->n != x0->n)) return set_error(HRV_EINVAL, "instnorm_stats: x1 extent mismatch");
  const int N = x0->n;
  const size_t need = hrv_instnorm_stats_workspace_bytes(x0, x1, h, w);
  if (!workspace || workspace_bytes < need) return set_error(HRV_EINVAL, "instnorm_stats: workspace too small (%zu < %zu)", workspace_bytes, need);
  cudaStream_t st = (cudaStream_t)stream;
  const int G = C / 8;
  const int PL = 256 / G;
  const long long HW = (long long)h * w;
  long long chunk;
  const unsigned gx = stats_blocks(HW, N, PL, chunk);
  double* acc = (double*)workspace;  // [N][C][2] raw sums, then the blocks' slabs
  double* slab = acc + (size_t)N * C * 2;
  HRV_LAUNCH_STORAGE(dt, instnorm_stats_kernel, dim3(gx, N), 256, (size_t)PL * C * 2 * sizeof(float), st, mk(x0), x0_shift,
                     mk(has1 ? x1 : nullptr), h, w, G, PL, (int)chunk, noise, noise_scale, slab);
  if ((rc = launch_ok("instnorm_stats"))) return rc;
  if ((rc = slab_sum(slab, N, (int)gx, C * 2, acc, C * 2, st, "instnorm_stats sum"))) return rc;
  instnorm_finalize_kernel<<<blocks_for(N * C, 256), 256, 0, st>>>(acc, N * C, 1.0 / (double)HW, eps, mean, rstd);
  return launch_ok("instnorm_finalize");
}

// Workspace of hrv_instnorm_stats2: the sums acc and nzacc, segment 0 (x0) slabs, segment 1 (x1) slabs, segment 0's noise-sum slabs.
static void stats2_plan(const hrv_tensor* x0, const hrv_tensor* x1, unsigned gx[2], long long chunk[2], size_t off[3], size_t& total) {
  const int N = x0->n;
  const bool has1 = x1 && x1->ptr;
  const int C = x0->c + (has1 ? x1->c : 0);
  size_t o = ((size_t)N * C * 4 + (size_t)N * 4) * sizeof(double);  // acc [N][C][4], nzacc [N][4]
  for (int seg = 0; seg < 2; ++seg) {
    gx[seg] = 0;
    chunk[seg] = 0;
    off[seg] = o;
    if (seg == 1 && !has1) continue;
    const hrv_tensor* xs = seg ? x1 : x0;
    const int G = xs->c / 8, PL = G > 0 && G <= 256 ? 256 / G : 1;
    gx[seg] = stats_blocks((long long)xs->h * xs->w, N, PL, chunk[seg]);
    o += (size_t)N * gx[seg] * xs->c * 4 * sizeof(double);
  }
  off[2] = o;
  total = o + (size_t)N * gx[0] * 4 * sizeof(double);
}

extern "C" size_t hrv_instnorm_stats2_workspace_bytes(const hrv_tensor* x0, const hrv_tensor* x1) {
  if (!x0) return 0;
  unsigned gx[2];
  long long chunk[2];
  size_t off[3], total;
  stats2_plan(x0, x1, gx, chunk, off, total);
  return total;
}

extern "C" int hrv_instnorm_stats2(const hrv_tensor* x0, int32_t x0_shift, const hrv_tensor* x1, int32_t h, int32_t w, const float* noise0,
                                   const float* noise_scale0, const float* noise1, const float* noise_scale1, float eps, float* mean0,
                                   float* rstd0, float* mean1, float* rstd1, void* workspace, size_t workspace_bytes, hrv_stream stream) {
  const int dt = storage_of(x0);
  int rc = check_vec(x0, "instnorm_stats2 x0", dt);
  if (rc) return rc;
  const bool has1 = x1 && x1->ptr;
  if (has1 && (rc = check_vec(x1, "instnorm_stats2 x1", dt))) return rc;
  const int C = x0->c + (has1 ? x1->c : 0);
  if ((x0->c % 8) || (C % 8)) return set_error(HRV_EINVAL, "instnorm_stats2: channel counts must be multiples of 8");
  if (x0->c / 8 > 256 || (has1 && x1->c / 8 > 256)) return set_error(HRV_EUNSUPPORTED, "instnorm_stats2: more than 2048 channels per source");
  if (x0_shift < 0 || x0_shift > 1) return set_error(HRV_EINVAL, "instnorm_stats2: x0_shift must be 0 or 1");
  if ((x0->h << x0_shift) != h || (x0->w << x0_shift) != w) return set_error(HRV_EINVAL, "instnorm_stats2: x0 extent mismatch");
  if (x0_shift && (w & 1)) return set_error(HRV_EINVAL, "instnorm_stats2: up-sampled width must be even");
  if (has1 && (x1->h != h || x1->w != w || x1->n != x0->n)) return set_error(HRV_EINVAL, "instnorm_stats2: x1 extent mismatch");
  if (!mean0 || !rstd0 || ((mean1 == nullptr) != (rstd1 == nullptr))) return set_error(HRV_EINVAL, "instnorm_stats2: outputs");
  if ((noise0 && !noise_scale0) || (noise1 && !noise_scale1)) return set_error(HRV_EINVAL, "instnorm_stats2: noise without noise_scale");
  const int N = x0->n;
  unsigned gx[2];
  long long chunk[2];
  size_t off[3], need;
  stats2_plan(x0, x1, gx, chunk, off, need);
  if (!workspace || workspace_bytes < need) return set_error(HRV_EINVAL, "instnorm_stats2: workspace too small (%zu < %zu)", workspace_bytes, need);
  cudaStream_t st = (cudaStream_t)stream;
  char* ws = (char*)workspace;
  double* nzslab = (double*)(ws + off[2]);
  for (int seg = 0; seg < (has1 ? 2 : 1); ++seg) {
    const hrv_tensor* xs = seg ? x1 : x0;
    const int shift = seg ? 0 : x0_shift;
    const int G = xs->c / 8, PL = 256 / G;
    // the noise-only sums are taken once, by the segment that walks the full-resolution grid exactly once per pixel: x0's walk covers
    // every full-resolution pixel through its footprint, so segment 0 always does it
    HRV_LAUNCH_STORAGE(dt, instnorm_stats2_kernel, dim3(gx[seg], N), 256, (size_t)PL * G * 8 * 4 * sizeof(float), st, mk(xs), shift,
                       w, G, PL, (int)chunk[seg], noise0, noise1, (double*)(ws + off[seg]), nzslab, seg == 0);
    if ((rc = launch_ok("instnorm_stats2"))) return rc;
  }
  double* acc = (double*)ws;
  double* nzacc = acc + (size_t)N * C * 4;
  if ((rc = slab_sum((const double*)(ws + off[0]), N, (int)gx[0], x0->c * 4, acc, C * 4, st, "instnorm_stats2 sum"))) return rc;
  if (has1 && (rc = slab_sum((const double*)(ws + off[1]), N, (int)gx[1], x1->c * 4, acc + (size_t)x0->c * 4, C * 4, st, "instnorm_stats2 sum"))) return rc;
  if ((rc = slab_sum(nzslab, N, (int)gx[0], 4, nzacc, 4, st, "instnorm_stats2 noise sum"))) return rc;
  instnorm_finalize2_kernel<<<blocks_for(N * C, 256), 256, 0, st>>>(acc, nzacc, N, C, 1.0 / ((double)h * w), eps, noise0 ? noise_scale0 : nullptr,
                                                                   noise1 ? noise_scale1 : nullptr, mean0, rstd0, mean1, rstd1);
  return launch_ok("instnorm_finalize2");
}

extern "C" int hrv_norm_apply_affine(const hrv_tensor* x, const float* mean, const float* rstd, const float* gamma, const float* beta,
                                     const hrv_tensor* res, int32_t act, const hrv_tensor* y, hrv_stream stream) {
  int rc;
  const int dt = storage_of(x);
  if ((rc = check_vec(x, "norm_apply x", dt)) || (rc = check_vec(y, "norm_apply y", dt))) return rc;
  const bool hr = res && res->ptr;
  if (hr && (rc = check_vec(res, "norm_apply res", dt))) return rc;
  if (!mean || !rstd) return set_error(HRV_EINVAL, "norm_apply: mean/rstd required");
  const int G = (x->c + 7) / 8;
  const long long total = (long long)x->n * x->h * x->w * G;
  HRV_LAUNCH_STORAGE(dt, instnorm_apply_kernel, blocks_for(total, 256), 256, 0, (cudaStream_t)stream, mk(x), mean, rstd, gamma, beta,
                     mk(hr ? res : nullptr), act, mk(y), total, G);
  return launch_ok("norm_apply");
}

extern "C" int hrv_instnorm_apply(const hrv_tensor* x, const float* mean, const float* rstd, int32_t act, const hrv_tensor* y,
                                  hrv_stream stream) {
  return hrv_norm_apply_affine(x, mean, rstd, nullptr, nullptr, nullptr, act, y, stream);
}

extern "C" int hrv_nchw_to_nhwc(const float* src, int32_t c, int32_t src_h, int32_t src_w, const hrv_tensor* dst, hrv_stream stream) {
  const int dt = storage_of(dst);
  int rc = check_vec(dst, "nchw_to_nhwc dst", dt);
  if (rc) return rc;
  const int G = (dst->c + 7) / 8;
  if (G * 8 > dst->pitch) return set_error(HRV_EINVAL, "nchw_to_nhwc: dst pitch too small for padded channels");
  const long long total = (long long)dst->n * dst->h * dst->w * G;
  HRV_LAUNCH_STORAGE(dt, nchw_to_nhwc_kernel, blocks_for(total, 256), 256, 0, (cudaStream_t)stream, src, c, src_h, src_w, mk(dst), G, total);
  return launch_ok("nchw_to_nhwc");
}

extern "C" int hrv_seg_softmax_cat(const float* input1, int32_t c1, const float* input2, int32_t c2, const float* seg, int32_t k,
                                   const float* cm, int32_t cm_channel, int32_t mode, int32_t softmax, const hrv_tensor* dst,
                                   float* seg_out, hrv_stream stream) {
  const int dt = storage_of(dst);
  int rc = check_vec(dst, "seg_softmax_cat dst", dt);
  if (rc) return rc;
  if (!input1 || !input2 || !seg || c1 < 1 || c2 < 1 || k < 1) return set_error(HRV_EINVAL, "seg_softmax_cat: null input or empty operand");
  if (dst->c != c1 + c2 + k) return set_error(HRV_EINVAL, "seg_softmax_cat: dst has %d channels, the operands %d + %d + %d", dst->c, c1, c2, k);
  if (mode < 0 || mode > 2) return set_error(HRV_EINVAL, "seg_softmax_cat: mode must be 0 (none), 1 (multiply by cm) or 2 (by cm > 0.5)");
  if (mode != 0 && (!cm || cm_channel < 0 || cm_channel >= k))
    return set_error(HRV_EINVAL, "seg_softmax_cat: mode %d needs cm and 0 <= cm_channel < %d", mode, k);
  const int G = (dst->c + 7) / 8;
  if (G * 8 > dst->pitch) return set_error(HRV_EINVAL, "seg_softmax_cat: dst pitch too small for padded channels");
  SegCatSrc S{input1, input2, seg, cm, c1, c2, k, mode != 0 ? cm_channel : -1, mode, softmax ? 1 : 0};
  const long long npix = (long long)dst->n * dst->h * dst->w;
  HRV_LAUNCH_STORAGE(dt, seg_softmax_cat_kernel, blocks_for(npix, 128), 128, 0, (cudaStream_t)stream, S, mk(dst), seg_out, G, npix);
  return launch_ok("seg_softmax_cat");
}

static int seg_iou_blocks(long long hw) {
  const long long b = (hw + SEG_IOU_THREADS - 1) / SEG_IOU_THREADS;
  return b < SEG_IOU_MAX_BLOCKS ? (int)b : SEG_IOU_MAX_BLOCKS;
}

extern "C" size_t hrv_seg_iou_workspace_bytes(int32_t n, int32_t h, int32_t w) {
  if (n < 1 || h < 1 || w < 1) return 0;
  return (size_t)n * seg_iou_blocks((long long)h * w) * SEG_IOU_WARPS * sizeof(int4);
}

extern "C" int hrv_seg_iou(const float* seg, int32_t k, const float* cm, const float* parse, int32_t n, int32_t h, int32_t w, float* iou,
                           void* workspace, size_t workspace_bytes, hrv_stream stream) {
  if (!seg || !cm || !parse || !iou) return set_error(HRV_EINVAL, "seg_iou: null argument");
  if (n < 1 || h < 1 || w < 1 || k <= SEG_IOU_CM_CHANNEL)
    return set_error(HRV_EINVAL, "seg_iou: need n, h, w >= 1 and k > %d (the composed cloth channel), got n=%d h=%d w=%d k=%d",
                     SEG_IOU_CM_CHANNEL, n, h, w, k);
  const long long hw = (long long)h * w;
  if ((long long)k * hw > 0x7fffffffLL) return set_error(HRV_EINVAL, "seg_iou: %d x %lld labels per sample overflow the int32 counts", k, hw);
  const size_t need = hrv_seg_iou_workspace_bytes(n, h, w);
  if (!workspace || workspace_bytes < need) return set_error(HRV_EINVAL, "seg_iou: workspace too small (%zu < %zu)", workspace_bytes, need);
  const int blocks = seg_iou_blocks(hw);
  cudaStream_t st = (cudaStream_t)stream;
  seg_iou_count_kernel<<<dim3(blocks, n), SEG_IOU_THREADS, 0, st>>>(seg, cm, parse, k, hw, (int4*)workspace);
  int rc = launch_ok("seg_iou");
  if (rc) return rc;
  seg_iou_finish_kernel<<<1, 32, 0, st>>>((const int4*)workspace, blocks * SEG_IOU_WARPS, n, iou);
  return launch_ok("seg_iou finish");
}

extern "C" int hrv_nhwc_to_nchw(const hrv_tensor* src, float* dst, hrv_stream stream) {
  if (!src || !src->ptr || !dst) return set_error(HRV_EINVAL, "nhwc_to_nchw: null");
  const long long npix = (long long)src->n * src->h * src->w;
  nhwc_to_nchw_kernel<<<blocks_for(npix, 256), 256, 0, (cudaStream_t)stream>>>(mk(src), dst, npix);
  return launch_ok("nhwc_to_nchw");
}

extern "C" int hrv_space_to_depth(const hrv_tensor* src, const hrv_tensor* dst, hrv_stream stream) {
  int rc;
  const int dt = storage_of(src);
  if ((rc = check_vec(src, "s2d src", dt)) || (rc = check_vec(dst, "s2d dst", dt))) return rc;
  const int G = (src->c + 7) / 8;
  if (dst->h != (src->h + 1) / 2 || dst->w != (src->w + 1) / 2 || dst->c < 4 * G * 8 || (dst->c % 8))
    return set_error(HRV_EINVAL, "s2d: dst must be ceil(h/2) x ceil(w/2) x (>= 4*roundup8(c))");
  const int Gd = dst->c / 8;
  const long long total = (long long)dst->n * dst->h * dst->w * Gd;
  HRV_LAUNCH_STORAGE(dt, space_to_depth_kernel, blocks_for(total, 256), 256, 0, (cudaStream_t)stream, mk(src), mk(dst), G, Gd, total);
  return launch_ok("space_to_depth");
}

extern "C" int hrv_avgpool3s2(const hrv_tensor* src, const hrv_tensor* dst, hrv_stream stream) {
  int rc;
  const int dt = storage_of(src);
  if ((rc = check_vec(src, "avgpool src", dt)) || (rc = check_vec(dst, "avgpool dst", dt))) return rc;
  if (dst->h != (src->h - 1) / 2 + 1 || dst->w != (src->w - 1) / 2 + 1) return set_error(HRV_EINVAL, "avgpool: dst extent");
  const int G = (src->c + 7) / 8;
  const long long total = (long long)dst->n * dst->h * dst->w * G;
  HRV_LAUNCH_STORAGE(dt, avgpool3s2_kernel, blocks_for(total, 256), 256, 0, (cudaStream_t)stream, mk(src), mk(dst), G, total);
  return launch_ok("avgpool3s2");
}

extern "C" int hrv_bilinear_up2_add(const hrv_tensor* a, const hrv_tensor* b, const hrv_tensor* dst, hrv_stream stream) {
  int rc;
  const int dt = storage_of(a);
  if ((rc = check_vec(a, "up2 a", dt)) || (rc = check_vec(dst, "up2 dst", dt))) return rc;
  const bool hb = b && b->ptr;
  if (hb && (rc = check_vec(b, "up2 b", dt))) return rc;
  if (dst->h != 2 * a->h || dst->w != 2 * a->w) return set_error(HRV_EINVAL, "up2: dst must be 2x");
  const int G = (a->c + 7) / 8;
  const long long total = (long long)dst->n * dst->h * dst->w * G;
  HRV_LAUNCH_STORAGE(dt, bilinear_up2_add_kernel, blocks_for(total, 256), 256, 0, (cudaStream_t)stream, mk(a), mk(hb ? b : nullptr), mk(dst), G, total);
  return launch_ok("bilinear_up2_add");
}

extern "C" int hrv_flow_warp(const float* flow_lo, const float* lin_x, const float* lin_y, const hrv_tensor* src, const hrv_tensor* dst,
                             float* flow_up, int32_t* idx_out, hrv_stream stream) {
  if (!flow_lo || !lin_x || !lin_y || !src || !dst || !src->ptr || !dst->ptr) return set_error(HRV_EINVAL, "flow_warp: null argument");
  if ((dst->h & 1) || (dst->w & 1)) return set_error(HRV_EINVAL, "flow_warp: output extent must be even");
  if (src->dtype == HRV_BF16 && (((uintptr_t)src->ptr & 15) || (src->pitch % 8))) return set_error(HRV_EINVAL, "flow_warp: src alignment");
  if (dst->dtype == HRV_BF16 && (((uintptr_t)dst->ptr & 15) || (dst->pitch % 8))) return set_error(HRV_EINVAL, "flow_warp: dst alignment");
  if (src->n != dst->n || src->c != dst->c) return set_error(HRV_EINVAL, "flow_warp: src/dst mismatch");
  const int G = (src->c + 7) / 8;
  const long long total = (long long)dst->n * dst->h * dst->w * G;
  // Python-float arithmetic of the reference ((iW/2 - 1.0)/2.0), rounded once to fp32 as torch does for a scalar divisor
  const float sx = (float)((dst->w / 2.0 - 1.0) / 2.0);
  const float sy = (float)((dst->h / 2.0 - 1.0) / 2.0);
  flow_warp_kernel<<<blocks_for(total, 256), 256, 0, (cudaStream_t)stream>>>(flow_lo, lin_x, lin_y, mk(src), mk(dst), flow_up, idx_out, sx, sy, G, total);
  return launch_ok("flow_warp");
}

// ------------------------------------------------------------------------------------------------ backward of the resampling ops
namespace hrv {

// Adjoint of F.interpolate(bilinear, x2, align_corners=False) along one axis: low-res index i receives from high-res
// d in {2i-1, 2i, 2i+1, 2i+2} with weights {0.25, 0.75, 0.75, 0.25}; the clamped border taps fold onto i (weights 1.0).
__device__ __forceinline__ void up2_adj(int i, int n, float (&wt)[4]) {
  wt[0] = i >= 1 ? 0.25f : 0.f;
  wt[1] = i == 0 ? 1.0f : 0.75f;
  wt[2] = i == n - 1 ? 1.0f : 0.75f;
  wt[3] = i <= n - 2 ? 0.25f : 0.f;
}

// thread = (low-res pixel, 8-channel group): da[n,y,x,:] = sum over the 4x4 high-res neighbourhood of wy*wx*dout
__global__ void bilinear_up2_bwd_kernel(View dout, View da, int G, long long total) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int g = (int)(idx % G);
  const long long pix = idx / G;
  const int x = (int)(pix % da.w);
  const int y = (int)((pix / da.w) % da.h);
  const int n = (int)(pix / ((long long)da.w * da.h));
  float wy[4], wx[4], acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  up2_adj(y, da.h, wy);
  up2_adj(x, da.w, wx);
  const __nv_bfloat16* base = reinterpret_cast<const __nv_bfloat16*>(dout.ptr) + (long long)n * dout.h * dout.w * dout.pitch + g * 8;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int Y = 2 * y - 1 + j;
    if (wy[j] == 0.f || Y < 0 || Y >= dout.h) continue;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int X = 2 * x - 1 + i;
      if (wx[i] == 0.f || X < 0 || X >= dout.w) continue;
      float f[8];
      unpack8(ldg16(base + ((long long)Y * dout.w + X) * dout.pitch), f);
      const float w = wy[j] * wx[i];
#pragma unroll
      for (int k = 0; k < 8; ++k) acc[k] = fmaf(w, f[k], acc[k]);
    }
  }
  *reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(const_cast<void*>(da.ptr)) + pix * da.pitch + g * 8) = pack8(acc);
}

// Backward of flow_warp_kernel.  thread = (dst pixel, 8-channel group): recomputes the sampling coordinates exactly as the
// forward, scatter-adds d_dst * w into d_src (fp32 accumulation buffer, atomics: the gather is irregular) and accumulates the
// analytic coordinate gradient (grid_sample border semantics: zero where the coordinate was clamped) into d_flow_up (fp32).
__global__ void flow_warp_bwd_kernel(const float* __restrict__ flow_lo, const float* __restrict__ lin_x, const float* __restrict__ lin_y,
                                     View src, View ddst, float* __restrict__ dsrc32, float* __restrict__ dflow_up, float sx, float sy,
                                     int G, long long total) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int g = (int)(idx % G);
  const long long pix = idx / G;
  const int W = ddst.w, H = ddst.h;
  const int x = (int)(pix % W);
  const int y = (int)((pix / W) % H);
  const int n = (int)(pix / ((long long)W * H));
  const int hl = H >> 1, wl = W >> 1;
  int xa, xb, ya, yb;
  float wxa, wxb, wya, wyb;
  up2_taps(x, wl, xa, xb, wxa, wxb);
  up2_taps(y, hl, ya, yb, wya, wyb);
  const float2* fl = reinterpret_cast<const float2*>(flow_lo) + (long long)n * hl * wl;
  const float2 f00 = __ldg(fl + (long long)ya * wl + xa), f01 = __ldg(fl + (long long)ya * wl + xb);
  const float2 f10 = __ldg(fl + (long long)yb * wl + xa), f11 = __ldg(fl + (long long)yb * wl + xb);
  const float fx = __fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(f00.x, wxa), __fmul_rn(f01.x, wxb)), wya), __fmul_rn(__fadd_rn(__fmul_rn(f10.x, wxa), __fmul_rn(f11.x, wxb)), wyb));
  const float fy = __fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(f00.y, wxa), __fmul_rn(f01.y, wxb)), wya), __fmul_rn(__fadd_rn(__fmul_rn(f10.y, wxa), __fmul_rn(f11.y, wxb)), wyb));
  const float gx = __fadd_rn(__fdiv_rn(fx, sx), __ldg(lin_x + x));
  const float gy = __fadd_rn(__fdiv_rn(fy, sy), __ldg(lin_y + y));
  const float ixr = __fdiv_rn(__fsub_rn(__fmul_rn(__fadd_rn(gx, 1.f), (float)src.w), 1.f), 2.f);
  const float iyr = __fdiv_rn(__fsub_rn(__fmul_rn(__fadd_rn(gy, 1.f), (float)src.h), 1.f), 2.f);
  const float ix = fminf(fmaxf(ixr, 0.f), (float)(src.w - 1)), iy = fminf(fmaxf(iyr, 0.f), (float)(src.h - 1));
  // clip_coordinates_set_grad: a coordinate ON the border counts as clamped too (torch: in <= 0 or in >= size-1 -> zero gradient)
  const float mx = (ixr <= 0.f || ixr >= (float)(src.w - 1)) ? 0.f : 1.f;
  const float my = (iyr <= 0.f || iyr >= (float)(src.h - 1)) ? 0.f : 1.f;
  const float fx0 = floorf(ix), fy0 = floorf(iy);
  const int x0 = (int)fx0, y0 = (int)fy0;
  const float tx = ix - fx0, ty = iy - fy0;
  const bool vx = x0 + 1 <= src.w - 1, vy = y0 + 1 <= src.h - 1;
  const int x1 = vx ? x0 + 1 : x0, y1 = vy ? y0 + 1 : y0;
  const float wx1 = vx ? tx : 0.f, wy1 = vy ? ty : 0.f, wx0 = 1.f - tx, wy0 = 1.f - ty;
  if (g * 8 >= ((src.c + 7) & ~7)) return;
  float d[8], a[8], b[8], c[8], e[8];
  unpack8(ldg16(reinterpret_cast<const __nv_bfloat16*>(ddst.ptr) + pix * ddst.pitch + g * 8), d);
  const long long ib = (long long)n * src.h * src.w;
  const __nv_bfloat16* sp = reinterpret_cast<const __nv_bfloat16*>(src.ptr) + g * 8;
  unpack8(ldg16(sp + (ib + (long long)y0 * src.w + x0) * src.pitch), a);
  unpack8(ldg16(sp + (ib + (long long)y0 * src.w + x1) * src.pitch), b);
  unpack8(ldg16(sp + (ib + (long long)y1 * src.w + x0) * src.pitch), c);
  unpack8(ldg16(sp + (ib + (long long)y1 * src.w + x1) * src.pitch), e);
  float dix = 0.f, diy = 0.f;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    // value = a*wy0*wx0 + b*wy0*wx1 + c*wy1*wx0 + e*wy1*wx1 ; taps outside the image carry zero weight AND zero derivative
    const float bb = vx ? b[k] : 0.f, cc = vy ? c[k] : 0.f, ee = (vx && vy) ? e[k] : 0.f;
    dix += d[k] * ((bb - a[k]) * wy0 + (ee - cc) * (vy ? ty : 0.f));
    diy += d[k] * ((cc - a[k]) * wx0 + (ee - bb) * (vx ? tx : 0.f));
  }
  if (dflow_up) {
    // d ix / d gx = src.w/2 ; d gx / d flow_up.x = 1/sx
    atomicAdd(dflow_up + pix * 2, dix * mx * (0.5f * (float)src.w) / sx);
    atomicAdd(dflow_up + pix * 2 + 1, diy * my * (0.5f * (float)src.h) / sy);
  }
  if (dsrc32) {
    const int cs = (src.c + 7) & ~7;
    float* o00 = dsrc32 + (ib + (long long)y0 * src.w + x0) * cs + g * 8;
    float* o01 = dsrc32 + (ib + (long long)y0 * src.w + x1) * cs + g * 8;
    float* o10 = dsrc32 + (ib + (long long)y1 * src.w + x0) * cs + g * 8;
    float* o11 = dsrc32 + (ib + (long long)y1 * src.w + x1) * cs + g * 8;
    const float w00 = wy0 * wx0, w01 = wy0 * wx1, w10 = wy1 * wx0, w11 = wy1 * wx1;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      atomicAdd(o00 + k, d[k] * w00);
      if (w01 != 0.f) atomicAdd(o01 + k, d[k] * w01);
      if (w10 != 0.f) atomicAdd(o10 + k, d[k] * w10);
      if (w11 != 0.f) atomicAdd(o11 + k, d[k] * w11);
    }
  }
}

// d_flow_lo[n,y,x,:] = adjoint of the x2 bilinear up-sampling applied to d_flow_up (2 fp32 channels)
__global__ void flow_up2_bwd_kernel(const float* __restrict__ dup, float* __restrict__ dlo, int N, int hl, int wl) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long total = (long long)N * hl * wl;
  if (idx >= total) return;
  const int x = (int)(idx % wl), y = (int)((idx / wl) % hl), n = (int)(idx / ((long long)wl * hl));
  float wy[4], wx[4], ax = 0.f, ay = 0.f;
  up2_adj(y, hl, wy);
  up2_adj(x, wl, wx);
  const int H = 2 * hl, W = 2 * wl;
  const float2* src = reinterpret_cast<const float2*>(dup) + (long long)n * H * W;
  for (int j = 0; j < 4; ++j) {
    const int Y = 2 * y - 1 + j;
    if (wy[j] == 0.f || Y < 0 || Y >= H) continue;
    for (int i = 0; i < 4; ++i) {
      const int X = 2 * x - 1 + i;
      if (wx[i] == 0.f || X < 0 || X >= W) continue;
      const float2 v = __ldg(src + (long long)Y * W + X);
      ax = fmaf(wy[j] * wx[i], v.x, ax);
      ay = fmaf(wy[j] * wx[i], v.y, ay);
    }
  }
  reinterpret_cast<float2*>(dlo)[idx] = make_float2(ax, ay);
}

// ---- ordered backward of flow_warp_kernel: d_src as a gather in a fixed order, d_flow_up without atomics.
// Pass 1, thread = (dst pixel p, 8-channel group g): recomputes the taps (warp_taps) and writes the group's share of the coordinate
// gradient to part[p][g]; the g == 0 thread also writes one sort entry per tap: key = source pixel index within the batch (the
// sentinel S = N*Hs*Ws for a zero-weight tap, so it sorts last), value = 4*p + tap, weight wts[4*p + tap].
__global__ void flow_warp_bwd_entries_kernel(const float* __restrict__ flow_lo, const float* __restrict__ lin_x, const float* __restrict__ lin_y,
                                             View src, View ddst, float sx, float sy, int G, long long total, unsigned* __restrict__ keys,
                                             unsigned* __restrict__ vals, float* __restrict__ wts, float2* __restrict__ part) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int g = (int)(idx % G);
  const long long pix = idx / G;
  const int W = ddst.w, H = ddst.h;
  const int x = (int)(pix % W);
  const int y = (int)((pix / W) % H);
  const int n = (int)(pix / ((long long)W * H));
  const WarpTaps t = warp_taps(flow_lo, lin_x, lin_y, n, x, y, H, W, src.h, src.w, sx, sy);
  const long long ib = (long long)n * src.h * src.w;
  if (keys && g == 0) {
    const unsigned sentinel = (unsigned)((long long)src.n * src.h * src.w);
    const long long tap_pix[4] = {ib + (long long)t.y0 * src.w + t.x0, ib + (long long)t.y0 * src.w + t.x1,
                                  ib + (long long)t.y1 * src.w + t.x0, ib + (long long)t.y1 * src.w + t.x1};
    const float w[4] = {t.wy0 * t.wx0, t.wy0 * t.wx1, t.wy1 * t.wx0, t.wy1 * t.wx1};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const long long e = 4 * pix + k;
      keys[e] = w[k] != 0.f ? (unsigned)tap_pix[k] : sentinel;
      vals[e] = (unsigned)e;
      wts[e] = w[k];
    }
  }
  if (!part) return;
  const float mx = (t.ixr <= 0.f || t.ixr >= (float)(src.w - 1)) ? 0.f : 1.f;
  const float my = (t.iyr <= 0.f || t.iyr >= (float)(src.h - 1)) ? 0.f : 1.f;
  float d[8], a[8], b[8], c[8], e[8];
  unpack8(ldg16(reinterpret_cast<const __nv_bfloat16*>(ddst.ptr) + pix * ddst.pitch + g * 8), d);
  const __nv_bfloat16* sp = reinterpret_cast<const __nv_bfloat16*>(src.ptr) + g * 8;
  unpack8(ldg16(sp + (ib + (long long)t.y0 * src.w + t.x0) * src.pitch), a);
  unpack8(ldg16(sp + (ib + (long long)t.y0 * src.w + t.x1) * src.pitch), b);
  unpack8(ldg16(sp + (ib + (long long)t.y1 * src.w + t.x0) * src.pitch), c);
  unpack8(ldg16(sp + (ib + (long long)t.y1 * src.w + t.x1) * src.pitch), e);
  float dix = 0.f, diy = 0.f;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    // value = a*wy0*wx0 + b*wy0*wx1 + c*wy1*wx0 + e*wy1*wx1 ; taps outside the image carry zero weight AND zero derivative
    const float bb = t.vx ? b[k] : 0.f, cc = t.vy ? c[k] : 0.f, ee = (t.vx && t.vy) ? e[k] : 0.f;
    dix += d[k] * ((bb - a[k]) * t.wy0 + (ee - cc) * t.wy1);
    diy += d[k] * ((cc - a[k]) * t.wx0 + (ee - bb) * t.wx1);
  }
  // d ix / d gx = src.w/2 ; d gx / d flow_up.x = 1/sx
  part[pix * G + g] = make_float2(dix * mx * (0.5f * (float)src.w) / sx, diy * my * (0.5f * (float)src.h) / sy);
}

// Pass 2, thread = dst pixel: dflow_up += the groups' partials, added in ascending group order.
__global__ void flow_warp_bwd_dflow_kernel(const float2* __restrict__ part, float2* __restrict__ dflow_up, int G, long long npix) {
  const long long pix = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= npix) return;
  float2 v = dflow_up[pix];
  for (int g = 0; g < G; ++g) {
    const float2 q = __ldg(part + pix * G + g);
    v.x = __fadd_rn(v.x, q.x);
    v.y = __fadd_rn(v.y, q.y);
  }
  dflow_up[pix] = v;
}

// Pass 3 (after the stable radix sort by key), thread = source pixel s in [0, S]: begin[s] = first sorted entry with key >= s.
__global__ void flow_warp_bwd_bounds_kernel(const unsigned* __restrict__ keys, long long m, unsigned* __restrict__ begin, long long S) {
  const long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (s > S) return;
  long long lo = 0, hi = m;
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    if ((long long)__ldg(keys + mid) < s) lo = mid + 1;
    else hi = mid;
  }
  begin[s] = (unsigned)lo;
}

// Pass 4, thread = (source pixel s, 8-channel group g): dsrc32[s] = sum of d_dst[p] * w over s's entries in ascending
// (dst pixel, tap) order — the stable sort kept that order.  __fmul_rn / __fadd_rn forbid FMA contraction, so the result equals a
// sequential fp32 sum in that order bit for bit.
__global__ void flow_warp_bwd_gather_kernel(View ddst, const unsigned* __restrict__ begin, const unsigned* __restrict__ vals,
                                            const float* __restrict__ wts, float* __restrict__ dsrc32, int G, long long total) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int g = (int)(idx % G);
  const long long s = idx / G;
  const unsigned b = __ldg(begin + s), e = __ldg(begin + s + 1);
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  const __nv_bfloat16* dp = reinterpret_cast<const __nv_bfloat16*>(ddst.ptr) + g * 8;
  for (unsigned i = b; i < e; ++i) {
    const unsigned v = __ldg(vals + i);
    const float w = __ldg(wts + v);
    float d[8];
    unpack8(ldg16(dp + (long long)(v >> 2) * ddst.pitch), d);
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[k] = __fadd_rn(acc[k], __fmul_rn(d[k], w));
  }
  float4* o = reinterpret_cast<float4*>(dsrc32 + s * (long long)G * 8 + g * 8);
  o[0] = make_float4(acc[0], acc[1], acc[2], acc[3]);
  o[1] = make_float4(acc[4], acc[5], acc[6], acc[7]);
}

// Workspace of hrv_flow_warp_bwd_ordered, 256-byte aligned pieces.
struct WarpBwdPlan {
  long long m, S, npix;
  int G, end_bit;
  size_t keys_in, keys_out, vals_in, vals_out, wts, begin, part, temp, temp_bytes, total;
};
static int warp_bwd_plan(const hrv_tensor* src, const hrv_tensor* ddst, WarpBwdPlan& p) {
  p.npix = (long long)ddst->n * ddst->h * ddst->w;
  p.m = 4 * p.npix;
  p.S = (long long)src->n * src->h * src->w;
  p.G = (src->c + 7) / 8;
  p.end_bit = log2i((int)(p.S + 1));
  if (p.end_bit < 1) p.end_bit = 1;
  p.temp_bytes = 0;
  cudaError_t e = cub::DeviceRadixSort::SortPairs(nullptr, p.temp_bytes, (const unsigned*)nullptr, (unsigned*)nullptr, (const unsigned*)nullptr,
                                                  (unsigned*)nullptr, (int)p.m, 0, p.end_bit);
  if (e != cudaSuccess) return set_error(HRV_ECUDA, "flow_warp_bwd_ordered: sort size query: %s", cudaGetErrorString(e));
  size_t o = 0;
  const size_t ent = align256((size_t)p.m * 4);
  p.keys_in = o; o += ent;
  p.keys_out = o; o += ent;
  p.vals_in = o; o += ent;
  p.vals_out = o; o += ent;
  p.wts = o; o += ent;
  p.begin = o; o += align256((size_t)(p.S + 1) * 4);
  p.part = o; o += align256((size_t)p.npix * p.G * sizeof(float2));
  p.temp = o; o += align256(p.temp_bytes);
  p.total = o;
  return HRV_OK;
}

}  // namespace hrv

extern "C" int hrv_bilinear_up2_bwd(const hrv_tensor* dout, const hrv_tensor* da, hrv_stream stream) {
  int rc;
  if ((rc = check_bf16_vec(dout, "up2_bwd dout")) || (rc = check_bf16_vec(da, "up2_bwd da"))) return rc;
  if (dout->h != 2 * da->h || dout->w != 2 * da->w) return set_error(HRV_EINVAL, "up2_bwd: dout must be 2x da");
  const int G = (da->c + 7) / 8;
  const long long total = (long long)da->n * da->h * da->w * G;
  bilinear_up2_bwd_kernel<<<blocks_for(total, 256), 256, 0, (cudaStream_t)stream>>>(mk(dout), mk(da), G, total);
  return launch_ok("bilinear_up2_bwd");
}

extern "C" int hrv_flow_warp_bwd(const float* flow_lo, const float* lin_x, const float* lin_y, const hrv_tensor* src, const hrv_tensor* ddst,
                                 float* dsrc32, float* dflow_up, float* dflow_lo, hrv_stream stream) {
  int rc;
  if (!flow_lo || !lin_x || !lin_y) return set_error(HRV_EINVAL, "flow_warp_bwd: null argument");
  if ((rc = check_bf16_vec(src, "flow_warp_bwd src")) || (rc = check_bf16_vec(ddst, "flow_warp_bwd ddst"))) return rc;
  if ((ddst->h & 1) || (ddst->w & 1) || src->n != ddst->n || src->c != ddst->c) return set_error(HRV_EINVAL, "flow_warp_bwd: shape mismatch");
  if (dflow_lo && !dflow_up) return set_error(HRV_EINVAL, "flow_warp_bwd: dflow_lo needs the dflow_up scratch buffer");
  const int G = (src->c + 7) / 8;
  const long long total = (long long)ddst->n * ddst->h * ddst->w * G;
  const float sx = (float)((ddst->w / 2.0 - 1.0) / 2.0), sy = (float)((ddst->h / 2.0 - 1.0) / 2.0);
  cudaStream_t st = (cudaStream_t)stream;
  flow_warp_bwd_kernel<<<blocks_for(total, 256), 256, 0, st>>>(flow_lo, lin_x, lin_y, mk(src), mk(ddst), dsrc32, dflow_up, sx, sy, G, total);
  if ((rc = launch_ok("flow_warp_bwd"))) return rc;
  if (dflow_lo) {
    const long long tl = (long long)ddst->n * (ddst->h / 2) * (ddst->w / 2);
    flow_up2_bwd_kernel<<<blocks_for(tl, 256), 256, 0, st>>>(dflow_up, dflow_lo, ddst->n, ddst->h / 2, ddst->w / 2);
    return launch_ok("flow_up2_bwd");
  }
  return HRV_OK;
}

extern "C" size_t hrv_flow_warp_bwd_ordered_workspace_bytes(const hrv_tensor* src, const hrv_tensor* ddst) {
  if (!src || !ddst) return 0;
  WarpBwdPlan p;
  return warp_bwd_plan(src, ddst, p) ? 0 : p.total;
}

extern "C" int hrv_flow_warp_bwd_ordered(const float* flow_lo, const float* lin_x, const float* lin_y, const hrv_tensor* src,
                                         const hrv_tensor* ddst, float* dsrc32, float* dflow_up, float* dflow_lo, void* workspace,
                                         size_t workspace_bytes, hrv_stream stream) {
  int rc;
  if (!flow_lo || !lin_x || !lin_y) return set_error(HRV_EINVAL, "flow_warp_bwd_ordered: null argument");
  if ((rc = check_bf16_vec(src, "flow_warp_bwd_ordered src")) || (rc = check_bf16_vec(ddst, "flow_warp_bwd_ordered ddst"))) return rc;
  if ((ddst->h & 1) || (ddst->w & 1) || src->n != ddst->n || src->c != ddst->c) return set_error(HRV_EINVAL, "flow_warp_bwd_ordered: shape mismatch");
  if (dflow_lo && !dflow_up) return set_error(HRV_EINVAL, "flow_warp_bwd_ordered: dflow_lo needs the dflow_up buffer");
  if (((uintptr_t)dsrc32 & 15)) return set_error(HRV_EINVAL, "flow_warp_bwd_ordered: dsrc32 needs 16-byte alignment");
  WarpBwdPlan p;
  if ((rc = warp_bwd_plan(src, ddst, p))) return rc;
  if (p.m >= (1LL << 32) || p.S >= (1LL << 31)) return set_error(HRV_EUNSUPPORTED, "flow_warp_bwd_ordered: more than 2^30 destination pixels");
  if (!workspace || workspace_bytes < p.total)
    return set_error(HRV_EINVAL, "flow_warp_bwd_ordered: workspace too small (%zu < %zu)", workspace_bytes, p.total);
  if (!dsrc32 && !dflow_up) return HRV_OK;
  char* ws = (char*)workspace;
  unsigned* keys_in = (unsigned*)(ws + p.keys_in);
  unsigned* keys_out = (unsigned*)(ws + p.keys_out);
  unsigned* vals_in = (unsigned*)(ws + p.vals_in);
  unsigned* vals_out = (unsigned*)(ws + p.vals_out);
  float* wts = (float*)(ws + p.wts);
  unsigned* begin = (unsigned*)(ws + p.begin);
  float2* part = (float2*)(ws + p.part);
  const float sx = (float)((ddst->w / 2.0 - 1.0) / 2.0), sy = (float)((ddst->h / 2.0 - 1.0) / 2.0);
  cudaStream_t st = (cudaStream_t)stream;
  const long long total = p.npix * p.G;
  flow_warp_bwd_entries_kernel<<<blocks_for(total, 256), 256, 0, st>>>(flow_lo, lin_x, lin_y, mk(src), mk(ddst), sx, sy, p.G, total,
                                                                       dsrc32 ? keys_in : nullptr, vals_in, wts, dflow_up ? part : nullptr);
  if ((rc = launch_ok("flow_warp_bwd_entries"))) return rc;
  if (dflow_up) {
    flow_warp_bwd_dflow_kernel<<<blocks_for(p.npix, 256), 256, 0, st>>>(part, (float2*)dflow_up, p.G, p.npix);
    if ((rc = launch_ok("flow_warp_bwd_dflow"))) return rc;
  }
  if (dsrc32) {
    size_t tb = p.temp_bytes;
    cudaError_t e = cub::DeviceRadixSort::SortPairs(ws + p.temp, tb, keys_in, keys_out, vals_in, vals_out, (int)p.m, 0, p.end_bit, st);
    if (e != cudaSuccess) return set_error(HRV_ECUDA, "flow_warp_bwd_ordered sort: %s", cudaGetErrorString(e));
    flow_warp_bwd_bounds_kernel<<<blocks_for(p.S + 1, 256), 256, 0, st>>>(keys_out, p.m, begin, p.S);
    if ((rc = launch_ok("flow_warp_bwd_bounds"))) return rc;
    flow_warp_bwd_gather_kernel<<<blocks_for(p.S * p.G, 256), 256, 0, st>>>(mk(ddst), begin, vals_out, wts, dsrc32, p.G, p.S * p.G);
    if ((rc = launch_ok("flow_warp_bwd_gather"))) return rc;
  }
  if (dflow_lo) {
    const long long tl = (long long)ddst->n * (ddst->h / 2) * (ddst->w / 2);
    flow_up2_bwd_kernel<<<blocks_for(tl, 256), 256, 0, st>>>(dflow_up, dflow_lo, ddst->n, ddst->h / 2, ddst->w / 2);
    return launch_ok("flow_up2_bwd");
  }
  return HRV_OK;
}

// ------------------------------------------------------------------------------------------------ weight packing
namespace hrv {
// One pass from the fp32 parameter layout (cout,cin,kh,kw) to the GEMM layout [taps][n_pad][cin_k] (zero padded), with optional
// 1/sigma scaling, (gamma,beta) row interleave of two parameters and the flip+transpose of the data-gradient convolution.
// kSplit = false: one plane of the flavour's 16-bit type.  kSplit = true (the 3xTF32 convolution of fp32 storage): fp32 planes
// hi = rna_tf32(v) at [0][taps][n_pad][cin_k] and lo = rna_tf32(v - hi) at [1][taps][n_pad][cin_k].
template <bool kSplit, typename D>
__global__ void pack_conv_weight_kernel(const float* __restrict__ w0, const float* __restrict__ w1, int cout, int cin, int kh, int kw,
                                        int transpose_flip, const float* __restrict__ inv_scale, D* __restrict__ dst,
                                        int n_pad, int cin_k, long long plane) {
  // thread = one (row n, K index c) of the GEMM operand; it walks the kh*kw taps, i.e. reads the taps of one (co,ci) pair from
  // CONTIGUOUS fp32 memory and writes one element per tap plane (coalesced across the threads of a warp, which vary c).
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= plane) return;
  const int c = (int)(idx % cin_k);
  const int n = (int)(idx / cin_k);
  const int inter = w1 ? 2 : 1;
  const int taps = kh * kw;
  const float* src = nullptr;
  if (!transpose_flip) {
    // GEMM row n = output channel (interleaved pair index), K index c = input channel
    if (n < cout * inter && c < cin) src = ((w1 && (n & 1)) ? w1 : w0) + ((long long)(n / inter) * cin + c) * taps;
  } else {
    // data-gradient conv: GEMM row n = original INPUT channel, K index c = original OUTPUT channel (interleaved), taps mirrored
    if (n < cin && c < cout * inter) src = ((w1 && (c & 1)) ? w1 : w0) + ((long long)(c / inter) * cin + n) * taps;
  }
  const float sc = inv_scale ? __ldg(inv_scale) : 1.f;
  for (int tap = 0; tap < taps; ++tap) {
    const float v = src ? __ldg(src + (transpose_flip ? taps - 1 - tap : tap)) * sc : 0.f;
    if constexpr (kSplit) {
      const float hi = rna_tf32(v);
      dst[(long long)tap * plane + idx] = hi;
      dst[(long long)(taps + tap) * plane + idx] = rna_tf32(v - hi);
    } else {
      dst[(long long)tap * plane + idx] = __float2bfloat16(v);
    }
  }
}
}  // namespace hrv

extern "C" int hrv_pack_conv_weight(const float* w0, const float* w1, int32_t cout, int32_t cin, int32_t kh, int32_t kw,
                                    int32_t transpose_flip, const float* inv_scale, void* dst, int32_t n_pad, int32_t cin_k,
                                    hrv_stream stream) {
  if (!w0 || !dst || cout < 1 || cin < 1 || kh < 1 || kw < 1) return set_error(HRV_EINVAL, "pack_conv_weight: bad arguments");
  const int inter = w1 ? 2 : 1;
  const int rows = transpose_flip ? cin : cout * inter, cols = transpose_flip ? cout * inter : cin;
  if (n_pad < rows || cin_k < cols) return set_error(HRV_EINVAL, "pack_conv_weight: destination too small (%d x %d for %d x %d)", n_pad, cin_k, rows, cols);
  const long long plane = (long long)n_pad * cin_k;
  pack_conv_weight_kernel<false><<<blocks_for(plane, 256), 256, 0, (cudaStream_t)stream>>>(w0, w1, cout, cin, kh, kw, transpose_flip, inv_scale,
                                                                                          (__nv_bfloat16*)dst, n_pad, cin_k, plane);
  return launch_ok("pack_conv_weight");
}

extern "C" int hrv_pack_conv_weight_tf32x2(const float* w0, const float* w1, int32_t cout, int32_t cin, int32_t kh, int32_t kw,
                                           int32_t transpose_flip, const float* inv_scale, void* dst, int32_t n_pad, int32_t cin_k,
                                           hrv_stream stream) {
  if (!w0 || !dst || cout < 1 || cin < 1 || kh < 1 || kw < 1) return set_error(HRV_EINVAL, "pack_conv_weight_tf32x2: bad arguments");
  const int inter = w1 ? 2 : 1;
  const int rows = transpose_flip ? cin : cout * inter, cols = transpose_flip ? cout * inter : cin;
  if (n_pad < rows || cin_k < cols)
    return set_error(HRV_EINVAL, "pack_conv_weight_tf32x2: destination too small (%d x %d for %d x %d)", n_pad, cin_k, rows, cols);
  const long long plane = (long long)n_pad * cin_k;
  pack_conv_weight_kernel<true><<<blocks_for(plane, 256), 256, 0, (cudaStream_t)stream>>>(w0, w1, cout, cin, kh, kw, transpose_flip, inv_scale,
                                                                                          (float*)dst, n_pad, cin_k, plane);
  return launch_ok("pack_conv_weight_tf32x2");
}
