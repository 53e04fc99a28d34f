// metrics.cu — the evaluation metrics of the reference's workflow (include/hrviton_sm100_metrics.h): the LPIPS AlexNet front end
// and per-layer distance (eval_models/networks_basic.py, eval_models/__init__.py), skimage's Gaussian SSIM as evaluate.py:67 calls
// it, and the Inception-v3 pieces behind the Inception Score, FID and KID (input resize, global pool, fp64 Gram products, KID subset
// sums, and the stride-1 pools and input of pytorch-fid's FID Inception).  fp32 and fp64 only, so this translation unit is compiled once (no 16-bit flavour).  No floating-point atomics: per-block
// partials land in slabs that a second kernel adds in a fixed order.
#include <type_traits>

#include "hrv_bilinear.cuh"
#include "hrv_host.h"

namespace hrv_metrics {
using hrv_host::set_error;

int launched(const char* what) {
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? HRV_OK : set_error(HRV_ECUDA, "%s: %s", what, cudaGetErrorString(e));
}
unsigned nblocks(long long total, int threads) { return (unsigned)((total + threads - 1) / threads); }

constexpr int kLpipsK = 11 * 11 * 3;  // conv1's im2col depth: (ky*11 + kx)*3 + ci

// ------------------------------------------------------------------------------------------------ LPIPS input
// dst[i,oy,ox,(ky*11+kx)*3+ci] = scaled(i, ci, 4*oy-2+ky, 4*ox-2+kx), zero outside the image (the zero padding of conv1 applies to the
// SCALED input) and in the pad channels [363, pitch).  scaled = (x - shift[ci]) / scale[ci], correctly rounded as torch computes it.
__global__ void lpips_input_kernel(const float* __restrict__ x, int H, int W, int Ho, int Wo, const float* __restrict__ shift,
                                   const float* __restrict__ scale, float* __restrict__ dst, int pitch, long long total) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int k = (int)(idx % pitch);
  const long long pix = idx / pitch;
  float v = 0.f;
  if (k < kLpipsK) {
    const int ox = (int)(pix % Wo), oy = (int)((pix / Wo) % Ho);
    const long long img = pix / ((long long)Wo * Ho);
    const int tap = k / 3, ci = k - tap * 3;
    const int ky = tap / 11, kx = tap - ky * 11;
    const int iy = 4 * oy - 2 + ky, ix = 4 * ox - 2 + kx;
    if (iy >= 0 && iy < H && ix >= 0 && ix < W) {
      const float xv = __ldg(x + ((img * 3 + ci) * H + iy) * W + ix);
      v = __fdiv_rn(__fsub_rn(xv, __ldg(shift + ci)), __ldg(scale + ci));
    }
  }
  dst[idx] = v;
}

// ------------------------------------------------------------------------------------------------ MaxPool2d(3, 2)
// Floor mode, no padding; torch's comparison (a NaN wins, the first of equal values stays), so the result is bit-exact.
__global__ void maxpool3s2_kernel(const float* __restrict__ x, int h, int w, int xp, float* __restrict__ y, int ho, int wo, int yp, int c,
                                  long long total) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int ch = (int)(idx % c);
  const long long pix = idx / c;
  const int ox = (int)(pix % wo), oy = (int)((pix / wo) % ho);
  const long long n = pix / ((long long)wo * ho);
  float m = -INFINITY;
#pragma unroll
  for (int dy = 0; dy < 3; ++dy)
#pragma unroll
    for (int dx = 0; dx < 3; ++dx) {
      const float v = __ldg(x + ((n * h + 2 * oy + dy) * w + 2 * ox + dx) * xp + ch);
      if (v > m || isnan(v)) m = v;
    }
  y[pix * yp + ch] = m;
}

// ------------------------------------------------------------------------------------------------ LPIPS distance of one layer
// One block per image pair (i, i + npair); each warp walks pixels, lanes walk channels.  Per pixel, in fp64:
//   n0 = sqrt(sum x0^2), n1 = sqrt(sum x1^2), d = sum_c w_c (x0_c/(n0+1e-10) - x1_c/(n1+1e-10))^2
// (normalize_tensor, the squared difference and the 1x1 `lin` convolution).  Lanes and warps meet through fixed shuffle trees and a
// fixed warp order, so the result does not depend on timing; out[i] = mean over pixels, rounded once to fp32 (spatial_average).
constexpr int kDistThreads = 512;
__global__ void __launch_bounds__(kDistThreads) lpips_dist_kernel(const float* __restrict__ f, int hw, int pitch, int c, int npair,
                                                                  const float* __restrict__ wl, float* __restrict__ out) {
  __shared__ double red[kDistThreads / 32];
  const int pair = blockIdx.x;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const float* f0 = f + (long long)pair * hw * pitch;
  const float* f1 = f + (long long)(pair + npair) * hw * pitch;
  double acc = 0.0;
  for (int p = warp; p < hw; p += kDistThreads / 32) {
    const float* a = f0 + (long long)p * pitch;
    const float* b = f1 + (long long)p * pitch;
    double s0 = 0.0, s1 = 0.0;
    for (int ch = lane; ch < c; ch += 32) {
      const double u = __ldg(a + ch), v = __ldg(b + ch);
      s0 = fma(u, u, s0);
      s1 = fma(v, v, s1);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      s0 += __shfl_xor_sync(0xffffffffu, s0, o);
      s1 += __shfl_xor_sync(0xffffffffu, s1, o);
    }
    const double r0 = 1.0 / (sqrt(s0) + 1e-10), r1 = 1.0 / (sqrt(s1) + 1e-10);
    double d = 0.0;
    for (int ch = lane; ch < c; ch += 32) {
      // both products rounded (no contraction into an fma): identical features give e = 0 exactly
      const double e = __dmul_rn((double)__ldg(a + ch), r0) - __dmul_rn((double)__ldg(b + ch), r1);
      d = fma((double)__ldg(wl + ch), e * e, d);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
    acc += d;  // every lane holds the same d
  }
  if (lane == 0) red[warp] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int i = 0; i < kDistThreads / 32; ++i) t += red[i];
    out[pair] = (float)(t / (double)hw);
  }
}

// ------------------------------------------------------------------------------------------------ Gaussian SSIM
// skimage.metrics.structural_similarity(gaussian_weights=True, sigma=1.5, truncate=3.5, use_sample_covariance=False) in fp64.
// Only the outputs the final crop keeps are computed: output (y, x) with 5 <= y < h-5, 5 <= x < w-5, whose 11x11 window lies inside
// the image, so the filter's border mode never matters.  A block owns a 32x8 tile of those outputs: it stages the 42x18 input halo in
// shared memory (as fp64), runs the horizontal pass for the five moments {x, y, xx, yy, xy} over the 18 rows, then every thread runs the
// vertical pass for its output and forms the SSIM value.  The block's sum goes to slab[n][tile]; ssim_finish_kernel adds the slabs in a
// fixed order and divides by the number of cropped outputs.
constexpr int kSsimR = 5, kSsimTW = 32, kSsimTH = 8, kSsimHW = kSsimTW + 2 * kSsimR, kSsimHH = kSsimTH + 2 * kSsimR;

__device__ __forceinline__ double ld_pix(const unsigned char* p, long long i) { return (double)__ldg(p + i); }
__device__ __forceinline__ double ld_pix(const float* p, long long i) { return (double)__ldg(p + i); }

template <typename T>
__global__ void __launch_bounds__(kSsimTW * kSsimTH) ssim_kernel(const T* __restrict__ im1, const T* __restrict__ im2, int h, int w,
                                                                 int tiles_x, double c1, double c2, double* __restrict__ slab) {
  __shared__ double sx[kSsimHH][kSsimHW], sy[kSsimHH][kSsimHW];
  __shared__ double hm[5][kSsimHH][kSsimTW];
  __shared__ double red[kSsimTW * kSsimTH / 32];
  __shared__ double c_gauss[2 * kSsimR + 1];
  const int n = blockIdx.y;
  const int tile = blockIdx.x;
  const int ty0 = (tile / tiles_x) * kSsimTH, tx0 = (tile % tiles_x) * kSsimTW;  // first cropped output of the tile, minus the crop
  const int t = threadIdx.x;
  const long long base = (long long)n * h * w;
  if (t <= 2 * kSsimR) {  // scipy.ndimage's 1-D Gaussian, sigma 1.5, radius int(3.5*1.5 + 0.5) = 5: exp(-x^2/(2 sigma^2)) / sum
    double sum = 0.0;
    for (int k = -kSsimR; k <= kSsimR; ++k) sum += exp(-0.5 / (1.5 * 1.5) * (double)(k * k));
    c_gauss[t] = exp(-0.5 / (1.5 * 1.5) * (double)((t - kSsimR) * (t - kSsimR))) / sum;
  }
  // input rows ty0 .. ty0+17, columns tx0 .. tx0+41 (output (ty0+5+j, tx0+5+i) reads rows ty0+j .. ty0+j+10)
  for (int i = t; i < kSsimHH * kSsimHW; i += blockDim.x) {
    const int r = i / kSsimHW, q = i - r * kSsimHW;
    const int y = ty0 + r, x = tx0 + q;
    double a = 0.0, b = 0.0;
    if (y < h && x < w) {
      a = ld_pix(im1, base + (long long)y * w + x);
      b = ld_pix(im2, base + (long long)y * w + x);
    }
    sx[r][q] = a;
    sy[r][q] = b;
  }
  __syncthreads();
  for (int i = t; i < kSsimHH * kSsimTW; i += blockDim.x) {
    const int r = i / kSsimTW, q = i - r * kSsimTW;
    double m0 = 0.0, m1 = 0.0, m2 = 0.0, m3 = 0.0, m4 = 0.0;
#pragma unroll
    for (int k = 0; k < 2 * kSsimR + 1; ++k) {
      const double g = c_gauss[k], a = sx[r][q + k], b = sy[r][q + k];
      m0 = fma(g, a, m0);
      m1 = fma(g, b, m1);
      m2 = fma(g, a * a, m2);
      m3 = fma(g, b * b, m3);
      m4 = fma(g, a * b, m4);
    }
    hm[0][r][q] = m0; hm[1][r][q] = m1; hm[2][r][q] = m2; hm[3][r][q] = m3; hm[4][r][q] = m4;
  }
  __syncthreads();
  const int j = t / kSsimTW, i = t - j * kSsimTW;
  const int oy = ty0 + kSsimR + j, ox = tx0 + kSsimR + i;
  double s = 0.0;
  if (oy < h - kSsimR && ox < w - kSsimR) {
    double ux = 0.0, uy = 0.0, uxx = 0.0, uyy = 0.0, uxy = 0.0;
#pragma unroll
    for (int k = 0; k < 2 * kSsimR + 1; ++k) {
      const double g = c_gauss[k];
      ux = fma(g, hm[0][j + k][i], ux);
      uy = fma(g, hm[1][j + k][i], uy);
      uxx = fma(g, hm[2][j + k][i], uxx);
      uyy = fma(g, hm[3][j + k][i], uyy);
      uxy = fma(g, hm[4][j + k][i], uxy);
    }
    const double vx = uxx - ux * ux, vy = uyy - uy * uy, vxy = uxy - ux * uy;  // cov_norm = 1 (use_sample_covariance=False)
    const double a1 = 2.0 * ux * uy + c1, a2 = 2.0 * vxy + c2;
    const double b1 = ux * ux + uy * uy + c1, b2 = vx + vy + c2;
    s = (a1 * a2) / (b1 * b2);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((t & 31) == 0) red[t >> 5] = s;
  __syncthreads();
  if (t == 0) {
    double tot = 0.0;
    for (int k = 0; k < kSsimTW * kSsimTH / 32; ++k) tot += red[k];
    slab[(long long)n * gridDim.x + tile] = tot;
  }
}

// One block per image: thread t adds its contiguous range of slabs in order, then a fixed shared-memory tree.
__global__ void __launch_bounds__(256) ssim_finish_kernel(const double* __restrict__ slab, int tiles, double inv_count, double* __restrict__ out) {
  __shared__ double part[256];
  const double* s = slab + (long long)blockIdx.x * tiles;
  const int k = (tiles + 255) / 256, b = threadIdx.x * k, e = min(b + k, tiles);
  double acc = 0.0;
  for (int i = b; i < e; ++i) acc += s[i];
  part[threadIdx.x] = acc;
  __syncthreads();
  for (int st = 128; st > 0; st >>= 1) {
    if (threadIdx.x < st) part[threadIdx.x] += part[threadIdx.x + st];
    __syncthreads();
  }
  if (threadIdx.x == 0) out[blockIdx.x] = part[0] * inv_count;
}

int ssim_tiles(int h, int w, int* tiles_x) {
  const int tx = (w - 2 * kSsimR + kSsimTW - 1) / kSsimTW, ty = (h - 2 * kSsimR + kSsimTH - 1) / kSsimTH;
  if (tiles_x) *tiles_x = tx;
  return tx * ty;
}

// ------------------------------------------------------------------------------------------------ Inception input resize
// F.interpolate(x, (oh, ow), mode='bilinear', align_corners=False, antialias=False), written as fp32 NHWC.  The source index, the
// weights and the blend are torch's own expressions in the same order (aten upsample_bilinear2d, accscalar_t = float), so the result is
// bit-identical.  The source reader gives the float value of one tap: fp32 NCHW as is, or uint8 NHWC as TF.to_tensor converts it
// (u8 / 255, correctly rounded).  kNormBefore maps every tap v to 2v - 1 before the blend (torchvision Inception on [0, 1] images),
// kNormAfter maps the blended value (pytorch-fid: F.interpolate, then 2x - 1); 2v is exact, so either is one rounding, as in torch.
// One thread per output element of the first 8-channel groups; channels [c, c8) are written as zeros.
struct NchwF32 {
  const float* p;
  int c, h, w;
  __device__ __forceinline__ float operator()(long long img, int ch, int y, int x) const { return __ldg(p + ((img * c + ch) * h + y) * w + x); }
};

struct NhwcU8 {
  const unsigned char* p;
  int c, h, w;
  __device__ __forceinline__ float operator()(long long img, int ch, int y, int x) const {
    return __fdiv_rn((float)__ldg(p + ((img * h + y) * w + x) * c + ch), 255.f);
  }
};

enum { kNormNone = 0, kNormBefore = 1, kNormAfter = 2 };

__device__ __forceinline__ float to_signed_unit(float v) { return __fsub_rn(__fmul_rn(2.f, v), 1.f); }

template <typename Src, int kNorm>
__global__ void resize_bilinear_kernel(Src src, float rh, float rw, float* __restrict__ dst, int oh, int ow, int pitch, int c8, long long total) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int ch = (int)(idx % c8);
  const long long pix = idx / c8;
  const int h = src.h, w = src.w;
  float val = 0.f;
  if (ch < src.c) {
    const int ox = (int)(pix % ow), oy = (int)((pix / ow) % oh);
    const long long img = pix / ((long long)ow * oh);
    const hrv_bilinear::Taps ty = hrv_bilinear::bilinear_taps(rh, oy, h), tx = hrv_bilinear::bilinear_taps(rw, ox, w);
    float v00 = src(img, ch, ty.i0, tx.i0), v01 = src(img, ch, ty.i0, tx.i1);
    float v10 = src(img, ch, ty.i1, tx.i0), v11 = src(img, ch, ty.i1, tx.i1);
    if (kNorm == kNormBefore) {
      v00 = to_signed_unit(v00); v01 = to_signed_unit(v01); v10 = to_signed_unit(v10); v11 = to_signed_unit(v11);
    }
    val = hrv_bilinear::bilinear_blend(ty, tx, v00, v01, v10, v11);
    if (kNorm == kNormAfter) val = to_signed_unit(val);
  }
  dst[pix * pitch + ch] = val;
}

// ------------------------------------------------------------------------------------------------ 3x3 stride-1 pool
// F.avg_pool2d(x, 3, 1, 1, count_include_pad=False) (kMode 0) or F.max_pool2d(x, 3, 1, 1) (kMode 1) on fp32 NHWC, y the same extent.
// As torch's CUDA kernels: the in-image taps in raster order, summed in fp32 from 0 and divided once by their count (correctly
// rounded), or compared with `v > m || isnan(v)` from -inf (NaN propagates, the first of equal values stays): bit-identical.  One
// thread per V consecutive channels of one output pixel (V = 4: 16-byte loads and stores, when pitches, channel offset and count allow).
template <int kMode, int V>
__global__ void pool3x3s1_kernel(const float* __restrict__ x, int h, int w, int xp, float* __restrict__ y, int yp, int cv, long long total) {
  using Vec = typename std::conditional<V == 4, float4, float>::type;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int cg = (int)(idx % cv);
  const long long pix = idx / cv;
  const int ox = (int)(pix % w), oy = (int)((pix / w) % h);
  const long long n = pix / ((long long)w * h);
  const int y0 = max(oy - 1, 0), y1 = min(oy + 2, h), x0 = max(ox - 1, 0), x1 = min(ox + 2, w);
  float acc[V];
#pragma unroll
  for (int i = 0; i < V; ++i) acc[i] = kMode == 0 ? 0.f : -INFINITY;
  for (int yy = y0; yy < y1; ++yy)
    for (int xx = x0; xx < x1; ++xx) {
      const Vec v = __ldg(reinterpret_cast<const Vec*>(x + ((n * h + yy) * w + xx) * xp) + cg);
      const float* vf = reinterpret_cast<const float*>(&v);
#pragma unroll
      for (int i = 0; i < V; ++i) {
        if (kMode == 0) acc[i] = __fadd_rn(acc[i], vf[i]);
        else if (vf[i] > acc[i] || isnan(vf[i])) acc[i] = vf[i];
      }
    }
  if (kMode == 0) {
    const float cnt = (float)((y1 - y0) * (x1 - x0));
#pragma unroll
    for (int i = 0; i < V; ++i) acc[i] = __fdiv_rn(acc[i], cnt);
  }
  Vec out;
#pragma unroll
  for (int i = 0; i < V; ++i) reinterpret_cast<float*>(&out)[i] = acc[i];
  reinterpret_cast<Vec*>(y + pix * yp)[cg] = out;
}

// ------------------------------------------------------------------------------------------------ global average pool
// y[n, ch] = (sum over the h*w pixels in raster order, in fp64) / (h*w), rounded once to fp32.  One thread per (n, ch): a warp reads
// 32 consecutive channels of one pixel.
__global__ void global_avgpool_kernel(const float* __restrict__ x, int hw, int pitch, int c, float* __restrict__ y, int ypitch,
                                      long long total) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int ch = (int)(idx % c);
  const long long n = idx / c;
  const float* p = x + n * hw * pitch + ch;
  double s = 0.0;
  for (int i = 0; i < hw; ++i) s += (double)__ldg(p + (long long)i * pitch);
  y[n * ypitch + ch] = (float)(s / (double)hw);
}

// ------------------------------------------------------------------------------------------------ fp64 Gram product
// C[i][j] (+)= sum_k A(i,k) * B(j,k) in fp64, A(i,k) = a[i*sam + k*sak], B(j,k) = b[j*sbn + k*sbk] (fp32 or fp64 elements).  A block
// owns a 64x64 tile of C and one K range (split z of the grid); every thread owns a 4x4 sub-tile (rows ty + 16r, columns tx + 16q) and
// adds its products in increasing k, one fma each (an fp32 x fp32 product is exact in fp64).  With one split the block writes C
// (c + acc when accumulating); with several, split z writes slab z and gram_finish_kernel adds the slabs in split order.
constexpr int kGramT = 64, kGramK = 16, kGramThreads = 256, kGramKPer = 512;

template <typename T>
__device__ __forceinline__ void gram_load(double (*s)[kGramT + 1], const T* __restrict__ g, long long si, long long sk, int i0, int ni, int k0,
                                          int k1, bool kfast) {
#pragma unroll
  for (int r = 0; r < kGramT * kGramK / kGramThreads; ++r) {
    const int e = threadIdx.x + r * kGramThreads;
    const int ii = kfast ? e / kGramK : e % kGramT, kk = kfast ? e % kGramK : e / kGramT;  // consecutive threads: consecutive addresses
    const int gi = i0 + ii, gk = k0 + kk;
    s[kk][ii] = (gi < ni && gk < k1) ? (double)__ldg(g + gi * si + gk * sk) : 0.0;
  }
}

template <typename T>
__global__ void __launch_bounds__(kGramThreads) gram_kernel(const T* __restrict__ a, long long sam, long long sak, const T* __restrict__ b,
                                                            long long sbn, long long sbk, int m, int n, int k, int kper, double* __restrict__ c,
                                                            long long ldc, int accumulate, double* __restrict__ slab) {
  __shared__ double As[kGramK][kGramT + 1], Bs[kGramK][kGramT + 1];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int j0 = blockIdx.x * kGramT, i0 = blockIdx.y * kGramT;
  const int kb = blockIdx.z * kper, ke = min(k, kb + kper);
  const bool a_kfast = sak == 1 && sam != 1, b_kfast = sbk == 1 && sbn != 1;
  double acc[4][4];
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int q = 0; q < 4; ++q) acc[r][q] = 0.0;
  for (int k0 = kb; k0 < ke; k0 += kGramK) {
    gram_load(As, a, sam, sak, i0, m, k0, ke, a_kfast);
    gram_load(Bs, b, sbn, sbk, j0, n, k0, ke, b_kfast);
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < kGramK; ++kk) {
      double ar[4], br[4];
#pragma unroll
      for (int r = 0; r < 4; ++r) ar[r] = As[kk][ty + 16 * r];
#pragma unroll
      for (int q = 0; q < 4; ++q) br[q] = Bs[kk][tx + 16 * q];
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int q = 0; q < 4; ++q) acc[r][q] = fma(ar[r], br[q], acc[r][q]);
    }
    __syncthreads();
  }
  double* s = slab ? slab + (long long)blockIdx.z * m * n : nullptr;
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int i = i0 + ty + 16 * r, j = j0 + tx + 16 * q;
      if (i >= m || j >= n) continue;
      if (s) s[(long long)i * n + j] = acc[r][q];
      else c[i * ldc + j] = accumulate ? c[i * ldc + j] + acc[r][q] : acc[r][q];
    }
}

__global__ void gram_finish_kernel(const double* __restrict__ slab, int splits, int m, int n, double* __restrict__ c, long long ldc, int accumulate) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long mn = (long long)m * n;
  if (idx >= mn) return;
  double s = slab[idx];
  for (int z = 1; z < splits; ++z) s += slab[z * mn + idx];
  double* p = c + (idx / n) * ldc + idx % n;
  *p = accumulate ? *p + s : s;
}

// Split-K only where the tiles alone leave most of the GPU idle and K is long; a function of the shape alone, so the summation order
// (and the result) does not depend on the device.
int gram_splits(int m, int n, int k, int* kper) {
  const long long tiles = (long long)((m + kGramT - 1) / kGramT) * ((n + kGramT - 1) / kGramT);
  int splits = 1;
  if (tiles < 128 && k >= 2 * kGramKPer) {
    splits = (int)((256 + tiles - 1) / tiles);
    splits = min(splits, min(64, k / kGramKPer));
  }
  const int per = ((k + splits - 1) / splits + kGramK - 1) / kGramK * kGramK;
  if (kper) *kper = per;
  return (k + per - 1) / per;
}

// ------------------------------------------------------------------------------------------------ KID subset sums
// Block (s, t) forms one sum of subset s over the cubic polynomial kernel k(g) = (g*gamma + 1)^3 of precomputed Gram entries:
// t = 0: sum_{i != j} k(Gxx[ix_i][ix_j]),  t = 1: sum_{i != j} k(Gyy[iy_i][iy_j]),  t = 2: sum_{i, j} k(Gxy[ix_i][iy_j]).
// Warp w walks the rows w, w + 16, ..., lanes the columns; fixed shuffle tree, then the warps in order.
constexpr int kKidThreads = 512;
__global__ void __launch_bounds__(kKidThreads) kid_sums_kernel(const double* __restrict__ gxx, const double* __restrict__ gyy,
                                                               const double* __restrict__ gxy, int na, int nb, const int* __restrict__ ix,
                                                               const int* __restrict__ iy, int m, double gamma, double* __restrict__ out) {
  __shared__ double red[kKidThreads / 32];
  const int s = blockIdx.x, t = blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const double* g = t == 0 ? gxx : (t == 1 ? gyy : gxy);
  const long long ld = t == 0 ? na : nb;
  const int* ri = (t == 1 ? iy : ix) + (long long)s * m;
  const int* ci = (t == 0 ? ix : iy) + (long long)s * m;
  double acc = 0.0;
  for (int i = warp; i < m; i += kKidThreads / 32) {
    const double* row = g + (long long)__ldg(ri + i) * ld;
    double r = 0.0;
    for (int j = lane; j < m; j += 32) {
      if (t < 2 && j == i) continue;
      const double v = fma(__ldg(row + __ldg(ci + j)), gamma, 1.0);
      r += v * v * v;
    }
    acc += r;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (lane == 0) red[warp] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double tot = 0.0;
    for (int w = 0; w < kKidThreads / 32; ++w) tot += red[w];
    out[(long long)s * 3 + t] = tot;
  }
}

}  // namespace hrv_metrics

using namespace hrv_metrics;

extern "C" int hrv_lpips_input(const float* x, int32_t n_img, int32_t h, int32_t w, const float* shift, const float* scale,
                               const hrv_tensor* dst, hrv_stream stream) {
  if (!x || !shift || !scale || !dst || !dst->ptr || n_img < 1 || h < 7 || w < 7)
    return set_error(HRV_EINVAL, "lpips_input: bad arguments (images need at least 7x7 pixels)");
  const int ho = (h + 4 - 11) / 4 + 1, wo = (w + 4 - 11) / 4 + 1;
  if (dst->dtype != HRV_F32 || dst->n != n_img || dst->h != ho || dst->w != wo || dst->c != kLpipsK || dst->pitch < kLpipsK ||
      (dst->pitch % 8) || ((uintptr_t)dst->ptr & 15))
    return set_error(HRV_EINVAL, "lpips_input: dst must be fp32 NHWC (%d,%d,%d,c=%d), pitch %% 8 == 0, 16-byte aligned", n_img, ho, wo, kLpipsK);
  const long long total = (long long)n_img * ho * wo * dst->pitch;
  lpips_input_kernel<<<nblocks(total, 256), 256, 0, (cudaStream_t)stream>>>(x, h, w, ho, wo, shift, scale, (float*)dst->ptr, dst->pitch, total);
  return launched("lpips_input");
}

extern "C" int hrv_maxpool3s2(const hrv_tensor* x, const hrv_tensor* y, hrv_stream stream) {
  if (!x || !y || !x->ptr || !y->ptr || x->dtype != HRV_F32 || y->dtype != HRV_F32 || x->h < 3 || x->w < 3)
    return set_error(HRV_EINVAL, "maxpool3s2: x and y must be fp32 NHWC, x at least 3x3");
  if (y->n != x->n || y->c != x->c || y->h != (x->h - 3) / 2 + 1 || y->w != (x->w - 3) / 2 + 1 || x->pitch < x->c || y->pitch < y->c)
    return set_error(HRV_EINVAL, "maxpool3s2: y must be (n, (h-3)/2+1, (w-3)/2+1, c)");
  const long long total = (long long)y->n * y->h * y->w * y->c;
  if (total)
    maxpool3s2_kernel<<<nblocks(total, 256), 256, 0, (cudaStream_t)stream>>>((const float*)x->ptr, x->h, x->w, x->pitch, (float*)y->ptr,
                                                                             y->h, y->w, y->pitch, y->c, total);
  return launched("maxpool3s2");
}

extern "C" int hrv_lpips_dist(const hrv_tensor* feat, const float* lin_w, float* out, hrv_stream stream) {
  if (!feat || !feat->ptr || !lin_w || !out || feat->dtype != HRV_F32 || feat->n < 2 || (feat->n & 1) || feat->pitch < feat->c || feat->c < 1)
    return set_error(HRV_EINVAL, "lpips_dist: feat must be fp32 NHWC holding 2N images (the N first images pair with the N last)");
  const int npair = feat->n / 2;
  lpips_dist_kernel<<<(unsigned)npair, kDistThreads, 0, (cudaStream_t)stream>>>((const float*)feat->ptr, feat->h * feat->w, feat->pitch,
                                                                                  feat->c, npair, lin_w, out);
  return launched("lpips_dist");
}

extern "C" size_t hrv_ssim_workspace_bytes(int32_t n, int32_t h, int32_t w) {
  if (n < 1 || h < 11 || w < 11) return 0;
  return (size_t)n * ssim_tiles(h, w, nullptr) * sizeof(double);
}

extern "C" int hrv_ssim(const void* im1, const void* im2, int32_t dtype, int32_t n, int32_t h, int32_t w, double data_range, double* out,
                        void* workspace, size_t workspace_bytes, hrv_stream stream) {
  if (!im1 || !im2 || !out || n < 1 || (dtype != HRV_SSIM_U8 && dtype != HRV_SSIM_F32) || !(data_range > 0.0))
    return set_error(HRV_EINVAL, "ssim: bad arguments");
  if (h < 11 || w < 11) return set_error(HRV_EINVAL, "ssim: the 11x11 window exceeds the %dx%d image", h, w);
  const size_t need = hrv_ssim_workspace_bytes(n, h, w);
  if (!workspace || workspace_bytes < need) return set_error(HRV_EINVAL, "ssim: workspace too small (%zu < %zu)", workspace_bytes, need);
  cudaStream_t st = (cudaStream_t)stream;
  int rc, tiles_x;
  const int tiles = ssim_tiles(h, w, &tiles_x);
  const double c1 = (0.01 * data_range) * (0.01 * data_range), c2 = (0.03 * data_range) * (0.03 * data_range);
  const dim3 grid((unsigned)tiles, (unsigned)n);
  double* slab = (double*)workspace;
  if (dtype == HRV_SSIM_U8)
    ssim_kernel<unsigned char><<<grid, kSsimTW * kSsimTH, 0, st>>>((const unsigned char*)im1, (const unsigned char*)im2, h, w, tiles_x, c1, c2, slab);
  else
    ssim_kernel<float><<<grid, kSsimTW * kSsimTH, 0, st>>>((const float*)im1, (const float*)im2, h, w, tiles_x, c1, c2, slab);
  if ((rc = launched("ssim"))) return rc;
  ssim_finish_kernel<<<(unsigned)n, 256, 0, st>>>(slab, tiles, 1.0 / ((double)(h - 2 * kSsimR) * (double)(w - 2 * kSsimR)), out);
  return launched("ssim finish");
}

extern "C" int hrv_resize_bilinear_nhwc(const float* x, int32_t n, int32_t c, int32_t h, int32_t w, int32_t unit_range, const hrv_tensor* dst,
                                        hrv_stream stream) {
  if (!x || !dst || !dst->ptr || n < 1 || c < 1 || h < 1 || w < 1)
    return set_error(HRV_EINVAL, "resize_bilinear_nhwc: bad arguments");
  const int c8 = (c + 7) / 8 * 8;
  if (dst->dtype != HRV_F32 || dst->n != n || dst->c != c || dst->h < 1 || dst->w < 1 || dst->pitch < c8)
    return set_error(HRV_EINVAL, "resize_bilinear_nhwc: dst must be fp32 NHWC (n=%d, oh, ow, c=%d) with pitch >= %d", n, c, c8);
  const long long total = (long long)n * dst->h * dst->w * c8;
  // torch's scale for an explicit output size: (float)in / out
  const float rh = (float)h / dst->h, rw = (float)w / dst->w;
  const NchwF32 src{x, c, h, w};
  if (unit_range)
    resize_bilinear_kernel<NchwF32, kNormBefore><<<nblocks(total, 256), 256, 0, (cudaStream_t)stream>>>(src, rh, rw, (float*)dst->ptr, dst->h,
                                                                                                         dst->w, dst->pitch, c8, total);
  else
    resize_bilinear_kernel<NchwF32, kNormNone><<<nblocks(total, 256), 256, 0, (cudaStream_t)stream>>>(src, rh, rw, (float*)dst->ptr, dst->h,
                                                                                                       dst->w, dst->pitch, c8, total);
  return launched("resize_bilinear_nhwc");
}

extern "C" int hrv_resize_bilinear_fid(const void* x, int32_t src, int32_t n, int32_t c, int32_t h, int32_t w, const hrv_tensor* dst,
                                       hrv_stream stream) {
  if (!x || !dst || !dst->ptr || n < 1 || c < 1 || h < 1 || w < 1 || (src != HRV_FID_SRC_F32_NCHW && src != HRV_FID_SRC_U8_NHWC))
    return set_error(HRV_EINVAL, "resize_bilinear_fid: bad arguments");
  const int c8 = (c + 7) / 8 * 8;
  if (dst->dtype != HRV_F32 || dst->n != n || dst->c != c || dst->h < 1 || dst->w < 1 || dst->pitch < c8)
    return set_error(HRV_EINVAL, "resize_bilinear_fid: dst must be fp32 NHWC (n=%d, oh, ow, c=%d) with pitch >= %d", n, c, c8);
  const long long total = (long long)n * dst->h * dst->w * c8;
  const float rh = (float)h / dst->h, rw = (float)w / dst->w;
  cudaStream_t st = (cudaStream_t)stream;
  if (src == HRV_FID_SRC_U8_NHWC)
    resize_bilinear_kernel<NhwcU8, kNormAfter><<<nblocks(total, 256), 256, 0, st>>>(NhwcU8{(const unsigned char*)x, c, h, w}, rh, rw,
                                                                                    (float*)dst->ptr, dst->h, dst->w, dst->pitch, c8, total);
  else
    resize_bilinear_kernel<NchwF32, kNormAfter><<<nblocks(total, 256), 256, 0, st>>>(NchwF32{(const float*)x, c, h, w}, rh, rw,
                                                                                     (float*)dst->ptr, dst->h, dst->w, dst->pitch, c8, total);
  return launched("resize_bilinear_fid");
}

extern "C" int hrv_pool3x3s1(const hrv_tensor* x, int32_t mode, const hrv_tensor* y, hrv_stream stream) {
  if (!x || !y || !x->ptr || !y->ptr || x->dtype != HRV_F32 || y->dtype != HRV_F32 || x->n < 1 || x->h < 1 || x->w < 1 || x->c < 1 ||
      (mode != HRV_POOL3X3_AVG_EXCL_PAD && mode != HRV_POOL3X3_MAX))
    return set_error(HRV_EINVAL, "pool3x3s1: x and y must be fp32 NHWC, mode 0 (average) or 1 (max)");
  if (y->n != x->n || y->h != x->h || y->w != x->w || y->c != x->c || x->pitch < x->c || y->pitch < y->c)
    return set_error(HRV_EINVAL, "pool3x3s1: y must have x's extent (%d,%d,%d,%d)", x->n, x->h, x->w, x->c);
  const bool vec4 = x->c % 4 == 0 && x->pitch % 4 == 0 && y->pitch % 4 == 0 && ((uintptr_t)x->ptr & 15) == 0 && ((uintptr_t)y->ptr & 15) == 0;
  const int cv = vec4 ? x->c / 4 : x->c;
  const long long total = (long long)x->n * x->h * x->w * cv;
  const unsigned nb = nblocks(total, 256);
  cudaStream_t st = (cudaStream_t)stream;
  const float* xp = (const float*)x->ptr;
  float* yp = (float*)y->ptr;
  if (mode == HRV_POOL3X3_AVG_EXCL_PAD) {
    if (vec4) pool3x3s1_kernel<0, 4><<<nb, 256, 0, st>>>(xp, x->h, x->w, x->pitch, yp, y->pitch, cv, total);
    else pool3x3s1_kernel<0, 1><<<nb, 256, 0, st>>>(xp, x->h, x->w, x->pitch, yp, y->pitch, cv, total);
  } else {
    if (vec4) pool3x3s1_kernel<1, 4><<<nb, 256, 0, st>>>(xp, x->h, x->w, x->pitch, yp, y->pitch, cv, total);
    else pool3x3s1_kernel<1, 1><<<nb, 256, 0, st>>>(xp, x->h, x->w, x->pitch, yp, y->pitch, cv, total);
  }
  return launched("pool3x3s1");
}

extern "C" int hrv_global_avgpool(const hrv_tensor* x, const hrv_tensor* y, hrv_stream stream) {
  if (!x || !y || !x->ptr || !y->ptr || x->dtype != HRV_F32 || y->dtype != HRV_F32 || x->h < 1 || x->w < 1 || x->c < 1 || x->pitch < x->c)
    return set_error(HRV_EINVAL, "global_avgpool: x and y must be fp32 NHWC");
  if (y->n != x->n || y->c != x->c || y->h != 1 || y->w != 1 || y->pitch < y->c)
    return set_error(HRV_EINVAL, "global_avgpool: y must be (n, 1, 1, c)");
  const long long total = (long long)x->n * x->c;
  global_avgpool_kernel<<<nblocks(total, 256), 256, 0, (cudaStream_t)stream>>>((const float*)x->ptr, x->h * x->w, x->pitch, x->c,
                                                                               (float*)y->ptr, y->pitch, total);
  return launched("global_avgpool");
}

extern "C" size_t hrv_gram_f64_workspace_bytes(int32_t m, int32_t n, int32_t k) {
  if (m < 1 || n < 1 || k < 1) return 0;
  const int splits = gram_splits(m, n, k, nullptr);
  return splits > 1 ? (size_t)splits * m * n * sizeof(double) : 0;
}

extern "C" int hrv_gram_f64(const void* a, int64_t sam, int64_t sak, const void* b, int64_t sbn, int64_t sbk, int32_t dtype, int32_t m, int32_t n,
                            int32_t k, double* c, int64_t ldc, int32_t accumulate, void* workspace, size_t workspace_bytes, hrv_stream stream) {
  if (!a || !b || !c || m < 1 || n < 1 || k < 1 || ldc < n || (dtype != HRV_GRAM_F32 && dtype != HRV_GRAM_F64))
    return set_error(HRV_EINVAL, "gram_f64: bad arguments");
  int kper;
  const int splits = gram_splits(m, n, k, &kper);
  const size_t need = hrv_gram_f64_workspace_bytes(m, n, k);
  if (need && (!workspace || workspace_bytes < need))
    return set_error(HRV_EINVAL, "gram_f64: workspace too small (%zu < %zu)", workspace_bytes, need);
  cudaStream_t st = (cudaStream_t)stream;
  double* slab = splits > 1 ? (double*)workspace : nullptr;
  const dim3 grid((unsigned)((n + kGramT - 1) / kGramT), (unsigned)((m + kGramT - 1) / kGramT), (unsigned)splits);
  if (dtype == HRV_GRAM_F32)
    gram_kernel<float><<<grid, kGramThreads, 0, st>>>((const float*)a, sam, sak, (const float*)b, sbn, sbk, m, n, k, kper, c, ldc, accumulate, slab);
  else
    gram_kernel<double><<<grid, kGramThreads, 0, st>>>((const double*)a, sam, sak, (const double*)b, sbn, sbk, m, n, k, kper, c, ldc, accumulate, slab);
  int rc = launched("gram_f64");
  if (rc || splits == 1) return rc;
  gram_finish_kernel<<<nblocks((long long)m * n, 256), 256, 0, st>>>(slab, splits, m, n, c, ldc, accumulate);
  return launched("gram_f64 finish");
}

extern "C" int hrv_kid_sums(const double* gxx, const double* gyy, const double* gxy, int32_t na, int32_t nb, const int32_t* ix, const int32_t* iy,
                            int32_t subsets, int32_t m, double gamma, double* out, hrv_stream stream) {
  if (!gxx || !gyy || !gxy || !ix || !iy || !out || subsets < 1 || m < 2 || m > na || m > nb)
    return set_error(HRV_EINVAL, "kid_sums: bad arguments (2 <= subset size <= the number of features of each set)");
  kid_sums_kernel<<<dim3((unsigned)subsets, 3), kKidThreads, 0, (cudaStream_t)stream>>>(gxx, gyy, gxy, na, nb, ix, iy, m, gamma, out);
  return launched("kid_sums");
}
