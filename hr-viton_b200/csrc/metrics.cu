// metrics.cu — the evaluation metrics of the reference's workflow (include/hrviton_sm100_metrics.h): the LPIPS AlexNet front end
// and per-layer distance (eval_models/networks_basic.py, eval_models/__init__.py) and skimage's Gaussian SSIM as evaluate.py:67 calls
// it.  fp32 and fp64 only, so this translation unit is compiled once (no 16-bit flavour).  No floating-point atomics: per-block
// partials land in slabs that a second kernel adds in a fixed order.
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
