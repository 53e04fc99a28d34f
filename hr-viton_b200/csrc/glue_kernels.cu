// glue_kernels.cu — data-movement / pooling kernels either side of the convolutions in the TRAINING step
// (SURVEY.md §8 rows N1/N2): space-to-depth backward, 2x2 max-pool (VGG19) forward/backward, 3x3/s2 average-pool backward
// (multi-scale discriminator), and the fused "upsample -> 15x15 Gaussian -> argmax -> 7-class one-hot" of the parse map
// (train_generator.py:247-273).  All HBM-bound: one 16-byte vector (8 bf16 channels) per thread, coalesced along channels.
#include "hrv_host.h"
#include "hrv_ptx.cuh"

namespace hrv {
namespace {

struct GView {
  const void* ptr;
  int n, h, w, c, pitch;
};
GView gv(const hrv_tensor* t) { return GView{t->ptr, t->n, t->h, t->w, t->c, t->pitch}; }

// dt: the storage type every tensor of the call must have (fp32 only where an entry point takes fp32 storage).
int check_vec(const hrv_tensor* t, const char* what, int dt = HRV_BF16) {
  if (!t || !t->ptr) return set_error(HRV_EINVAL, "%s: null tensor", what);
  if (t->dtype != dt)
    return dt == HRV_BF16 ? set_error(HRV_EINVAL, "%s: must be bf16 NHWC", what)
                          : set_error(HRV_EINVAL, "%s: must be fp32 like the call's other tensors (one storage type per call)", what);
  if (((uintptr_t)t->ptr & 15) || (t->pitch % 8) || t->pitch < t->c) return set_error(HRV_EINVAL, "%s: needs a 16-byte aligned ptr and pitch %% 8 == 0", what);
  return HRV_OK;
}
int launched(const char* what) {
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? HRV_OK : set_error(HRV_ECUDA, "%s: %s", what, cudaGetErrorString(e));
}
unsigned nblocks(long long total, int threads) { return (unsigned)((total + threads - 1) / threads); }

__device__ __forceinline__ uint4 ld16(const __nv_bfloat16* p) { return __ldg(reinterpret_cast<const uint4*>(p)); }
__device__ __forceinline__ void st16(__nv_bfloat16* p, const uint4& v) { *reinterpret_cast<uint4*>(p) = v; }
__device__ __forceinline__ void un8(const uint4& u, float (&f)[8]) {
  f[0] = bf16_lo(u.x); f[1] = bf16_hi(u.x); f[2] = bf16_lo(u.y); f[3] = bf16_hi(u.y);
  f[4] = bf16_lo(u.z); f[5] = bf16_hi(u.z); f[6] = bf16_lo(u.w); f[7] = bf16_hi(u.w);
}
__device__ __forceinline__ uint4 pk8(const float (&f)[8]) {
  return make_uint4(pack_bf16(f[0], f[1]), pack_bf16(f[2], f[3]), pack_bf16(f[4], f[5]), pack_bf16(f[6], f[7]));
}
__device__ __forceinline__ const __nv_bfloat16* at(const GView& v, int n, int y, int x) {
  return reinterpret_cast<const __nv_bfloat16*>(v.ptr) + (((long long)n * v.h + y) * v.w + x) * v.pitch;
}
__device__ __forceinline__ __nv_bfloat16* at_w(const GView& v, int n, int y, int x) { return const_cast<__nv_bfloat16*>(at(v, n, y, x)); }

// ---------------------------------------------------------------------------------------------- space-to-depth backward
// dx[n,y,x,g*8..] = d[n, y/2, x/2, ((y&1)*2 + (x&1)) * C8 + g*8..]     thread = (dx pixel, channel group)
__global__ void space_to_depth_bwd_kernel(GView d, GView dx, int G, long long total) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int g = (int)(idx % G);
  const long long pix = idx / G;
  const int x = (int)(pix % dx.w), y = (int)((pix / dx.w) % dx.h), n = (int)(pix / ((long long)dx.w * dx.h));
  const int sub = ((y & 1) << 1) | (x & 1);
  st16(at_w(dx, n, y, x) + g * 8, ld16(at(d, n, y >> 1, x >> 1) + (sub * G + g) * 8));
}

// ---------------------------------------------------------------------------------------------- 2x2 max-pool (stride 2, floor)
__global__ void maxpool2_fwd_kernel(GView x, GView y, int G, long long total) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int g = (int)(idx % G);
  const long long pix = idx / G;
  const int X = (int)(pix % y.w), Y = (int)((pix / y.w) % y.h), n = (int)(pix / ((long long)y.w * y.h));
  const __nv_bfloat16* p = at(x, n, 2 * Y, 2 * X) + g * 8;
  const long long row = (long long)x.w * x.pitch;
  const uint4 a = ld16(p), b = ld16(p + x.pitch), c = ld16(p + row), d = ld16(p + row + x.pitch);
  float fa[8], fb[8], fc[8], fd[8], o[8];
  un8(a, fa); un8(b, fb); un8(c, fc); un8(d, fd);
#pragma unroll
  for (int i = 0; i < 8; ++i) o[i] = fmaxf(fmaxf(fa[i], fb[i]), fmaxf(fc[i], fd[i]));
  st16(at_w(y, n, Y, X) + g * 8, pk8(o));
}
// The gradient goes to the FIRST maximum of the window in row-major order (what the library's index-based backward does).
__global__ void maxpool2_bwd_kernel(GView x, GView dy, GView dx, int G, long long total, int relu_gate) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int g = (int)(idx % G);
  const long long pix = idx / G;
  const int X = (int)(pix % dy.w), Y = (int)((pix / dy.w) % dy.h), n = (int)(pix / ((long long)dy.w * dy.h));
  const __nv_bfloat16* p = at(x, n, 2 * Y, 2 * X) + g * 8;
  const long long row = (long long)x.w * x.pitch;
  float f[4][8], gy[8], o[4][8];
  un8(ld16(p), f[0]); un8(ld16(p + x.pitch), f[1]); un8(ld16(p + row), f[2]); un8(ld16(p + row + x.pitch), f[3]);
  un8(ld16(at(dy, n, Y, X) + g * 8), gy);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    int best = 0;
    float m = f[0][i];
#pragma unroll
    for (int k = 1; k < 4; ++k)
      if (f[k][i] > m) { m = f[k][i]; best = k; }
#pragma unroll
    for (int k = 0; k < 4; ++k) o[k][i] = (k == best && !(relu_gate && m <= 0.f)) ? gy[i] : 0.f;
  }
  __nv_bfloat16* q = at_w(dx, n, 2 * Y, 2 * X) + g * 8;
  const long long qrow = (long long)dx.w * dx.pitch;
  st16(q, pk8(o[0])); st16(q + dx.pitch, pk8(o[1])); st16(q + qrow, pk8(o[2])); st16(q + qrow + dx.pitch, pk8(o[3]));
}

// ---------------------------------------------------------------------------------------------- avg-pool 3x3/s2/p1 backward
// count_include_pad=False: dx[y,x] = sum over windows (Y,X) containing (y,x) of dy[Y,X] / valid(Y,X).  thread = (dx pixel, group)
__global__ void avgpool3s2_bwd_kernel(GView dy, GView dx, int G, long long total) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int g = (int)(idx % G);
  const long long pix = idx / G;
  const int x = (int)(pix % dx.w), y = (int)((pix / dx.w) % dx.h), n = (int)(pix / ((long long)dx.w * dx.h));
  float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  const int Y0 = y >> 1, Y1 = (y & 1) ? Y0 + 1 : Y0, X0 = x >> 1, X1 = (x & 1) ? X0 + 1 : X0;
  for (int Y = Y0; Y <= Y1; ++Y) {
    if (Y >= dy.h) continue;
    const int rows = min(2 * Y + 1, dx.h - 1) - max(2 * Y - 1, 0) + 1;
    for (int X = X0; X <= X1; ++X) {
      if (X >= dy.w) continue;
      const int cols = min(2 * X + 1, dx.w - 1) - max(2 * X - 1, 0) + 1;
      float v[8];
      un8(ld16(at(dy, n, Y, X) + g * 8), v);
      const float inv = 1.f / (float)(rows * cols);
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] += v[i] * inv;
    }
  }
  st16(at_w(dx, n, y, x) + g * 8, pk8(acc));
}

// ---------------------------------------------------------------------------------------------- parse map: up -> blur -> argmax
// seg: fp32 NCHW (n,C,h,w) low-resolution class scores.  For every output pixel of the (H,W) grid:
//   u_c   = bilinear(seg_c) (align_corners=False, F.interpolate semantics)              train_generator.py:247
//   b_c   = 15x15 Gaussian(sigma 3), zero padding, separable                               train_generator.py:154,247
//   k     = argmax_c b_c  (first maximum)                                                  train_generator.py:248
// outputs: idx (n,H,W) int64 and/or onehot (n,groups,H,W) fp32 with onehot[group_of[k]] = 1   train_generator.py:251-273
constexpr int kTile = 32, kHalo = 7, kU = kTile + 2 * kHalo;  // 46
struct ParseArgs {
  const float* seg;
  long long* idx;
  float* onehot;
  float* overlap;       // optional (n,1,H,W): sum over the classes in occl_mask of softmax_c(blurred scores)  (remove_overlap's operand)
  unsigned occl_mask;
  int n, C, h, w, H, W, groups;
  float sy, sx;
  float g[15];
  int group_of[32];
};
__global__ void __launch_bounds__(256) parse_blur_argmax_kernel(const __grid_constant__ ParseArgs a) {
  __shared__ float U[kU][kU + 1];
  __shared__ float Hb[kU][kTile + 1];
  const int n = blockIdx.z, ty0 = blockIdx.y * kTile, tx0 = blockIdx.x * kTile;
  const int tid = threadIdx.x;
  const int col = tid & 31, rq = tid >> 5;  // thread owns output rows rq, rq+8, rq+16, rq+24 of column col
  float best[4] = {-INFINITY, -INFINITY, -INFINITY, -INFINITY};
  int arg[4] = {0, 0, 0, 0};
  float sm_all[4] = {0.f, 0.f, 0.f, 0.f}, sm_sel[4] = {0.f, 0.f, 0.f, 0.f};  // online softmax sums relative to the running maximum `best`
  for (int c = 0; c < a.C; ++c) {
    const float* s = a.seg + ((long long)n * a.C + c) * a.h * a.w;
    for (int i = tid; i < kU * kU; i += 256) {
      const int uy = i / kU, ux = i - uy * kU;
      const int Y = ty0 + uy - kHalo, X = tx0 + ux - kHalo;
      float v = 0.f;
      if (Y >= 0 && Y < a.H && X >= 0 && X < a.W) {
        const float fy = fmaxf(a.sy * ((float)Y + 0.5f) - 0.5f, 0.f), fx = fmaxf(a.sx * ((float)X + 0.5f) - 0.5f, 0.f);
        const int y0 = (int)fy, x0 = (int)fx;
        const int y1 = min(y0 + 1, a.h - 1), x1 = min(x0 + 1, a.w - 1);
        const float ly = fy - (float)y0, lx = fx - (float)x0;
        const float v00 = __ldg(s + y0 * a.w + x0), v01 = __ldg(s + y0 * a.w + x1), v10 = __ldg(s + y1 * a.w + x0), v11 = __ldg(s + y1 * a.w + x1);
        v = (1.f - ly) * ((1.f - lx) * v00 + lx * v01) + ly * ((1.f - lx) * v10 + lx * v11);
      }
      U[uy][ux] = v;
    }
    __syncthreads();
    for (int i = tid; i < kU * kTile; i += 256) {
      const int uy = i >> 5, x = i & 31;
      float acc = 0.f;
#pragma unroll
      for (int k = 0; k < 15; ++k) acc = fmaf(a.g[k], U[uy][x + k], acc);
      Hb[uy][x] = acc;
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int y = rq + 8 * j;
      float acc = 0.f;
#pragma unroll
      for (int k = 0; k < 15; ++k) acc = fmaf(a.g[k], Hb[y + k][col], acc);
      if (a.overlap) {  // softmax over classes without storing the blurred planes: rescale the sums when the maximum moves
        const float m_new = fmaxf(best[j], acc);
        const float scale = __expf(best[j] - m_new), e = __expf(acc - m_new);
        sm_all[j] = sm_all[j] * scale + e;
        sm_sel[j] = sm_sel[j] * scale + (((a.occl_mask >> c) & 1u) ? e : 0.f);
      }
      if (acc > best[j]) { best[j] = acc; arg[j] = c; }
    }
    // U / Hb are rewritten by the next channel: the barrier after the U fill separates Hb readers from Hb writers,
    // but U writers of channel c+1 must wait for the horizontal pass of channel c -> already ordered by the 2nd barrier.
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int Y = ty0 + rq + 8 * j, X = tx0 + col;
    if (Y < a.H && X < a.W) {
      const long long p = ((long long)n * a.H + Y) * a.W + X;
      if (a.idx) a.idx[p] = arg[j];
      if (a.overlap) a.overlap[p] = sm_sel[j] / sm_all[j];
      if (a.onehot) {
        const int grp = a.group_of[arg[j]];
        for (int q = 0; q < a.groups; ++q) a.onehot[(((long long)n * a.groups + q) * a.H + Y) * a.W + X] = (q == grp) ? 1.f : 0.f;
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------- stand-alone Gaussian blur
// tgm.image.GaussianBlur((k,k),(sigma,sigma)) on fp32 NCHW planes (train_generator.py:181,247; test_generator.py:91,185): separable,
// zero padding k/2, normalised 1-D taps — the same arithmetic as the fused parse kernel above, without the resize / arg-max.
// One block = one 32x32 output tile of one plane.  Used by the torchgeometry shim that lets the reference scripts run unchanged.
constexpr int kBlurMaxR = 15, kBU = kTile + 2 * kBlurMaxR;  // up to 31 taps
struct BlurArgs {
  const float* src;
  float* dst;
  int planes, H, W, r;
  float g[2 * kBlurMaxR + 1];
};
__global__ void __launch_bounds__(256) gaussian_blur_kernel(const __grid_constant__ BlurArgs a) {
  __shared__ float U[kBU][kBU + 1];
  __shared__ float Hb[kBU][kTile + 1];
  const int plane = blockIdx.z, ty0 = blockIdx.y * kTile, tx0 = blockIdx.x * kTile, tid = threadIdx.x;
  const int r = a.r, UU = kTile + 2 * r, taps = 2 * r + 1;
  const float* s = a.src + (long long)plane * a.H * a.W;
  for (int i = tid; i < UU * UU; i += 256) {
    const int uy = i / UU, ux = i - uy * UU;
    const int Y = ty0 + uy - r, X = tx0 + ux - r;
    U[uy][ux] = (Y >= 0 && Y < a.H && X >= 0 && X < a.W) ? __ldg(s + (long long)Y * a.W + X) : 0.f;
  }
  __syncthreads();
  for (int i = tid; i < UU * kTile; i += 256) {
    const int uy = i >> 5, x = i & 31;
    float acc = 0.f;
    for (int k = 0; k < taps; ++k) acc = fmaf(a.g[k], U[uy][x + k], acc);
    Hb[uy][x] = acc;
  }
  __syncthreads();
  const int col = tid & 31, rq = tid >> 5;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int y = rq + 8 * j, Y = ty0 + y, X = tx0 + col;
    float acc = 0.f;
    for (int k = 0; k < taps; ++k) acc = fmaf(a.g[k], Hb[y + k][col], acc);
    if (Y < a.H && X < a.W) a.dst[(long long)plane * a.H * a.W + (long long)Y * a.W + X] = acc;
  }
}

// ---------------------------------------------------------------------------------------------- hi-res flow warp (planar fp32)
// train_generator.py:232-238 / test_generator.py:170-176: the 128x96 appearance flow is up-sampled to the cloth's resolution
// (F.interpolate(size=(H,W), bilinear, align_corners=False), any scale), divided by ((wl-1)/2, (hl-1)/2) [correctly rounded fp32
// division], added to the linspace base grid and used to grid_sample (bilinear, border) the cloth / cloth mask.  One thread = one
// output pixel, looping over the few channels (3 + 1): planar reads and writes are coalesced along x.
__global__ void __launch_bounds__(256) flow_warp_nchw_kernel(const float* __restrict__ flow_lo, int hl, int wl, const float* __restrict__ lin_x,
                                                            const float* __restrict__ lin_y, const float* __restrict__ src, int C, int Hs, int Ws,
                                                            float* __restrict__ dst, int H, int W, float div_x, float div_y, float sc_y,
                                                            float sc_x, float* __restrict__ grid_out, const float* __restrict__ mask_src,
                                                            const float* __restrict__ overlap, float* __restrict__ mask_out, int composite,
                                                            long long npix) {
  const long long pix = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= npix) return;
  const int x = (int)(pix % W), y = (int)((pix / W) % H), n = (int)(pix / ((long long)W * H));
  // F.interpolate source coordinate: max(scale * (d + 0.5) - 0.5, 0), scale = in/out (area_pixel_compute_source_index)
  const float fy = fmaxf(__fsub_rn(__fmul_rn(sc_y, __fadd_rn((float)y, 0.5f)), 0.5f), 0.f);
  const float fx = fmaxf(__fsub_rn(__fmul_rn(sc_x, __fadd_rn((float)x, 0.5f)), 0.5f), 0.f);
  const int y0 = (int)fy, x0 = (int)fx;
  const int y1 = min(y0 + 1, hl - 1), x1 = min(x0 + 1, wl - 1);
  const float ly = __fsub_rn(fy, (float)y0), lx = __fsub_rn(fx, (float)x0);
  const float hy = __fsub_rn(1.f, ly), hx = __fsub_rn(1.f, lx);
  const float2* fl = reinterpret_cast<const float2*>(flow_lo) + (long long)n * hl * wl;
  const float2 f00 = __ldg(fl + (long long)y0 * wl + x0), f01 = __ldg(fl + (long long)y0 * wl + x1);
  const float2 f10 = __ldg(fl + (long long)y1 * wl + x0), f11 = __ldg(fl + (long long)y1 * wl + x1);
  // torch upsample_bilinear2d: w_y0 * (w_x0 * v00 + w_x1 * v01) + w_y1 * (w_x0 * v10 + w_x1 * v11)
  const float ux = __fadd_rn(__fmul_rn(hy, __fadd_rn(__fmul_rn(hx, f00.x), __fmul_rn(lx, f01.x))), __fmul_rn(ly, __fadd_rn(__fmul_rn(hx, f10.x), __fmul_rn(lx, f11.x))));
  const float uy = __fadd_rn(__fmul_rn(hy, __fadd_rn(__fmul_rn(hx, f00.y), __fmul_rn(lx, f01.y))), __fmul_rn(ly, __fadd_rn(__fmul_rn(hx, f10.y), __fmul_rn(lx, f11.y))));
  const float gx = __fadd_rn(__fdiv_rn(ux, div_x), __ldg(lin_x + x));
  const float gy = __fadd_rn(__fdiv_rn(uy, div_y), __ldg(lin_y + y));
  if (grid_out) reinterpret_cast<float2*>(grid_out)[pix] = make_float2(gx, gy);
  float ix = __fdiv_rn(__fsub_rn(__fmul_rn(__fadd_rn(gx, 1.f), (float)Ws), 1.f), 2.f);
  float iy = __fdiv_rn(__fsub_rn(__fmul_rn(__fadd_rn(gy, 1.f), (float)Hs), 1.f), 2.f);
  ix = fminf(fmaxf(ix, 0.f), (float)(Ws - 1));
  iy = fminf(fmaxf(iy, 0.f), (float)(Hs - 1));
  const float bx = floorf(ix), by = floorf(iy);
  const int sx0 = (int)bx, sy0 = (int)by;
  const float tx = __fsub_rn(ix, bx), ty = __fsub_rn(iy, by);
  const int sx1 = min(sx0 + 1, Ws - 1), sy1 = min(sy0 + 1, Hs - 1);
  const float wx1 = (sx0 + 1 <= Ws - 1) ? tx : 0.f, wy1 = (sy0 + 1 <= Hs - 1) ? ty : 0.f;
  const float wx0 = 1.f - tx, wy0 = 1.f - ty;
  const float w00 = wy0 * wx0, w01 = wy0 * wx1, w10 = wy1 * wx0, w11 = wy1 * wx1;
  const long long plane_s = (long long)Hs * Ws, plane_d = (long long)H * W;
  const long long o00 = (long long)sy0 * Ws + sx0, o01 = (long long)sy0 * Ws + sx1, o10 = (long long)sy1 * Ws + sx0, o11 = (long long)sy1 * Ws + sx1;
  float wm = 1.f;
  if (mask_src) {  // the cloth mask rides along: warped with the same taps, occlusion-corrected, optionally composited into the cloth
    const float* mp = mask_src + (long long)n * plane_s;
    wm = __ldg(mp + o00) * w00 + __ldg(mp + o01) * w01 + __ldg(mp + o10) * w10 + __ldg(mp + o11) * w11;
    if (overlap) wm = wm - __ldg(overlap + pix) * wm;  // remove_overlap (train_generator.py:26-31, test_generator.py:19-24)
    if (mask_out) mask_out[pix] = wm;
  }
  const float* sp = src + (long long)n * C * plane_s;
  float* dp = dst + (long long)n * C * plane_d + (long long)y * W + x;
  for (int c = 0; c < C; ++c, sp += plane_s, dp += plane_d) {
    float v = __ldg(sp + o00) * w00 + __ldg(sp + o01) * w01 + __ldg(sp + o10) * w10 + __ldg(sp + o11) * w11;
    if (composite) v = v * wm + (1.f - wm);  // warped_cloth * mask + white * (1 - mask)  (train_generator.py:244, test_generator.py:178)
    *dp = v;
  }
}

// ---------------------------------------------------------------------------------------------- hi-res flow warp backward
// d flow_lo of flow_warp_nchw_kernel (without overlap / composite), in three gathers with fixed summation orders:
//   1. thread = hi-res pixel: the analytic coordinate gradient of grid_sample (bilinear, border; a coordinate clamped or exactly on
//      the border gets none), summing the C channels and then the mask in that order, times d ix / d flow = (size/2) / div;
//   2. thread = (n, hi-res row y, lo-res column X): R[y][X] = sum over hi-res columns x (ascending) of wx(x, X) * dhi[y][x];
//   3. thread = (n, Y, X): dflow_lo[Y][X] = sum over hi-res rows y (ascending) of wy(y, Y) * R[y][X]
// — 2 and 3 are the adjoint of F.interpolate(size, bilinear, align_corners=False), row then column.
__device__ __forceinline__ void resize_taps(float sc, int d, int n_lo, int& i0, int& i1, float& l, float& h) {
  const float f = fmaxf(__fsub_rn(__fmul_rn(sc, __fadd_rn((float)d, 0.5f)), 0.5f), 0.f);
  i0 = (int)f;
  i1 = min(i0 + 1, n_lo - 1);
  l = __fsub_rn(f, (float)i0);
  h = __fsub_rn(1.f, l);
}
__global__ void __launch_bounds__(256) flow_warp_nchw_bwd_coord_kernel(const float* __restrict__ flow_lo, int hl, int wl, const float* __restrict__ lin_x,
                                                                      const float* __restrict__ lin_y, const float* __restrict__ src, int C, int Hs, int Ws,
                                                                      const float* __restrict__ d_dst, int H, int W, float div_x, float div_y,
                                                                      float sc_y, float sc_x, const float* __restrict__ mask_src,
                                                                      const float* __restrict__ d_mask, float2* __restrict__ dhi, long long npix) {
  const long long pix = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= npix) return;
  const int x = (int)(pix % W), y = (int)((pix / W) % H), n = (int)(pix / ((long long)W * H));
  int y0, y1, x0, x1;
  float ly, hy, lx, hx;
  resize_taps(sc_y, y, hl, y0, y1, ly, hy);
  resize_taps(sc_x, x, wl, x0, x1, lx, hx);
  const float2* fl = reinterpret_cast<const float2*>(flow_lo) + (long long)n * hl * wl;
  const float2 f00 = __ldg(fl + (long long)y0 * wl + x0), f01 = __ldg(fl + (long long)y0 * wl + x1);
  const float2 f10 = __ldg(fl + (long long)y1 * wl + x0), f11 = __ldg(fl + (long long)y1 * wl + x1);
  const float ux = __fadd_rn(__fmul_rn(hy, __fadd_rn(__fmul_rn(hx, f00.x), __fmul_rn(lx, f01.x))), __fmul_rn(ly, __fadd_rn(__fmul_rn(hx, f10.x), __fmul_rn(lx, f11.x))));
  const float uy = __fadd_rn(__fmul_rn(hy, __fadd_rn(__fmul_rn(hx, f00.y), __fmul_rn(lx, f01.y))), __fmul_rn(ly, __fadd_rn(__fmul_rn(hx, f10.y), __fmul_rn(lx, f11.y))));
  const float gx = __fadd_rn(__fdiv_rn(ux, div_x), __ldg(lin_x + x));
  const float gy = __fadd_rn(__fdiv_rn(uy, div_y), __ldg(lin_y + y));
  const float ixr = __fdiv_rn(__fsub_rn(__fmul_rn(__fadd_rn(gx, 1.f), (float)Ws), 1.f), 2.f);
  const float iyr = __fdiv_rn(__fsub_rn(__fmul_rn(__fadd_rn(gy, 1.f), (float)Hs), 1.f), 2.f);
  const float ix = fminf(fmaxf(ixr, 0.f), (float)(Ws - 1)), iy = fminf(fmaxf(iyr, 0.f), (float)(Hs - 1));
  const float mx = (ixr <= 0.f || ixr >= (float)(Ws - 1)) ? 0.f : 1.f;
  const float my = (iyr <= 0.f || iyr >= (float)(Hs - 1)) ? 0.f : 1.f;
  const float bx = floorf(ix), by = floorf(iy);
  const int sx0 = (int)bx, sy0 = (int)by;
  const float tx = __fsub_rn(ix, bx), ty = __fsub_rn(iy, by);
  const bool vx = sx0 + 1 <= Ws - 1, vy = sy0 + 1 <= Hs - 1;
  const int sx1 = vx ? sx0 + 1 : sx0, sy1 = vy ? sy0 + 1 : sy0;
  const float wx0 = 1.f - tx, wy0 = 1.f - ty, wx1 = vx ? tx : 0.f, wy1 = vy ? ty : 0.f;
  const long long plane_s = (long long)Hs * Ws, plane_d = (long long)H * W;
  const long long o00 = (long long)sy0 * Ws + sx0, o01 = (long long)sy0 * Ws + sx1, o10 = (long long)sy1 * Ws + sx0, o11 = (long long)sy1 * Ws + sx1;
  const long long dpix = (long long)y * W + x;
  float dix = 0.f, diy = 0.f;
  // value = a*wy0*wx0 + b*wy0*wx1 + c*wy1*wx0 + e*wy1*wx1 ; taps outside the image carry zero weight AND zero derivative
  for (int ch = 0; ch <= C; ++ch) {
    const float* sp;
    float d;
    if (ch < C) {
      if (!d_dst) continue;
      sp = src + ((long long)n * C + ch) * plane_s;
      d = __ldg(d_dst + ((long long)n * C + ch) * plane_d + dpix);
    } else {
      if (!d_mask) break;
      sp = mask_src + (long long)n * plane_s;
      d = __ldg(d_mask + (long long)n * plane_d + dpix);
    }
    const float a = __ldg(sp + o00), b = vx ? __ldg(sp + o01) : 0.f, c = vy ? __ldg(sp + o10) : 0.f, e = (vx && vy) ? __ldg(sp + o11) : 0.f;
    dix = __fadd_rn(dix, __fmul_rn(d, __fadd_rn(__fmul_rn(__fsub_rn(b, a), wy0), __fmul_rn(__fsub_rn(e, c), wy1))));
    diy = __fadd_rn(diy, __fmul_rn(d, __fadd_rn(__fmul_rn(__fsub_rn(c, a), wx0), __fmul_rn(__fsub_rn(e, b), wx1))));
  }
  dhi[pix] = make_float2(dix * mx * (0.5f * (float)Ws) / div_x, diy * my * (0.5f * (float)Hs) / div_y);
}

// First hi-res index d whose lower resize tap i0(d) is >= target (i0 is non-decreasing in d).
__device__ __forceinline__ int first_hi(float sc, int target, int n_hi, int n_lo) {
  int d = max(0, (int)(((float)target + 0.5f) / sc - 0.5f) - 2);
  int i0, i1;
  float l, h;
  while (d > 0) {
    resize_taps(sc, d - 1, n_lo, i0, i1, l, h);
    if (i0 < target) break;
    --d;
  }
  while (d < n_hi) {
    resize_taps(sc, d, n_lo, i0, i1, l, h);
    if (i0 >= target) break;
    ++d;
  }
  return d;
}

// Adjoint of the resize along one axis, as a gather onto lo-res index L: sum over hi-res d (ascending) whose taps i0 / i1 are L.
// in: element (d) at in[d * stride]; float2 values.
__device__ __forceinline__ float2 resize_adjoint(const float2* __restrict__ in, long long stride, float sc, int L, int n_hi, int n_lo) {
  float2 acc = make_float2(0.f, 0.f);
  for (int d = first_hi(sc, L - 1, n_hi, n_lo); d < n_hi; ++d) {
    int i0, i1;
    float l, h;
    resize_taps(sc, d, n_lo, i0, i1, l, h);
    if (i0 > L) break;
    const float2 v = in[(long long)d * stride];
    if (i0 == L) { acc.x = __fadd_rn(acc.x, __fmul_rn(h, v.x)); acc.y = __fadd_rn(acc.y, __fmul_rn(h, v.y)); }
    if (i1 == L) { acc.x = __fadd_rn(acc.x, __fmul_rn(l, v.x)); acc.y = __fadd_rn(acc.y, __fmul_rn(l, v.y)); }
  }
  return acc;
}
__global__ void __launch_bounds__(256) resize_adjoint_rows_kernel(const float2* __restrict__ dhi, int H, int W, int wl, float sc_x,
                                                                 float2* __restrict__ rows, long long total) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int X = (int)(i % wl);
  const long long ny = i / wl;  // n * H + y
  rows[i] = resize_adjoint(dhi + ny * W, 1, sc_x, X, W, wl);
}
__global__ void __launch_bounds__(256) resize_adjoint_cols_kernel(const float2* __restrict__ rows, int H, int hl, int wl, float sc_y,
                                                                 float2* __restrict__ dlo, long long total) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int X = (int)(i % wl), Y = (int)((i / wl) % hl), n = (int)(i / ((long long)wl * hl));
  dlo[i] = resize_adjoint(rows + (long long)n * H * wl + X, wl, sc_y, Y, H, hl);
}

// ---------------------------------------------------------------------------------------------- label map -> one-hot planes
// Input feeding (SURVEY.md 8f N4; cp_dataset.py:150-172 builds the 13-channel one-hot parse map on the CPU and ships it as fp32):
// the host ships ONE byte per pixel, this kernel expands it on the device.  out[n,c,p] = (label[n,p] == c).  thread = pixel.
__global__ void __launch_bounds__(256) onehot_u8_kernel(const unsigned char* __restrict__ lab, float* __restrict__ out, int C, long long hw, long long npix) {
  const long long pix = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= npix) return;
  const long long n = pix / hw, p = pix - n * hw;
  const int l = (int)__ldg(lab + pix);
  float* o = out + n * C * hw + p;
  for (int c = 0; c < C; ++c) o[(long long)c * hw] = (c == l) ? 1.f : 0.f;
}

// ---------------------------------------------------------------------------------------------- im2col for tiny-Cin convolutions
// dst[n,y,x, tap*C + ci] = src[n, y+ky-pad, x+kx-pad, ci] (zero outside / beyond taps*C).  A 3x3 convolution over a 7-channel
// label map (SPADE's mlp_shared, network_generator.py:182-184) becomes ONE K=64 GEMM block per pixel tile instead of nine K=16
// taps, and its weight gradient a plain 1x1 GEMM.  thread = (pixel, 8-channel group of dst)
// E = the raw storage element: unsigned short (either 16-bit type, moved as bits) or float (fp32 storage).
template <typename E>
__global__ void im2col_kernel(GView src, GView dst, int kh, int kw, int pad, int Gd, long long total) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int g = (int)(idx % Gd);
  const long long pix = idx / Gd;
  const int x = (int)(pix % dst.w), y = (int)((pix / dst.w) % dst.h), n = (int)(pix / ((long long)dst.w * dst.h));
  const int K = kh * kw * src.c;
  const E* s = reinterpret_cast<const E*>(src.ptr);
  E v[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int j = g * 8 + i;
    E o = 0;
    if (j < K) {
      const int tap = j / src.c, ci = j - tap * src.c;
      const int ky = tap / kw, kx = tap - ky * kw;
      const int sy = y + ky - pad, sx = x + kx - pad;
      if (sy >= 0 && sy < src.h && sx >= 0 && sx < src.w) o = __ldg(s + (((long long)n * src.h + sy) * src.w + sx) * src.pitch + ci);
    }
    v[i] = o;
  }
  if constexpr (sizeof(E) == 2) {
    uint4 o4;
    o4.x = v[0] | ((unsigned)v[1] << 16); o4.y = v[2] | ((unsigned)v[3] << 16); o4.z = v[4] | ((unsigned)v[5] << 16); o4.w = v[6] | ((unsigned)v[7] << 16);
    st16(at_w(dst, n, y, x) + g * 8, o4);
  } else {
    float4* o = reinterpret_cast<float4*>(reinterpret_cast<float*>(const_cast<void*>(dst.ptr)) + (((long long)n * dst.h + y) * dst.w + x) * dst.pitch + g * 8);
    o[0] = make_float4(v[0], v[1], v[2], v[3]);
    o[1] = make_float4(v[4], v[5], v[6], v[7]);
  }
}

// 3x3 / 7-channel specialisation (the SPADE label map): thread = pixel; nine 16-byte loads (one per tap, the 8th lane is the
// buffer's zero pad channel), the 63 values are re-packed with compile-time indices, eight 16-byte stores (128 contiguous bytes).
__device__ __forceinline__ uint32_t half_of(const uint4& u, int ci) {
  const uint32_t w = ci < 2 ? u.x : (ci < 4 ? u.y : (ci < 6 ? u.z : u.w));
  return (ci & 1) ? (w >> 16) : (w & 0xFFFFu);
}
__global__ void __launch_bounds__(256) im2col3x3_c7_kernel(GView src, GView dst, long long npix) {
  const long long pix = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= npix) return;
  const int x = (int)(pix % dst.w), y = (int)((pix / dst.w) % dst.h), n = (int)(pix / ((long long)dst.w * dst.h));
  uint4 t[9];
#pragma unroll
  for (int tap = 0; tap < 9; ++tap) {
    const int sy = y + tap / 3 - 1, sx = x + tap % 3 - 1;
    t[tap] = (sy >= 0 && sy < src.h && sx >= 0 && sx < src.w) ? ld16(at(src, n, sy, sx)) : make_uint4(0, 0, 0, 0);
  }
  __nv_bfloat16* o = at_w(dst, n, y, x);
#pragma unroll
  for (int g = 0; g < 8; ++g) {
    uint32_t w[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int j0 = g * 8 + 2 * q, j1 = j0 + 1;
      const uint32_t lo = j0 < 63 ? half_of(t[j0 / 7], j0 % 7) : 0u;
      const uint32_t hi = j1 < 63 ? half_of(t[j1 / 7], j1 % 7) : 0u;
      w[q] = lo | (hi << 16);
    }
    st16(o + g * 8, make_uint4(w[0], w[1], w[2], w[3]));
  }
}

// ---------------------------------------------------------------------------------------------- L1 feature loss
// sum |a - b| over the (n,h,w,c) views (every block writes its fp64 partial to slab[blockIdx.x]; l1_finish_kernel adds them in
// a fixed order), and its gradient da = sign(a - b) * (*gscale).
__global__ void __launch_bounds__(256) l1_fwd_kernel(GView a, GView b, int G, long long total, double* __restrict__ slab) {
  float acc = 0.f;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const int g = (int)(idx % G);
    const long long pix = idx / G;
    float fa[8], fb[8];
    un8(ld16(reinterpret_cast<const __nv_bfloat16*>(a.ptr) + pix * a.pitch + g * 8), fa);
    un8(ld16(reinterpret_cast<const __nv_bfloat16*>(b.ptr) + pix * b.pitch + g * 8), fb);
    const int lim = min(8, a.c - g * 8);
#pragma unroll
    for (int i = 0; i < 8; ++i)
      if (i < lim) acc += fabsf(fa[i] - fb[i]);
  }
  __shared__ float red[8];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int i = 0; i < 8; ++i) t += (double)red[i];
    slab[blockIdx.x] = t;
  }
}
// One block of 256 threads: thread t adds the slabs of its contiguous range [t*k, (t+1)*k) in order, then a fixed shared-memory
// tree combines the 256 partials — the same order on every launch, without one thread walking thousands of slabs serially.
__global__ void __launch_bounds__(256) l1_finish_kernel(const double* __restrict__ slab, int nb, double* __restrict__ out) {
  __shared__ double part[256];
  const int k = (nb + 255) / 256, b = threadIdx.x * k, e = min(b + k, nb);
  double t = 0.0;
#pragma unroll 4
  for (int i = b; i < e; ++i) t += slab[i];
  part[threadIdx.x] = t;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if (threadIdx.x < s) part[threadIdx.x] += part[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) *out = part[0];
}
__global__ void l1_bwd_kernel(GView a, GView b, GView da, int G, long long total, const float* __restrict__ gscale, int relu_gate) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int g = (int)(idx % G);
  const long long pix = idx / G;
  const float gs = __ldg(gscale);
  float fa[8], fb[8], o[8];
  un8(ld16(reinterpret_cast<const __nv_bfloat16*>(a.ptr) + pix * a.pitch + g * 8), fa);
  un8(ld16(reinterpret_cast<const __nv_bfloat16*>(b.ptr) + pix * b.pitch + g * 8), fb);
  const int lim = min(8, a.c - g * 8);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const float d = fa[i] - fb[i];
    o[i] = (i < lim && !(relu_gate && fa[i] <= 0.f)) ? (d > 0.f ? gs : (d < 0.f ? -gs : 0.f)) : 0.f;
  }
  st16(reinterpret_cast<__nv_bfloat16*>(const_cast<void*>(da.ptr)) + pix * da.pitch + g * 8, pk8(o));
}

// ---------------------------------------------------------------------------------------------- loss-scaling gradient pass
// g *= *inv_scale in place over a device table of fp32 segments; found_inf = 1 if any input element is inf or NaN.  Each segment is
// cut into chunks of kUnChunk float4 starting at its first 16-byte boundary; chunk k of the concatenated chunk sequence belongs to
// block k % gridDim.x, so large and small segments spread over all blocks without a prefix-sum table.  Every block walks the whole
// table, staged through shared memory kUnThreads descriptors at a time.  The block that owns a segment's chunk 0 also handles the
// (at most 3 + 3) elements before the first and after the last 16-byte boundary.
constexpr int kUnThreads = 256, kUnVec = 4;
constexpr long long kUnChunk = (long long)kUnThreads * kUnVec;  // float4 per chunk: 16 KiB
__device__ __forceinline__ bool nonfinite(float v) { return (__float_as_uint(v) & 0x7f800000u) == 0x7f800000u; }
__device__ __forceinline__ void unscale1(float& v, float s, bool& bad) {
  bad |= nonfinite(v);
  v = __fmul_rn(v, s);
}
// the table's pointers come through shared memory: the explicit .global accesses spare the generic-address check
__device__ __forceinline__ void unscale_at(float* p, float s, bool& bad) {
  float v = __ldcg(p);
  unscale1(v, s, bad);
  __stcg(p, v);
}

__global__ void __launch_bounds__(kUnThreads) grad_unscale_check_kernel(const hrv_grad_segment* __restrict__ segs, int nseg,
                                                                        const float* __restrict__ inv_scale, float* __restrict__ found_inf) {
  __shared__ hrv_grad_segment tab[kUnThreads];
  const float s = __ldg(inv_scale);
  const unsigned G = gridDim.x;
  bool bad = false;
  unsigned long long base = 0;  // chunks of all earlier segments
  for (int s0 = 0; s0 < nseg; s0 += kUnThreads) {
    const int cnt = min(kUnThreads, nseg - s0);
    __syncthreads();
    if ((int)threadIdx.x < cnt) tab[threadIdx.x] = segs[s0 + threadIdx.x];
    __syncthreads();
    for (int i = 0; i < cnt; ++i) {
      float* p = tab[i].ptr;
      const long long n = tab[i].n;
      const long long head = min(n, (long long)((((uintptr_t)0 - (uintptr_t)p) & 15) >> 2));
      const long long nv = (n - head) >> 2, tail = n - head - 4 * nv;
      const long long nc = nv ? (nv + kUnChunk - 1) / kUnChunk : (n ? 1 : 0);
      const unsigned r = (unsigned)(base % G);
      long long c = blockIdx.x >= r ? blockIdx.x - r : blockIdx.x + G - r;  // first chunk of this segment owned by this block
      base += nc;
      if (c == 0) {
        if ((long long)threadIdx.x < head) unscale_at(p + threadIdx.x, s, bad);
        if ((long long)threadIdx.x < tail) unscale_at(p + head + 4 * nv + threadIdx.x, s, bad);
      }
      float4* q = reinterpret_cast<float4*>(p + head);
      for (; c < nc; c += G) {
        const long long b = c * kUnChunk, lim = min(kUnChunk, nv - b);
        float4 v[kUnVec];
#pragma unroll
        for (int u = 0; u < kUnVec; ++u) {
          const long long j = threadIdx.x + u * kUnThreads;
          if (j < lim) v[u] = __ldcg(q + b + j);
        }
#pragma unroll
        for (int u = 0; u < kUnVec; ++u) {
          const long long j = threadIdx.x + u * kUnThreads;
          if (j < lim) {
            unscale1(v[u].x, s, bad); unscale1(v[u].y, s, bad); unscale1(v[u].z, s, bad); unscale1(v[u].w, s, bad);
            __stcg(q + b + j, v[u]);
          }
        }
      }
    }
  }
  if (__syncthreads_or(bad) && threadIdx.x == 0) *found_inf = 1.f;
}

}  // namespace
}  // namespace hrv

using namespace hrv;

extern "C" int hrv_space_to_depth_bwd(const hrv_tensor* d, const hrv_tensor* dx, hrv_stream stream) {
  int rc;
  if ((rc = check_vec(d, "s2d_bwd d")) || (rc = check_vec(dx, "s2d_bwd dx"))) return rc;
  const int G = (dx->c + 7) / 8;
  if (d->n != dx->n || d->h != (dx->h + 1) / 2 || d->w != (dx->w + 1) / 2 || d->pitch < 4 * G * 8 || dx->pitch < G * 8)
    return set_error(HRV_EINVAL, "s2d_bwd: extents (d %dx%dx%d for dx %dx%dx%d)", d->h, d->w, d->c, dx->h, dx->w, dx->c);
  const long long total = (long long)dx->n * dx->h * dx->w * G;
  if (total) space_to_depth_bwd_kernel<<<nblocks(total, 256), 256, 0, (cudaStream_t)stream>>>(gv(d), gv(dx), G, total);
  return launched("space_to_depth_bwd");
}

extern "C" int hrv_maxpool2_fwd(const hrv_tensor* x, const hrv_tensor* y, hrv_stream stream) {
  int rc;
  if ((rc = check_vec(x, "maxpool x")) || (rc = check_vec(y, "maxpool y"))) return rc;
  if (y->n != x->n || y->h != x->h / 2 || y->w != x->w / 2 || y->c != x->c) return set_error(HRV_EINVAL, "maxpool: y must be (n, h/2, w/2, c)");
  const int G = (x->c + 7) / 8;
  const long long total = (long long)y->n * y->h * y->w * G;
  if (total) maxpool2_fwd_kernel<<<nblocks(total, 256), 256, 0, (cudaStream_t)stream>>>(gv(x), gv(y), G, total);
  return launched("maxpool2_fwd");
}

extern "C" int hrv_maxpool2_bwd(const hrv_tensor* x, const hrv_tensor* dy, const hrv_tensor* dx, int32_t relu_gate, hrv_stream stream) {
  int rc;
  if ((rc = check_vec(x, "maxpool_bwd x")) || (rc = check_vec(dy, "maxpool_bwd dy")) || (rc = check_vec(dx, "maxpool_bwd dx"))) return rc;
  if (dy->n != x->n || dy->h != x->h / 2 || dy->w != x->w / 2 || dy->c != x->c || dx->n != x->n || dx->h != x->h || dx->w != x->w || dx->c != x->c)
    return set_error(HRV_EINVAL, "maxpool_bwd: extents");
  if ((x->h | x->w) & 1) {  // rows / columns the floor-mode pool never reads get a zero gradient
    cudaError_t e = cudaMemsetAsync(const_cast<void*>(dx->ptr), 0, (size_t)dx->n * dx->h * dx->w * dx->pitch * 2, (cudaStream_t)stream);
    if (e != cudaSuccess) return set_error(HRV_ECUDA, "maxpool_bwd memset: %s", cudaGetErrorString(e));
  }
  const int G = (x->c + 7) / 8;
  const long long total = (long long)dy->n * dy->h * dy->w * G;
  if (total) maxpool2_bwd_kernel<<<nblocks(total, 256), 256, 0, (cudaStream_t)stream>>>(gv(x), gv(dy), gv(dx), G, total, relu_gate);
  return launched("maxpool2_bwd");
}

extern "C" int hrv_avgpool3s2_bwd(const hrv_tensor* dy, const hrv_tensor* dx, hrv_stream stream) {
  int rc;
  if ((rc = check_vec(dy, "avgpool_bwd dy")) || (rc = check_vec(dx, "avgpool_bwd dx"))) return rc;
  if (dy->n != dx->n || dy->h != (dx->h - 1) / 2 + 1 || dy->w != (dx->w - 1) / 2 + 1) return set_error(HRV_EINVAL, "avgpool_bwd: extents");
  const int G = (dx->c + 7) / 8;
  if (dy->pitch < G * 8) return set_error(HRV_EINVAL, "avgpool_bwd: dy has fewer channel groups than dx");
  const long long total = (long long)dx->n * dx->h * dx->w * G;
  if (total) avgpool3s2_bwd_kernel<<<nblocks(total, 256), 256, 0, (cudaStream_t)stream>>>(gv(dy), gv(dx), G, total);
  return launched("avgpool3s2_bwd");
}

extern "C" int hrv_parse_blur_argmax(const float* seg, int32_t n, int32_t c, int32_t h, int32_t w, int32_t H, int32_t W,
                                     const int32_t* group_of, int32_t groups, int64_t* idx, float* onehot, uint32_t occl_mask,
                                     float* overlap, hrv_stream stream) {
  if (!seg || (!idx && !onehot && !overlap) || n < 1 || c < 1 || c > 32 || h < 1 || w < 1 || H < 1 || W < 1)
    return set_error(HRV_EINVAL, "parse_blur_argmax: bad arguments (c must be <= 32)");
  if (onehot && (!group_of || groups < 1)) return set_error(HRV_EINVAL, "parse_blur_argmax: onehot needs group_of / groups");
  ParseArgs a;
  memset(&a, 0, sizeof(a));
  a.seg = seg; a.idx = (long long*)idx; a.onehot = onehot; a.overlap = overlap; a.occl_mask = occl_mask;
  a.n = n; a.C = c; a.h = h; a.w = w; a.H = H; a.W = W; a.groups = groups;
  a.sy = (float)h / (float)H; a.sx = (float)w / (float)W;
  double g[15], sum = 0;
  for (int k = 0; k < 15; ++k) { g[k] = (double)expf(-(float)((k - 7) * (k - 7)) / 18.f); sum += g[k]; }
  float fsum = 0.f;
  for (int k = 0; k < 15; ++k) fsum += (float)g[k];
  (void)sum;
  for (int k = 0; k < 15; ++k) a.g[k] = (float)g[k] / fsum;
  for (int k = 0; k < c; ++k) {
    a.group_of[k] = group_of ? group_of[k] : k;
    if (onehot && (a.group_of[k] < 0 || a.group_of[k] >= groups)) return set_error(HRV_EINVAL, "parse_blur_argmax: group_of[%d] out of range", k);
  }
  dim3 grid((W + kTile - 1) / kTile, (H + kTile - 1) / kTile, n);
  parse_blur_argmax_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(a);
  return launched("parse_blur_argmax");
}

extern "C" int hrv_onehot_u8(const uint8_t* labels, int32_t n, int32_t classes, int32_t h, int32_t w, float* out, hrv_stream stream) {
  if (!labels || !out || n < 1 || classes < 1 || h < 1 || w < 1) return set_error(HRV_EINVAL, "onehot_u8: bad arguments");
  const long long hw = (long long)h * w, npix = hw * n;
  onehot_u8_kernel<<<nblocks(npix, 256), 256, 0, (cudaStream_t)stream>>>(labels, out, classes, hw, npix);
  return launched("onehot_u8");
}

extern "C" int hrv_gaussian_blur(const float* src, int32_t planes, int32_t h, int32_t w, int32_t ksize, float sigma, float* dst,
                                 hrv_stream stream) {
  if (!src || !dst || planes < 1 || h < 1 || w < 1 || ksize < 1 || !(ksize & 1) || ksize > 2 * kBlurMaxR + 1 || !(sigma > 0.f))
    return set_error(HRV_EINVAL, "gaussian_blur: odd ksize <= %d, sigma > 0", 2 * kBlurMaxR + 1);
  BlurArgs a;
  memset(&a, 0, sizeof(a));
  a.src = src; a.dst = dst; a.planes = planes; a.H = h; a.W = w; a.r = ksize / 2;
  float g[2 * kBlurMaxR + 1], fsum = 0.f;
  for (int k = 0; k < ksize; ++k) { g[k] = expf(-(float)((k - a.r) * (k - a.r)) / (2.f * sigma * sigma)); fsum += g[k]; }
  for (int k = 0; k < ksize; ++k) a.g[k] = g[k] / fsum;
  dim3 grid((w + kTile - 1) / kTile, (h + kTile - 1) / kTile, planes);
  gaussian_blur_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(a);
  return launched("gaussian_blur");
}

extern "C" int hrv_flow_warp_nchw(const float* flow_lo, int32_t n, int32_t hl, int32_t wl, const float* lin_x, const float* lin_y,
                                  const float* src, int32_t c, int32_t hs, int32_t ws, float* dst, int32_t h, int32_t w, float div_x,
                                  float div_y, float* grid_out, const float* mask_src, const float* overlap, float* mask_out,
                                  int32_t composite, hrv_stream stream) {
  if (!flow_lo || !lin_x || !lin_y || !src || !dst || n < 1 || hl < 1 || wl < 1 || c < 1 || hs < 1 || ws < 1 || h < 1 || w < 1)
    return set_error(HRV_EINVAL, "flow_warp_nchw: bad arguments");
  if ((overlap || mask_out || composite) && !mask_src) return set_error(HRV_EINVAL, "flow_warp_nchw: overlap / mask_out / composite need mask_src");
  const long long npix = (long long)n * h * w;
  flow_warp_nchw_kernel<<<nblocks(npix, 256), 256, 0, (cudaStream_t)stream>>>(flow_lo, hl, wl, lin_x, lin_y, src, c, hs, ws, dst, h, w, div_x,
                                                                             div_y, (float)hl / (float)h, (float)wl / (float)w, grid_out, mask_src,
                                                                             overlap, mask_out, composite, npix);
  return launched("flow_warp_nchw");
}

extern "C" size_t hrv_flow_warp_nchw_bwd_workspace_bytes(int32_t n, int32_t h, int32_t w, int32_t wl) {
  if (n < 1 || h < 1 || w < 1 || wl < 1) return 0;
  return ((size_t)n * h * w + (size_t)n * h * wl) * sizeof(float2);
}

extern "C" int hrv_flow_warp_nchw_bwd(const float* flow_lo, int32_t n, int32_t hl, int32_t wl, const float* lin_x, const float* lin_y,
                                      const float* src, int32_t c, int32_t hs, int32_t ws, const float* d_dst, int32_t h, int32_t w,
                                      float div_x, float div_y, const float* mask_src, const float* d_mask, float* d_flow_lo,
                                      void* workspace, size_t workspace_bytes, hrv_stream stream) {
  if (!flow_lo || !lin_x || !lin_y || !d_flow_lo || n < 1 || hl < 1 || wl < 1 || c < 0 || hs < 1 || ws < 1 || h < 1 || w < 1)
    return set_error(HRV_EINVAL, "flow_warp_nchw_bwd: bad arguments");
  if ((d_dst && (!src || c < 1)) || (d_mask && !mask_src) || (!d_dst && !d_mask))
    return set_error(HRV_EINVAL, "flow_warp_nchw_bwd: d_dst needs src, d_mask needs mask_src, and one of them is required");
  const size_t need = hrv_flow_warp_nchw_bwd_workspace_bytes(n, h, w, wl);
  if (!workspace || workspace_bytes < need) return set_error(HRV_EINVAL, "flow_warp_nchw_bwd: workspace too small (%zu < %zu)", workspace_bytes, need);
  cudaStream_t st = (cudaStream_t)stream;
  float2* dhi = (float2*)workspace;
  float2* rows = dhi + (size_t)n * h * w;
  const float sc_y = (float)hl / (float)h, sc_x = (float)wl / (float)w;
  const long long npix = (long long)n * h * w;
  flow_warp_nchw_bwd_coord_kernel<<<nblocks(npix, 256), 256, 0, st>>>(flow_lo, hl, wl, lin_x, lin_y, d_dst ? src : nullptr, d_dst ? c : 0, hs, ws,
                                                                      d_dst, h, w, div_x, div_y, sc_y, sc_x, mask_src, d_mask, dhi, npix);
  int rc;
  if ((rc = launched("flow_warp_nchw_bwd"))) return rc;
  const long long nr = (long long)n * h * wl, nl = (long long)n * hl * wl;
  resize_adjoint_rows_kernel<<<nblocks(nr, 256), 256, 0, st>>>(dhi, h, w, wl, sc_x, rows, nr);
  if ((rc = launched("resize_adjoint_rows"))) return rc;
  resize_adjoint_cols_kernel<<<nblocks(nl, 256), 256, 0, st>>>(rows, h, hl, wl, sc_y, (float2*)d_flow_lo, nl);
  return launched("resize_adjoint_cols");
}

extern "C" int hrv_im2col(const hrv_tensor* src, const hrv_tensor* dst, int32_t kh, int32_t kw, int32_t pad, hrv_stream stream) {
  int rc;
  const bool f32 = src && src->dtype == HRV_F32;  // fp32 storage: the generic kernel on 4-byte elements, dst fp32 as well
  const int dt = f32 ? HRV_F32 : HRV_BF16;
  if ((rc = check_vec(src, "im2col src", dt)) || (rc = check_vec(dst, "im2col dst", dt))) return rc;
  if (kh < 1 || kw < 1 || dst->n != src->n || dst->h != src->h || dst->w != src->w || dst->c < kh * kw * src->c || (dst->c % 8))
    return set_error(HRV_EINVAL, "im2col: dst must be (n,h,w, >= kh*kw*c, multiple of 8)");
  const int Gd = dst->c / 8;
  const long long total = (long long)dst->n * dst->h * dst->w * Gd;
  const long long npix = (long long)dst->n * dst->h * dst->w;
  if (f32) {
    if (total) im2col_kernel<float><<<nblocks(total, 256), 256, 0, (cudaStream_t)stream>>>(gv(src), gv(dst), kh, kw, pad, Gd, total);
  } else if (kh == 3 && kw == 3 && pad == 1 && src->c == 7 && dst->c == 64) {
    if (npix) im2col3x3_c7_kernel<<<nblocks(npix, 256), 256, 0, (cudaStream_t)stream>>>(gv(src), gv(dst), npix);
  } else if (total) {
    im2col_kernel<unsigned short><<<nblocks(total, 256), 256, 0, (cudaStream_t)stream>>>(gv(src), gv(dst), kh, kw, pad, Gd, total);
  }
  return launched("im2col");
}

static int l1_check(const hrv_tensor* a, const hrv_tensor* b) {
  int rc;
  if ((rc = check_vec(a, "l1 a")) || (rc = check_vec(b, "l1 b"))) return rc;
  if (a->n != b->n || a->h != b->h || a->w != b->w || a->c != b->c) return set_error(HRV_EINVAL, "l1: shape mismatch");
  return HRV_OK;
}

static long long l1_blocks(const hrv_tensor* a) {
  const long long total = (long long)a->n * a->h * a->w * ((a->c + 7) / 8);
  const long long want = (total + 255) / 256, cap = (long long)sm_count() * 16;
  return want < cap ? want : cap;
}

extern "C" size_t hrv_l1_sum_workspace_bytes(const hrv_tensor* a) { return a ? (size_t)l1_blocks(a) * sizeof(double) : 0; }

extern "C" int hrv_l1_sum(const hrv_tensor* a, const hrv_tensor* b, double* sum, void* workspace, size_t workspace_bytes, hrv_stream stream) {
  int rc;
  if ((rc = l1_check(a, b))) return rc;
  if (!sum) return set_error(HRV_EINVAL, "l1_sum: null accumulator");
  const long long nb = l1_blocks(a);
  if (nb && (!workspace || workspace_bytes < (size_t)nb * sizeof(double)))
    return set_error(HRV_EINVAL, "l1_sum: workspace too small (%zu < %zu)", workspace_bytes, (size_t)nb * sizeof(double));
  cudaStream_t st = (cudaStream_t)stream;
  const int G = (a->c + 7) / 8;
  const long long total = (long long)a->n * a->h * a->w * G;
  if (nb) l1_fwd_kernel<<<(unsigned)nb, 256, 0, st>>>(gv(a), gv(b), G, total, (double*)workspace);
  if ((rc = launched("l1_sum"))) return rc;
  l1_finish_kernel<<<1, 256, 0, st>>>((const double*)workspace, (int)nb, sum);
  return launched("l1_sum finish");
}

extern "C" int hrv_l1_bwd(const hrv_tensor* a, const hrv_tensor* b, const float* gscale, const hrv_tensor* da, int32_t relu_gate, hrv_stream stream) {
  int rc;
  if ((rc = l1_check(a, b)) || (rc = l1_check(a, da))) return rc;
  if (!gscale) return set_error(HRV_EINVAL, "l1_bwd: null gscale");
  const int G = (a->c + 7) / 8;
  const long long total = (long long)a->n * a->h * a->w * G;
  if (total) l1_bwd_kernel<<<nblocks(total, 256), 256, 0, (cudaStream_t)stream>>>(gv(a), gv(b), gv(da), G, total, gscale, relu_gate);
  return launched("l1_bwd");
}

extern "C" int hrv_grad_unscale_check(const hrv_grad_segment* segments, int32_t num_segments, const float* inv_scale, float* found_inf,
                                      hrv_stream stream) {
  if (!segments || num_segments < 0 || !inv_scale || !found_inf) return set_error(HRV_EINVAL, "grad_unscale_check: bad arguments");
  if (num_segments == 0) return HRV_OK;
  // 8 blocks of 256 threads per SM (the thread limit), 4 x 16 bytes in flight per thread
  grad_unscale_check_kernel<<<(unsigned)sm_count() * 8, kUnThreads, 0, (cudaStream_t)stream>>>(segments, num_segments, inv_scale, found_inf);
  return launched("grad_unscale_check");
}
