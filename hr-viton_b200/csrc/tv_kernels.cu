// tv_kernels.cu — the stage-1 flow TV loss, plain and edge-aware (train_condition.py:183-232: --edgeawaretv last_only|weighted,
// --add_lasttv), forward and backward for up to HRV_TV_MAX_FLOWS flows in one call each.  The forward adds per-block partial sums in a
// fixed order; the backward is a gather on both sides (flow pixels read their neighbour pairs, mask pixels read the few flow-resolution
// pixels whose bilinear taps touch them), so there are no atomics and every run gives the same bits.  fp32 only: the TU is compiled in
// both library flavours, identically.
#include "hrv_bilinear.cuh"
#include "hrv_host.h"

namespace hrv {
namespace {

using hrv_bilinear::Taps;
using hrv_bilinear::bilinear_taps;

constexpr int kTvThreads = 256;
constexpr int kTvBlocks = 64;  // blocks per flow of the forward sums: fixed, so the summation order depends on the shapes alone
constexpr float kEdge = -150.f;

struct TvFlow {
  const float* flow;  // [n][h][w][2]
  float* dflow;
  float* m;   // workspace: F.interpolate(mask, (h, w)) [n][h][w]
  float* dm;  // workspace: its gradient
  int h, w;
  float we, wp;
};
struct TvArgs {
  TvFlow f[HRV_TV_MAX_FLOWS];
  int nflows, n;
  const float* mask;  // [n][mh][mw] or NULL
  int mh, mw;
  double* slab;  // [nflows][kTvBlocks][4]: {sum |D_y| e_y, sum |D_x| e_x, sum |D_y|, sum |D_x|}
  const float* dloss;
  float* dmask;
};

__device__ __forceinline__ float sgnf(float v) { return v > 0.f ? 1.f : (v < 0.f ? -1.f : 0.f); }

// m_i = F.interpolate(mask, (h_i, w_i), 'bilinear', align_corners=False).  grid (pixel blocks, flow)
__global__ void __launch_bounds__(kTvThreads) tv_mask_down_kernel(const __grid_constant__ TvArgs a) {
  const TvFlow& f = a.f[blockIdx.y];
  const long long npix = (long long)a.n * f.h * f.w;
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= npix) return;
  const int x = (int)(p % f.w), y = (int)((p / f.w) % f.h), n = (int)(p / ((long long)f.w * f.h));
  const Taps ty = bilinear_taps((float)a.mh / f.h, y, a.mh), tx = bilinear_taps((float)a.mw / f.w, x, a.mw);
  const float* src = a.mask + (long long)n * a.mh * a.mw;
  const float* r0 = src + (long long)ty.i0 * a.mw;
  const float* r1 = src + (long long)ty.i1 * a.mw;
  f.m[p] = hrv_bilinear::bilinear_blend(ty, tx, __ldg(r0 + tx.i0), __ldg(r0 + tx.i1), __ldg(r1 + tx.i0), __ldg(r1 + tx.i1));
}

__device__ __forceinline__ float edge(const float* m, long long p, long long q) { return expf(kEdge * fabsf(m[q] - m[p])); }

// Per-block sums of the four TV numerators of flow blockIdx.y: thread = pixel (grid-stride over kTvBlocks blocks), each pixel owns the
// pairs (y, y+1) and (x, x+1); fp32 per thread, fp64 across the warp and the block in a fixed tree.
__global__ void __launch_bounds__(kTvThreads) tv_sums_kernel(const __grid_constant__ TvArgs a) {
  const TvFlow& f = a.f[blockIdx.y];
  const long long npix = (long long)a.n * f.h * f.w;
  const float2* fl = reinterpret_cast<const float2*>(f.flow);
  float s[4] = {0.f, 0.f, 0.f, 0.f};
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < npix; p += (long long)kTvBlocks * blockDim.x) {
    const int x = (int)(p % f.w), y = (int)((p / f.w) % f.h);
    const float2 v = __ldg(fl + p);
    if (y < f.h - 1) {
      const long long q = p + f.w;
      const float2 u = __ldg(fl + q);
      const float d0 = fabsf(u.x - v.x), d1 = fabsf(u.y - v.y);
      const float e = a.mask ? edge(f.m, p, q) : 1.f;
      s[0] += d0 * e + d1 * e;
      s[2] += d0 + d1;
    }
    if (x < f.w - 1) {
      const long long q = p + 1;
      const float2 u = __ldg(fl + q);
      const float d0 = fabsf(u.x - v.x), d1 = fabsf(u.y - v.y);
      const float e = a.mask ? edge(f.m, p, q) : 1.f;
      s[1] += d0 * e + d1 * e;
      s[3] += d0 + d1;
    }
  }
  __shared__ double red[kTvThreads / 32][4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    double t = (double)s[k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5][k] = t;
  }
  __syncthreads();
  if (threadIdx.x < 4) {
    double t = 0.0;
    for (int wgrp = 0; wgrp < kTvThreads / 32; ++wgrp) t += red[wgrp][threadIdx.x];
    a.slab[((long long)blockIdx.y * kTvBlocks + blockIdx.x) * 4 + threadIdx.x] = t;
  }
}

// One warp: lane i < nflows adds flow i's slabs in block order and forms its term; lane 0 adds the terms in flow order.
__global__ void tv_finish_kernel(const __grid_constant__ TvArgs a, float* __restrict__ loss, float* __restrict__ terms) {
  __shared__ double term[HRV_TV_MAX_FLOWS];
  const int i = threadIdx.x;
  if (i < a.nflows) {
    const TvFlow& f = a.f[i];
    double s[4] = {0.0, 0.0, 0.0, 0.0};
    for (int b = 0; b < kTvBlocks; ++b)
      for (int k = 0; k < 4; ++k) s[k] += a.slab[((long long)i * kTvBlocks + b) * 4 + k];
    const double dy = 2.0 * a.n * (f.h - 1) * f.w, dx = 2.0 * a.n * f.h * (f.w - 1);
    term[i] = (double)f.we * (s[0] / dy + s[1] / dx) + (double)f.wp * (s[2] / dy + s[3] / dx);
    if (terms) terms[i] = (float)term[i];
  }
  __syncwarp();
  if (i == 0) {
    double t = 0.0;
    for (int k = 0; k < a.nflows; ++k) t += term[k];
    *loss = (float)t;
  }
}

// dflow and d m_i of flow blockIdx.y: thread = pixel p, gathering over the (up to four) pairs that contain p.  For the pair (p, q),
// q the next pixel along an axis with mean divisor D:  d loss / d|D f_c| = g (we e + wp) / D, and, with the mask,
// d loss / d(m[q] - m[p]) = -150 sgn(m[q] - m[p]) e (|D f_0| + |D f_1|) g we / D.
__global__ void __launch_bounds__(kTvThreads) tv_bwd_flow_kernel(const __grid_constant__ TvArgs a) {
  const TvFlow& f = a.f[blockIdx.y];
  const long long npix = (long long)a.n * f.h * f.w;
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= npix) return;
  const int x = (int)(p % f.w), y = (int)((p / f.w) % f.h);
  const float g = __ldg(a.dloss);
  const float cy = g / (2.f * a.n * (f.h - 1) * f.w), cx = g / (2.f * a.n * f.h * (f.w - 1));
  const float2* fl = reinterpret_cast<const float2*>(f.flow);
  float df0 = 0.f, df1 = 0.f, dm = 0.f;
  // (lo, hi) is the pair, sign = +1 when p is hi (d(f[hi] - f[lo]) / d f[p] = +1), -1 when p is lo
  auto pair = [&](long long lo, long long hi, float c, float sign) {
    const float2 u = __ldg(fl + lo), w = __ldg(fl + hi);
    const float d0 = w.x - u.x, d1 = w.y - u.y;
    float e = 1.f, dmd = 0.f;
    if (a.mask) {
      const float md = f.m[hi] - f.m[lo];
      e = expf(kEdge * fabsf(md));
      dmd = (c * f.we) * (fabsf(d0) + fabsf(d1)) * e * kEdge * sgnf(md);
    }
    const float k = c * (f.we * e + f.wp);
    df0 += sign * (sgnf(d0) * k);
    df1 += sign * (sgnf(d1) * k);
    dm += sign * dmd;
  };
  if (y < f.h - 1) pair(p, p + f.w, cy, -1.f);
  if (y > 0) pair(p - f.w, p, cy, 1.f);
  if (x < f.w - 1) pair(p, p + 1, cx, -1.f);
  if (x > 0) pair(p - 1, p, cx, 1.f);
  reinterpret_cast<float2*>(f.dflow)[p] = make_float2(df0, df1);
  if (a.mask) f.dm[p] = dm;
}

// First output index d (of n_out) whose lower tap i0(d) is >= target (i0 is non-decreasing in d).
__device__ __forceinline__ int first_out(float scale, int target, int n_out, int n_in) {
  int d = max(0, (int)(((float)target + 0.5f) / scale - 0.5f) - 2);
  while (d > 0 && bilinear_taps(scale, d - 1, n_in).i0 >= target) --d;
  while (d < n_out && bilinear_taps(scale, d, n_in).i0 < target) ++d;
  return d;
}

// dmask[n][Y][X] = sum over flows i (in order) of the adjoint of the interpolation applied to d m_i: rows y (ascending) whose taps
// include Y, each the sum over columns x (ascending) whose taps include X of wx * dm_i[y][x], times wy.  A tap counts once per
// coincidence (i0 == i1 == Y at the last row adds both lambdas), as torch's backward adds both.
__global__ void __launch_bounds__(kTvThreads) tv_bwd_mask_kernel(const __grid_constant__ TvArgs a) {
  const long long npix = (long long)a.n * a.mh * a.mw;
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= npix) return;
  const int X = (int)(p % a.mw), Y = (int)((p / a.mw) % a.mh), n = (int)(p / ((long long)a.mw * a.mh));
  float acc = 0.f;
  for (int i = 0; i < a.nflows; ++i) {
    const TvFlow& f = a.f[i];
    const float sy = (float)a.mh / f.h, sx = (float)a.mw / f.w;
    const float* dm = f.dm + (long long)n * f.h * f.w;
    const int x_first = first_out(sx, X - 1, f.w, a.mw);
    for (int y = first_out(sy, Y - 1, f.h, a.mh); y < f.h; ++y) {
      const Taps ty = bilinear_taps(sy, y, a.mh);
      if (ty.i0 > Y) break;
      const float wy = (ty.i0 == Y ? ty.l0 : 0.f) + (ty.i1 == Y ? ty.l1 : 0.f);
      if (wy == 0.f) continue;
      float row = 0.f;
      for (int x = x_first; x < f.w; ++x) {
        const Taps tx = bilinear_taps(sx, x, a.mw);
        if (tx.i0 > X) break;
        const float wx = (tx.i0 == X ? tx.l0 : 0.f) + (tx.i1 == X ? tx.l1 : 0.f);
        row += wx * dm[(long long)y * f.w + x];
      }
      acc += wy * row;
    }
  }
  a.dmask[p] = acc;
}

int launched(const char* what) {
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? HRV_OK : set_error(HRV_ECUDA, "%s: %s", what, cudaGetErrorString(e));
}

size_t align256(size_t v) { return (v + 255) / 256 * 256; }

// Validates the call and lays the workspace out: slabs, then m_i and d m_i of every flow.
int tv_setup(const hrv_tv_flow* flows, int nflows, int n, const float* mask, int mh, int mw, void* workspace, size_t workspace_bytes,
             TvArgs& a, long long& max_pix, const char* what) {
  if (!flows || nflows < 1 || nflows > HRV_TV_MAX_FLOWS || n < 1)
    return set_error(HRV_EINVAL, "%s: need 1..%d flows and n >= 1, got %d flows, n=%d", what, HRV_TV_MAX_FLOWS, nflows, n);
  if (mask && (mh < 1 || mw < 1)) return set_error(HRV_EINVAL, "%s: mask extent %dx%d", what, mh, mw);
  const size_t need = hrv_flow_tv_workspace_bytes(flows, nflows, n);
  if (!workspace || workspace_bytes < need) return set_error(HRV_EINVAL, "%s: workspace too small (%zu < %zu)", what, workspace_bytes, need);
  memset(&a, 0, sizeof(a));
  a.nflows = nflows;
  a.n = n;
  a.mask = mask;
  a.mh = mh;
  a.mw = mw;
  char* ws = (char*)workspace;
  a.slab = (double*)ws;
  ws += align256((size_t)nflows * kTvBlocks * 4 * sizeof(double));
  max_pix = 0;
  for (int i = 0; i < nflows; ++i) {
    const hrv_tv_flow& s = flows[i];
    if (!s.flow || s.h < 2 || s.w < 2) return set_error(HRV_EINVAL, "%s: flow %d is null or smaller than 2x2 (%dx%d)", what, i, s.h, s.w);
    const long long npix = (long long)n * s.h * s.w;
    if (npix > 0x7fffffffLL) return set_error(HRV_EINVAL, "%s: flow %d has too many pixels", what, i);
    TvFlow& f = a.f[i];
    f.flow = s.flow;
    f.h = s.h;
    f.w = s.w;
    f.we = s.edge_weight;
    f.wp = s.plain_weight;
    f.m = (float*)ws;
    ws += align256((size_t)npix * sizeof(float));
    f.dm = (float*)ws;
    ws += align256((size_t)npix * sizeof(float));
    if (npix > max_pix) max_pix = npix;
  }
  return HRV_OK;
}

unsigned nblocks(long long total) { return (unsigned)((total + kTvThreads - 1) / kTvThreads); }

}  // namespace

extern "C" size_t hrv_flow_tv_workspace_bytes(const hrv_tv_flow* flows, int32_t nflows, int32_t n) {
  if (!flows || nflows < 1 || nflows > HRV_TV_MAX_FLOWS || n < 1) return 0;
  size_t b = align256((size_t)nflows * kTvBlocks * 4 * sizeof(double));
  for (int i = 0; i < nflows; ++i) b += 2 * align256((size_t)n * (flows[i].h > 0 ? flows[i].h : 0) * (flows[i].w > 0 ? flows[i].w : 0) * sizeof(float));
  return b;
}

extern "C" int hrv_flow_tv(const hrv_tv_flow* flows, int32_t nflows, int32_t n, const float* mask, int32_t mh, int32_t mw, float* loss,
                           float* terms, float* const* mask_down, void* workspace, size_t workspace_bytes, hrv_stream stream) {
  TvArgs a;
  long long max_pix;
  int rc;
  if ((rc = tv_setup(flows, nflows, n, mask, mh, mw, workspace, workspace_bytes, a, max_pix, "flow_tv"))) return rc;
  if (!loss) return set_error(HRV_EINVAL, "flow_tv: null loss");
  if (mask_down && !mask) return set_error(HRV_EINVAL, "flow_tv: mask_down without mask");
  for (int i = 0; mask_down && i < nflows; ++i) {
    if (!mask_down[i]) return set_error(HRV_EINVAL, "flow_tv: mask_down[%d] is null", i);
    a.f[i].m = mask_down[i];  // the down-sampled mask goes to the caller's buffer instead of the workspace
  }
  cudaStream_t st = (cudaStream_t)stream;
  if (mask) {
    tv_mask_down_kernel<<<dim3(nblocks(max_pix), nflows), kTvThreads, 0, st>>>(a);
    if ((rc = launched("flow_tv mask"))) return rc;
  }
  tv_sums_kernel<<<dim3(kTvBlocks, nflows), kTvThreads, 0, st>>>(a);
  if ((rc = launched("flow_tv sums"))) return rc;
  tv_finish_kernel<<<1, 32, 0, st>>>(a, loss, terms);
  return launched("flow_tv finish");
}

extern "C" int hrv_flow_tv_bwd(const hrv_tv_flow* flows, int32_t nflows, int32_t n, const float* mask, int32_t mh, int32_t mw,
                               const float* dloss, float* const* dflows, float* dmask, void* workspace, size_t workspace_bytes,
                               hrv_stream stream) {
  TvArgs a;
  long long max_pix;
  int rc;
  if ((rc = tv_setup(flows, nflows, n, mask, mh, mw, workspace, workspace_bytes, a, max_pix, "flow_tv_bwd"))) return rc;
  if (!dloss || !dflows) return set_error(HRV_EINVAL, "flow_tv_bwd: null dloss or dflows");
  if (!mask && dmask) return set_error(HRV_EINVAL, "flow_tv_bwd: dmask without mask");
  for (int i = 0; i < nflows; ++i) {
    if (!dflows[i]) return set_error(HRV_EINVAL, "flow_tv_bwd: dflows[%d] is null", i);
    a.f[i].dflow = dflows[i];
  }
  a.dloss = dloss;
  a.dmask = dmask;
  cudaStream_t st = (cudaStream_t)stream;
  if (mask) {
    tv_mask_down_kernel<<<dim3(nblocks(max_pix), nflows), kTvThreads, 0, st>>>(a);
    if ((rc = launched("flow_tv_bwd mask"))) return rc;
  }
  tv_bwd_flow_kernel<<<dim3(nblocks(max_pix), nflows), kTvThreads, 0, st>>>(a);
  if ((rc = launched("flow_tv_bwd flow"))) return rc;
  if (dmask) {
    tv_bwd_mask_kernel<<<nblocks((long long)n * mh * mw), kTvThreads, 0, st>>>(a);
    return launched("flow_tv_bwd mask adjoint");
  }
  return HRV_OK;
}

}  // namespace hrv
