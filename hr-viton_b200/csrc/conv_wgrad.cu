// conv_wgrad.cu — convolution weight gradient on wgmma:  dW[co,ci,ky,kx] += sum_{n,y,x} dY[n,y,x,co] * X[n,y+ky-pad,x+kx-pad,ci]
//
// GEMM view per tap (ky, kx):  D[co, ci] (M = 128 output channels over two consumer warpgroups, N = BN = 64 or 128 input channels,
// fp32 accumulators in registers), K = pixels.  Both operands are channel-contiguous in NHWC memory, i.e. *MN-major* for the MMA
// (K = pixels is the strided index): a TMA box {64 channels, PX pixels} lands as PX rows of 128 B (SWIZZLE_128B) = K-rows of a
// 64-wide MN block; blocks of 64 channels sit LBO bytes apart, 8-row K groups SBO = 1024 B apart.
// Grid = (co tiles) x (ci tiles) x KH x KW x splits; each CTA streams its share of the (n, y, x-segment) chunks (one dY box pair and
// the X box shifted by its tap per chunk) and finally writes its fp32 partial tile into slab `split` of the workspace
// [splits][cout][cin][KH][KW]; wgrad_reduce_kernel then sums the slabs in a FIXED order into dW — the result is bit-reproducible run
// to run (fp32 atomics would not be).
// Replaces the weight-gradient half of nn.Conv2d's backward (networks.py / network_generator.py convolutions, stage-2 training).
#include <stdlib.h>

#include "hrv_host.h"
#include "hrv_ptx.cuh"

namespace hrv {

constexpr int kWgThreads = 288;  // warpgroups 0, 1: MMA + epilogue (64 output channels each), warp 8: TMA producer
constexpr int kPX = 64;          // pixels (K) per pipeline stage
constexpr uint32_t kWgSmem = 110u * 1024u;  // two CTAs per SM (plus 1 KB reserved per CTA)

struct alignas(64) WgradArgs {
  CUtensorMap tmDY;  // dY (N,OH,OW,cout) box {64, kPX, 1, 1}
  CUtensorMap tmX;   // X  (N,H,W,cin)    box {64, kPX, 1, 1}
  int Nimg, OH, OW, xsegs;
  int KH, KW, pad;
  int cout, cin, BN, stages, splits;
  int m_tiles, n_tiles;
  float* dw;  // (cout, cin, KH, KW) fp32 (splits == 1: written directly) or the workspace [splits][cout][cin][KH][KW]
};

// dw[i] = sum_{s < splits} ws[s][i], slabs added in increasing s: deterministic.  float4 per thread.
__global__ void __launch_bounds__(256) wgrad_reduce_kernel(const float* __restrict__ ws, float* __restrict__ dw, long long n4, long long slab4, int splits) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  float4 acc = __ldg(reinterpret_cast<const float4*>(ws) + i);
  for (int s = 1; s < splits; ++s) {
    const float4 v = __ldg(reinterpret_cast<const float4*>(ws) + (long long)s * slab4 + i);
    acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
  }
  reinterpret_cast<float4*>(dw)[i] = acc;
}
__global__ void __launch_bounds__(256) wgrad_reduce1_kernel(const float* __restrict__ ws, float* __restrict__ dw, long long n, int splits) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float acc = __ldg(ws + i);
  for (int s = 1; s < splits; ++s) acc += __ldg(ws + (long long)s * n + i);
  dw[i] = acc;
}

template <int BN>
__global__ void __launch_bounds__(kWgThreads, 2) conv_wgrad_kernel(const __grid_constant__ WgradArgs a) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  constexpr uint32_t kBlk = kPX * 128u;                                     // one 64-channel block of kPX pixel rows: 8 KB
  constexpr uint32_t stage_bytes = kBlk * (2u + BN / 64);                  // dY: co blocks 0, 1; X: BN / 64 ci blocks
  const uint32_t stage0 = base + 1024u;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int S = a.stages;

  // tile coordinates
  int bid = blockIdx.x;
  const int split = bid % a.splits; bid /= a.splits;
  const int kx = bid % a.KW; bid /= a.KW;
  const int ky = bid % a.KH; bid /= a.KH;
  const int nt = bid % a.n_tiles;
  const int mt = bid / a.n_tiles;
  const int m0 = mt * 128, n0 = nt * a.BN;
  const int chunks_total = a.Nimg * a.OH * a.xsegs;
  const int my_chunks = (chunks_total - split + a.splits - 1) / a.splits;  // chunks split, split+splits, ...

  if (threadIdx.x == 0) {
    for (int s = 0; s < S; ++s) { mbar_init(bar_full(base, s), 1); mbar_init(bar_empty(base, s), 8); }  // one arrival per consumer warp
    fence_mbar_init();
  }
  __syncthreads();

  if (warp == 8) {
    // ===================================================== TMA producer (one lane)
    if (lane == 0) {
      tma_prefetch_desc(&a.tmDY);
      tma_prefetch_desc(&a.tmX);
      StageRing ring(stage0, stage_bytes, S);
      int c = split;
      for (int i = 0; i < my_chunks; ++i, c += a.splits) {
        const int xs = c % a.xsegs;
        int r = c / a.xsegs;
        const int y = r % a.OH;
        const int n = r / a.OH;
        const uint32_t full = bar_full(base, ring.stage), sa = ring.addr;
        mbar_wait(bar_empty(base, ring.stage), ring.phase ^ 1u);
        mbar_arrive_expect_tx(full, stage_bytes);
        tma_load_4d(sa, &a.tmDY, full, m0, xs * kPX, y, n);
        tma_load_4d(sa + kBlk, &a.tmDY, full, m0 + 64, xs * kPX, y, n);
        for (int b = 0; b < BN / 64; ++b)
          tma_load_4d(sa + (2u + b) * kBlk, &a.tmX, full, n0 + 64 * b, xs * kPX - a.pad + kx, y + ky - a.pad, n);
        ring.next();
      }
    }
    return;
  }

  // ===================================================== consumers: warpgroup wg owns output channels m0 + [64 wg, 64 wg + 64)
  // Both operands are MN-major (channels contiguous, K = pixels strided): LBO = 64-channel block stride, SBO = 8 pixel rows.
  const int wg = warp >> 2;
  float acc[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
  {
    StageRing ring(stage0, stage_bytes, S);
    int prev = 0;
    for (int i = 0; i < my_chunks; ++i) {
      mbar_wait(bar_full(base, ring.stage), ring.phase);
      wgmma_fence();
      const uint32_t sdy = ring.addr + (uint32_t)wg * kBlk, sx = ring.addr + 2u * kBlk;
#pragma unroll
      for (int kk = 0; kk < kPX / 16; ++kk) {  // 16 pixel rows per instruction
        const uint64_t da = make_wgmma_desc(sdy + kk * 2048u, 1024, 1, kBlk);
        const uint64_t db = make_wgmma_desc(sx + kk * 2048u, 1024, 1, kBlk);
        const uint32_t accf = (uint32_t)((i | kk) != 0);
        wgmma_nx<BN, 1, 1>(acc, da, db, accf);
      }
      wgmma_commit();
      wgmma_wait<1>();
      if (i > 0 && lane == 0) mbar_arrive(bar_empty(base, prev));
      prev = ring.stage;
      ring.next();
    }
    wgmma_wait<0>();
    fence_regs(acc);
  }

  // ===================================================== epilogue: fp32 partial tile -> dW[(co*cin+ci)*KH*KW + ky*KW + kx] of this split's slab
  // wgmma fragment: thread (warp w, lane l) holds rows (co) 16 (w % 4) + l / 4 and that + 8, columns (ci) 8 j + 2 (l % 4) + {0, 1}.
  float* const slab = a.dw + (long long)split * a.cout * a.cin * a.KH * a.KW;  // this CTA's private slab: plain stores, no atomics
  const int co_base = m0 + wg * 64 + (warp & 3) * 16 + (lane >> 2);
  const int ci_base = n0 + 2 * (lane & 3);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int co = co_base + 8 * h;
    if (co >= a.cout) continue;
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int ci = ci_base + 8 * j + e;
        // a split without work (more splits than chunks) writes zeros: acc was never touched
        if (ci < a.cin) slab[(((long long)co * a.cin + ci) * a.KH + ky) * a.KW + kx] = acc[4 * j + 2 * h + e];
      }
    }
  }
}

}  // namespace hrv

using namespace hrv;

// Split-K factor: two CTAs per SM are resident, CTAs of one launch take equal time, so the launch costs
// waves * (chunks per CTA + fixed prologue/epilogue) with waves = ceil(grid / (2 SMs)).  Pick the split that minimises it — a grid
// that spills a few CTAs into an extra wave (e.g. 270 CTAs on 2 x 132 slots) costs a whole wave.
static int wgrad_splits(int tiles, int chunks) {
  const int sms = 2 * sm_count();
  int splits = 1;
  const long long kFixed = 16;  // prologue + epilogue, in units of one 64-pixel chunk step
  long long best = -1;
  int smax = 8 * sms / tiles + 1;
  if (smax > chunks) smax = chunks;
  if (smax < 1) smax = 1;
  for (int sp = 1; sp <= smax; ++sp) {
    const long long waves = ((long long)tiles * sp + sms - 1) / sms;
    const long long cost = waves * ((chunks + sp - 1) / sp + kFixed);
    if (best < 0 || cost < best) { best = cost; splits = sp; }
  }
  const char* env = getenv("HRV_WGRAD_SPLITS");  // A/B runs
  if (env && atoi(env) > 0) splits = atoi(env) < chunks ? atoi(env) : (chunks > 0 ? chunks : 1);
  return splits;
}
static void wgrad_geometry(const hrv_tensor* x, const hrv_tensor* dy, int kh, int kw, int* tiles, int* chunks, int* bn, int* m_tiles, int* n_tiles) {
  *bn = x->c <= 64 ? 64 : 128;
  *m_tiles = (dy->c + 127) / 128;
  *n_tiles = (x->c + *bn - 1) / *bn;
  *chunks = x->n * dy->h * ((dy->w + kPX - 1) / kPX);
  *tiles = *m_tiles * *n_tiles * kh * kw;
}

extern "C" size_t hrv_conv2d_wgrad_workspace_bytes(const hrv_tensor* x, const hrv_tensor* dy, int32_t kh, int32_t kw) {
  if (!x || !dy || kh < 1 || kw < 1) return 0;
  int tiles, chunks, bn, mt, nt;
  wgrad_geometry(x, dy, kh, kw, &tiles, &chunks, &bn, &mt, &nt);
  const int splits = wgrad_splits(tiles, chunks);
  return splits > 1 ? (size_t)splits * dy->c * x->c * kh * kw * sizeof(float) : 0;
}

extern "C" int hrv_conv2d_wgrad(const hrv_tensor* x, const hrv_tensor* dy, int32_t kh, int32_t kw, int32_t pad, float* dw,
                                void* workspace, size_t workspace_bytes, hrv_stream stream) {
  if (!x || !dy || !x->ptr || !dy->ptr || !dw) return set_error(HRV_EINVAL, "wgrad: null argument");
  if (x->dtype != HRV_BF16 || dy->dtype != HRV_BF16) return set_error(HRV_EINVAL, "wgrad: x and dy must be bf16 NHWC");
  if (((uintptr_t)x->ptr & 15) || ((uintptr_t)dy->ptr & 15) || (x->pitch % 8) || (dy->pitch % 8))
    return set_error(HRV_EINVAL, "wgrad: 16-byte alignment and pitch %% 8 == 0 required");
  if (kh < 1 || kw < 1 || kw > 4 || x->n != dy->n) return set_error(HRV_EINVAL, "wgrad: bad geometry");
  if (dy->h > x->h + 2 * pad - kh + 1 || dy->w > x->w + 2 * pad - kw + 1) return set_error(HRV_EINVAL, "wgrad: dy extent exceeds the conv output extent");  // smaller = cropped output
  WgradArgs a;
  memset(&a, 0, sizeof(a));
  a.Nimg = x->n; a.OH = dy->h; a.OW = dy->w; a.xsegs = (dy->w + kPX - 1) / kPX;
  a.KH = kh; a.KW = kw; a.pad = pad; a.cout = dy->c; a.cin = x->c;
  int tiles, chunks;
  wgrad_geometry(x, dy, kh, kw, &tiles, &chunks, &a.BN, &a.m_tiles, &a.n_tiles);
  const int splits = wgrad_splits(tiles, chunks);
  const long long dw_elems = (long long)dy->c * x->c * kh * kw;
  if (splits > 1) {
    const size_t need = (size_t)splits * dw_elems * sizeof(float);
    if (!workspace || workspace_bytes < need || ((uintptr_t)workspace & 15))
      return set_error(HRV_EINVAL, "wgrad: workspace too small or misaligned (%zu < %zu): ask hrv_conv2d_wgrad_workspace_bytes", workspace_bytes, need);
    a.dw = (float*)workspace;  // CTAs write slabs; wgrad_reduce_kernel sums them into dw in a fixed order
  } else {
    a.dw = dw;                 // one CTA per output element: plain stores straight into dw
  }
  a.splits = splits;
  const uint32_t stage_bytes = kPX * 128u * (2u + (uint32_t)(a.BN / 64));
  int stages = (int)((kWgSmem - 2048u) / stage_bytes);
  if (stages > 16) stages = 16;
  a.stages = stages;
  int rc = encode_nhwc_map(&a.tmDY, *dy, 64, kPX, 1, 1);
  if (!rc) rc = encode_nhwc_map(&a.tmX, *x, 64, kPX, 1, 1);
  if (rc) return rc;
  const size_t smem = 2048 + (size_t)stages * stage_bytes;
  const int grid = tiles * splits;
  cudaStream_t st = (cudaStream_t)stream;
  rc = a.BN == 128 ? launch_dyn_smem<conv_wgrad_kernel<128>>("conv_wgrad", grid, kWgThreads, smem, kWgSmem, st, a)
                   : launch_dyn_smem<conv_wgrad_kernel<64>>("conv_wgrad", grid, kWgThreads, smem, kWgSmem, st, a);
  if (rc) return rc;
  if (splits > 1) {
    if ((dw_elems % 4) || ((uintptr_t)dw & 15)) {  // slabs not 16-byte aligned: scalar reduction (tiny layers, e.g. 13 -> 13 channels)
      wgrad_reduce1_kernel<<<(unsigned)((dw_elems + 255) / 256), 256, 0, st>>>((const float*)workspace, dw, dw_elems, splits);
    } else {
      const long long n4 = dw_elems / 4;
      wgrad_reduce_kernel<<<(unsigned)((n4 + 255) / 256), 256, 0, st>>>((const float*)workspace, dw, n4, n4, splits);
    }
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return set_error(HRV_ECUDA, "wgrad_reduce launch: %s", cudaGetErrorString(e));
  }
  return HRV_OK;
}
