// conv_wgrad.cu — convolution weight gradient on wgmma:  dW[co,ci,ky,kx] += sum_{n,y,x} dY[n,y,x,co] * X[n,y+ky-pad,x+kx-pad,ci]
//
// GEMM view per tap (ky, kx):  D[m, n] with K = pixels.  Per layer the host puts one operand on the 128-row M side (two consumer
// warpgroups of 64 rows, A from shared memory) and the other on the BN-column N side, fp32 accumulators in registers: M = cout and
// N = cin, or M = cin and N = cout (the X box, shifted by the tap, then feeds A).  N is cut into 128-, 64- or 32-column tiles, the
// last one optionally narrower; wgrad_plan picks the orientation and tiling that issue the fewest MMA columns.  The gamma|beta
// layers (128 -> 160) become M = cin, N = 128 + 32: exact, where M = cout would pad 160 rows to 256.
// Both operands are channel-contiguous in NHWC memory, i.e. *MN-major* for the MMA (K = pixels is the strided index): a TMA box
// {64 channels, PX pixels} lands as PX rows of 128 B (SWIZZLE_128B) = K-rows of a 64-wide MN block; blocks of 64 channels sit
// LBO bytes apart, 8-row K groups SBO = 1024 B apart.  A 32-column tile is a {32 channels, PX pixels} box of 64-byte rows
// (SWIZZLE_64B, SBO = 512 B): the canonical MN-major layout of a 32-column operand.
// Grid = (M tiles) x (N tiles) x KH x KW x splits; each CTA streams its share of the (n, y, x-segment) chunks (one dY box set and
// the X box set shifted by its tap per chunk) and finally writes its fp32 partial tile into slab `split` of the workspace
// [splits][cout][cin][KH][KW]; wgrad_reduce_kernel then sums the slabs in a FIXED order into dW — the result is bit-reproducible run
// to run (fp32 atomics would not be).
// Replaces the weight-gradient half of nn.Conv2d's backward (networks.py / network_generator.py convolutions, stage-2 training).
#include <stdlib.h>

#include "hrv_host.h"
#include "hrv_ptx.cuh"

namespace hrv {

constexpr int kWgThreads = 288;  // warpgroups 0, 1: MMA + epilogue (64 M rows each), warp 8: TMA producer
constexpr int kPX = 64;          // pixels (K) per pipeline stage
constexpr uint32_t kWgSmem = 110u * 1024u;  // two CTAs per SM (plus 1 KB reserved per CTA)
constexpr uint32_t kBlk = kPX * 128u;       // one 64-channel SWIZZLE_128B block of kPX pixel rows: 8 KB
constexpr uint32_t kTail = kPX * 64u;       // one 32-channel SWIZZLE_64B block of kPX pixel rows: 4 KB

// Stage of a W-column tile (W = 32, 64, 128): A blocks 0, 1 (128 M rows), then W / 64 N blocks of 64 channels or one of 32.
__host__ __device__ constexpr uint32_t wgrad_stage_bytes(int w) { return 2u * kBlk + (w == 32 ? kTail : kBlk * (uint32_t)(w / 64)); }
__host__ __device__ constexpr int wgrad_stages(int w) { return (kWgSmem - 2048u) / wgrad_stage_bytes(w) < 16 ? (kWgSmem - 2048u) / wgrad_stage_bytes(w) : 16; }

struct alignas(64) WgradArgs {
  CUtensorMap tmA;   // M-side operand (dY, or X when a_is_x) box {64, kPX, 1, 1}
  CUtensorMap tmB;   // N-side operand box {64, kPX, 1, 1}
  CUtensorMap tmBt;  // N-side operand box {32, kPX, 1, 1}, SWIZZLE_64B (32-wide tiles only)
  int Nimg, OH, OW, xsegs;
  int KH, KW, pad;
  int cout, cin, splits;
  int a_is_x;  // 1: M = input channels, N = output channels; 0: M = output channels, N = input channels
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

// One (M tile, N tile, tap, split) work item of width W in {32, 64, 128}.  64 and 128 read the N operand as W / 64 SWIZZLE_128B
// blocks; 32 reads one SWIZZLE_64B block (the canonical MN-major layout of a 32-column operand; 128-byte rows would need 64).
template <int W>
__device__ __forceinline__ void wgrad_tile(const WgradArgs& a, uint32_t base, int m0, int n0, int ky, int kx, int split) {
  constexpr uint32_t stage_bytes = wgrad_stage_bytes(W);
  constexpr int S = wgrad_stages(W);
  const uint32_t stage0 = base + 1024u;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
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
      const CUtensorMap* tmb = W == 32 ? &a.tmBt : &a.tmB;
      tma_prefetch_desc(&a.tmA);
      tma_prefetch_desc(tmb);
      // pixel offsets of each operand's box: the X box moves with the tap, the dY box does not
      const int ax = a.a_is_x ? kx - a.pad : 0, ay = a.a_is_x ? ky - a.pad : 0;
      const int bx = a.a_is_x ? 0 : kx - a.pad, by = a.a_is_x ? 0 : ky - a.pad;
      StageRing ring(stage0, stage_bytes, S);
      int c = split;
      for (int i = 0; i < my_chunks; ++i, c += a.splits) {
        const int x0 = (c % a.xsegs) * kPX;
        int r = c / a.xsegs;
        const int y = r % a.OH;
        const int n = r / a.OH;
        const uint32_t full = bar_full(base, ring.stage), sa = ring.addr;
        mbar_wait(bar_empty(base, ring.stage), ring.phase ^ 1u);
        mbar_arrive_expect_tx(full, stage_bytes);
        tma_load_4d(sa, &a.tmA, full, m0, x0 + ax, y + ay, n);
        tma_load_4d(sa + kBlk, &a.tmA, full, m0 + 64, x0 + ax, y + ay, n);
#pragma unroll
        for (int b = 0; b < (W + 63) / 64; ++b) tma_load_4d(sa + (2u + b) * kBlk, tmb, full, n0 + 64 * b, x0 + bx, y + by, n);
        ring.next();
      }
    }
    return;
  }

  // ===================================================== consumers: warpgroup wg owns M rows m0 + [64 wg, 64 wg + 64)
  // Both operands are MN-major (channels contiguous, K = pixels strided): LBO = 64-channel block stride, SBO = 8 pixel rows.
  const int wg = warp >> 2;
  float acc[W / 2];
#pragma unroll
  for (int i = 0; i < W / 2; ++i) acc[i] = 0.f;
  {
    StageRing ring(stage0, stage_bytes, S);
    int prev = 0;
    for (int i = 0; i < my_chunks; ++i) {
      mbar_wait(bar_full(base, ring.stage), ring.phase);
      wgmma_fence();
      const uint32_t sa = ring.addr + (uint32_t)wg * kBlk, sb = ring.addr + 2u * kBlk;
#pragma unroll
      for (int kk = 0; kk < kPX / 16; ++kk) {  // 16 pixel rows per instruction
        const uint64_t da = make_wgmma_desc(sa + kk * 2048u, 1024, 1, kBlk);
        const uint32_t accf = (uint32_t)((i | kk) != 0);
        if constexpr (W == 32) wgmma_n32<1, 1>(acc, da, make_wgmma_desc(sb + kk * 1024u, 512, 2, kTail), accf);
        else wgmma_nx<W, 1, 1>(acc, da, make_wgmma_desc(sb + kk * 2048u, 1024, 1, kBlk), accf);
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
  // wgmma fragment: thread (warp w, lane l) holds rows (M) 16 (w % 4) + l / 4 and that + 8, columns (N) 8 j + 2 (l % 4) + {0, 1}.
  float* const slab = a.dw + (long long)split * a.cout * a.cin * a.KH * a.KW;  // this CTA's private slab: plain stores, no atomics
  const long long ci_stride = (long long)a.KH * a.KW, co_stride = (long long)a.cin * ci_stride;
  const long long m_stride = a.a_is_x ? ci_stride : co_stride, n_stride = a.a_is_x ? co_stride : ci_stride;
  const int m_count = a.a_is_x ? a.cin : a.cout, n_count = a.a_is_x ? a.cout : a.cin;
  float* const tap = slab + ky * a.KW + kx;
  const int m_base = m0 + wg * 64 + (warp & 3) * 16 + (lane >> 2);
  const int n_base = n0 + 2 * (lane & 3);
  // a split without work (more splits than chunks) writes zeros: acc was never touched
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int m = m_base + 8 * h;
    if (m >= m_count) continue;
    float* const row = tap + m * m_stride;
#pragma unroll
    for (int j = 0; j < W / 8; ++j) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int n = n_base + 8 * j + e;
        if (n < n_count) row[n * n_stride] = acc[4 * j + 2 * h + e];
      }
    }
  }
}

// N tiles 0 .. n_tiles - 2 are BN wide; the last is BT wide when BT != 0 (e.g. 160 columns = 128 + 32: a 160-wide tile's 80
// accumulators do not fit the 96 registers a thread gets at two 288-thread CTAs per SM).
template <int BN, int BT>
__global__ void __launch_bounds__(kWgThreads, 2) conv_wgrad_kernel(const __grid_constant__ WgradArgs a) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  // Split slowest: the CTAs of all taps and tiles of one split read the same pixel chunks, and with consecutive block indices they
  // run in the same wave, so each chunk comes from HBM about once and from L2 after that.  With the split fastest they sat a split
  // count apart and each re-read the (far larger than L2) full-resolution X and dY from HBM.
  int bid = blockIdx.x;
  const int kx = bid % a.KW; bid /= a.KW;
  const int ky = bid % a.KH; bid /= a.KH;
  const int nt = bid % a.n_tiles; bid /= a.n_tiles;
  const int mt = bid % a.m_tiles;
  const int split = bid / a.m_tiles;
  if constexpr (BT != 0) {
    if (nt == a.n_tiles - 1) {
      wgrad_tile<BT>(a, base, mt * 128, nt * BN, ky, kx, split);
      return;
    }
  }
  wgrad_tile<BN>(a, base, mt * 128, nt * BN, ky, kx, split);
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

struct WgradPlan {
  int a_is_x, bn, bt, m_tiles, n_tiles, tiles, chunks;
};
// Orientation and N tiling of one layer: the choice that issues the fewest MMA columns, each tile charged kTileCost columns more
// for what it repeats whatever its width (the A box stream, the barrier handshakes, the epilogue).  N is covered by BN-wide tiles,
// the last of them optionally narrower (BT).  Ties keep M = cout and the wider tile.
static WgradPlan wgrad_plan(const hrv_tensor* x, const hrv_tensor* dy, int kh, int kw) {
  static const int kTiling[][2] = {{128, 0}, {128, 64}, {128, 32}, {64, 0}, {32, 0}};  // {BN, BT}
  const long long kTileCost = 32;
  WgradPlan best{};
  long long best_cost = -1;
  for (int a_is_x = 0; a_is_x < 2; ++a_is_x) {
    const int cm = a_is_x ? x->c : dy->c, cn = a_is_x ? dy->c : x->c;
    const int mt = (cm + 127) / 128;
    for (const auto& t : kTiling) {
      const int bn = t[0], bt = t[1], rem = cn % bn;
      if (bt && (rem == 0 || rem > bt)) continue;  // the narrow last tile must exist and suffice
      const int nt = bt ? cn / bn + 1 : (cn + bn - 1) / bn;
      const long long cost = (long long)mt * ((long long)(bt ? nt - 1 : nt) * (bn + kTileCost) + (bt ? bt + kTileCost : 0));
      if (best_cost < 0 || cost < best_cost) { best_cost = cost; best = WgradPlan{a_is_x, bn, bt, mt, nt, 0, 0}; }
    }
  }
  best.chunks = x->n * dy->h * ((dy->w + kPX - 1) / kPX);
  best.tiles = best.m_tiles * best.n_tiles * kh * kw;
  return best;
}

extern "C" size_t hrv_conv2d_wgrad_workspace_bytes(const hrv_tensor* x, const hrv_tensor* dy, int32_t kh, int32_t kw) {
  if (!x || !dy || kh < 1 || kw < 1) return 0;
  const WgradPlan p = wgrad_plan(x, dy, kh, kw);
  const int splits = wgrad_splits(p.tiles, p.chunks);
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
  const WgradPlan p = wgrad_plan(x, dy, kh, kw);
  a.a_is_x = p.a_is_x; a.m_tiles = p.m_tiles; a.n_tiles = p.n_tiles;
  const int splits = wgrad_splits(p.tiles, p.chunks);
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
  const hrv_tensor& ta = p.a_is_x ? *x : *dy;
  const hrv_tensor& tb = p.a_is_x ? *dy : *x;
  int rc = encode_nhwc_map(&a.tmA, ta, 64, kPX, 1, 1);
  if (!rc) rc = encode_nhwc_map(&a.tmB, tb, 64, kPX, 1, 1);
  if (!rc && (p.bn == 32 || p.bt == 32)) rc = encode_nhwc_map(&a.tmBt, tb, 32, kPX, 1, 1, CU_TENSOR_MAP_SWIZZLE_64B);
  if (rc) return rc;
  size_t smem = 2048 + (size_t)wgrad_stages(p.bn) * wgrad_stage_bytes(p.bn);
  if (p.bt) {
    const size_t tail = 2048 + (size_t)wgrad_stages(p.bt) * wgrad_stage_bytes(p.bt);
    if (tail > smem) smem = tail;
  }
  const int grid = p.tiles * splits;
  cudaStream_t st = (cudaStream_t)stream;
  switch (p.bn * 1000 + p.bt) {
    case 32000: rc = launch_dyn_smem<conv_wgrad_kernel<32, 0>>("conv_wgrad", grid, kWgThreads, smem, kWgSmem, st, a); break;
    case 64000: rc = launch_dyn_smem<conv_wgrad_kernel<64, 0>>("conv_wgrad", grid, kWgThreads, smem, kWgSmem, st, a); break;
    case 128000: rc = launch_dyn_smem<conv_wgrad_kernel<128, 0>>("conv_wgrad", grid, kWgThreads, smem, kWgSmem, st, a); break;
    case 128032: rc = launch_dyn_smem<conv_wgrad_kernel<128, 32>>("conv_wgrad", grid, kWgThreads, smem, kWgSmem, st, a); break;
    default: rc = launch_dyn_smem<conv_wgrad_kernel<128, 64>>("conv_wgrad", grid, kWgThreads, smem, kWgSmem, st, a); break;
  }
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
