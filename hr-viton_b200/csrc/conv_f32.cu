// conv_f32.cu — the fp32 reference-precision convolution: NHWC fp32 implicit GEMM in 3xTF32 on sm_90a (wgmma .tf32 + TMA + mbarrier).
//
//   Same GEMM view and pipeline shape as conv_igemm.cu (M = 128 output pixels per tile, N = BNT = 64 or 128 output channels, K walked
//   tap by tap), with fp32 storage throughout:
//   A operand:  one TMA 4-D box {32 ch, TW, TH, TN} of the fp32 NHWC input per (tap, channel chunk) = one 128-byte SWIZZLE_128B row per
//               pixel; TMA zero fill is the convolution's zero padding.
//   B operand:  one TMA box {32, BNT, 1, 2} of the pre-split weights [2][taps][n_pad][cin_k] (hrv_pack_conv_weight_tf32x2): plane 0 =
//               hi = rna_tf32(w), plane 1 = lo = rna_tf32(w - hi), both landing in the same stage.
//   Split:      once a stage has landed, each consumer warpgroup rewrites its 64 A rows in place as hi = rna_tf32(a) and writes
//               lo = rna_tf32(a - hi) into a scratch tile (ping-pong: the previous stage's MMAs may still read the other one).  The split
//               is elementwise, so the 128B swizzle carries over unchanged.
//   MMA:        three wgmma m64nBNTk8 .tf32 chains into the same fp32 accumulators, small terms first: lo*B_hi, hi*B_lo, hi*B_hi.
//               Each TF32 x TF32 product is exact in fp32, so the result carries ~21 significant bits of every operand (the lo*lo term,
//               ~2^-22 relative, is dropped) — indistinguishable from an fp32 convolution at the 1e-3 output tolerance, where one TF32
//               pass is not (DESIGN.md §4).
//   Pipeline:   one CTA per SM (the three chains triple the MMA work per stage; the stage ring is as deep as 227 KB allows).
//   Epilogues:  LINEAR and SPADE with the semantics of conv_igemm.cu on fp32 storage.  The gate residual modes and gamma_out belong to the
//               backward pass and are refused: fp32 storage is inference-only.
#include <stdlib.h>

#include "hrv_host.h"
#include "hrv_ptx.cuh"

namespace hrv {
namespace {

constexpr int kMaxStages = 8;
constexpr int kConsumers = 2;                        // consumer warpgroups (64 pixels each)
constexpr int kThreads = 128 * kConsumers + 32;      // + one producer warp
constexpr uint32_t kRowBytes = 128;                  // 32 fp32 channels: one SWIZZLE_128B row
constexpr uint32_t kABytes = 128 * kRowBytes;        // 128 pixels
constexpr uint32_t kWgBytes = 64 * kRowBytes;        // one consumer warpgroup's 64 rows
constexpr uint32_t kScratch = 2 * kConsumers * kWgBytes;  // lo tiles, two per consumer (ping-pong)
constexpr uint32_t kSmemMax = 227u * 1024u;          // one CTA per SM

struct Tf32Args {
  CUtensorMap tmA;
  CUtensorMap tmB;
  int Nimg, Hout, Wout;
  int tw_log, th_log;
  int tiles_x, tiles_y, tiles_n;
  int KH, KW, off_y, off_x, chunks;
  int stages, n_gemm;
  int epi, act;
  const float* scale;
  const float* shift;
  float* out;
  int out_pitch, out_layout, out_c, store_c;
  const float* res;
  int res_pitch, res_c;
  const float* x0;
  int x0_c, x0_pitch, x0_shift;
  const float* x1;
  int x1_pitch;
  const float* mean;
  const float* rstd;
  const float* noise;
  const float* noise_scale;
  int C_mod;
};

struct Pix {
  int x, y, n;
  bool valid;
  long long pix;
};

// LINEAR epilogue of GEMM columns (c, c+1) of one pixel: out = act(acc*scale + shift (+ res)).  NHWC outputs whose pitch has room write
// the pad channels up to the next multiple of 8 as the 16-bit path does (act(0) + res); NCHW outputs stop at out_c.
__device__ __forceinline__ void epi_linear2(const Tf32Args& a, const Pix& p, int c, float v0, float v1) {
  if (!p.valid || c >= a.store_c) return;
  float f[2] = {v0, v1};
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int j = c + i;
    const bool in = j < a.n_gemm;
    const float sc = in ? (a.scale ? __ldg(a.scale + j) : 1.f) : 0.f;
    const float sh = (in && a.shift) ? __ldg(a.shift + j) : 0.f;
    f[i] = fmaf(f[i], sc, sh);
    if (a.res && j < a.res_c) f[i] += __ldg(a.res + p.pix * a.res_pitch + j);
    f[i] = apply_act(f[i], a.act);
  }
  if (a.out_layout == 0) {
    float* op = a.out + p.pix * a.out_pitch + c;
    op[0] = f[0];
    if (c + 1 < a.store_c) op[1] = f[1];
  } else {
    const long long hw = (long long)a.Hout * a.Wout;
#pragma unroll
    for (int i = 0; i < 2; ++i)
      if (c + i < a.out_c) a.out[((long long)p.n * a.out_c + c + i) * hw + (long long)p.y * a.Wout + p.x] = f[i];
  }
}

// SPADE epilogue of channel ch of one pixel; g, b = the (gamma, beta) accumulators of columns 2ch, 2ch+1.
__device__ __forceinline__ void epi_spade1(const Tf32Args& a, const Pix& p, long long pix0, float nz, int ch, float g, float b) {
  if (!p.valid || ch >= a.C_mod) return;
  const float xs = (ch < a.x0_c) ? __ldg(a.x0 + pix0 * a.x0_pitch + ch) : __ldg(a.x1 + p.pix * a.x1_pitch + (ch - a.x0_c));
  const float mu = __ldg(a.mean + (long long)p.n * a.C_mod + ch);
  const float rs = __ldg(a.rstd + (long long)p.n * a.C_mod + ch);
  const float ns = a.noise_scale ? __ldg(a.noise_scale + ch) : 0.f;
  const float gm = g + (a.shift ? __ldg(a.shift + 2 * ch) : 0.f);
  const float bt = b + (a.shift ? __ldg(a.shift + 2 * ch + 1) : 0.f);
  const float xn = (fmaf(nz, ns, xs) - mu) * rs;
  a.out[p.pix * a.out_pitch + ch] = apply_act(fmaf(xn, 1.f + gm, bt), a.act);
}

template <int BNT>
__device__ __forceinline__ void mma_tile(float (&d)[BNT / 2], uint64_t da, uint64_t db, uint32_t scale_d) {
  if constexpr (BNT == 64) wgmma_tf32_n64(d, da, db, scale_d);
  else wgmma_tf32_n128(d, da, db, scale_d);
}

__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t threads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}

// hi/lo split of one warpgroup's 64 rows (8 KB): thread t handles four 16-byte vectors.
__device__ __forceinline__ void split_rows(uint32_t hi_rows, uint32_t lo_rows, int t) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const uint32_t off = (uint32_t)(i * 128 + t) * 16u;
    float v[4];
    asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v[0]), "=f"(v[1]), "=f"(v[2]), "=f"(v[3]) : "r"(hi_rows + off) : "memory");
    float h[4], l[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      h[j] = rna_tf32(v[j]);
      l[j] = rna_tf32(v[j] - h[j]);
    }
    asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(hi_rows + off), "f"(h[0]), "f"(h[1]), "f"(h[2]), "f"(h[3]) : "memory");
    asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(lo_rows + off), "f"(l[0]), "f"(l[1]), "f"(l[2]), "f"(l[3]) : "memory");
  }
}

}  // namespace

template <int BNT>
__global__ void __launch_bounds__(kThreads, 1) conv_tf32x3_kernel(const __grid_constant__ Tf32Args a) {
  constexpr uint32_t B_PLANE = (uint32_t)BNT * kRowBytes;
  constexpr uint32_t STAGE = kABytes + 2 * B_PLANE;  // all parts multiples of 1024 B: every operand starts at swizzle phase 0
  constexpr int R = BNT / 2;                         // accumulator registers per consumer thread

  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  auto bar_full = [&](int s) { return base + 8u * s; };
  auto bar_empty = [&](int s) { return base + 128u + 8u * s; };
  const uint32_t scratch = base + 1024u;
  const uint32_t stage0 = scratch + kScratch;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int S = a.stages;
  const int KT = a.KH * a.KW * a.chunks;
  const int nt = blockIdx.x % a.tiles_n;
  int mt = blockIdx.x / a.tiles_n;
  const int tx = mt % a.tiles_x;
  mt /= a.tiles_x;
  const int ty = mt % a.tiles_y;
  const int ti = mt / a.tiles_y;

  if (threadIdx.x == 0) {
    for (int s = 0; s < S; ++s) {
      mbar_init(bar_full(s), 1);
      mbar_init(bar_empty(s), 4 * kConsumers);  // one arrival per consumer warp
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp == 4 * kConsumers) {
    // ===================================================== TMA producer (one lane)
    if (lane == 0) {
      tma_prefetch_desc(&a.tmA);
      tma_prefetch_desc(&a.tmB);
      const int x0 = (tx << a.tw_log) - a.off_x;
      const int y0 = (ty << a.th_log) - a.off_y;
      const int n0 = ti << (7 - a.tw_log - a.th_log);
      int st = 0, ky = 0, kx = 0, kc = 0, tap = 0;
      uint32_t ph = 0, sa = stage0;
      for (int k = 0; k < KT; ++k) {
        mbar_wait(bar_empty(st), ph ^ 1u);
        mbar_arrive_expect_tx(bar_full(st), STAGE);
        tma_load_4d(sa, &a.tmA, bar_full(st), kc * 32, x0 + kx, y0 + ky, n0);
        tma_load_4d(sa + kABytes, &a.tmB, bar_full(st), kc * 32, nt * BNT, tap, 0);  // hi and lo planes
        if (++kc == a.chunks) {
          kc = 0;
          ++tap;
          if (++kx == a.KW) { kx = 0; ++ky; }
        }
        sa += STAGE;
        if (++st == S) { st = 0; ph ^= 1u; sa = stage0; }
      }
    }
    return;
  }

  // ===================================================== consumers: warpgroup wg computes pixels [64 wg, 64 wg + 64) of the tile
  // The tensor cores add into their accumulators with truncation; chained over a whole K walk (hundreds of MMAs) that bias alone would
  // cost ~20x the rounding error of an fp32 sum.  So each stage (12 MMAs) starts a fresh partial tile, and the partials are summed in
  // fp32 registers with round-to-nearest adds (the promotion is what makes the result fp32-class, not just the operand split).
  const int wg = warp >> 2;
  const int t = threadIdx.x & 127;
  float acc[R], part[R];
#pragma unroll
  for (int i = 0; i < R; ++i) acc[i] = 0.f;
  {
    int st = 0;
    uint32_t ph = 0, sa = stage0;
    for (int k = 0; k < KT; ++k) {
      mbar_wait(bar_full(st), ph);
      const uint32_t a_hi = sa + (uint32_t)wg * kWgBytes;
      // ping-pong lo tile: the other warpgroup-local tile may still be named by the previous stage's descriptors
      const uint32_t a_lo = scratch + (uint32_t)((k & 1) * kConsumers + wg) * kWgBytes;
      split_rows(a_hi, a_lo, t);
      fence_proxy_async();        // generic-proxy writes -> visible to the wgmma (async proxy) reads
      named_bar_sync(1 + wg, 128);  // every row of this warpgroup is split before its MMAs read any
      wgmma_fence();
      const uint32_t b_hi = sa + kABytes, b_lo = b_hi + B_PLANE;
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {  // K = 8 per instruction: +32 bytes inside the 128-byte swizzle row
        const uint64_t dah = make_wgmma_desc(a_hi + 32u * kk, 8 * kRowBytes, 1);
        const uint64_t dal = make_wgmma_desc(a_lo + 32u * kk, 8 * kRowBytes, 1);
        const uint64_t dbh = make_wgmma_desc(b_hi + 32u * kk, 8 * kRowBytes, 1);
        const uint64_t dbl = make_wgmma_desc(b_lo + 32u * kk, 8 * kRowBytes, 1);
        mma_tile<BNT>(part, dal, dbh, (uint32_t)(kk != 0));
        mma_tile<BNT>(part, dah, dbl, 1u);
        mma_tile<BNT>(part, dah, dbh, 1u);
      }
      wgmma_commit();
      wgmma_wait<0>();  // this stage's MMAs are done: its smem can be refilled and its partial promoted
      if (lane == 0) mbar_arrive(bar_empty(st));
      fence_regs(part);
#pragma unroll
      for (int i = 0; i < R; ++i) acc[i] += part[i];
      sa += STAGE;
      if (++st == S) { st = 0; ph ^= 1u; sa = stage0; }
    }
  }

  // ===================================================== epilogue straight from the accumulator registers (fragment as in conv_igemm.cu)
  const int tw_mask = (1 << a.tw_log) - 1, th_mask = (1 << a.th_log) - 1;
  const int r_base = wg * 64 + (warp & 3) * 16 + (lane >> 2);
  const int n_base = nt * BNT + 2 * (lane & 3);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int r = r_base + 8 * h;
    Pix p;
    p.x = (tx << a.tw_log) + (r & tw_mask);
    p.y = (ty << a.th_log) + ((r >> a.tw_log) & th_mask);
    p.n = (ti << (7 - a.tw_log - a.th_log)) + (r >> (a.tw_log + a.th_log));
    p.valid = (p.x < a.Wout) && (p.y < a.Hout) && (p.n < a.Nimg);
    p.pix = ((long long)p.n * a.Hout + p.y) * a.Wout + p.x;
    if (a.epi == 0) {
#pragma unroll
      for (int j = 0; j < BNT / 8; ++j) epi_linear2(a, p, n_base + 8 * j, acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
    } else {
      const int sh0 = a.x0_shift;
      const long long pix0 = ((long long)p.n * (a.Hout >> sh0) + (p.y >> sh0)) * (a.Wout >> sh0) + (p.x >> sh0);
      const float nz = (p.valid && a.noise) ? __ldg(a.noise + p.pix) : 0.f;
#pragma unroll
      for (int j = 0; j < BNT / 8; ++j) epi_spade1(a, p, pix0, nz, (n_base + 8 * j) >> 1, acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
    }
  }
}

namespace {

template <int BNT>
int launch_tf32x3(const Tf32Args& args, int grid, size_t smem, cudaStream_t st) {
  static bool attr_done = false;
  if (!attr_done) {
    cudaError_t e = cudaFuncSetAttribute(conv_tf32x3_kernel<BNT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemMax);
    if (e != cudaSuccess) return set_error(HRV_ECUDA, "cudaFuncSetAttribute(conv_tf32x3): %s", cudaGetErrorString(e));
    attr_done = true;
  }
  conv_tf32x3_kernel<BNT><<<grid, kThreads, smem, st>>>(args);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(HRV_ECUDA, "conv_tf32x3 launch: %s", cudaGetErrorString(e));
  return HRV_OK;
}

}  // namespace
}  // namespace hrv

namespace hrv_host {

int conv2d_fwd_tf32x3(const hrv_conv_params* p, hrv_stream stream) {
  using namespace hrv;
  const hrv_tensor& in = p->in;
  const hrv_tensor& out = p->out;
  if (((uintptr_t)in.ptr & 15) || (in.pitch % 8) || in.pitch < in.c)
    return set_error(HRV_EINVAL, "conv(fp32): input needs 16-byte aligned ptr and pitch %% 8 == 0 (pitch=%d c=%d)", in.pitch, in.c);
  if (p->bk != 64 && p->bk != 32 && p->bk != 16) return set_error(HRV_EINVAL, "conv(fp32): bk must be 64/32/16");
  if (p->bn < 16 || p->bn > 256 || (p->bn % 16)) return set_error(HRV_EINVAL, "conv(fp32): bn=%d must be a multiple of 16 in [16,256]", p->bn);
  if (p->kh < 1 || p->kw < 1 || p->n_gemm < 1) return set_error(HRV_EINVAL, "conv(fp32): bad kh/kw/n_gemm");
  if (out.n != in.n) return set_error(HRV_EINVAL, "conv(fp32): batch mismatch");
  if (((uintptr_t)p->wpack & 15)) return set_error(HRV_EINVAL, "conv(fp32): wpack must be 16-byte aligned");
  if (out.dtype != HRV_F32 || !out.ptr || ((uintptr_t)out.ptr & 3))
    return set_error(HRV_EINVAL, "conv(fp32): an fp32 input needs an fp32 output (one storage type per call)");
  if (p->res.ptr && p->res.dtype != HRV_F32) return set_error(HRV_EINVAL, "conv(fp32): the residual must be fp32 (one storage type per call)");
  if (p->res.ptr && p->res_mode != HRV_RES_ADD)
    return set_error(HRV_EUNSUPPORTED, "conv(fp32): the gate residual modes belong to the backward pass; fp32 storage is inference-only");
  if (p->out_layout != HRV_NHWC && p->out_layout != HRV_NCHW) return set_error(HRV_EINVAL, "conv(fp32): out_layout %d", p->out_layout);

  Tf32Args a;
  memset(&a, 0, sizeof(a));
  a.Nimg = out.n; a.Hout = out.h; a.Wout = out.w;
  const int bnt = p->n_gemm <= 64 ? 64 : 128;
  const int TW = pick_pow2(out.w, 128);
  const int TH = pick_pow2(out.h, 128 / TW);
  const int TN = 128 / (TW * TH);
  a.tw_log = log2i(TW); a.th_log = log2i(TH);
  a.tiles_x = (out.w + TW - 1) / TW;
  a.tiles_y = (out.h + TH - 1) / TH;
  const int tiles_img = (out.n + TN - 1) / TN;
  a.tiles_n = (p->n_gemm + bnt - 1) / bnt;
  a.KH = p->kh; a.KW = p->kw; a.off_y = p->off_y; a.off_x = p->off_x;
  a.chunks = (in.c + 31) / 32;
  a.n_gemm = p->n_gemm;
  a.epi = p->epi; a.act = p->act;
  a.scale = p->scale; a.shift = p->shift;
  a.out = (float*)out.ptr; a.out_pitch = out.pitch; a.out_layout = p->out_layout; a.out_c = out.c;
  const int c8 = (out.c + 7) & ~7;
  a.store_c = (p->out_layout == HRV_NHWC && out.pitch >= c8) ? c8 : out.c;
  if (p->res.ptr) {
    a.res = (const float*)p->res.ptr; a.res_pitch = p->res.pitch;
    a.res_c = p->res.pitch >= a.store_c ? a.store_c : out.c;
  }

  if (p->epi == HRV_EPI_SPADE) {
    const int C = p->x0.c + (p->x1.ptr ? p->x1.c : 0);
    if (p->n_gemm != 2 * C) return set_error(HRV_EINVAL, "conv(fp32 spade): n_gemm=%d must equal 2*(x0.c+x1.c)=%d", p->n_gemm, 2 * C);
    if (p->x0.dtype != HRV_F32 || (p->x1.ptr && p->x1.dtype != HRV_F32))
      return set_error(HRV_EINVAL, "conv(fp32 spade): x0/x1 must be fp32 (one storage type per call)");
    if (p->gamma_out.ptr) return set_error(HRV_EUNSUPPORTED, "conv(fp32 spade): gamma_out belongs to the backward pass; fp32 storage is inference-only");
    if ((p->x0.c % 8) || (C % 8) || p->out_layout != HRV_NHWC || !p->mean || !p->rstd || !p->x0.ptr)
      return set_error(HRV_EINVAL, "conv(fp32 spade): channel counts must be multiples of 8, output NHWC, mean/rstd/x0 set");
    if (p->x0_shift && ((out.h & 1) || (out.w & 1) || p->x0.h * 2 != out.h || p->x0.w * 2 != out.w))
      return set_error(HRV_EINVAL, "conv(fp32 spade): x0_shift needs x0 at exactly half resolution");
    if (!p->x0_shift && (p->x0.h != out.h || p->x0.w != out.w)) return set_error(HRV_EINVAL, "conv(fp32 spade): x0 extent mismatch");
    if (out.c != C) return set_error(HRV_EINVAL, "conv(fp32 spade): out.c must equal C");
    a.x0 = (const float*)p->x0.ptr; a.x0_c = p->x0.c; a.x0_pitch = p->x0.pitch; a.x0_shift = p->x0_shift ? 1 : 0;
    a.x1 = (const float*)p->x1.ptr; a.x1_pitch = p->x1.pitch;
    a.mean = p->mean; a.rstd = p->rstd; a.noise = p->noise; a.noise_scale = p->noise_scale; a.C_mod = C;
  } else if (p->epi != HRV_EPI_LINEAR) {
    return set_error(HRV_EINVAL, "conv(fp32): unknown epilogue %d", p->epi);
  }

  // ---- pipeline: as many stages as fit next to the lo scratch tiles in one SM's shared memory, at most one per K step
  const uint32_t stage_bytes = kABytes + 2u * (uint32_t)bnt * kRowBytes;
  const int KT = p->kh * p->kw * a.chunks;
  int stages = (int)((kSmemMax - 2048u - kScratch) / stage_bytes);
  if (stages > kMaxStages) stages = kMaxStages;
  if (stages > KT) stages = KT < 2 ? 2 : KT;
  a.stages = stages;
  const size_t smem = 2048 + kScratch + (size_t)stages * stage_bytes;  // 1 KB alignment slack + 1 KB of barriers

  // ---- tensor maps
  const int elem = 4;
  const int taps = p->kh * p->kw;
  {
    cuuint64_t dims[4] = {(cuuint64_t)in.c, (cuuint64_t)in.w, (cuuint64_t)in.h, (cuuint64_t)in.n};
    cuuint64_t strides[3] = {(cuuint64_t)in.pitch * elem, (cuuint64_t)in.w * in.pitch * elem, (cuuint64_t)in.h * in.w * in.pitch * elem};
    cuuint32_t box[4] = {32, (cuuint32_t)TW, (cuuint32_t)TH, (cuuint32_t)TN};
    cuuint32_t es[4] = {1, 1, 1, 1};
    int rc = encode_tensor_map(&a.tmA, 4, in.ptr, dims, strides, box, es, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_DATA_TYPE_FLOAT32);
    if (rc) return rc;
  }
  {
    // pre-split weights [2][taps][n_pad][cin_k] as laid out by hrv_pack_conv_weight_tf32x2 for this (bk, bn)
    const cuuint64_t cin_k = (cuuint64_t)((in.c + p->bk - 1) / p->bk) * p->bk;
    const cuuint64_t n_pad = (cuuint64_t)((p->n_gemm + p->bn - 1) / p->bn) * p->bn;
    cuuint64_t dims[4] = {cin_k, n_pad, (cuuint64_t)taps, 2};
    cuuint64_t strides[3] = {cin_k * elem, n_pad * cin_k * elem, (cuuint64_t)taps * n_pad * cin_k * elem};
    cuuint32_t box[4] = {32, (cuuint32_t)bnt, 1, 2};
    cuuint32_t es[4] = {1, 1, 1, 1};
    int rc = encode_tensor_map(&a.tmB, 4, const_cast<void*>(p->wpack), dims, strides, box, es, CU_TENSOR_MAP_SWIZZLE_128B,
                               CU_TENSOR_MAP_DATA_TYPE_FLOAT32);
    if (rc) return rc;
  }
  const long long total = (long long)a.tiles_n * a.tiles_x * a.tiles_y * tiles_img;
  if (total > 0x7FFFFFFFLL) return set_error(HRV_EINVAL, "conv(fp32): too many tiles");
  cudaStream_t st = (cudaStream_t)stream;
  return bnt == 64 ? launch_tf32x3<64>(a, (int)total, smem, st) : launch_tf32x3<128>(a, (int)total, smem, st);
}

}  // namespace hrv_host
