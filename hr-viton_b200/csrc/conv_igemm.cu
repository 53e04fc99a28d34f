// conv_igemm.cu — NHWC convolution as an im2col-free implicit GEMM on sm_90a (wgmma + TMA + mbarrier).
//
//   GEMM view:  M = output pixels (128 per tile = TN x TH x TW box), N = output channels (BNT = 64 or 128 per tile),
//               K = taps x input channels, walked tap by tap in chunks of 64 channels.
//   A operand:  one TMA 4-D box {64 ch, TW, TH, TN} of the NHWC input per (tap, channel chunk), shifted by the tap offset;
//               TMA zero-fills out-of-range pixels (= the convolution's zero padding) and channels past the input's or the packed
//               weight's channel count, so every layer runs on 64-channel K blocks whatever block size its weights were packed with.
//   B operand:  one TMA box {64, BNT} of the packed weights [taps][n_pad][cin_k] (K-major); rows past n_pad are zero fill.
//   MMA:        wgmma.mma_async m64nBNTk16, bf16 (fp16 flavour: f16) operands from 128B-swizzled shared memory, fp32 accumulators in
//               the registers of the consumer warpgroups.
//   Pipeline:   one CTA per (pixel tile, N tile), two CTAs per SM (the epilogue of one overlaps the mainloop of the other).
//               Warp 8 = TMA producer, warpgroups 0 / 1 = consumers for pixels 0-63 / 64-127 of the tile.  A ring of `stages`
//               (A + B) stages with full (transaction count) / empty (one arrival per consumer warp) mbarriers.
//   Epilogues:  LINEAR  out = act(acc*scale + shift (+ residual))      (bias / folded BatchNorm / residual / tanh)
//               SPADE   out = act((x + noise*ns - mean)*rstd*(1+gamma) + beta), gamma/beta = interleaved GEMM columns: a thread's
//                       accumulator pair (2j, 2j+1) is (gamma, beta) of one channel, so the SPADE modulation never leaves registers
//                       (network_generator.py:115-121,170-171).
//
// Replaces nn.Conv2d at networks.py:60-93,178-192 and network_generator.py:97-99,132-135,184-201,263-272.
#include <stdlib.h>

#include "hrv_host.h"
#include "hrv_ptx.cuh"

namespace hrv {

constexpr int kMaxStages = 16;
constexpr int kConsumers = 2;                       // consumer warpgroups (64 pixels each)
constexpr int kThreads = 128 * kConsumers + 32;     // + one producer warp
constexpr uint32_t kRowBytes = 128;                 // 64 channels of 2 bytes: one SWIZZLE_128B row
constexpr uint32_t kABytes = 128 * kRowBytes;       // 128 pixels
constexpr uint32_t kSmemPerCta = 110u * 1024u;      // two CTAs per SM (plus 1 KB reserved per CTA)

struct alignas(64) ConvArgs {
  CUtensorMap tmA;
  CUtensorMap tmB;
  int Nimg, Hout, Wout;
  int tw_log, th_log;
  int tiles_x, tiles_y, tiles_img, tiles_n;
  int KH, KW, off_y, off_x, chunks;
  int stages, n_gemm;
  int epi, act;
  const float* scale;
  const float* shift;
  void* out;
  int out_pitch, out_dtype, out_layout, out_c;
  const void* res;
  int res_pitch, res_dtype, res_mode;  // res_mode: 0 add, 1 ReLU gate, 2 LeakyReLU(0.2) gate (bf16 res only)
  const __nv_bfloat16* x0;
  int x0_c, x0_pitch, x0_shift;
  const __nv_bfloat16* x1;
  int x1_pitch;
  const float* mean;
  const float* rstd;
  const float* noise;
  const float* noise_scale;
  int C_mod;
  __nv_bfloat16* gamma_out;
  int gamma_pitch;
};

// One output pixel as seen by an epilogue thread.
struct EpiPix {
  int x, y, n;
  bool valid;
  long long pix;
};

// LINEAR epilogue of two adjacent GEMM columns (c, c+1) of one pixel: out = act(acc*scale + shift (+ res | * act'(res))).
// bf16 NHWC outputs also write the pad channels up to the next multiple of 8 (as act(0) + res), fp32 outputs stop at out_c.
__device__ __forceinline__ void epi_linear2(const ConvArgs& a, const EpiPix& p, int c, float v0, float v1) {
  const bool bf16_nhwc = a.out_dtype == 0 && a.out_layout == 0;
  const int store_c = bf16_nhwc ? ((a.out_c + 7) & ~7) : a.out_c;
  if (!p.valid || c >= store_c) return;
  float f[2] = {v0, v1};
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int j = c + i;
    const bool in = j < a.n_gemm;
    const float sc = in ? (a.scale ? __ldg(a.scale + j) : 1.f) : 0.f;
    const float sh = (in && a.shift) ? __ldg(a.shift + j) : 0.f;
    f[i] = fmaf(f[i], sc, sh);
  }
  if (a.res) {
    if (a.res_dtype == 0) {
      const uint32_t rv = __ldg(reinterpret_cast<const unsigned int*>(reinterpret_cast<const __nv_bfloat16*>(a.res) + p.pix * a.res_pitch + c));
      const float rf[2] = {bf16_lo(rv), bf16_hi(rv)};
      if (a.res_mode == 0) {
        f[0] += rf[0]; f[1] += rf[1];
      } else {  // activation backward of the layer below, fused: multiply by act'(its saved output)
        const float slope = a.res_mode == 1 ? 0.f : 0.2f;
#pragma unroll
        for (int i = 0; i < 2; ++i) f[i] = rf[i] > 0.f ? f[i] : f[i] * slope;
      }
    } else {
      const float* rp = reinterpret_cast<const float*>(a.res) + p.pix * a.res_pitch + c;
#pragma unroll
      for (int i = 0; i < 2; ++i)
        if (c + i < a.out_c) f[i] += __ldg(rp + i);
    }
  }
  f[0] = apply_act(f[0], a.act);
  f[1] = apply_act(f[1], a.act);
  if (a.out_dtype == 0) {  // c even, pitch % 8 == 0: a 4-byte store
    *reinterpret_cast<uint32_t*>(reinterpret_cast<__nv_bfloat16*>(a.out) + p.pix * a.out_pitch + c) = pack_bf16(f[0], f[1]);
  } else if (a.out_layout == 0) {
    float* op = reinterpret_cast<float*>(a.out) + p.pix * a.out_pitch + c;
    op[0] = f[0];
    if (c + 1 < a.out_c) op[1] = f[1];
  } else {  // fp32 NCHW
    float* op = reinterpret_cast<float*>(a.out);
    const long long hw = (long long)a.Hout * a.Wout;
#pragma unroll
    for (int i = 0; i < 2; ++i)
      if (c + i < a.out_c) op[((long long)p.n * a.out_c + c + i) * hw + (long long)p.y * a.Wout + p.x] = f[i];
  }
}

// SPADE epilogue of one channel ch of one pixel; g, b = the (gamma, beta) accumulators of columns 2ch, 2ch+1.
__device__ __forceinline__ void epi_spade1(const ConvArgs& a, const EpiPix& p, long long pix0, float nz, int ch, float g, float b) {
  if (!p.valid || ch >= a.C_mod) return;
  const __nv_bfloat16* xp = (ch < a.x0_c) ? (a.x0 + pix0 * a.x0_pitch + ch) : (a.x1 + p.pix * a.x1_pitch + (ch - a.x0_c));
  const float xs = __bfloat162float(*xp);
  const float mu = __ldg(a.mean + (long long)p.n * a.C_mod + ch);
  const float rs = __ldg(a.rstd + (long long)p.n * a.C_mod + ch);
  const float ns = a.noise_scale ? __ldg(a.noise_scale + ch) : 0.f;
  const float gm = g + (a.shift ? __ldg(a.shift + 2 * ch) : 0.f);
  const float bt = b + (a.shift ? __ldg(a.shift + 2 * ch + 1) : 0.f);
  const float xn = (fmaf(nz, ns, xs) - mu) * rs;
  const float o = apply_act(fmaf(xn, 1.f + gm, bt), a.act);
  if (a.gamma_out) a.gamma_out[p.pix * a.gamma_pitch + ch] = __float2bfloat16(gm);  // training: gamma for the backward pass
  reinterpret_cast<__nv_bfloat16*>(a.out)[p.pix * a.out_pitch + ch] = __float2bfloat16(o);
}

template <int BNT>
__device__ __forceinline__ void wgmma_tile(float (&d)[BNT / 2], uint64_t da, uint64_t db, uint32_t scale_d) {
  if constexpr (BNT == 64) wgmma_n64<0, 0>(d, da, db, scale_d);
  else wgmma_n128<0, 0>(d, da, db, scale_d);
}

template <int BNT>
__global__ void __launch_bounds__(kThreads, 2) conv_wgmma_kernel(const __grid_constant__ ConvArgs a) {
  constexpr uint32_t B_BYTES = (uint32_t)BNT * kRowBytes;
  constexpr uint32_t STAGE = kABytes + B_BYTES;  // both parts multiples of 1024 B: every operand starts at swizzle phase 0
  constexpr int R = BNT / 2;                     // accumulator registers per consumer thread

  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  auto bar_full = [&](int s) { return base + 8u * s; };
  auto bar_empty = [&](int s) { return base + 128u + 8u * s; };
  const uint32_t stage0 = base + 1024u;

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
        tma_load_4d(sa, &a.tmA, bar_full(st), kc * 64, x0 + kx, y0 + ky, n0);
        tma_load_3d(sa + kABytes, &a.tmB, bar_full(st), kc * 64, nt * BNT, tap);
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
  const int wg = warp >> 2;
  float acc[R];
#pragma unroll
  for (int i = 0; i < R; ++i) acc[i] = 0.f;
  {
    int st = 0, prev = 0;
    uint32_t ph = 0, sa = stage0;
    for (int k = 0; k < KT; ++k) {
      mbar_wait(bar_full(st), ph);
      wgmma_fence();
      const uint32_t a_row0 = sa + (uint32_t)wg * (64u * kRowBytes);
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {  // K = 16 per instruction: +32 bytes inside the 128-byte swizzle row
        const uint64_t da = make_wgmma_desc(a_row0 + 32u * kk, 8 * kRowBytes, 1);
        const uint64_t db = make_wgmma_desc(sa + kABytes + 32u * kk, 8 * kRowBytes, 1);
        wgmma_tile<BNT>(acc, da, db, (uint32_t)((k | kk) != 0));
      }
      wgmma_commit();
      wgmma_wait<1>();  // the MMAs of the previous stage have finished reading it
      if (k > 0 && lane == 0) mbar_arrive(bar_empty(prev));
      prev = st;
      sa += STAGE;
      if (++st == S) { st = 0; ph ^= 1u; sa = stage0; }
    }
    wgmma_wait<0>();
    fence_regs(acc);
  }

  // ===================================================== epilogue straight from the accumulator registers
  // wgmma m64nN fragment: thread (warp w, lane l) holds rows 16 (w % 4) + l / 4 and that + 8, columns 8 j + 2 (l % 4) + {0, 1}.
  const int tw_mask = (1 << a.tw_log) - 1, th_mask = (1 << a.th_log) - 1;
  const int r_base = wg * 64 + (warp & 3) * 16 + (lane >> 2);
  const int n_base = nt * BNT + 2 * (lane & 3);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int r = r_base + 8 * h;
    EpiPix p;
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

// ------------------------------------------------------------------------------------------------ host side

template <int BNT>
static int launch_conv(const ConvArgs& args, int grid, size_t smem, cudaStream_t st) {
  static bool attr_done = false;
  if (!attr_done) {
    cudaError_t e = cudaFuncSetAttribute(conv_wgmma_kernel<BNT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemPerCta);
    if (e != cudaSuccess) return set_error(HRV_ECUDA, "cudaFuncSetAttribute(conv_wgmma): %s", cudaGetErrorString(e));
    attr_done = true;
  }
  conv_wgmma_kernel<BNT><<<grid, kThreads, smem, st>>>(args);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(HRV_ECUDA, "conv_wgmma launch: %s", cudaGetErrorString(e));
  return HRV_OK;
}

}  // namespace hrv

using namespace hrv;

extern "C" int hrv_conv2d_fwd(const hrv_conv_params* p, hrv_stream stream) {
  if (!p) return set_error(HRV_EINVAL, "conv: null params");
  const hrv_tensor& in = p->in;
  const hrv_tensor& out = p->out;
  if (in.dtype == HRV_F32) return conv2d_fwd_tf32x3(p, stream);  // fp32 storage: the 3xTF32 kernel of conv_f32.cu
  if (in.dtype != HRV_BF16) return set_error(HRV_EINVAL, "conv: input must be bf16 NHWC");
  if (((uintptr_t)in.ptr & 15) || (in.pitch % 8) || in.pitch < in.c)
    return set_error(HRV_EINVAL, "conv: input needs 16-byte aligned ptr and pitch %% 8 == 0 (pitch=%d c=%d)", in.pitch, in.c);
  if (p->bk != 64 && p->bk != 32 && p->bk != 16) return set_error(HRV_EINVAL, "conv: bk must be 64/32/16");
  if (p->bn < 16 || p->bn > 256 || (p->bn % 16)) return set_error(HRV_EINVAL, "conv: bn=%d must be a multiple of 16 in [16,256]", p->bn);
  if (p->kh < 1 || p->kw < 1 || p->n_gemm < 1) return set_error(HRV_EINVAL, "conv: bad kh/kw/n_gemm");
  if (out.n != in.n) return set_error(HRV_EINVAL, "conv: batch mismatch");
  if (((uintptr_t)p->wpack & 15)) return set_error(HRV_EINVAL, "conv: wpack must be 16-byte aligned");
  if (out.dtype == HRV_BF16 && (p->out_layout != HRV_NHWC || ((uintptr_t)out.ptr & 15) || (out.pitch % 8)))
    return set_error(HRV_EINVAL, "conv: bf16 output must be NHWC, 16-byte aligned, pitch %% 8 == 0");
  if (p->res.ptr && p->res.dtype == HRV_BF16 && (((uintptr_t)p->res.ptr & 15) || (p->res.pitch % 8)))
    return set_error(HRV_EINVAL, "conv: bf16 residual must be 16-byte aligned with pitch %% 8 == 0");

  ConvArgs a;
  memset(&a, 0, sizeof(a));
  a.Nimg = out.n; a.Hout = out.h; a.Wout = out.w;
  // N tile: 64 columns for narrow GEMMs, else 128 (a 64 x 128 fp32 accumulator is 64 registers per thread, which keeps two CTAs
  // resident per SM).  Independent of the packing's bn: the weight map's row extent is the packed n_pad, rows past it are zero fill.
  const int bnt = p->n_gemm <= 64 ? 64 : 128;
  const int TW = pick_pow2(out.w, 128);
  const int TH = pick_pow2(out.h, 128 / TW);
  const int TN = 128 / (TW * TH);
  a.tw_log = log2i(TW); a.th_log = log2i(TH);
  a.tiles_x = (out.w + TW - 1) / TW;
  a.tiles_y = (out.h + TH - 1) / TH;
  a.tiles_img = (out.n + TN - 1) / TN;
  a.tiles_n = (p->n_gemm + bnt - 1) / bnt;
  a.KH = p->kh; a.KW = p->kw; a.off_y = p->off_y; a.off_x = p->off_x;
  a.chunks = (in.c + 63) / 64;
  a.n_gemm = p->n_gemm;
  a.epi = p->epi; a.act = p->act;
  a.scale = p->scale; a.shift = p->shift;
  a.out = out.ptr; a.out_pitch = out.pitch; a.out_dtype = out.dtype; a.out_layout = p->out_layout; a.out_c = out.c;
  a.res = p->res.ptr; a.res_pitch = p->res.pitch; a.res_dtype = p->res.dtype; a.res_mode = p->res.ptr ? p->res_mode : 0;
  if (a.res_mode < 0 || a.res_mode > 2) return set_error(HRV_EINVAL, "conv: res_mode %d", a.res_mode);
  if (a.res_mode && (p->res.dtype != HRV_BF16 || out.dtype != HRV_BF16 || p->out_layout != HRV_NHWC || p->epi != HRV_EPI_LINEAR || p->act != HRV_ACT_NONE))
    return set_error(HRV_EINVAL, "conv: gate modes need a bf16 res, a bf16 NHWC output, the LINEAR epilogue and no activation");

  if (p->epi == HRV_EPI_SPADE) {
    const int C = p->x0.c + (p->x1.ptr ? p->x1.c : 0);
    if (p->n_gemm != 2 * C) return set_error(HRV_EINVAL, "conv(spade): n_gemm=%d must equal 2*(x0.c+x1.c)=%d", p->n_gemm, 2 * C);
    if ((p->x0.c % 8) || (C % 8) || out.dtype != HRV_BF16 || !p->mean || !p->rstd || !p->x0.ptr)
      return set_error(HRV_EINVAL, "conv(spade): channel counts must be multiples of 8, output bf16, mean/rstd/x0 set");
    if (((uintptr_t)p->x0.ptr & 15) || (p->x0.pitch % 8) || (p->x1.ptr && (((uintptr_t)p->x1.ptr & 15) || (p->x1.pitch % 8))))
      return set_error(HRV_EINVAL, "conv(spade): x0/x1 alignment");
    if (p->x0_shift && ((out.h & 1) || (out.w & 1) || p->x0.h * 2 != out.h || p->x0.w * 2 != out.w))
      return set_error(HRV_EINVAL, "conv(spade): x0_shift needs x0 at exactly half resolution");
    if (!p->x0_shift && (p->x0.h != out.h || p->x0.w != out.w)) return set_error(HRV_EINVAL, "conv(spade): x0 extent mismatch");
    if (out.c != C) return set_error(HRV_EINVAL, "conv(spade): out.c must equal C");
    a.x0 = (const __nv_bfloat16*)p->x0.ptr; a.x0_c = p->x0.c; a.x0_pitch = p->x0.pitch; a.x0_shift = p->x0_shift ? 1 : 0;
    a.x1 = (const __nv_bfloat16*)p->x1.ptr; a.x1_pitch = p->x1.pitch;
    a.mean = p->mean; a.rstd = p->rstd; a.noise = p->noise; a.noise_scale = p->noise_scale; a.C_mod = C;
    if (p->gamma_out.ptr) {
      if (p->gamma_out.dtype != HRV_BF16 || ((uintptr_t)p->gamma_out.ptr & 15) || (p->gamma_out.pitch % 8) || p->gamma_out.c != C)
        return set_error(HRV_EINVAL, "conv(spade): gamma_out must be bf16 (n,h,w,C), 16-byte aligned");
      a.gamma_out = (__nv_bfloat16*)p->gamma_out.ptr; a.gamma_pitch = p->gamma_out.pitch;
    }
  } else if (p->epi != HRV_EPI_LINEAR) {
    return set_error(HRV_EINVAL, "conv: unknown epilogue %d", p->epi);
  }

  // ---- pipeline: as many stages as fit in half of an SM's shared memory (two CTAs per SM), at most one per K step
  const uint32_t stage_bytes = kABytes + (uint32_t)bnt * kRowBytes;
  const int KT = p->kh * p->kw * a.chunks;
  int stages = (int)((kSmemPerCta - 2048u) / stage_bytes);
  if (stages > kMaxStages) stages = kMaxStages;
  if (stages > KT) stages = KT < 2 ? 2 : KT;
  a.stages = stages;
  const size_t smem = 2048 + (size_t)stages * stage_bytes;  // 1 KB alignment slack + 1 KB of barriers

  // ---- tensor maps
  const int elem = 2;
  const int taps = p->kh * p->kw;
  {
    cuuint64_t dims[4] = {(cuuint64_t)in.c, (cuuint64_t)in.w, (cuuint64_t)in.h, (cuuint64_t)in.n};
    cuuint64_t strides[3] = {(cuuint64_t)in.pitch * elem, (cuuint64_t)in.w * in.pitch * elem, (cuuint64_t)in.h * in.w * in.pitch * elem};
    cuuint32_t box[4] = {64, (cuuint32_t)TW, (cuuint32_t)TH, (cuuint32_t)TN};
    cuuint32_t es[4] = {1, 1, 1, 1};
    int rc = encode_tensor_map(&a.tmA, 4, in.ptr, dims, strides, box, es, CU_TENSOR_MAP_SWIZZLE_128B);
    if (rc) return rc;
  }
  {
    // packed weights [taps][n_pad][cin_k] as laid out by hrv_pack_conv_weight for this (bk, bn)
    const cuuint64_t cin_k = (cuuint64_t)((in.c + p->bk - 1) / p->bk) * p->bk;
    const cuuint64_t n_pad = (cuuint64_t)((p->n_gemm + p->bn - 1) / p->bn) * p->bn;
    cuuint64_t dims[3] = {cin_k, n_pad, (cuuint64_t)taps};
    cuuint64_t strides[2] = {cin_k * elem, n_pad * cin_k * elem};
    cuuint32_t box[3] = {64, (cuuint32_t)bnt, 1};
    cuuint32_t es[3] = {1, 1, 1};
    int rc = encode_tensor_map(&a.tmB, 3, const_cast<void*>(p->wpack), dims, strides, box, es, CU_TENSOR_MAP_SWIZZLE_128B);
    if (rc) return rc;
  }
  const long long total = (long long)a.tiles_n * a.tiles_x * a.tiles_y * a.tiles_img;
  if (total > 0x7FFFFFFFLL) return set_error(HRV_EINVAL, "conv: too many tiles");
  cudaStream_t st = (cudaStream_t)stream;
  return bnt == 64 ? launch_conv<64>(a, (int)total, smem, st) : launch_conv<128>(a, (int)total, smem, st);
}
