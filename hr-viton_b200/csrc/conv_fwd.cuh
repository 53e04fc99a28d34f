// conv_fwd.cuh — what the two forward convolution kernels share: conv_wgmma_kernel (conv_igemm.cu, 16-bit storage) and
// conv_tf32x3_kernel (conv_f32.cu, fp32 storage).  Both are NHWC implicit GEMMs with the same tiling and warp roles:
//
//   GEMM view:  M = output pixels (128 per tile = TN x TH x TW box), N = output channels (BNT = 64 or 128 per tile),
//               K = taps x input channels, walked tap by tap in K blocks of one 128-byte SWIZZLE_128B row per pixel (64 16-bit or
//               32 fp32 channels).
//   A operand:  one TMA 4-D box {K block, TW, TH, TN} of the NHWC input per (tap, K block), shifted by the tap offset; TMA zero-fills
//               out-of-range pixels (= the convolution's zero padding) and channels past the input's or the packed weight's channel
//               count, so every layer runs on full K blocks whatever block size its weights were packed with.
//   B operand:  one TMA box {K block, BNT} per weight plane of the packed weights [planes][taps][n_pad][cin_k] (K-major); rows past
//               n_pad are zero fill.
//   Pipeline:   warp 8 = TMA producer, warpgroups 0 / 1 = consumers for pixels 0-63 / 64-127 of the tile.  A ring of `stages`
//               (A + B) stages with full (transaction count) / empty (one arrival per consumer warp) mbarriers.
//   Epilogues:  staged: the accumulators go through an fp32 tile in the idle stage ring and leave in row order, as 16-byte vectors.
//               LINEAR  out = act(acc*scale + shift (+ residual))      (bias / folded BatchNorm / residual / tanh)
//               SPADE   out = act((x + noise*ns - mean)*rstd*(1+gamma) + beta), gamma/beta = interleaved GEMM columns (2k, 2k+1)
//                       of channel k, so one 8-channel group of the modulation is 16 adjacent tile columns
//                       (network_generator.py:115-121,170-171).
//               The gate residual modes and gamma_out serve the backward pass and exist on 16-bit storage only.
//
// Shared memory of a CTA: 1 KB of mbarriers (full at +0, empty at +128, halo at +256), then `scratch` bytes the kernel owns, then
// the halo slots (halo main loop only) and the stage ring (together at least the 128 x BNT fp32 epilogue tile).
#pragma once
#include "hrv_host.h"
#include "hrv_ptx.cuh"

namespace hrv {

constexpr int kConvConsumers = 2;                        // consumer warpgroups (64 pixels each)
constexpr int kConvThreads = 128 * kConvConsumers + 32;  // + one producer warp
constexpr uint32_t kConvRowBytes = 128;                  // one K block of one pixel / weight row: one SWIZZLE_128B row
constexpr uint32_t kConvABytes = 128 * kConvRowBytes;    // 128 pixels

// Halo main loop of conv_wgmma_kernel (16-bit storage, chosen by conv_fwd from the shape): the tile is 2 rows x kHaloTW pixels of
// one image, and the producer loads its input halo once per K chunk c, as the TMA box {64 ch, kHaloTW + KW - 1, 2 + KH - 1, 1}, into
// its own 1024-byte aligned slot with its own full barrier (bar_halo).  The stage ring behind the slots carries only B boxes.  Every
// tap then reads its A operand out of the slot: warpgroup w's 64 pixels are one contiguous run of halo row w + ky from pixel kx.
constexpr int kHaloTW = 64;
__host__ __device__ constexpr uint32_t halo_box_bytes(int kh, int kw) { return kConvRowBytes * (uint32_t)(kHaloTW + kw - 1) * (uint32_t)(1 + kh); }
__host__ __device__ constexpr uint32_t halo_slot_bytes(int kh, int kw) { return (halo_box_bytes(kh, kw) + 1023u) & ~1023u; }
__device__ __forceinline__ uint32_t bar_halo(uint32_t bars, int c) { return bars + 256u + 8u * c; }

// T = activation storage: __nv_bfloat16 (__half in the fp16 flavour) or float.
template <typename T>
constexpr bool kStorage16 = sizeof(T) == 2;

template <typename T>
struct alignas(64) ConvArgs {
  CUtensorMap tmA;
  CUtensorMap tmB;
  int Nimg, Hout, Wout;
  int tw_log, th_log;
  int tiles_x, tiles_y, tiles_n;
  int KH, KW, off_y, off_x, chunks;
  int halo;                        // conv_wgmma_kernel's halo main loop (tmA boxes the tile's halo; stage ring = B boxes only)
  int stages, n_gemm;
  int epi, act;
  const float* scale;
  const float* shift;
  void* out;                       // T NHWC; on 16-bit storage also fp32 NHWC / NCHW
  int out_pitch, out_dtype, out_layout, out_c;
  int store_c;                     // LINEAR writes channels [0, store_c): out_c, or up to the next multiple of 8 (pad channels)
  int out_vec;                     // out is the storage type, NHWC, 16-byte aligned, pitch and store_c multiples of 8: 8-channel stores
  const void* res;                 // T NHWC; on 16-bit storage also fp32 NHWC
  int res_pitch, res_dtype, res_c;  // an fp32 residual is added to channels [0, res_c)
  int res_mode;                    // 0 add, 1 ReLU gate, 2 LeakyReLU(0.2) gate (16-bit res only)
  const T* x0;
  int x0_c, x0_pitch, x0_shift;
  const T* x1;
  int x1_pitch;
  const float* mean;
  const float* rstd;
  const float* noise;
  const float* noise_scale;
  int C_mod;
  T* gamma_out;                    // 16-bit storage only
  int gamma_pitch;
};

// Tile of one CTA (N tile, pixel tile (x, y), image group) and the 1024-byte aligned start of its shared memory.
struct ConvTile {
  int nt, tx, ty, ti;
  uint32_t bars;
};

// Decodes the CTA's tile and initialises the barrier ring; every thread of the CTA calls it.
template <typename T>
__device__ __forceinline__ ConvTile conv_prologue(const ConvArgs<T>& a) {
  extern __shared__ uint8_t smem_raw[];
  ConvTile t;
  t.bars = (smem_u32(smem_raw) + 1023u) & ~1023u;
  t.nt = blockIdx.x % a.tiles_n;
  int mt = blockIdx.x / a.tiles_n;
  t.tx = mt % a.tiles_x;
  mt /= a.tiles_x;
  t.ty = mt % a.tiles_y;
  t.ti = mt / a.tiles_y;
  const int S = a.stages;
  if (threadIdx.x == 0) {
    for (int s = 0; s < S; ++s) {
      mbar_init(bar_full(t.bars, s), 1);
      mbar_init(bar_empty(t.bars, s), 4 * kConvConsumers);  // one arrival per consumer warp
    }
    for (int c = 0; c < (a.halo ? a.chunks : 0); ++c) mbar_init(bar_halo(t.bars, c), 1);
    fence_mbar_init();
  }
  __syncthreads();
  return t;
}

// TMA producer (one lane): per K step one A box of KB channels and the B box of PLANES weight planes into the next stage.
template <int BNT, int KB, int PLANES, typename T>
__device__ __forceinline__ void conv_produce(const ConvArgs<T>& a, const ConvTile& t, uint32_t stage0) {
  constexpr uint32_t STAGE = kConvABytes + PLANES * (uint32_t)BNT * kConvRowBytes;
  tma_prefetch_desc(&a.tmA);
  tma_prefetch_desc(&a.tmB);
  const int KT = a.KH * a.KW * a.chunks;
  const int x0 = (t.tx << a.tw_log) - a.off_x;
  const int y0 = (t.ty << a.th_log) - a.off_y;
  const int n0 = t.ti << (7 - a.tw_log - a.th_log);
  int ky = 0, kx = 0, kc = 0, tap = 0;
  StageRing ring(stage0, STAGE, a.stages);
  for (int k = 0; k < KT; ++k) {
    const uint32_t full = bar_full(t.bars, ring.stage);
    mbar_wait(bar_empty(t.bars, ring.stage), ring.phase ^ 1u);
    mbar_arrive_expect_tx(full, STAGE);
    tma_load_4d(ring.addr, &a.tmA, full, kc * KB, x0 + kx, y0 + ky, n0);
    if constexpr (PLANES == 1) tma_load_3d(ring.addr + kConvABytes, &a.tmB, full, kc * KB, t.nt * BNT, tap);
    else tma_load_4d(ring.addr + kConvABytes, &a.tmB, full, kc * KB, t.nt * BNT, tap, 0);  // all planes in one box
    if (++kc == a.chunks) {
      kc = 0;
      ++tap;
      if (++kx == a.KW) { kx = 0; ++ky; }
    }
    ring.next();
  }
}

// ------------------------------------------------------------------------------------------------ epilogue
// The epilogue runs after the main loop and is staged through the stage ring (halo slots first in the halo main loop), which is idle
// by then (the producer issued exactly KT loads, plus one halo box per chunk, and the consumers waited on all of them):
//   1. each consumer thread writes its wgmma fragment into an fp32 [128 pixels][BNT] tile at the start of the ring;
//   2. the 256 consumer threads walk the tile in row order.  A thread owns one 8-channel group (8 LINEAR columns, or 16 interleaved
//      SPADE gamma/beta columns) and visits every (256 / threads per pixel)-th pixel, so x, the residual, out and gamma_out move as
//      16-byte vectors of consecutive channels and the per-channel constants are loaded once.  fp32 outputs that are not the storage
//      type (flows, discriminator logits, NCHW heads) keep one element per store, with lanes along pixels so that NCHW rows coalesce.
// Tile layout: XOR swizzle, no padding.  Row r is BNT floats; its 16-byte chunk q is stored at chunk q ^ (r & 7).  A fragment store
// (8 rows x 32 bytes per warp) then hits every bank twice (2 wavefronts, the minimum for 256 bytes), and a row-order 16-byte load
// (32 / G rows x G groups per warp, G a power of two) hits every bank four times (4 wavefronts, the minimum for 512 bytes).

constexpr uint32_t kEpiBar = 3;  // named barrier of the 256 consumer threads (conv_f32.cu uses 1 and 2 in its main loop)

__host__ __device__ constexpr uint32_t conv_tile_bytes(int bnt) { return 128u * (uint32_t)bnt * 4u; }

// Byte offset of element (pixel r, tile column c) in the staged tile.
template <int BNT>
__device__ __forceinline__ uint32_t tile_off(int r, int c) {
  return (uint32_t)r * (BNT * 4u) + ((((uint32_t)c >> 2) ^ ((uint32_t)r & 7u)) << 4) + (((uint32_t)c & 3u) << 2);
}

// One output pixel: row r of the tile.
struct EpiPix {
  int x, y, n;
  bool valid;
  long long pix;
};

template <typename T>
__device__ __forceinline__ EpiPix epi_pix(const ConvArgs<T>& a, const ConvTile& t, int r) {
  EpiPix p;
  p.x = (t.tx << a.tw_log) + (r & ((1 << a.tw_log) - 1));
  p.y = (t.ty << a.th_log) + ((r >> a.tw_log) & ((1 << a.th_log) - 1));
  p.n = (t.ti << (7 - a.tw_log - a.th_log)) + (r >> (a.tw_log + a.th_log));
  p.valid = (p.x < a.Wout) && (p.y < a.Hout) && (p.n < a.Nimg);
  p.pix = ((long long)p.n * a.Hout + p.y) * a.Wout + p.x;
  return p;
}

// Eight consecutive activations <-> fp32 (16-byte aligned).
__device__ __forceinline__ void ld8(const __nv_bfloat16* p, float (&v)[8]) {
  const uint4 u = __ldg(reinterpret_cast<const uint4*>(p));
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) { v[2 * i] = bf16_lo(w[i]); v[2 * i + 1] = bf16_hi(w[i]); }
}
__device__ __forceinline__ void ld8(const float* p, float (&v)[8]) {
  const float4 u = __ldg(reinterpret_cast<const float4*>(p)), w = __ldg(reinterpret_cast<const float4*>(p) + 1);
  v[0] = u.x; v[1] = u.y; v[2] = u.z; v[3] = u.w; v[4] = w.x; v[5] = w.y; v[6] = w.z; v[7] = w.w;
}
__device__ __forceinline__ void st8(__nv_bfloat16* p, const float (&v)[8]) {
  *reinterpret_cast<uint4*>(p) = make_uint4(pack_bf16(v[0], v[1]), pack_bf16(v[2], v[3]), pack_bf16(v[4], v[5]), pack_bf16(v[6], v[7]));
}
__device__ __forceinline__ void st8(float* p, const float (&v)[8]) {
  reinterpret_cast<float4*>(p)[0] = make_float4(v[0], v[1], v[2], v[3]);
  reinterpret_cast<float4*>(p)[1] = make_float4(v[4], v[5], v[6], v[7]);
}

// LINEAR scale / shift of GEMM column j; columns past n_gemm (pad channels) become act(0) (+ res).
template <typename T>
__device__ __forceinline__ void lin_coef(const ConvArgs<T>& a, int j, float& sc, float& sh) {
  const bool in = j < a.n_gemm;
  sc = in ? (a.scale ? __ldg(a.scale + j) : 1.f) : 0.f;
  sh = (in && a.shift) ? __ldg(a.shift + j) : 0.f;
}

// Threads per pixel of the row pass: `groups` 8-channel groups rounded up to a power of two (returned as log2).
__device__ __forceinline__ int groups_log(int groups) { return groups <= 1 ? 0 : 32 - __clz(groups - 1); }

// LINEAR into a storage-type NHWC output (a.out_vec): out = act(acc*scale + shift (+ res | * act'(res))), 8 channels per access.
template <int BNT, typename T>
__device__ __forceinline__ void epi_linear_rows(const ConvArgs<T>& a, const ConvTile& t, uint32_t tile, int tid) {
  const int col0 = t.nt * BNT;
  const int groups = (min(BNT, a.store_c - col0) + 7) >> 3;  // store_c % 8 == 0 here
  if (groups <= 0) return;
  const int gl = groups_log(groups);
  const int g = tid & ((1 << gl) - 1);
  if (g >= groups) return;
  const int c = col0 + 8 * g;
  float sc[8], sh[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) lin_coef(a, c + i, sc[i], sh[i]);
  for (int r = tid >> gl; r < 128; r += 256 >> gl) {
    const EpiPix p = epi_pix(a, t, r);
    if (!p.valid) continue;
    float f[8];
    ld_shared_v4(tile + tile_off<BNT>(r, 8 * g), f);
    ld_shared_v4(tile + tile_off<BNT>(r, 8 * g + 4), f + 4);
#pragma unroll
    for (int i = 0; i < 8; ++i) f[i] = fmaf(f[i], sc[i], sh[i]);
    if (a.res) {
      bool res_st = false;
      if constexpr (kStorage16<T>) {
        res_st = a.res_dtype == HRV_BF16;
        if (res_st) {
          float rf[8];
          ld8(static_cast<const T*>(a.res) + p.pix * a.res_pitch + c, rf);
          if (a.res_mode == 0) {
#pragma unroll
            for (int i = 0; i < 8; ++i) f[i] += rf[i];
          } else {  // activation backward of the layer below, fused: multiply by act'(its saved output)
            const float slope = a.res_mode == 1 ? 0.f : 0.2f;
#pragma unroll
            for (int i = 0; i < 8; ++i) f[i] = rf[i] > 0.f ? f[i] : f[i] * slope;
          }
        }
      }
      if (!res_st) {
        const float* rp = static_cast<const float*>(a.res) + p.pix * a.res_pitch + c;
#pragma unroll
        for (int i = 0; i < 8; ++i)
          if (c + i < a.res_c) f[i] += __ldg(rp + i);
      }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) f[i] = apply_act(f[i], a.act);
    st8(static_cast<T*>(a.out) + p.pix * a.out_pitch + c, f);
  }
}

// LINEAR into an fp32 output that is not the storage type (or not 16-byte aligned): one element per store, lanes along pixels.
template <int BNT, typename T>
__device__ __forceinline__ void epi_linear_f32(const ConvArgs<T>& a, const ConvTile& t, uint32_t tile, int tid) {
  const int col0 = t.nt * BNT;
  const int ncols = min(BNT, a.store_c - col0);
  const int r = tid & 127;
  const EpiPix p = epi_pix(a, t, r);
  if (!p.valid) return;
  float* const out = static_cast<float*>(a.out);
  const long long hw = (long long)a.Hout * a.Wout;
  for (int cl = tid >> 7; cl < ncols; cl += 2) {
    const int c = col0 + cl;
    float sc, sh;
    lin_coef(a, c, sc, sh);
    float f = fmaf(ld_shared_f32(tile + tile_off<BNT>(r, cl)), sc, sh);
    if (a.res) {
      bool res_st = false;
      if constexpr (kStorage16<T>) {
        res_st = a.res_dtype == HRV_BF16;
        if (res_st) {
          const float rf = __bfloat162float(static_cast<const T*>(a.res)[p.pix * a.res_pitch + c]);
          if (a.res_mode == 0) f += rf;
          else f = rf > 0.f ? f : f * (a.res_mode == 1 ? 0.f : 0.2f);
        }
      }
      if (!res_st && c < a.res_c) f += __ldg(static_cast<const float*>(a.res) + p.pix * a.res_pitch + c);
    }
    f = apply_act(f, a.act);
    if (a.out_layout == HRV_NHWC) out[p.pix * a.out_pitch + c] = f;
    else out[((long long)p.n * a.out_c + c) * hw + (long long)p.y * a.Wout + p.x] = f;
  }
}

// SPADE: out = act((x + noise*ns - mean)*rstd*(1+gamma) + beta); tile columns (2k, 2k+1) are (gamma, beta) of channel k.
template <int BNT, typename T>
__device__ __forceinline__ void epi_spade_rows(const ConvArgs<T>& a, const ConvTile& t, uint32_t tile, int tid) {
  const int ch0 = t.nt * (BNT / 2);
  const int groups = min(BNT / 2, a.C_mod - ch0) >> 3;  // C_mod % 8 == 0
  if (groups <= 0) return;
  const int gl = groups_log(groups);
  const int g = tid & ((1 << gl) - 1);
  if (g >= groups) return;
  const int ch = ch0 + 8 * g;
  float ns[8], gs[8], bs[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    ns[i] = a.noise_scale ? __ldg(a.noise_scale + ch + i) : 0.f;
    gs[i] = a.shift ? __ldg(a.shift + 2 * (ch + i)) : 0.f;
    bs[i] = a.shift ? __ldg(a.shift + 2 * (ch + i) + 1) : 0.f;
  }
  const bool in_x0 = ch < a.x0_c;  // x0_c % 8 == 0: a group never straddles x0 / x1
  const int sh0 = a.x0_shift;
  int n_cur = -1;
  float mu[8], rs[8];
  for (int r = tid >> gl; r < 128; r += 256 >> gl) {
    const EpiPix p = epi_pix(a, t, r);
    if (!p.valid) continue;
    if (p.n != n_cur) {  // a tile spans several images at small resolutions
      n_cur = p.n;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        mu[i] = __ldg(a.mean + (long long)p.n * a.C_mod + ch + i);
        rs[i] = __ldg(a.rstd + (long long)p.n * a.C_mod + ch + i);
      }
    }
    float xs[8];
    if (in_x0) {
      const long long pix0 = ((long long)p.n * (a.Hout >> sh0) + (p.y >> sh0)) * (a.Wout >> sh0) + (p.x >> sh0);
      ld8(a.x0 + pix0 * a.x0_pitch + ch, xs);
    } else {
      ld8(a.x1 + p.pix * a.x1_pitch + (ch - a.x0_c), xs);
    }
    const float nz = a.noise ? __ldg(a.noise + p.pix) : 0.f;
    float v[16];
#pragma unroll
    for (int q = 0; q < 4; ++q) ld_shared_v4(tile + tile_off<BNT>(r, 16 * g + 4 * q), v + 4 * q);
    float o[8], gm[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      gm[i] = v[2 * i] + gs[i];
      const float bt = v[2 * i + 1] + bs[i];
      const float xn = (fmaf(nz, ns[i], xs[i]) - mu[i]) * rs[i];
      o[i] = apply_act(fmaf(xn, 1.f + gm[i], bt), a.act);
    }
    if constexpr (kStorage16<T>) {
      if (a.gamma_out) st8(a.gamma_out + p.pix * a.gamma_pitch + ch, gm);  // training: gamma for the backward pass
    }
    st8(static_cast<T*>(a.out) + p.pix * a.out_pitch + ch, o);
  }
}

// Epilogue of the 256 consumer threads after their main loops (each warpgroup has run wgmma_wait<0>); `tile` = start of the stage
// ring.  wgmma m64nN fragment: thread (warp w, lane l) holds rows 16 (w % 4) + l / 4 and that + 8 of its warpgroup's 64, columns
// 8 j + 2 (l % 4) + {0, 1}.
template <int BNT, typename T>
__device__ __forceinline__ void conv_epilogue(const ConvArgs<T>& a, const ConvTile& t, const float (&acc)[BNT / 2], uint32_t tile) {
  const int tid = threadIdx.x;  // 0..255
  const int warp = tid >> 5, lane = tid & 31;
  named_bar_sync(kEpiBar, 4 * 32 * kConvConsumers);  // both warpgroups' MMAs are done reading the ring
  fence_proxy_async();
  const int r0 = (warp >> 2) * 64 + (warp & 3) * 16 + (lane >> 2);
  const int c0 = 2 * (lane & 3);
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int j = 0; j < BNT / 8; ++j)
      st_shared_v2(tile + tile_off<BNT>(r0 + 8 * h, 8 * j + c0), acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
  named_bar_sync(kEpiBar, 4 * 32 * kConvConsumers);
  if (a.epi == HRV_EPI_SPADE) epi_spade_rows<BNT>(a, t, tile, tid);
  else if (a.out_vec) epi_linear_rows<BNT>(a, t, tile, tid);
  else epi_linear_f32<BNT>(a, t, tile, tid);
}

// ------------------------------------------------------------------------------------------------ host side

// What a kernel supplies to the shared host setup.
struct ConvBudget {
  uint32_t smem;     // dynamic shared memory one CTA may use
  int max_stages;
  uint32_t scratch;  // bytes between the barriers and the stage ring
  int kblock;        // K-block width in channels
  int planes;        // weight planes per stage
};

// Validates `p` for storage T, picks the tiling, sizes the stage ring, encodes both tensor maps and launches kKernel64 or kKernel128
// (the kernel's instances for N tiles of 64 / 128 columns).  Errors are prefixed "conv" / "conv(spade)" on 16-bit storage and
// "conv(fp32)" / "conv(fp32 spade)" on fp32 storage.
template <typename T, auto kKernel64, auto kKernel128>
int conv_fwd(const hrv_conv_params* p, const ConvBudget& budget, const char* name, hrv_stream stream) {
  constexpr bool f32 = !kStorage16<T>;
  constexpr int storage = f32 ? HRV_F32 : HRV_BF16;
  const char* const pre = f32 ? "conv(fp32)" : "conv";
  const char* const spre = f32 ? "conv(fp32 spade)" : "conv(spade)";
  const hrv_tensor& in = p->in;
  const hrv_tensor& out = p->out;
  if (((uintptr_t)in.ptr & 15) || (in.pitch % 8) || in.pitch < in.c)
    return set_error(HRV_EINVAL, "%s: input needs 16-byte aligned ptr and pitch %% 8 == 0 (pitch=%d c=%d)", pre, in.pitch, in.c);
  if (p->bk != 64 && p->bk != 32 && p->bk != 16) return set_error(HRV_EINVAL, "%s: bk must be 64/32/16", pre);
  if (p->bn < 16 || p->bn > 256 || (p->bn % 16)) return set_error(HRV_EINVAL, "%s: bn=%d must be a multiple of 16 in [16,256]", pre, p->bn);
  if (p->kh < 1 || p->kw < 1 || p->n_gemm < 1) return set_error(HRV_EINVAL, "%s: bad kh/kw/n_gemm", pre);
  if (out.n != in.n) return set_error(HRV_EINVAL, "%s: batch mismatch", pre);
  if (((uintptr_t)p->wpack & 15)) return set_error(HRV_EINVAL, "%s: wpack must be 16-byte aligned", pre);
  if (!(out.dtype == storage || (!f32 && out.dtype == HRV_F32)) || !out.ptr || ((uintptr_t)out.ptr & 3))
    return set_error(HRV_EINVAL, "%s: the output must be non-null and %s", pre, f32 ? "fp32 (one storage type per call)" : "bf16 or fp32");
  if (p->out_layout != HRV_NHWC && p->out_layout != HRV_NCHW) return set_error(HRV_EINVAL, "%s: out_layout %d", pre, p->out_layout);
  if (out.dtype == HRV_BF16 && (p->out_layout != HRV_NHWC || ((uintptr_t)out.ptr & 15) || (out.pitch % 8)))
    return set_error(HRV_EINVAL, "%s: bf16 output must be NHWC, 16-byte aligned, pitch %% 8 == 0", pre);
  const int res_mode = p->res.ptr ? p->res_mode : 0;
  if (p->res.ptr) {
    if (!(p->res.dtype == storage || (!f32 && p->res.dtype == HRV_F32)))
      return set_error(HRV_EINVAL, "%s: the residual must be %s", pre, f32 ? "fp32 (one storage type per call)" : "bf16 or fp32");
    if (p->res.dtype == HRV_BF16 && (((uintptr_t)p->res.ptr & 15) || (p->res.pitch % 8)))
      return set_error(HRV_EINVAL, "%s: bf16 residual must be 16-byte aligned with pitch %% 8 == 0", pre);
  }
  if (res_mode < 0 || res_mode > 2) return set_error(HRV_EINVAL, "%s: res_mode %d", pre, res_mode);
  if (f32 && res_mode)
    return set_error(HRV_EUNSUPPORTED, "%s: the gate residual modes belong to the backward pass; fp32 storage is inference-only", pre);
  if (res_mode && (p->res.dtype != HRV_BF16 || out.dtype != HRV_BF16 || p->out_layout != HRV_NHWC || p->epi != HRV_EPI_LINEAR ||
                   p->act != HRV_ACT_NONE))
    return set_error(HRV_EINVAL, "%s: gate modes need a bf16 res, a bf16 NHWC output, the LINEAR epilogue and no activation", pre);

  ConvArgs<T> a;
  memset(&a, 0, sizeof(a));
  a.Nimg = out.n; a.Hout = out.h; a.Wout = out.w;
  // N tile: 64 columns for narrow GEMMs, else 128 (a 64 x 128 fp32 accumulator is 64 registers per thread).  Independent of the
  // packing's bn: the weight map's row extent is the packed n_pad, rows past it are zero fill.
  const int bnt = p->n_gemm <= 64 ? 64 : 128;
  a.chunks = (in.c + budget.kblock - 1) / budget.kblock;
  // Halo main loop (16-bit storage): for every kernel with more than one tap whose output rows split into 64-pixel runs and whose halo
  // slots leave room for at least two B stages.  A 3x3 layer stages each input pixel once per chunk instead of once per tap.
  const uint32_t halo_slot = halo_slot_bytes(p->kh, p->kw);
  const uint32_t b_stage = (uint32_t)(budget.planes * bnt) * kConvRowBytes;
  a.halo = !f32 && p->kh * p->kw > 1 && out.w % kHaloTW == 0 &&
           (uint64_t)a.chunks * halo_slot + 2u * b_stage <= budget.smem - 2048u - budget.scratch;
  const int TW = a.halo ? kHaloTW : pick_pow2(out.w, 128);
  const int TH = a.halo ? 2 : pick_pow2(out.h, 128 / TW);
  const int TN = 128 / (TW * TH);
  a.tw_log = log2i(TW); a.th_log = log2i(TH);
  a.tiles_x = (out.w + TW - 1) / TW;
  a.tiles_y = (out.h + TH - 1) / TH;
  const int tiles_img = (out.n + TN - 1) / TN;
  a.tiles_n = (p->n_gemm + bnt - 1) / bnt;
  a.KH = p->kh; a.KW = p->kw; a.off_y = p->off_y; a.off_x = p->off_x;
  a.n_gemm = p->n_gemm;
  a.epi = p->epi; a.act = p->act;
  a.scale = p->scale; a.shift = p->shift;
  a.out = out.ptr; a.out_pitch = out.pitch; a.out_dtype = out.dtype; a.out_layout = p->out_layout; a.out_c = out.c;
  // NHWC outputs in the storage type carry pad channels up to the next multiple of 8: written as act(0) (+ res) where the pitch has
  // room.  Other outputs stop at out_c.
  const int c8 = (out.c + 7) & ~7;
  a.store_c = (p->out_layout == HRV_NHWC && out.dtype == storage && out.pitch >= c8) ? c8 : out.c;
  // Always true for 16-bit outputs (their alignment is validated above).  Other outputs are written one element per store.
  a.out_vec = p->out_layout == HRV_NHWC && out.dtype == storage && !((uintptr_t)out.ptr & 15) && !(out.pitch % 8) && !(a.store_c % 8);
  if (p->res.ptr) {
    a.res = p->res.ptr; a.res_pitch = p->res.pitch; a.res_dtype = p->res.dtype; a.res_mode = res_mode;
    a.res_c = (p->res.dtype == storage && p->res.pitch >= a.store_c) ? a.store_c : out.c;
  }

  if (p->epi == HRV_EPI_SPADE) {
    const int C = p->x0.c + (p->x1.ptr ? p->x1.c : 0);
    if (p->n_gemm != 2 * C) return set_error(HRV_EINVAL, "%s: n_gemm=%d must equal 2*(x0.c+x1.c)=%d", spre, p->n_gemm, 2 * C);
    if (p->x0.dtype != storage || (p->x1.ptr && p->x1.dtype != storage))
      return set_error(HRV_EINVAL, "%s: x0/x1 must be %s (one storage type per call)", spre, f32 ? "fp32" : "bf16");
    if (f32 && p->gamma_out.ptr)
      return set_error(HRV_EUNSUPPORTED, "%s: gamma_out belongs to the backward pass; fp32 storage is inference-only", spre);
    if ((p->x0.c % 8) || (C % 8) || out.dtype != storage || p->out_layout != HRV_NHWC || !p->mean || !p->rstd || !p->x0.ptr)
      return set_error(HRV_EINVAL, "%s: channel counts must be multiples of 8, output %s NHWC, mean/rstd/x0 set", spre, f32 ? "fp32" : "bf16");
    if (((uintptr_t)p->x0.ptr & 15) || (p->x0.pitch % 8) || (p->x1.ptr && (((uintptr_t)p->x1.ptr & 15) || (p->x1.pitch % 8))))
      return set_error(HRV_EINVAL, "%s: x0/x1 alignment", spre);
    if (!a.out_vec) return set_error(HRV_EINVAL, "%s: the output needs a 16-byte aligned ptr and pitch %% 8 == 0", spre);
    if (p->x0_shift && ((out.h & 1) || (out.w & 1) || p->x0.h * 2 != out.h || p->x0.w * 2 != out.w))
      return set_error(HRV_EINVAL, "%s: x0_shift needs x0 at exactly half resolution", spre);
    if (!p->x0_shift && (p->x0.h != out.h || p->x0.w != out.w)) return set_error(HRV_EINVAL, "%s: x0 extent mismatch", spre);
    if (out.c != C) return set_error(HRV_EINVAL, "%s: out.c must equal C", spre);
    a.x0 = (const T*)p->x0.ptr; a.x0_c = p->x0.c; a.x0_pitch = p->x0.pitch; a.x0_shift = p->x0_shift ? 1 : 0;
    a.x1 = (const T*)p->x1.ptr; a.x1_pitch = p->x1.pitch;
    a.mean = p->mean; a.rstd = p->rstd; a.noise = p->noise; a.noise_scale = p->noise_scale; a.C_mod = C;
    if (p->gamma_out.ptr) {
      if (p->gamma_out.dtype != HRV_BF16 || ((uintptr_t)p->gamma_out.ptr & 15) || (p->gamma_out.pitch % 8) || p->gamma_out.c != C)
        return set_error(HRV_EINVAL, "%s: gamma_out must be bf16 (n,h,w,C), 16-byte aligned", spre);
      a.gamma_out = (T*)p->gamma_out.ptr; a.gamma_pitch = p->gamma_out.pitch;
    }
  } else if (p->epi != HRV_EPI_LINEAR) {
    return set_error(HRV_EINVAL, "%s: unknown epilogue %d", pre, p->epi);
  }

  // ---- pipeline: as many stages as fit in the budget next to the scratch, at most one per K step; the ring also holds the
  //      epilogue tile.  The halo main loop's stages hold B boxes only, behind the halo slots.
  const uint32_t halo_bytes = a.halo ? (uint32_t)a.chunks * halo_slot : 0u;
  const uint32_t stage_bytes = a.halo ? b_stage : kConvABytes + b_stage;
  const int KT = p->kh * p->kw * a.chunks;
  int stages = (int)((budget.smem - 2048u - budget.scratch - halo_bytes) / stage_bytes);
  if (stages > budget.max_stages) stages = budget.max_stages;
  if (stages > KT) stages = KT < 2 ? 2 : KT;
  a.stages = stages;
  const size_t ring_stages = halo_bytes + (size_t)stages * stage_bytes;
  const size_t ring = ring_stages > conv_tile_bytes(bnt) ? ring_stages : conv_tile_bytes(bnt);
  const size_t smem = 2048 + budget.scratch + ring;  // 1 KB alignment slack + 1 KB of barriers

  // ---- tensor maps: the input (the tile's box, or its halo), and the packed weights [planes][taps][n_pad][cin_k] as laid out for
  //      this (bk, bn)
  int rc = a.halo ? encode_nhwc_map(&a.tmA, in, budget.kblock, TW + p->kw - 1, TH + p->kh - 1, 1)
                  : encode_nhwc_map(&a.tmA, in, budget.kblock, TW, TH, TN);
  if (rc) return rc;
  const cuuint64_t elem = sizeof(T);
  const cuuint64_t cin_k = (cuuint64_t)((in.c + p->bk - 1) / p->bk) * p->bk;
  const cuuint64_t n_pad = (cuuint64_t)((p->n_gemm + p->bn - 1) / p->bn) * p->bn;
  const cuuint64_t taps = (cuuint64_t)(p->kh * p->kw);
  const cuuint64_t dims[4] = {cin_k, n_pad, taps, (cuuint64_t)budget.planes};
  const cuuint64_t strides[3] = {cin_k * elem, n_pad * cin_k * elem, taps * n_pad * cin_k * elem};
  const cuuint32_t box[4] = {(cuuint32_t)budget.kblock, (cuuint32_t)bnt, 1, (cuuint32_t)budget.planes};
  const cuuint32_t es[4] = {1, 1, 1, 1};
  rc = encode_tensor_map(&a.tmB, budget.planes == 1 ? 3 : 4, const_cast<void*>(p->wpack), dims, strides, box, es, CU_TENSOR_MAP_SWIZZLE_128B,
                         f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16);
  if (rc) return rc;

  const long long total = (long long)a.tiles_n * a.tiles_x * a.tiles_y * tiles_img;
  if (total > 0x7FFFFFFFLL) return set_error(HRV_EINVAL, "%s: too many tiles", pre);
  cudaStream_t st = (cudaStream_t)stream;
  return bnt == 64 ? launch_dyn_smem<kKernel64>(name, (int)total, kConvThreads, smem, budget.smem, st, a)
                   : launch_dyn_smem<kKernel128>(name, (int)total, kConvThreads, smem, budget.smem, st, a);
}

}  // namespace hrv
