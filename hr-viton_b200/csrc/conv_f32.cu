// conv_f32.cu — the fp32 reference-precision convolution: NHWC fp32 implicit GEMM in 3xTF32 on sm_90a (wgmma .tf32 + TMA + mbarrier).
//
//   Tiling, TMA producer, epilogues and host setup are shared with the 16-bit kernel (conv_fwd.cuh).  What is this kernel's own:
//   K blocks:   32 fp32 channels (one 128-byte SWIZZLE_128B row per pixel).  Two weight planes, both in one TMA box {32, BNT, 1, 2} of
//               the pre-split weights [2][taps][n_pad][cin_k] (hrv_pack_conv_weight_tf32x2): plane 0 = hi = rna_tf32(w), plane 1 =
//               lo = rna_tf32(w - hi).
//   Split:      once a stage has landed, each consumer warpgroup rewrites its 64 A rows in place as hi = rna_tf32(a) and writes
//               lo = rna_tf32(a - hi) into a scratch tile (ping-pong: the previous stage's MMAs may still read the other one).  The split
//               is elementwise, so the 128B swizzle carries over unchanged.
//   MMA:        three wgmma m64nBNTk8 .tf32 chains into the same fp32 accumulators, small terms first: lo*B_hi, hi*B_lo, hi*B_hi.
//               Each TF32 x TF32 product is exact in fp32, so the result carries ~21 significant bits of every operand (the lo*lo term,
//               ~2^-22 relative, is dropped) — indistinguishable from an fp32 convolution at the 1e-3 output tolerance, where one TF32
//               pass is not (DESIGN.md §4).
//   Occupancy:  one CTA per SM (the three chains triple the MMA work per stage; the stage ring is as deep as 227 KB allows).
//   Epilogues:  LINEAR and SPADE on fp32 storage; the gate residual modes and gamma_out are refused: fp32 storage is inference-only.
#include "conv_fwd.cuh"

namespace hrv {

constexpr uint32_t kWgBytes = 64 * kConvRowBytes;                // one consumer warpgroup's 64 rows
constexpr uint32_t kScratch = 2 * kConvConsumers * kWgBytes;     // lo tiles, two per consumer (ping-pong)
constexpr ConvBudget kBudget32 = {227u * 1024u, 8, kScratch, 32, 2};  // one CTA per SM

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

template <int BNT>
__global__ void __launch_bounds__(kConvThreads, 1) conv_tf32x3_kernel(const __grid_constant__ ConvArgs<float> a) {
  constexpr uint32_t B_PLANE = (uint32_t)BNT * kConvRowBytes;
  constexpr uint32_t STAGE = kConvABytes + 2 * B_PLANE;  // all parts multiples of 1024 B: every operand starts at swizzle phase 0
  constexpr int R = BNT / 2;                             // accumulator registers per consumer thread

  const ConvTile tile = conv_prologue(a);
  const uint32_t scratch = tile.bars + 1024u;
  const uint32_t stage0 = scratch + kScratch;
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (warp == 4 * kConvConsumers) {
    if (lane == 0) conv_produce<BNT, 32, 2>(a, tile, stage0);
    return;
  }

  // ===================================================== consumers: warpgroup wg computes pixels [64 wg, 64 wg + 64) of the tile
  // The tensor cores add into their accumulators with truncation; chained over a whole K walk (hundreds of MMAs) that bias alone would
  // cost ~20x the rounding error of an fp32 sum.  So each stage (12 MMAs) starts a fresh partial tile, and the partials are summed in
  // fp32 registers with round-to-nearest adds (the promotion is what makes the result fp32-class, not just the operand split).
  const int wg = warp >> 2;
  const int t = threadIdx.x & 127;
  const int KT = a.KH * a.KW * a.chunks;
  float acc[R], part[R];
#pragma unroll
  for (int i = 0; i < R; ++i) acc[i] = 0.f;
  {
    StageRing ring(stage0, STAGE, a.stages);
    for (int k = 0; k < KT; ++k) {
      mbar_wait(bar_full(tile.bars, ring.stage), ring.phase);
      const uint32_t a_hi = ring.addr + (uint32_t)wg * kWgBytes;
      // ping-pong lo tile: the other warpgroup-local tile may still be named by the previous stage's descriptors
      const uint32_t a_lo = scratch + (uint32_t)((k & 1) * kConvConsumers + wg) * kWgBytes;
      split_rows(a_hi, a_lo, t);
      fence_proxy_async();        // generic-proxy writes -> visible to the wgmma (async proxy) reads
      named_bar_sync(1 + wg, 128);  // every row of this warpgroup is split before its MMAs read any
      wgmma_fence();
      const uint32_t b_hi = ring.addr + kConvABytes, b_lo = b_hi + B_PLANE;
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {  // K = 8 per instruction: +32 bytes inside the 128-byte swizzle row
        const uint64_t dah = make_wgmma_desc(a_hi + 32u * kk, 8 * kConvRowBytes, 1);
        const uint64_t dal = make_wgmma_desc(a_lo + 32u * kk, 8 * kConvRowBytes, 1);
        const uint64_t dbh = make_wgmma_desc(b_hi + 32u * kk, 8 * kConvRowBytes, 1);
        const uint64_t dbl = make_wgmma_desc(b_lo + 32u * kk, 8 * kConvRowBytes, 1);
        wgmma_tf32_nx<BNT>(part, dal, dbh, (uint32_t)(kk != 0));
        wgmma_tf32_nx<BNT>(part, dah, dbl, 1u);
        wgmma_tf32_nx<BNT>(part, dah, dbh, 1u);
      }
      wgmma_commit();
      wgmma_wait<0>();  // this stage's MMAs are done: its smem can be refilled and its partial promoted
      if (lane == 0) mbar_arrive(bar_empty(tile.bars, ring.stage));
      fence_regs(part);
#pragma unroll
      for (int i = 0; i < R; ++i) acc[i] += part[i];
      ring.next();
    }
  }
  conv_epilogue<BNT>(a, tile, acc, stage0);
}

}  // namespace hrv

namespace hrv_host {

int conv2d_fwd_tf32x3(const hrv_conv_params* p, hrv_stream stream) {
  using namespace hrv;
  return conv_fwd<float, conv_tf32x3_kernel<64>, conv_tf32x3_kernel<128>>(p, kBudget32, "conv_tf32x3", stream);
}

}  // namespace hrv_host
