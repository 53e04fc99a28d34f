// conv_igemm.cu — NHWC convolution on 16-bit storage as an im2col-free implicit GEMM on sm_90a (wgmma + TMA + mbarrier).
//
//   Tiling, TMA producer, epilogues and host setup are shared with the fp32 kernel (conv_fwd.cuh).  What is this kernel's own:
//   K blocks:   64 channels of 2 bytes; one weight plane, TMA box {64, BNT}.
//   MMA:        wgmma.mma_async m64nBNTk16, bf16 (fp16 flavour: f16) operands from 128B-swizzled shared memory, fp32 accumulators in
//               the registers of the consumer warpgroups, one wgmma group kept in flight before a stage is released.
//   Halo loop:  3x3 / 2x2 layers whose output rows split into 64-pixel runs and whose halo fits next to two B stages (conv_fwd.cuh)
//               stage each chunk's input halo once per tile and read every tap's A operand out of it.  The wgmma sequence of every
//               output element is that of the tap-by-tap loop, so both loops give bit-identical results.
//   Occupancy:  two CTAs per SM (the epilogue of one overlaps the mainloop of the other): <= 110 KB of shared memory and <= 112
//               registers per thread.
//
// Replaces nn.Conv2d at networks.py:60-93,178-192 and network_generator.py:97-99,132-135,184-201,263-272.
#include "conv_fwd.cuh"

namespace hrv {

constexpr ConvBudget kBudget16 = {110u * 1024u, 16, 0, 64, 1};  // two CTAs per SM (plus 1 KB reserved per CTA)

// TMA producer of the halo main loop (one lane): the halo box of every K chunk into its slot, then per K step (tap outer, chunk
// inner, as conv_produce) the B box into the next stage behind the slots.
template <int BNT>
__device__ __forceinline__ void conv_produce_halo(const ConvArgs<__nv_bfloat16>& a, const ConvTile& t, uint32_t slots) {
  constexpr uint32_t BSTAGE = (uint32_t)BNT * kConvRowBytes;
  tma_prefetch_desc(&a.tmA);
  tma_prefetch_desc(&a.tmB);
  const uint32_t slot = halo_slot_bytes(a.KH, a.KW);
  const int x0 = (t.tx << a.tw_log) - a.off_x;
  const int y0 = (t.ty << a.th_log) - a.off_y;
  for (int c = 0; c < a.chunks; ++c) {
    mbar_arrive_expect_tx(bar_halo(t.bars, c), halo_box_bytes(a.KH, a.KW));
    tma_load_4d(slots + c * slot, &a.tmA, bar_halo(t.bars, c), c * 64, x0, y0, t.ti);
  }
  const int KT = a.KH * a.KW * a.chunks;
  int kc = 0, tap = 0;
  StageRing ring(slots + a.chunks * slot, BSTAGE, a.stages);
  for (int k = 0; k < KT; ++k) {
    const uint32_t full = bar_full(t.bars, ring.stage);
    mbar_wait(bar_empty(t.bars, ring.stage), ring.phase ^ 1u);
    mbar_arrive_expect_tx(full, BSTAGE);
    tma_load_3d(ring.addr, &a.tmB, full, kc * 64, t.nt * BNT, tap);
    if (++kc == a.chunks) { kc = 0; ++tap; }
    ring.next();
  }
}

template <int BNT>
__global__ void __launch_bounds__(kConvThreads, 2) conv_wgmma_kernel(const __grid_constant__ ConvArgs<__nv_bfloat16> a) {
  constexpr uint32_t STAGE = kConvABytes + (uint32_t)BNT * kConvRowBytes;  // both parts multiples of 1024 B: swizzle phase 0
  constexpr int R = BNT / 2;                                               // accumulator registers per consumer thread

  const ConvTile t = conv_prologue(a);
  const uint32_t stage0 = t.bars + 1024u;
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (warp == 4 * kConvConsumers) {
    if (lane == 0) {
      if (a.halo) conv_produce_halo<BNT>(a, t, stage0);
      else conv_produce<BNT, 64, 1>(a, t, stage0);
    }
    return;
  }

  // ===================================================== consumers: warpgroup wg computes pixels [64 wg, 64 wg + 64) of the tile
  const int wg = warp >> 2;
  const int KT = a.KH * a.KW * a.chunks;
  // Halo loop: slot c holds halo rows of (kHaloTW + KW - 1) pixels; the A operand of tap (ky, kx) starts at pixel kx of row wg + ky,
  // a whole number of 128-byte rows past the slot's 1024-byte boundary (make_wgmma_desc: the swizzle follows the absolute address).
  const uint32_t slot = a.halo ? halo_slot_bytes(a.KH, a.KW) : 0u;
  const uint32_t halo_row = (uint32_t)(kHaloTW + a.KW - 1) * kConvRowBytes;
  float acc[R];
#pragma unroll
  for (int i = 0; i < R; ++i) acc[i] = 0.f;
  {
    StageRing ring(stage0 + a.chunks * slot, a.halo ? (uint32_t)BNT * kConvRowBytes : STAGE, a.stages);
    uint32_t a_tap = stage0 + (uint32_t)wg * halo_row;  // halo loop: A of (ky, kx, chunk 0)
    int kx = 0, kc = 0;
    int prev = 0;
    for (int k = 0; k < KT; ++k) {
      uint32_t a_row0, b0;
      if (a.halo) {
        if (k < a.chunks) mbar_wait(bar_halo(t.bars, k), 0);  // the first tap walks every chunk: wait for each slot once
        a_row0 = a_tap + kc * slot;
        b0 = ring.addr;
        if (++kc == a.chunks) {
          kc = 0;
          a_tap += kConvRowBytes;
          if (++kx == a.KW) { kx = 0; a_tap += halo_row - a.KW * kConvRowBytes; }
        }
      } else {
        a_row0 = ring.addr + (uint32_t)wg * (64u * kConvRowBytes);
        b0 = ring.addr + kConvABytes;
      }
      mbar_wait(bar_full(t.bars, ring.stage), ring.phase);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {  // K = 16 per instruction: +32 bytes inside the 128-byte swizzle row
        const uint64_t da = make_wgmma_desc(a_row0 + 32u * kk, 8 * kConvRowBytes, 1);
        const uint64_t db = make_wgmma_desc(b0 + 32u * kk, 8 * kConvRowBytes, 1);
        wgmma_nx<BNT>(acc, da, db, (uint32_t)((k | kk) != 0));
      }
      wgmma_commit();
      wgmma_wait<1>();  // the MMAs of the previous stage have finished reading it
      if (k > 0 && lane == 0) mbar_arrive(bar_empty(t.bars, prev));
      prev = ring.stage;
      ring.next();
    }
    wgmma_wait<0>();
    fence_regs(acc);
  }
  conv_epilogue<BNT>(a, t, acc, stage0);
}

}  // namespace hrv

using namespace hrv;

extern "C" int hrv_conv2d_fwd(const hrv_conv_params* p, hrv_stream stream) {
  if (!p) return set_error(HRV_EINVAL, "conv: null params");
  if (p->in.dtype == HRV_F32) return conv2d_fwd_tf32x3(p, stream);  // fp32 storage: the 3xTF32 kernel of conv_f32.cu
  if (p->in.dtype != HRV_BF16) return set_error(HRV_EINVAL, "conv: input must be bf16 NHWC");
  return conv_fwd<__nv_bfloat16, conv_wgmma_kernel<64>, conv_wgmma_kernel<128>>(p, kBudget16, "conv_wgmma", stream);
}
