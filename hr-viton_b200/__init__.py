"""hrviton_b200 — H100-native (sm_90a) hot path of HR-VITON.

On disk this package lives in ``hr-viton_b200/``; import it through
``hrv_loader.load()`` (see /hrv_loader.py).  Contents:

  csrc/       hand-written CUDA (wgmma/TMA implicit-GEMM conv, fused
              InstanceNorm/SPADE/warp kernels) + the C-ABI (include/hrviton_sm100.h)
  capi.py     ctypes binding of the C-ABI; fails loudly when the .so is missing
  ops.py      NHWC-bf16 tensor views + thin op wrappers over the C-ABI
  synth.py    deterministic synthetic weights / inputs (tests, golden, bench)
  data.py     the VITON-HD loader: PIL decoding in the workers, resize / composite / assembly on the GPU
  tocg.py / spade.py / disc.py   host-side orchestration of the three networks
"""
__all__ = ["capi", "ops", "synth"]
