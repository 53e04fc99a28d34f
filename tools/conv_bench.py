"""Micro-benchmark of hrv_conv2d_fwd on the SPADE-generator layer shapes (device-resident, CUDA events).
Usage: python tools/conv_bench.py [batch]"""
import os, sys, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import hrv_loader; hrv_loader.load()
from hrviton_b200 import ops
from hrviton_b200.ops import Act
B = int(sys.argv[1]) if len(sys.argv) > 1 else 4
REPS = int(sys.argv[2]) if len(sys.argv) > 2 else 10  # 1 => single launch per case (ncu captures)
cases = [  # cin, cout(n_gemm), k, h, w, spade
    (128, 160, 3, 1024, 768, True), (128, 288, 3, 512, 384, True), (128, 544, 3, 256, 192, True), (128, 64, 3, 1024, 768, True),
    (80, 32, 3, 1024, 768, False), (80, 32, 1, 1024, 768, False), (32, 32, 3, 1024, 768, False), (144, 64, 3, 512, 384, False),
    (7, 384, 3, 1024, 768, False), (9, 16, 3, 1024, 768, False), (32, 3, 3, 1024, 768, False), (1040, 512, 3, 64, 48, False),
    (272, 128, 3, 256, 192, False), (528, 256, 3, 128, 96, False),
    (64, 384, 1, 1024, 768, False), (64, 128, 1, 1024, 768, False), (160, 128, 3, 1024, 768, False), (192, 128, 3, 1024, 768, False)]
for cin, cout, k, h, w, spade in cases:
    x = Act(torch.randn(B, h, w, ops.round_up(cin, 8), device="cuda").to(torch.bfloat16), c=cin)
    wt = torch.randn(cout // (2 if spade else 1), cin, k, k, device="cuda") * 0.05
    if spade:
        C = cout // 2
        pw = ops.pack_weight(wt, (k // 2, k // 2), interleave=wt.clone())
        x0 = Act(torch.randn(B, h, w, C, device="cuda").to(torch.bfloat16))
        mean = torch.zeros(B, C, device="cuda"); rstd = torch.ones(B, C, device="cuda")
        noise = torch.randn(B, h, w, device="cuda"); ns = torch.zeros(C, device="cuda"); sh = torch.zeros(2 * C, device="cuda")
        out = Act.empty(B, h, w, C)
        fn = lambda: ops.conv2d_spade(x, pw, out, x0, 0, None, mean, rstd, noise, ns, sh, 2)
    else:
        pw = ops.pack_weight(wt, (k // 2, k // 2))
        out = Act.empty(B, h, w, cout)
        fn = lambda: ops.conv2d(x, pw, out)
    for _ in range(3 if REPS > 1 else 0): fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(REPS): fn()
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / REPS
    fl = 2.0 * cin * cout * k * k * B * h * w
    print("%4d->%4d k%d %4dx%-4d %s  %7.3f ms  %7.1f TFLOP/s" % (cin, cout, k, h, w, "spade " if spade else "linear", ms, fl / ms / 1e9), flush=True)

# weight-gradient kernel on the same layer shapes
for cin, cout, k, h, w in [(128, 160, 3, 1024, 768), (128, 288, 3, 512, 384), (80, 32, 3, 1024, 768), (1040, 512, 3, 64, 48), (256, 256, 3, 256, 192),
                          (64, 128, 1, 1024, 768), (7, 128, 3, 1024, 768), (160, 128, 3, 1024, 768), (64, 64, 3, 1024, 768)]:
    x = Act(torch.randn(B, h, w, ops.round_up(cin, 8), device="cuda").to(torch.bfloat16), c=cin)
    dy = Act(torch.randn(B, h, w, ops.round_up(cout, 8), device="cuda").to(torch.bfloat16), c=cout)
    fn = lambda: ops.conv2d_wgrad(x, dy, k, k, k // 2)
    for _ in range(3 if REPS > 1 else 0): fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(REPS): fn()
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / REPS
    print("wgrad %4d->%4d k%d %4dx%-4d          %7.3f ms  %7.1f TFLOP/s" % (cin, cout, k, h, w, ms, 2.0 * cin * cout * k * k * B * h * w / ms / 1e9), flush=True)
