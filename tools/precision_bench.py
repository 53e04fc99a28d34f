"""Inference time of the three storage precisions in one run: SPADEGenerator 1024x768 (batch 8 by default) and the ConditionGenerator
at 256x192, alternating bf16 / fp16 / fp32 round by round (CUDA events after warm-up; the median round is reported).  A separate
profiled pass per precision brackets every convolution launch with events and reports the convolutions' algorithmic TFLOP/s against
the data-sheet peak of the tensor-core format they run on (H100 SXM, dense: 989 BF16/FP16; 495 TF32, i.e. 165 useful at three
passes for the 3xTF32 fp32 mode).  Prints the card name and power limit first; one JSON line per precision.
Usage: python tools/precision_bench.py [--batch 8] [--tocg-batch 8] [--iters 5] [--rounds 3] [--out FILE]"""
import argparse
import json
import os
import subprocess
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import hrv_loader  # noqa: E402

hrv_loader.load()
from hrviton_b200 import ops  # noqa: E402

PEAK_TFLOPS = {"bf16": 989.0, "fp16": 989.0, "fp32": 495.0 / 3}  # useful rate: 3xTF32 issues three TF32 MMAs per product
MODES = ("bf16", "fp16", "fp32")


def card():
    name = torch.cuda.get_device_name()
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=60).stdout.strip().splitlines()
        return name, q[torch.cuda.current_device()] if q else "n/a"
    except (OSError, subprocess.SubprocessError):
        return name, "n/a"


def build(h, w):
    import network_generator
    import networks
    opt = types.SimpleNamespace(norm_G="spectralaliasinstance", gen_semantic_nc=7, ngf=64, num_upsampling_layers="most", fine_height=h,
                                fine_width=w, cuda=True, warp_feature="T1", out_layer="relu")
    torch.manual_seed(0)
    G = network_generator.SPADEGenerator(opt, 9).cuda().eval()
    G.init_weights("xavier", 0.02)
    G.noise_source = lambda b, hh, ww: torch.randn(b, hh, ww, device="cuda")
    T = networks.ConditionGenerator(opt, 4, 16, 13, ngf=96, norm_layer=torch.nn.BatchNorm2d).cuda().eval()
    return G, T


def timed(fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def conv_rate(fn):
    """(conv launches, conv ms, algorithmic TFLOP/s of the convolutions) over one profiled call."""
    ops.PROFILE = []
    try:
        fn()
        torch.cuda.synchronize()
        conv = [(work, e0.elapsed_time(e1)) for kind, work, e0, e1, _ in ops.PROFILE if kind in ("conv", "conv_spade")]
    finally:
        ops.PROFILE = None
    flops, ms = sum(c[0] for c in conv), sum(c[1] for c in conv)
    return len(conv), ms, flops / ms / 1e9 if ms > 0 else 0.0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--tocg-batch", type=int, default=8)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("precision_bench: no GPU (there is no CPU measurement path)")
    name, smi = card()
    print("card: %s | nvidia-smi name, power.limit, clocks.max.sm: %s" % (name, smi), flush=True)
    G, T = build(1024, 768)
    g = torch.Generator().manual_seed(1)
    x = torch.randn(a.batch, 9, 1024, 768, generator=g).cuda()
    seg = torch.zeros(a.batch, 7, 1024, 768).scatter_(1, torch.randint(0, 7, (a.batch, 1, 1024, 768), generator=g), 1.0).cuda()
    i1 = torch.randn(a.tocg_batch, 4, 256, 192, generator=g).cuda()
    i2 = torch.randn(a.tocg_batch, 16, 256, 192, generator=g).cuda()
    run_g = lambda: G(x, seg)
    run_t = lambda: T(i1, i2)
    times = {m: {"gen": [], "tocg": []} for m in MODES}
    with torch.no_grad():
        for m in MODES:  # warm-up: packs the weights of every precision, loads the kernels
            ops.set_precision(m)
            run_g(), run_t(), run_g(), run_t()
        torch.cuda.synchronize()
        for _ in range(a.rounds):  # alternate the precisions: drift of the shared host affects all three alike
            for m in MODES:
                ops.set_precision(m)
                run_g(), run_t()  # repack after the switch, outside the timed window
                torch.cuda.synchronize()
                times[m]["gen"].append(timed(run_g, a.iters))
                times[m]["tocg"].append(timed(run_t, a.iters))
        results = []
        for m in MODES:
            ops.set_precision(m)
            run_g()
            torch.cuda.synchronize()
            n_conv, conv_ms, tflops = conv_rate(run_g)
            med = lambda v: sorted(v)[len(v) // 2]
            r = {"precision": m, "card": name, "nvidia_smi": smi,
                 "gen_1024x768_b%d_ms" % a.batch: round(med(times[m]["gen"]), 3),
                 "gen_img_per_s": round(a.batch * 1000.0 / med(times[m]["gen"]), 2),
                 "tocg_256x192_b%d_ms" % a.tocg_batch: round(med(times[m]["tocg"]), 3),
                 "gen_conv_launches": n_conv, "gen_conv_ms": round(conv_ms, 3), "gen_conv_tflops": round(tflops, 1),
                 "gen_conv_share_of_datasheet_peak": round(tflops / PEAK_TFLOPS[m], 3), "datasheet_peak_tflops": PEAK_TFLOPS[m],
                 "rounds_gen_ms": [round(v, 3) for v in times[m]["gen"]]}
            results.append(r)
            print(json.dumps(r), flush=True)
        ops.set_precision("bf16")
    base = results[0]["gen_1024x768_b%d_ms" % a.batch]
    print("fp32 / bf16 generator time: %.2fx" % (results[2]["gen_1024x768_b%d_ms" % a.batch] / base))
    if a.out:
        with open(a.out, "w") as f:
            json.dump({"card": name, "nvidia_smi": smi, "results": results}, f, indent=1)


if __name__ == "__main__":
    main()
