"""What dynamic loss scaling costs the fp16 stage-2 training step, and where the scale settles.

    HRV_PRECISION=fp16 python tools/loss_scale_bench.py [--batch 8] [--rounds 3] [--steps 20] [--settle 200]

The bench.py train_stage2 workload (1024x768, the same models and synthetic batch) runs as one CUDA graph per step in fp16
storage, in turn without (loss_scale=None) and with loss_scale="dynamic": each round captures one trainer, times --steps replays
with CUDA events, and releases the graph before the next trainer captures.  A third arm runs loss_scale="dynamic" with S pinned
to 1: the same launches as the scaled step on the same (underflowing) data as the unscaled one, so that its difference to "none"
is the cost of the scaling passes themselves and its difference to "dynamic" is the cost of computing on gradients that are no
longer flushed to zero.  hrv_grad_unscale_check alone is timed over G's gradients.  Then the scaled trainer runs --settle more
replays; the loss scales and the number of skipped (non-finite) steps are counted on the device.  Prints one JSON line, with the
card's name and power limit."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402  (workload definition: shapes, generator, discriminator options)
import hrv_loader  # noqa: E402

hrv_loader.load()
import torch  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--settle", type=int, default=200)
    args = ap.parse_args()
    from hrviton_b200 import ops, train_step
    if ops.get_precision() != "fp16":
        raise SystemExit("run with HRV_PRECISION=fp16: loss scaling addresses fp16 storage")
    assert torch.cuda.is_available(), "loss_scale_bench needs a GPU"
    os.environ.setdefault("HRV_VGG_RANDOM_INIT", "1")
    import types

    import network_generator
    import networks
    dev = torch.device("cuda", 0)
    H, W = bench.H, bench.W
    torch.manual_seed(0)
    tocg = networks.ConditionGenerator(types.SimpleNamespace(warp_feature="T1", out_layer="relu", cuda=True), 4, 16, 13, ngf=96,
                                       norm_layer=torch.nn.BatchNorm2d)
    with torch.no_grad():
        for mod in tocg.modules():
            if isinstance(mod, torch.nn.BatchNorm2d):
                mod.running_mean.normal_(0, 0.1)
                mod.running_var.uniform_(0.5, 1.5)
    tocg = tocg.to(dev).eval()
    dopt = bench.gen_opt()
    dopt.ndf, dopt.norm_D, dopt.n_layers_D, dopt.num_D, dopt.no_ganFeat_loss = 64, "spectralinstance", 3, 2, False
    vgg = networks.Vgg19().to(dev).eval()
    batch = train_step.synthetic_batch(args.batch, H, W, dev, seed=100)

    def trainer(loss_scale):
        g = bench.build_generator(dev).train()
        d = network_generator.MultiscaleDiscriminator(dopt)
        d.init_weights("xavier", 0.02)
        tr = train_step.Stage2Trainer(tocg, g, d.to(dev).train(), vgg, loss_scale=loss_scale)
        tr.step(batch, H, W)  # lazy initialisation (optimizer state, caches, gradient tensors) before any capture
        return tr

    trainers = {"none": trainer(None), "dynamic": trainer("dynamic"), "dynamic_s1": trainer("dynamic")}
    for sc in trainers["dynamic_s1"].scalers.values():
        sc.scale.fill_(1.0)
        sc.growth_interval = 1 << 30
    times = {k: [] for k in trainers}
    for _ in range(args.rounds):
        for name, tr in trainers.items():
            tr.capture(batch, H, W)
            tr.replay()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.steps):
                tr.replay()
            e1.record()
            torch.cuda.synchronize()
            times[name].append(e0.elapsed_time(e1) / args.steps)
            tr.release_graph()
    tr = trainers["dynamic"]
    grads = tr.scalers["G"].gradients(tr.opt_g)
    one, found = torch.ones((), device=dev), torch.zeros((), device=dev)
    table = ops.grad_unscale_check(grads, one, found)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(50):
        ops.grad_unscale_check(grads, one, found, table)
    e1.record()
    torch.cuda.synchronize()
    kernel_ms = e0.elapsed_time(e1) / 50
    numel = sum(g.numel() for g in grads)
    tr.capture(batch, H, W)
    skipped = {k: torch.zeros((), device=dev) for k in tr.scalers}
    for _ in range(args.settle):
        tr.replay()
        for k, sc in tr.scalers.items():
            skipped[k] += sc.found_inf
    torch.cuda.synchronize()
    adam_steps = max(int(s["step"]) for s in tr.opt_g.state.values())
    med = {k: statistics.median(v) for k, v in times.items()}
    print(json.dumps({
        "tool": "loss_scale_bench", "card": card(), "batch": args.batch, "shape": [H, W], "precision": "fp16",
        "step_ms": {k: [round(t, 2) for t in v] for k, v in times.items()}, "median_ms": {k: round(v, 2) for k, v in med.items()},
        "overhead_ms": round(med["dynamic"] - med["none"], 3), "overhead_pct": round(100.0 * (med["dynamic"] / med["none"] - 1.0), 3),
        "passes_ms (dynamic_s1 - none)": round(med["dynamic_s1"] - med["none"], 3),
        "unscale_kernel": {"ms": round(kernel_ms, 4), "G_grad_elements": numel, "GB_per_s": round(8.0 * numel / kernel_ms / 1e6, 1)},
        "settle_steps": args.settle, "scale_after_settle": {k: float(sc.scale) for k, sc in tr.scalers.items()},
        "skipped_steps": {k: int(v) for k, v in skipped.items()}, "adam_step_count_G": adam_steps}))


if __name__ == "__main__":
    main()
