"""What discriminator rejection costs: the reference's torch glue against pipeline.rejection_scores and pipeline.ConditionGraph,
and what scoring adds to a try-on request served from pipeline.TryOnGraph.

    python tools/rejection_bench.py [--batches 1,4,16] [--tryon-batches 1,4] [--precision bf16|fp16|fp32] [--rounds 3] [--calls 20]

Scoring a condition at 256x192 (tocg forward + discriminator), three arms on the same drop-in modules and inputs:
    glue    tocg -> torch soft-max / ones_like / slice-assign / multiply / torch.cat -> D(nchw) -> D_logit (test_condition.py:99-123,
            with its two numpy round trips replaced by device thresholds),
    eager   pipeline.rejection_scores (one fused kernel builds the discriminator's NHWC input),
    graph   pipeline.ConditionGraph.
At 1024x768: pipeline.TryOnGraph with and without discriminator=, i.e. what the score adds to a request.  Every shape of every arm
is warmed up (the graph arms capture there), the arms' scores are asserted to agree, then the arms are timed alternately for
--rounds rounds.  Columns as tools/inference_graph_bench.py: device_ms (CUDA events around --calls back-to-back calls, per call),
host_ms (host time to issue one call), latency_ms (one call + synchronize, median).  Medians over the rounds are printed as a table
and as one JSON line, with the card's name and power limit."""
import argparse
import json
import os
import statistics
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bench  # noqa: E402  (the flagship workload's shapes and generator)
import hrv_loader  # noqa: E402
from inference_graph_bench import card, measure  # noqa: E402

hrv_loader.load()
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402


def glue_scores(tocg, D, inputs, norm_const):
    """The reference's scoring glue (test_condition.py:99-123, 'warp_grad'), thresholds on the device."""
    from hrviton_b200 import pipeline
    with torch.no_grad():
        input1 = torch.cat([inputs["cloth"], (inputs["cloth_mask"] > 0.5).float()], 1)
        input2 = torch.cat([inputs["parse_agnostic"], inputs["densepose"]], 1)
        _, fake_segmap, _, warped_cm = tocg(input1, input2)
        cloth_mask = torch.ones_like(fake_segmap)
        cloth_mask[:, 3:4, :, :] = warped_cm
        fake_segmap = fake_segmap * cloth_mask
        l = pipeline.d_logit(D(torch.cat((input1, input2, F.softmax(fake_segmap, dim=1)), dim=1)))
        return l / (1 - l) / norm_const


def run_arms(name, fns, scores, args, results, tol):
    outs = {}
    for arm, fn in fns.items():
        fn()  # warm-up (the graph arms capture here)
        torch.cuda.manual_seed(1)
        fn()
        outs[arm] = scores[arm]().clone()
    first = next(iter(outs))
    for arm, s in outs.items():
        d = float((s - outs[first]).abs().max())
        assert d <= tol[arm], "%s: arm %s scores differ from %s by %.3e" % (name, arm, first, d)
    times = {arm: [] for arm in fns}
    for _ in range(args.rounds):
        for arm, fn in fns.items():
            times[arm].append(measure(fn, args.calls))
    med = {arm: {k: round(statistics.median(r[k] for r in rs), 3) for k in rs[0]} for arm, rs in times.items()}
    results[name] = {"median": med, "rounds": {arm: [{k: round(v, 3) for k, v in r.items()} for r in rs] for arm, rs in times.items()}}
    print("%-16s " % name + " | ".join("%s: device %7.3f ms  host %7.3f ms  latency %7.3f ms" % (
        arm, m["device_ms"], m["host_ms"], m["latency_ms"]) for arm, m in med.items()), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,4,16")
    ap.add_argument("--tryon-batches", default="1,4")
    ap.add_argument("--precision", default="bf16", choices=["bf16", "fp16", "fp32"])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--calls", type=int, default=20)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "rejection_bench needs a GPU"
    import networks
    from hrviton_b200 import ops, pipeline, train_step
    ops.set_precision(args.precision)
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    tocg = networks.ConditionGenerator(types.SimpleNamespace(warp_feature="T1", out_layer="relu", cuda=True), 4, 16, 13, ngf=96,
                                       norm_layer=torch.nn.BatchNorm2d)
    with torch.no_grad():
        for mod in tocg.modules():
            if isinstance(mod, torch.nn.BatchNorm2d):
                mod.running_mean.normal_(0, 0.1)
                mod.running_var.uniform_(0.5, 1.5)
    tocg = tocg.to(dev).eval()
    D = networks.define_D(input_nc=33, Ddownx2=True, Ddropout=True, n_layers_D=3, spectral=False, num_D=2).to(dev).eval()
    M = 0.5  # any positive constant: the arithmetic does not depend on its value
    # the scores agree bit for bit between eager and graph; the glue arm differs by torch's soft-max and 16-bit rounding of D's input
    tol = {"glue": 0.0, "eager": 5e-2 if args.precision != "fp32" else 1e-3, "graph": 5e-2 if args.precision != "fp32" else 1e-3}
    name = card()
    results = {}
    for b in [int(v) for v in args.batches.split(",")]:
        batch = train_step.synthetic_batch(b, 256, 192, dev, seed=100)
        cond = pipeline.ConditionGraph(tocg, D, M)
        last = {}
        arm = lambda key, fn: (lambda: last.__setitem__(key, fn()))
        fns = {"glue": arm("glue", lambda: glue_scores(tocg, D, batch, M)),
               "eager": arm("eager", lambda: pipeline.rejection_scores(tocg, D, batch, M)[0]),
               "graph": arm("graph", lambda: cond(batch)[0])}
        run_arms("score_256x192_b%d" % b, fns, {k: (lambda k=k: last[k]) for k in fns}, args, results, tol)
        assert torch.equal(last["eager"], last["graph"])
        cond.release()
    g = bench.build_generator(dev)
    H, W = bench.H, bench.W
    for b in [int(v) for v in args.tryon_batches.split(",") if v]:
        batch = train_step.synthetic_batch(b, H, W, dev, seed=100)
        plain, scored = pipeline.TryOnGraph(tocg, g), pipeline.TryOnGraph(tocg, g, discriminator=D, norm_const=M)
        last = {}
        arm = lambda key, fn: (lambda: last.__setitem__(key, fn()))
        fns = {"tryon": arm("tryon", lambda: plain(batch)), "tryon+score": arm("tryon+score", lambda: scored(batch))}
        run_arms("tryon_%dx%d_b%d" % (H, W, b), fns, {k: (lambda k=k: last[k][0]) for k in fns}, args, results,
                 {"tryon": 0.0, "tryon+score": 0.0})  # the images must be identical
        plain.release()
        scored.release()
    print(json.dumps({"tool": "rejection_bench", "card": name, "precision": args.precision, "rounds": args.rounds, "calls": args.calls,
                      "results": results}))


if __name__ == "__main__":
    main()
