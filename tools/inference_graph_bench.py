"""Eager versus CUDA-graph replay of try-on inference: how much of a call's latency is host-side orchestration.

    python tools/inference_graph_bench.py [--batches 1,4,16] [--precision bf16|fp16|fp32] [--rounds 3] [--calls 20]

Two workloads at 1024x768 on the bench.py models and synthetic inputs: the end-to-end pipeline (pipeline.tryon_forward with
occlusion handling, against pipeline.TryOnGraph) and the SPADEGenerator forward alone (generator(x, seg) under no_grad, against
pipeline.GeneratorGraph).  For every batch size both arms are warmed up (the graph arm captures its shape), checked to return
the same output from the same torch seed, then timed alternately, eager then graph, for --rounds rounds.  Each round of an arm
reports
    device_ms   CUDA events around --calls back-to-back calls, per call (the GPU-side time of a stream of calls),
    host_ms     host wall time to issue one call, measured over the same back-to-back calls (no synchronisation inside),
    latency_ms  wall time of one call followed by torch.cuda.synchronize(), median over --calls calls: what a caller that serves
                one request at a time waits.
Medians over the rounds are printed as a table and as one JSON line, with the card's name and power limit."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402  (workload definition: shapes, generator options and weights, synthetic generator inputs)
import hrv_loader  # noqa: E402

hrv_loader.load()
import torch  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def measure(fn, calls):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    t0 = time.perf_counter()
    for _ in range(calls):
        fn()
    t1 = time.perf_counter()
    e1.record()
    torch.cuda.synchronize()
    lat = []
    for _ in range(calls):
        t = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        lat.append(time.perf_counter() - t)
    return {"device_ms": e0.elapsed_time(e1) / calls, "host_ms": 1e3 * (t1 - t0) / calls, "latency_ms": 1e3 * statistics.median(lat)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,4,16")
    ap.add_argument("--precision", default="bf16", choices=["bf16", "fp16", "fp32"])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--calls", type=int, default=20)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "inference_graph_bench needs a GPU"
    import networks
    from hrviton_b200 import ops, pipeline, train_step
    ops.set_precision(args.precision)
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
    g = bench.build_generator(dev)
    name = card()
    results = {}
    for b in [int(v) for v in args.batches.split(",")]:
        batch = train_step.synthetic_batch(b, H, W, dev, seed=100)
        x, seg = (t.to(dev) for t in bench.synth_batch(b, "cpu", 100))
        tryon, gen = pipeline.TryOnGraph(tocg, g), pipeline.GeneratorGraph(g)

        def gen_eager():
            with torch.no_grad():
                return g(x, seg)
        arms = {"pipeline": {"eager": lambda: pipeline.tryon_forward(tocg, g, batch, occlusion=True)[0], "graph": lambda: tryon(batch)[0]},
                "gen_fwd": {"eager": gen_eager, "graph": lambda: gen(x, seg)}}
        for wl, fns in arms.items():
            outs = {}
            for arm, fn in fns.items():
                fn()  # warm-up (the graph arm captures here)
                torch.cuda.manual_seed(1)
                outs[arm] = fn().clone()
            times = {arm: [] for arm in fns}
            for _ in range(args.rounds):
                for arm, fn in fns.items():
                    times[arm].append(measure(fn, args.calls))
            med = {arm: {k: round(statistics.median(r[k] for r in rs), 3) for k in rs[0]} for arm, rs in times.items()}
            results["%s_b%d" % (wl, b)] = {"batch": b, "outputs_equal": bool(torch.equal(outs["eager"], outs["graph"])), "median": med,
                                           "rounds": {arm: [{k: round(v, 3) for k, v in r.items()} for r in rs] for arm, rs in times.items()}}
            print("%-9s b%-3d  eager: device %8.3f ms  host %8.3f ms  latency %8.3f ms | graph: device %8.3f ms  host %8.3f ms  "
                  "latency %8.3f ms | latency x%.2f  outputs equal %s"
                  % (wl, b, med["eager"]["device_ms"], med["eager"]["host_ms"], med["eager"]["latency_ms"], med["graph"]["device_ms"],
                     med["graph"]["host_ms"], med["graph"]["latency_ms"], med["eager"]["latency_ms"] / med["graph"]["latency_ms"],
                     results["%s_b%d" % (wl, b)]["outputs_equal"]), flush=True)
        tryon.release()
        gen.release()
        del batch, x, seg
    print(json.dumps({"tool": "inference_graph_bench", "card": name, "shape": [H, W], "precision": args.precision,
                      "rounds": args.rounds, "calls": args.calls, "results": results}))


if __name__ == "__main__":
    main()
