"""Is stage-2 training loader-bound?  Measures the reference's CPDataLoader and hrviton_b200.data.VitonHDLoader on a synthetic
VITON-HD tree, then stage-2 graph steps fed by each.

    python tools/loader_bench.py [--seconds 30] [--samples 256] [--workers 2 4 8] [--sizes 1024x768 256x192] [--skip-stage2] [--out DIR]

1. Loader throughput (samples/s, batches of 8, over --seconds after a warm-up) at 1024x768 and 256x192 for each worker count, and the
   host-to-device bytes per sample: the reference's CPDataLoader (from oracle/_ref, skipped when absent; its batches moved to the GPU as
   the training scripts do) and VitonHDLoader (device tensors ready).
2. Stage2Trainer graph steps at 1024x768, batch 8, fed by BatchFeeder over one synthetic batch and by VitonHDLoader with 4 workers,
   alternated in rounds; each round first drains the batches the idle loader queued, then times --steps steps.  The loader-fed step
   time against the synthetic one answers the question.
The tree is written once to a temporary directory (64 seeded samples, replicated to --samples names: every file is decoded anew)."""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import hrv_loader  # noqa: E402

hrv_loader.load()
import torch  # noqa: E402

from hrviton_b200 import data, synth, train_step  # noqa: E402

UNIQUE = 64


def write_tree(root, n):
    names = synth.write_vitonhd(root, UNIQUE, seed=0)
    base = os.path.join(root, "train")
    for i in range(UNIQUE, n):
        src, dst = names[i % UNIQUE][:-4], "%06d_00" % i
        for d in os.listdir(base):
            for f in os.listdir(os.path.join(base, d)):
                if f.startswith(src):
                    shutil.copyfile(os.path.join(base, d, f), os.path.join(base, d, f.replace(src, dst)))
    with open(os.path.join(root, "pairs.txt"), "w") as f:
        f.write("".join("%06d_00.jpg %06d_00.jpg\n" % (i, (i + 1) % n) for i in range(n)))


def device_line():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return {"device": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip().splitlines()[0] if q.stdout else None,
            "cpus": os.cpu_count()}


def timed(next_batch, batch, seconds, warm=3):
    for _ in range(warm):
        next_batch()
    torch.cuda.synchronize()
    t0, n = time.perf_counter(), 0
    while True:
        next_batch()
        n += batch
        if time.perf_counter() - t0 >= seconds:
            break
    torch.cuda.synchronize()
    return n / (time.perf_counter() - t0)


def reference_loader(root, fh, fw, batch, workers):
    import hrv_env
    if hrv_env.reference_dir() is None:
        return None, None
    cp = hrv_env.load_reference_script("cp_dataset")
    opt = types.SimpleNamespace(dataroot=root, datamode="train", data_list="pairs.txt", fine_height=fh, fine_width=fw, semantic_nc=13,
                                shuffle=True, batch_size=batch, workers=workers)
    loader = cp.CPDataLoader(opt, cp.CPDataset(opt))
    nbytes = [0]

    def next_batch():
        b = loader.next_batch()
        tensors = [v for v in b.values() if torch.is_tensor(v)] + [t for v in b.values() if isinstance(v, dict) for t in v.values()
                                                                    if torch.is_tensor(t)]
        nbytes[0] = sum(t.numel() * t.element_size() for t in tensors)
        return [t.cuda(non_blocking=True) for t in tensors]
    return loader, (next_batch, nbytes)


def stage2(root, batch, rounds, steps, results):
    import network_generator
    import networks
    h, w = 1024, 768
    gopt = types.SimpleNamespace(norm_G="spectralaliasinstance", gen_semantic_nc=7, ngf=64, num_upsampling_layers="most", fine_height=h,
                                 fine_width=w, cuda=True, ndf=64, norm_D="spectralinstance", n_layers_D=3, num_D=2, no_ganFeat_loss=False,
                                 init_type="xavier", init_variance=0.02)
    torch.manual_seed(0)
    tocg = networks.ConditionGenerator(types.SimpleNamespace(warp_feature="T1", out_layer="relu", cuda=True), 4, 16, 13, ngf=96,
                                       norm_layer=torch.nn.BatchNorm2d)
    G = network_generator.SPADEGenerator(gopt, 9)
    D = network_generator.MultiscaleDiscriminator(gopt)
    for m, seed in ((tocg, 1), (G, 2), (D, 3)):
        sd = m.state_dict()
        synth.fill_state_dict(sd, seed)
        m.load_state_dict(sd)
    tr = train_step.Stage2Trainer(tocg.cuda().eval(), G.cuda().train(), D.cuda().train(), networks.Vgg19().cuda().eval())
    batch_cpu = train_step.synthetic_batch(batch, h, w, "cpu", seed=100)
    feeder = train_step.BatchFeeder(batch_cpu, torch.device("cuda"))
    loader = data.VitonHDLoader(root, "train", "pairs.txt", h, w, batch, workers=4, keys=data.STAGE2_KEYS)
    tr.step({k: v.cuda() for k, v in batch_cpu.items()}, h, w)
    tr.capture({k: v.cuda() for k, v in batch_cpu.items()}, h, w)
    feeder.prefetch()
    for _ in range(3):  # warm both feeds (the loader's workers start here)
        tr.replay(feeder=feeder)
        tr.replay(feeder=loader)
    # While one feed runs, the idle loader's workers fill its queue: prefetch_factor (2) x 4 workers batches, plus the staged slot.
    # Each round first drains that backlog untimed, so the timed steps see only what the workers deliver while the step runs.
    drain = 2 * 4 + 4
    times = {"BatchFeeder (one synthetic batch)": [], "VitonHDLoader (4 workers)": []}
    for _ in range(rounds):
        for name, f in (("BatchFeeder (one synthetic batch)", feeder), ("VitonHDLoader (4 workers)", loader)):
            for _ in range(drain):
                tr.replay(feeder=f)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(steps):
                tr.replay(feeder=f)
            torch.cuda.synchronize()
            times[name].append((time.perf_counter() - t0) / steps * 1e3)
    tr.release_graph()
    for name, t in times.items():
        ms = sorted(t)[len(t) // 2]
        line = {"stage2_1024x768_b%d" % batch: name, "ms_per_step_median": round(ms, 2), "ms_per_round": [round(v, 2) for v in t],
                "img_s": round(batch * 1e3 / ms, 2)}
        print(json.dumps(line), flush=True)
        results.append(line)
    del loader


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=30.0)
    ap.add_argument("--samples", type=int, default=256)
    ap.add_argument("--workers", type=int, nargs="+", default=[2, 4, 8])
    ap.add_argument("--sizes", nargs="*", default=["1024x768", "256x192"], help="fine sizes of the throughput part")
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--steps", type=int, default=100, help="timed stage-2 steps per round, after the loader's backlog is drained")
    ap.add_argument("--out", default=None, help="directory for loader_bench.json")
    ap.add_argument("--skip-stage2", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "loader_bench needs a GPU"
    os.environ.setdefault("HRV_VGG_RANDOM_INIT", "1")
    results = [device_line()]
    print(json.dumps(results[0]), flush=True)
    root = tempfile.mkdtemp(prefix="vitonhd_")
    try:
        t0 = time.perf_counter()
        write_tree(root, args.samples)
        print(json.dumps({"tree": "%d samples at 1024x768 written in %.1f s" % (args.samples, time.perf_counter() - t0)}), flush=True)
        for fh, fw in (tuple(int(v) for v in s.split("x")) for s in args.sizes):
            for workers in args.workers:
                ref, hooks = reference_loader(root, fh, fw, args.batch, workers)
                arms = []
                if ref is not None:
                    arms.append(("CPDataLoader (reference)", hooks[0], lambda: hooks[1][0]))
                ours = data.VitonHDLoader(root, "train", "pairs.txt", fh, fw, args.batch, workers=workers)
                arms.append(("VitonHDLoader", ours.next_batch, lambda: ours.bytes_per_step))
                for name, nb, nbytes in arms:
                    rate = timed(nb, args.batch, args.seconds)
                    line = {"loader": name, "size": "%dx%d" % (fh, fw), "workers": workers, "batch": args.batch,
                            "samples_per_s": round(rate, 2), "h2d_mb_per_sample": round(nbytes() / args.batch / 1e6, 2)}
                    print(json.dumps(line), flush=True)
                    results.append(line)
                del ref, hooks, ours, arms
        if not args.skip_stage2:
            stage2(root, args.batch, args.rounds, args.steps, results)
    finally:
        shutil.rmtree(root, ignore_errors=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "loader_bench.json"), "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
