"""Times the stage-2 graph step with the options of train_generator.py, and the loader's --GT keys (one process, one GPU).

    python tools/stage2_options_bench.py [--batch 8] [--steps 10] [--rounds 3] [--seconds 10]

1. The captured stage-2 step (Stage2Trainer.capture / replay) at 1024x768, bf16 storage, on synthetic weights and batches, for the
   default options (the README's --occlusion), --GT, --no_vgg_loss, --no_ganFeat_loss and --clothmask_composition detach.  Every
   round captures each option set, times --steps replays with CUDA events and releases the graph, so the options alternate within the
   run: the spread between rounds is the noise of the number.
2. data.VitonHDLoader at 1024x768, batches of --batch, 4 workers, in samples/s: the keys a --GT run reads (train_step.GT_KEYS) against
   data.STAGE2_KEYS, alternating, on a synthetic VITON-HD tree in a temporary directory.
Prints one line per measurement and the GPU's name and power limit."""
import argparse
import os
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

from hrviton_b200 import data, ops, synth, train_step  # noqa: E402

H, W = 1024, 768
OPTIONS = (("default", {}), ("GT", {"gt": True}), ("no_vgg_loss", {"no_vgg_loss": True}), ("no_ganFeat_loss", {"no_ganFeat_loss": True}),
           ("detach", {"clothmask_composition": "detach"}))


def networks_():
    import network_generator
    import networks
    gopt = types.SimpleNamespace(norm_G="spectralaliasinstance", gen_semantic_nc=7, ngf=64, num_upsampling_layers="most", fine_height=H,
                                 fine_width=W, cuda=True, ndf=64, norm_D="spectralinstance", n_layers_D=3, num_D=2, no_ganFeat_loss=False,
                                 init_type="xavier", init_variance=0.02)
    tocg = networks.ConditionGenerator(types.SimpleNamespace(warp_feature="T1", out_layer="relu", cuda=True), 4, 16, 13, ngf=96,
                                       norm_layer=torch.nn.BatchNorm2d)
    G, D = network_generator.SPADEGenerator(gopt, 9), network_generator.MultiscaleDiscriminator(gopt)
    for m, seed in ((tocg, 3), (G, 4), (D, 5)):
        sd = m.state_dict()
        synth.fill_state_dict(sd, seed)
        m.load_state_dict(sd)
    return tocg.cuda().eval(), G.cuda().train(), D.cuda().train(), networks.Vgg19().cuda().eval()


def timed(fn, steps):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def bench_steps(n, steps, rounds):
    os.environ["HRV_VGG_RANDOM_INIT"] = "1"
    ops.set_precision("bf16")
    tocg, G, D, vgg = networks_()
    batches = {gt: (train_step.synthetic_batch_gt if gt else train_step.synthetic_batch)(n, H, W, "cuda", seed=1) for gt in (False, True)}
    ms = {name: [] for name, _ in OPTIONS}
    for _ in range(rounds):
        for name, kw in OPTIONS:
            kw = dict(kw)
            no_feat = kw.pop("no_ganFeat_loss", False)
            D.no_ganFeat_loss = no_feat  # the discriminator's option, as build() sets it
            gt = kw.get("gt", False)
            tr = train_step.Stage2Trainer(None if gt else tocg, G, D, None if kw.get("no_vgg_loss") else vgg, occlusion=not gt,
                                          tensor_lr=True, **kw)
            tr.capture(batches[gt], H, W, rollback=True)
            ms[name].append(timed(tr.replay, steps))
            tr.release_graph()
            del tr
            torch.cuda.empty_cache()
    for name, _ in OPTIONS:
        print("stage2 graph step %-16s n=%d %dx%d bf16: %s ms per step (rounds of %d)"
              % (name, n, H, W, " / ".join("%.1f" % m for m in ms[name]), steps), flush=True)


def bench_loader(n, seconds, rounds):
    with tempfile.TemporaryDirectory() as root:
        synth.write_vitonhd(root, 32, seed=0)
        res = {"GT_KEYS": [], "STAGE2_KEYS": []}
        for _ in range(rounds):
            for name, keys in (("GT_KEYS", train_step.GT_KEYS), ("STAGE2_KEYS", data.STAGE2_KEYS)):
                loader = data.VitonHDLoader(root, "train", "pairs.txt", H, W, n, workers=4, keys=keys)
                try:
                    for _ in range(3):
                        loader.next_batch()
                    torch.cuda.synchronize()
                    t0, k = time.perf_counter(), 0
                    while time.perf_counter() - t0 < seconds:
                        loader.next_batch()
                        k += n
                    torch.cuda.synchronize()
                    res[name].append(k / (time.perf_counter() - t0))
                finally:
                    loader.close()
        for name, v in res.items():
            print("loader %-11s %dx%d b=%d workers=4 cpus=%d: %s samples/s" % (name, H, W, n, os.cpu_count(), " / ".join("%.1f" % x for x in v)),
                  flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--seconds", type=float, default=10.0)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("stage2_options_bench needs a GPU")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print("gpu:", q.stdout.strip() or torch.cuda.get_device_name(), flush=True)
    os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")  # read when the first cuBLAS handle is made
    torch.use_deterministic_algorithms(True)  # as train.py runs the step
    bench_steps(a.batch, a.steps, a.rounds)
    bench_loader(a.batch, a.seconds, a.rounds)


if __name__ == "__main__":
    main()
