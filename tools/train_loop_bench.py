"""Cost of the training driver (hrviton_b200.train_loop.TrainRun) over the bare loader-fed graph loop, stage 2 at 1024x768, batch 8.

Both arms replay the same captured trainer fed by the same VitonHDLoader, alternated round by round in one process:
  bare:   for _ in range(steps): trainer.replay(feeder=loader)
  driver: run.train(until=run.step + steps)   (schedule, display, save and LPIPS hooks on; none of their steps in the window)
Then one save step (model files + state file) and one evaluation (LPIPS over --eval-samples test try-ons, batch 1) are timed on
their own.  Prints one JSON line with the card and its power limit, and writes it to --out.

    python tools/train_loop_bench.py --samples 32 --steps 50 --rounds 4"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--samples", type=int, default=32, help="synthetic training samples written (1024x768)")
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--workers", type=int, default=4)
    ap.add_argument("--steps", type=int, default=50, help="steps per arm per round")
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--eval-samples", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    os.environ.setdefault("HRV_VGG_RANDOM_INIT", "1")
    os.environ.setdefault("HRV_ALEX_RANDOM_INIT", "1")
    import torch

    import hrv_loader
    hrv_loader.load()
    import networks
    from hrviton_b200 import metrics, synth, train_loop
    if not torch.cuda.is_available():
        raise SystemExit("train_loop_bench.py measures on a GPU; none is visible")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    tmp = tempfile.mkdtemp(prefix="trainloop_bench_")
    synth.write_vitonhd(tmp, a.samples, seed=1, datamode="train")
    synth.write_vitonhd(tmp, a.eval_samples, seed=2, datamode="test", pairs="test_pairs.txt")
    tocg = networks.ConditionGenerator(argparse.Namespace(warp_feature="T1", out_layer="relu", cuda=True), 4, 16, 13, ngf=96,
                                       norm_layer=torch.nn.BatchNorm2d)
    sd = tocg.state_dict()
    synth.fill_state_dict(sd, 3)
    torch.save(sd, os.path.join(tmp, "tocg.pth"))
    heads = metrics.PNetLin(pretrained=False).state_dict()
    synth.fill_state_dict({k: v for k, v in heads.items() if not k.startswith("scaling_layer.")}, 4)  # the constant input scaling stays
    for k in heads:
        if k.startswith("lin"):  # LPIPS heads are non-negative
            heads[k].abs_()
    os.makedirs(os.path.join(tmp, "eval_models", "weights", "v0.1"))
    torch.save(heads, os.path.join(tmp, "eval_models", "weights", "v0.1", "alex.pth"))
    os.chdir(tmp)  # PerceptualLoss reads ./eval_models/weights/v0.1/alex.pth
    opt = train_loop.parse_args("stage2", ["--name", "bench", "--dataroot", tmp, "--data_list", "pairs.txt", "-b", str(a.batch), "-j",
                                           str(a.workers), "--checkpoint_dir", os.path.join(tmp, "ckpt"), "--tocg_checkpoint",
                                           os.path.join(tmp, "tocg.pth"), "--test_dataroot", tmp, "--test_data_list", "test_pairs.txt",
                                           "--occlusion", "--keep_step", "100000", "--decay_step", "100000", "--display_count", "100000",
                                           "--save_count", "100000", "--lpips_count", "100000"])
    run = train_loop.build(opt, log=lambda *x: None)
    run.lpips_samples = a.eval_samples
    run.start()
    tr, loader = run.trainer, run.loader

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3

    def bare():
        for _ in range(a.steps):
            tr.replay(feeder=loader)

    def driver():
        run.train(until=run.step + a.steps)

    for _ in range(3):  # warm: the loader's queue, the first replays
        tr.replay(feeder=loader)
    res = {"bare": [], "driver": []}
    for r in range(a.rounds):
        for name, fn in (("bare", bare), ("driver", driver)) if r % 2 == 0 else (("driver", driver), ("bare", bare)):
            res[name].append(timed(fn) / a.steps)
    save_ms = timed(run.save)
    run.evaluate()  # first evaluation captures the try-on graph
    tr.replay(feeder=loader)  # weights change between evaluations, as in training: the next evaluation captures again
    eval_ms = timed(run.evaluate)
    tr.release_graph()
    if run._tryon is not None:
        run._tryon.release()
    out = {"gpu": gpu, "batch": a.batch, "size": "1024x768", "steps_per_round": a.steps, "rounds": a.rounds,
           "bare_ms_per_step": [round(x, 2) for x in res["bare"]], "driver_ms_per_step": [round(x, 2) for x in res["driver"]],
           "bare_mean": round(sum(res["bare"]) / a.rounds, 2), "driver_mean": round(sum(res["driver"]) / a.rounds, 2),
           "save_step_ms": round(save_ms, 1), "eval_ms": round(eval_ms, 1), "eval_samples": a.eval_samples,
           "eval_ms_per_sample": round(eval_ms / a.eval_samples, 2)}
    line = json.dumps(out)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
