"""Times the stage-1 training step (the train_stage1 workload of bench.py: tocg + stage-1 D + VGG losses + Adam, one CUDA graph per
step) with plain nn.BatchNorm2d and with sync_batchnorm.SynchronizedBatchNorm2d, alternating the two in rounds.

With one process SynchronizedBatchNorm2d takes the per-rank path: the two arms run the same kernels, must produce bit-identical
results, and must time alike.  Under torchrun with N >= 2 ranks the difference between the arms is the cost of SyncBN's 68 small
fp64 all-reduces per step (34 layers, one in forward and one in backward), captured into the step's graph with the gradient buckets.

    python tools/syncbn_bench.py [--batch 4] [--height 1024 --width 768] [--steps 10] [--rounds 3]
    torchrun --nproc_per_node N tools/syncbn_bench.py ...

Prints one JSON line (rank 0) with the median ms per step of each arm, the GPU model and its power limit."""
import argparse
import contextlib
import io
import json
import os
import subprocess
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import hrv_loader  # noqa: E402

hrv_loader.load()
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402


def _gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name()


def _trainer(norm_layer, batch, world):
    import networks
    from hrviton_b200 import ddp, train_step
    torch.manual_seed(0)
    topt = types.SimpleNamespace(warp_feature="T1", out_layer="relu", cuda=True)
    tocg = networks.ConditionGenerator(topt, 4, 16, 13, ngf=96, norm_layer=norm_layer).cuda().train()
    with contextlib.redirect_stdout(io.StringIO()):
        D = networks.define_D(input_nc=33, Ddownx2=True, Ddropout=True, n_layers_D=3, spectral=False, num_D=2)
    D = D.cuda().train()
    reducers = {}
    if world > 1:
        ddp.broadcast_module_state(tocg)
        ddp.broadcast_module_state(D)
        ddp.syncbn_group()
        reducers = {"G": ddp.GradBucketReducer(list(tocg.parameters())), "D": ddp.GradBucketReducer(list(D.parameters()))}
    tr = train_step.Stage1Trainer(tocg, D, networks.Vgg19().cuda().eval(), reducers=reducers)
    tr.capture(batch)  # two eager warm-up steps (optimizer state, NCCL communicators, buckets), then the captured step
    return tr


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--batch", type=int, default=4, help="per-rank batch")
    ap.add_argument("--height", type=int, default=1024)
    ap.add_argument("--width", type=int, default=768)
    ap.add_argument("--steps", type=int, default=10, help="replays per arm per round")
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    os.environ.setdefault("HRV_VGG_RANDOM_INIT", "1")
    assert torch.cuda.is_available(), "syncbn_bench needs a GPU"
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    if world > 1:
        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", "0")))
        dist.init_process_group("nccl", device_id=torch.device("cuda", torch.cuda.current_device()))
    else:
        torch.cuda.set_device(0)
    from hrviton_b200 import ddp, train_step
    batch = train_step.synthetic_batch_stage1(args.batch, args.height, args.width, "cuda", seed=100 + rank)
    arms = {"batchnorm": _trainer(torch.nn.BatchNorm2d, batch, world), "syncbn": _trainer(ddp.SynchronizedBatchNorm2d, batch, world)}
    outs = {}
    for name, tr in arms.items():  # the third step of each arm, from identical starting states and dropout seeds
        torch.manual_seed(1)
        outs[name] = {k: v.clone() for k, v in tr.replay().items()}
    torch.cuda.synchronize()
    identical = all(torch.equal(outs["batchnorm"][k], outs["syncbn"][k]) for k in outs["batchnorm"])
    times = {name: [] for name in arms}
    for _ in range(args.rounds):
        for name, tr in arms.items():
            if world > 1:
                dist.barrier()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.steps):
                tr.replay()
            e1.record()
            torch.cuda.synchronize()
            times[name].append(e0.elapsed_time(e1) / args.steps)
    med = {name: sorted(t)[len(t) // 2] for name, t in times.items()}
    if rank == 0:
        print(json.dumps({"tool": "syncbn_bench", "world_size": world, "per_rank_batch": args.batch, "size": [args.height, args.width],
                          "ms_per_step": med, "rounds_ms": times, "syncbn_overhead_ms": med["syncbn"] - med["batchnorm"],
                          "third_step_bit_identical": identical, "gpu": _gpu_info()}))
    for tr in arms.values():
        tr.release_graph()
    if world > 1:
        dist.destroy_process_group()
    if world == 1 and not identical:
        sys.exit("with one process SynchronizedBatchNorm2d must give the BatchNorm2d step bit for bit")


if __name__ == "__main__":
    main()
