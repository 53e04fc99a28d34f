"""Times the stage-1 flow TV and the stage-1 graph step with the loss options of train_condition.py (one process, one GPU).

    python tools/tv_bench.py [--batch 8] [--iters 200] [--steps 20]

1. The fused TV (hrv_flow_tv forward, hrv_flow_tv_bwd backward, through autograd_tocg.flow_tv) against the reference's torch expression
   (train_condition.py's TV lines, eager, deterministic mode off: its interpolate backward is refused in deterministic mode) on the tocg's
   five flows of a 256x192 input, for --edgeawaretv last_only and weighted --add_lasttv.
2. The captured stage-1 step (Stage1Trainer.capture / replay) at 256x192 for the default options, weighted + add_lasttv, no_GAN_loss
   and G_D_seperate.
Prints one line per measurement and the GPU's name and power limit."""
import argparse
import contextlib
import io
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import hrv_loader  # noqa: E402

hrv_loader.load()
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from hrviton_b200 import autograd_tocg, synth, train_step  # noqa: E402

FLOWS = [(8, 6), (16, 12), (32, 24), (64, 48), (128, 96)]


def torch_tv(flow_list, mask, mode, add_lasttv):
    """train_condition.py:201-232 restated with the same torch ops."""
    loss = 0
    idx = [len(flow_list) - 1] if mode == "last_only" else range(len(flow_list))
    for i in idx:
        flow = flow_list[i]
        down = F.interpolate(mask, flow.shape[1:3], mode="bilinear").permute(0, 2, 3, 1)
        y = torch.abs(flow[:, 1:] - flow[:, :-1]) * torch.exp(-150 * torch.abs(down[:, 1:] - down[:, :-1]))
        x = torch.abs(flow[:, :, 1:] - flow[:, :, :-1]) * torch.exp(-150 * torch.abs(down[:, :, 1:] - down[:, :, :-1]))
        s = 1.0 if mode == "last_only" else 2.0 ** (4 - i)
        loss = loss + y.mean() / s + x.mean() / s
    if add_lasttv:
        flow = flow_list[-1]
        loss = loss + torch.abs(flow[:, 1:] - flow[:, :-1]).mean() + torch.abs(flow[:, :, 1:] - flow[:, :, :-1]).mean()
    return loss


def timed(fn, iters):
    for _ in range(10):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def bench_tv(n, iters):
    g = torch.Generator().manual_seed(0)
    flows = [torch.randn(n, h, w, 2, generator=g).cuda().requires_grad_() for h, w in FLOWS]
    mask = torch.rand(n, 1, 256, 192, generator=g).cuda().requires_grad_()
    for mode, add in (("last_only", False), ("weighted", True)):
        for name, f in (("fused", lambda: autograd_tocg.flow_tv(flows, mask, mode, add)), ("torch", lambda: torch_tv(flows, mask, mode, add))):
            fwd = timed(f, iters)

            def fb():
                loss = f()
                torch.autograd.grad(loss, flows + [mask], allow_unused=True)  # last_only reads one flow
            both = timed(fb, iters)
            print("tv %-9s %s+add_lasttv=%d n=%d: forward %.4f ms, forward+backward %.4f ms (backward %.4f ms)"
                  % (mode, name, add, n, fwd, both, both - fwd), flush=True)


def bench_steps(n, steps):
    import networks
    os.environ["HRV_VGG_RANDOM_INIT"] = "1"
    opt = __import__("types").SimpleNamespace(warp_feature="T1", out_layer="relu", cuda=True)
    batches = [train_step.synthetic_batch_stage1(n, 256, 192, "cuda", seed=s) for s in range(2)]
    for name, kw in (("default", {}), ("weighted+add_lasttv", {"edgeawaretv": "weighted", "add_lasttv": True}),
                     ("no_GAN_loss", {"no_gan_loss": True}), ("G_D_seperate", {"g_d_separate": True})):
        torch.manual_seed(0)
        tocg = networks.ConditionGenerator(opt, 4, 16, 13, ngf=96, norm_layer=torch.nn.BatchNorm2d)
        sd = tocg.state_dict()
        synth.fill_state_dict(sd, 3)
        tocg.load_state_dict(sd)
        with contextlib.redirect_stdout(io.StringIO()):
            D = networks.define_D(input_nc=33, Ddownx2=True, Ddropout=True, n_layers_D=3, spectral=False, num_D=2)
        tr = train_step.Stage1Trainer(tocg.cuda().train(), D.cuda().train(), networks.Vgg19().cuda().eval(), tensor_lr=True, **kw)
        tr.capture(batches[0], rollback=True)
        ms = []
        for r in range(3):  # rounds: the spread between them is the noise of the number
            ms.append(timed(lambda: tr.replay(batches[1]), steps))
        tr.release_graph()
        print("stage1 graph step %-20s n=%d: %s ms per step (rounds of %d)" % (name, n, " / ".join("%.2f" % m for m in ms), steps), flush=True)
        del tr, tocg, D
        torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--steps", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tv_bench needs a GPU")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print("gpu:", q.stdout.strip() or torch.cuda.get_device_name(), flush=True)
    bench_tv(a.batch, a.iters)
    bench_steps(a.batch, a.steps)


if __name__ == "__main__":
    main()
