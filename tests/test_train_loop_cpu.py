"""CPU: the training driver's host logic (hrviton_b200.train_loop) — the LR schedule against torch's LambdaLR with the reference's
lambda, the state file round trip, model files read by networks.load_checkpoint and by test_generator.py's strict load_checkpoint_G,
and the command line's refusals."""
import collections
import os

import pytest
import torch

import hrv_env
from hrviton_b200 import train_loop, train_step


@pytest.mark.parametrize("load_step,keep_step,decay_step,interval", [(0, 100000, 100000, 1000), (0, 7, 5, 1), (3, 7, 5, 1),
                                                                     (2500, 5000, 4000, 1000), (9, 7, 20, 3), (0, 4, 0, 2)])
def test_schedule_equals_lambdalr(load_step, keep_step, decay_step, interval):
    """train_generator.py:155-159,596-598 run as written: lr of every step, across keep_step and to the end of decay."""
    p = torch.nn.Parameter(torch.zeros(1))
    opt = torch.optim.Adam([p], lr=1.0)
    sched = torch.optim.lr_scheduler.LambdaLR(opt, lr_lambda=lambda step: 1.0 - max(0, step * interval + load_step - keep_step)
                                              / float(decay_step + 1))
    end = keep_step + decay_step
    stride = max(1, (end - load_step) // 3000)  # every step of the short schedules, a sample of the long one plus every boundary
    steps = sorted(set(range(load_step, end, stride)) | {s for s in range(load_step, end) if s % interval in (0, interval - 1)})
    want = {}
    opt.step()  # as the reference's loop: the optimiser steps before the scheduler
    for step in range(load_step, end):
        want[step] = opt.param_groups[0]["lr"]
        if (step + 1) % interval == 0:
            sched.step()
    for step in steps:
        assert train_loop.lr_factor(step, load_step, keep_step, decay_step, interval) == want[step], step
    assert want[end - 1] < 1.0 or decay_step == 0


class _Loader:
    seed, batch_size = 7, 2

    def __init__(self):
        self.pos = (3, 5)

    def position(self):
        return self.pos

    def start_at(self, epoch, index):
        self.pos = (epoch, index)


class _Trainer(train_step._TrainState, train_step._LossScaling):
    """A trainer's state surface on CPU modules: the real optimisers (fused Adam, device-tensor lr) and state_dict code."""
    _captured = None

    def __init__(self, seed, g_lr=2e-4, occlusion=True):
        torch.manual_seed(seed)
        self.tocg, self.D = torch.nn.Sequential(torch.nn.Linear(4, 3), torch.nn.BatchNorm1d(3)), torch.nn.Linear(3, 2)
        self.G = self.tocg  # the stage-2 role of the trained generator
        self._make_optimizers(self.tocg.parameters(), self.D.parameters(), g_lr, 1e-4, (0.5, 0.999), True)
        self.scalers = {}
        self.occlusion = occlusion
        self.replays = 0

    def replay(self, feeder=None):
        self.replays += 1
        return {"loss": torch.zeros(())}

    def step(self):
        x = torch.randn(5, 4)
        for opt, loss in ((self.opt_g, self.tocg(x).square().mean()), (self.opt_d, self.D(torch.randn(5, 3)).square().mean())):
            opt.zero_grad()
            loss.backward()
            opt.step()


def _fake_cuda_rng(monkeypatch):
    box = {"state": torch.arange(16, dtype=torch.uint8)}
    monkeypatch.setattr(torch.cuda, "get_rng_state", lambda *a: box["state"].clone())
    monkeypatch.setattr(torch.cuda, "set_rng_state", lambda s, *a: box.update(state=s.clone()))
    return box


def test_state_file_round_trip(tmp_path, monkeypatch):
    cuda_rng = _fake_cuda_rng(monkeypatch)
    a = _Trainer(1)
    for _ in range(3):
        a.step()
    a.set_lr_factor(0.25)
    run = train_loop.TrainRun("stage1", a, _Loader(), str(tmp_path), keep_step=10, load_step=0)
    run.step = 4
    torch.manual_seed(123)
    cpu_rng = torch.get_rng_state()
    path = run.save()
    assert sorted(os.listdir(tmp_path)) == ["D_step_000004.pth", "state_step_000004.pth", "tocg_step_000004.pth"]
    st = torch.load(path, weights_only=False)
    assert st["step"] == 4 and st["loader"] == {"seed": 7, "epoch": 3, "index": 5, "batch_size": 2} and st["trainer"]["lr_factor"] == 0.25

    b = _Trainer(2)  # other weights, no optimiser state yet
    torch.manual_seed(0)
    cuda_rng["state"] = torch.zeros(16, dtype=torch.uint8)
    loader = _Loader()
    loader.pos = (0, 0)
    rb = train_loop.TrainRun("stage1", b, loader, str(tmp_path), keep_step=10)
    rb.resume(path)
    assert rb.step == 4 and loader.pos == (3, 5) and b.lr_factor == 0.25
    assert torch.equal(torch.get_rng_state(), cpu_rng) and torch.equal(cuda_rng["state"], torch.arange(16, dtype=torch.uint8))
    for x, y in ((a.tocg, b.tocg), (a.D, b.D)):
        sx, sy = x.state_dict(), y.state_dict()
        assert all(torch.equal(sx[k], sy[k]) for k in sx)
    for oa, ob in ((a.opt_g, b.opt_g), (a.opt_d, b.opt_d)):
        assert ob.param_groups[0]["lr"] is b._lr["G" if ob is b.opt_g else "D"]  # the trainer's own lr tensor, not the file's
        for pa, pb in zip(oa.param_groups[0]["params"], ob.param_groups[0]["params"]):
            for k in ("step", "exp_avg", "exp_avg_sq"):
                assert torch.equal(oa.state[pa][k], ob.state[pb][k]), k
    assert float(b._lr["G"]) == float(a._lr["G"]) and float(b._lr["D"]) == float(a._lr["D"])
    a.step()  # one more step from the same state: the same result
    torch.set_rng_state(cpu_rng)
    b.step()
    assert all(torch.equal(x, y) for x, y in zip(a.tocg.state_dict().values(), b.tocg.state_dict().values()))

    with pytest.raises(ValueError, match="stage1 state"):
        train_loop.TrainRun("stage2", _Trainer(3), _Loader(), str(tmp_path), keep_step=10).resume(path)
    other = _Loader()
    other.seed = 8
    with pytest.raises(ValueError, match="seed"):
        train_loop.TrainRun("stage1", _Trainer(3), other, str(tmp_path), keep_step=10).resume(path)
    # a resume with other flags would not continue the saved run
    with pytest.raises(ValueError, match="base_lr"):
        train_loop.TrainRun("stage1", _Trainer(3, g_lr=1e-3), _Loader(), str(tmp_path), keep_step=10).resume(path)
    with pytest.raises(ValueError, match="occlusion"):
        train_loop.TrainRun("stage1", _Trainer(3, occlusion=False), _Loader(), str(tmp_path), keep_step=10).resume(path)


class _FrozenTocgTrainer(_Trainer):
    """Stage-2 roles: a frozen tocg besides the trained G and D."""

    def __init__(self, seed, tocg_seed):
        super().__init__(seed)
        self.tocg = torch.nn.Linear(4, 4)
        with torch.no_grad():
            self.tocg.weight.copy_(torch.randn(4, 4, generator=torch.Generator().manual_seed(tocg_seed)))
            self.tocg.bias.zero_()


def test_resume_refuses_another_frozen_tocg(tmp_path, monkeypatch):
    _fake_cuda_rng(monkeypatch)
    run = train_loop.TrainRun("stage2", _FrozenTocgTrainer(1, 5), _Loader(), str(tmp_path), keep_step=10, decay_step=10)
    run.step = 2
    path = run.save()
    assert sorted(os.listdir(tmp_path)) == ["dis_step_000002.pth", "gen_step_000002.pth", "state_step_000002.pth"]
    train_loop.TrainRun("stage2", _FrozenTocgTrainer(2, 5), _Loader(), str(tmp_path), keep_step=10, decay_step=10).resume(path)
    with pytest.raises(ValueError, match="tocg_sha256"):
        train_loop.TrainRun("stage2", _FrozenTocgTrainer(2, 6), _Loader(), str(tmp_path), keep_step=10, decay_step=10).resume(path)


def test_stage2_rank1_trains_without_an_evaluator(tmp_path, monkeypatch):
    """Under torchrun only rank 0 builds the LPIPS evaluator: the other ranks construct the run and train through the evaluation
    steps without it; rank 0 without an evaluator is refused."""
    monkeypatch.setattr(train_loop, "_dist", lambda: (object(), 1, 2))
    tr = _Trainer(1)
    run = train_loop.TrainRun("stage2", tr, _Loader(), str(tmp_path), keep_step=10, decay_step=10, lpips_count=1, save_count=100,
                              display_count=100, evaluator=None)
    run.evaluate = None  # any call would raise
    run.train(until=3)
    assert run.step == 3 and tr.replays == 3 and run.lpips == []
    monkeypatch.setattr(train_loop, "_dist", lambda: (object(), 0, 2))
    with pytest.raises(ValueError, match="evaluator"):
        train_loop.TrainRun("stage2", _Trainer(1), _Loader(), str(tmp_path), keep_step=10, decay_step=10, lpips_count=1)


def test_model_files_load_with_the_reference_loaders(tmp_path):
    import network_generator
    import networks
    from helpers import gen_opt, tocg_opt
    tocg = networks.ConditionGenerator(tocg_opt(), 4, 16, 13, ngf=96, norm_layer=torch.nn.BatchNorm2d)
    G = network_generator.SPADEGenerator(gen_opt(512, 384), 9)
    for i, m in enumerate((tocg, G)):
        with torch.no_grad():
            for t in m.state_dict().values():
                if t.is_floating_point():
                    t.copy_(torch.randn(t.shape, generator=torch.Generator().manual_seed(i)))
    train_loop.save_model(tocg, str(tmp_path / "tocg_step_000010.pth"))
    train_loop.save_model(G, str(tmp_path / "gen_step_000010.pth"))

    t2 = networks.ConditionGenerator(tocg_opt(), 4, 16, 13, ngf=96, norm_layer=torch.nn.BatchNorm2d)
    networks.load_checkpoint(t2, str(tmp_path / "tocg_step_000010.pth"), tocg_opt(False))
    assert all(torch.equal(a, b) for a, b in zip(tocg.state_dict().values(), t2.state_dict().values()))

    # test_generator.py:77-86: keys renamed, _metadata carried over, strict=True
    sd = torch.load(str(tmp_path / "gen_step_000010.pth"))
    assert isinstance(sd, collections.OrderedDict) and list(sd) == list(G.state_dict())
    new = collections.OrderedDict([(k.replace("ace", "alias").replace(".Spade", ""), v) for (k, v) in sd.items()])
    new._metadata = collections.OrderedDict([(k.replace("ace", "alias").replace(".Spade", ""), v) for (k, v) in sd._metadata.items()])
    g2 = network_generator.SPADEGenerator(gen_opt(512, 384), 9)
    g2.load_state_dict(new, strict=True)
    assert all(torch.equal(a, b) for a, b in zip(G.state_dict().values(), g2.state_dict().values()))

    if hrv_env.reference_dir() is None:
        return
    tg = hrv_env.load_reference_script("test_generator")  # the reference's own function and SPADEGenerator
    ref = tg.SPADEGenerator(gen_opt(512, 384), 9)
    tg.load_checkpoint_G(ref, str(tmp_path / "gen_step_000010.pth"), gen_opt(512, 384, cuda=False))
    assert all(torch.equal(a, b) for a, b in zip(G.state_dict().values(), ref.state_dict().values()))


@pytest.mark.parametrize("stage,argv,match", [
    ("stage2", ["--name", "x", "--tocg_checkpoint", "{ckpt}", "--bogus", "1"], "unrecognized"),
    ("stage2", ["--name", "x"], "tocg_checkpoint"),
    ("stage2", ["--name", "x", "--tocg_checkpoint", "{ckpt}", "-b", "0"], "batch_size"),
    ("stage2", ["--name", "x", "--tocg_checkpoint", "{ckpt}", "--lpips_count", "0"], "lpips_count"),
    ("stage2", ["--name", "x", "--tocg_checkpoint", "{ckpt}", "--load_step", "5", "--keep_step", "2", "--decay_step", "3"], "nothing to train"),
    ("stage2", ["--name", "x", "--tocg_checkpoint", "{ckpt}", "--fine_height", "512"], "fine_height"),
    ("stage2", ["--name", "x", "--tocg_checkpoint", "{root}/missing.pth"], "does not exist"),
    ("stage2", ["--name", "x", "--tocg_checkpoint", "{ckpt}", "--G_lr", "-1"], "G_lr"),
    ("stage2", ["--name", "x", "--tocg_checkpoint", "{ckpt}", "--resume", "{ckpt}", "--load_step", "3"], "resume"),
    ("stage2", ["--name", "x", "--tocg_checkpoint", "{ckpt}", "--resume", "{root}/none.pth"], "not a file"),
    ("stage1", ["--decay_step", "3"], "unrecognized"),
    ("stage1", ["--lpips_count", "3"], "unrecognized"),
    ("stage1", ["--dataroot", "{root}/nowhere"], "does not exist"),
    ("stage1", ["--save_count", "-1"], "save_count"),
])
def test_cli_refuses_bad_flags(tmp_path, capsys, stage, argv, match):
    ckpt = tmp_path / "tocg.pth"
    ckpt.write_bytes(b"")
    argv = [a.format(root=tmp_path, ckpt=ckpt) for a in argv]
    with pytest.raises(SystemExit) as e:
        train_loop.parse_args(stage, ["--dataroot", str(tmp_path)] + argv)
    assert e.value.code == 2
    assert match in capsys.readouterr().err


def test_cli_accepts_the_reference_flags(tmp_path):
    ckpt = tmp_path / "tocg.pth"
    ckpt.write_bytes(b"")
    opt = train_loop.parse_args("stage2", ["--name", "x", "--dataroot", str(tmp_path), "--data_list", "p.txt", "-b", "4", "-j", "2",
                                           "--fine_height", "512", "--fine_width", "384", "--keep_step", "10", "--decay_step", "10",
                                           "--load_step", "5", "--save_count", "5", "--display_count", "1", "--lpips_count", "5",
                                           "--G_lr", "0.001", "--D_lr", "0.002", "--tocg_checkpoint", str(ckpt), "--occlusion", "--fp16"])
    assert (opt.batch_size, opt.workers, opt.fine_height, opt.load_step, opt.fp16, opt.occlusion, opt.G_lr) == (4, 2, 512, 5, True, True, 0.001)
    opt = train_loop.parse_args("stage1", ["--dataroot", str(tmp_path), "--batch-size", "3"])
    assert (opt.batch_size, opt.fine_height, opt.fine_width, opt.keep_step, opt.tocg_checkpoint) == (3, 256, 192, 300000, "")
    with pytest.raises(SystemExit):
        train_loop.main(["stage3"])
