"""GPU: the training driver (hrviton_b200.train_loop, tools/train.py).

The central check: a run of N steps equals k steps, a save, and a fresh process that resumes from the state file and trains the
remaining N - k steps, bit for bit (every parameter, BatchNorm and spectral-norm buffer, Adam's exp_avg / exp_avg_sq / step, the loss
scalers, the generators, every per-step loss), for stage 1 and stage 2, in bf16 and in fp16 with dynamic loss scaling, with a stage-2
schedule that crosses keep_step after the save.  Also: capture(rollback=True) leaves every state as it was, the device-tensor lr at
factor 1 equals today's trainer, and the driver's LPIPS equals PerceptualLoss on the same outputs accumulated as train_generator.py
accumulates it.

The runs are subprocesses executing this file (`python test_train_loop_gpu.py <out> <stage> <flags>`), so each starts from a clean
process as a resumed job does."""
import json
import os
import subprocess
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for _p in (ROOT, HERE):
    if _p not in sys.path:
        sys.path.insert(0, _p)
import hrv_loader  # noqa: E402

hrv_loader.load()

pytestmark = pytest.mark.gpu
N_TRAIN, N_TEST, BATCH = 6, 2, 2
SIZES = {"stage1": (256, 192), "stage2": (512, 384)}


def _env(tmp):
    env = dict(os.environ, HRV_VGG_RANDOM_INIT="1", HRV_ALEX_RANDOM_INIT="1", CUBLAS_WORKSPACE_CONFIG=":4096:8",
               PYTHONPATH=os.pathsep.join([ROOT, HERE]))
    env.pop("WORLD_SIZE", None)
    return env


@pytest.fixture(scope="module")
def tree(tmp_path_factory):
    """A synthetic VITON-HD tree, a tocg checkpoint and the LPIPS heads where PerceptualLoss looks for them (./eval_models/...)."""
    import networks
    from helpers import tocg_opt
    from hrviton_b200 import metrics, synth
    root = tmp_path_factory.mktemp("trainloop")
    synth.write_vitonhd(str(root), N_TRAIN, seed=31, datamode="train")
    synth.write_vitonhd(str(root), N_TEST, seed=32, datamode="test", pairs="test_pairs.txt")
    tocg = networks.ConditionGenerator(tocg_opt(), 4, 16, 13, ngf=96, norm_layer=torch.nn.BatchNorm2d)
    sd = tocg.state_dict()
    synth.fill_state_dict(sd, 3)
    torch.save(sd, str(root / "tocg.pth"))
    heads = metrics.PNetLin(pretrained=False).state_dict()
    synth.fill_state_dict({k: v for k, v in heads.items() if not k.startswith("scaling_layer.")}, 4)  # the constant input scaling stays
    for k in heads:
        if k.startswith("lin"):  # LPIPS heads are non-negative
            heads[k].abs_()
    os.makedirs(str(root / "eval_models" / "weights" / "v0.1"))
    torch.save(heads, str(root / "eval_models" / "weights" / "v0.1" / "alex.pth"))
    return root


def _flags(tree, stage, name, fp16, extra=()):
    h, w = SIZES[stage]
    f = ["--name", name, "--dataroot", str(tree), "--data_list", "pairs.txt", "-b", str(BATCH), "-j", "1", "--fine_height", str(h),
         "--fine_width", str(w), "--checkpoint_dir", str(tree / "ckpt"), "--display_count", "1000", "--occlusion", "--seed", "3"]
    if stage == "stage1":
        f += ["--keep_step", "6", "--save_count", "4"]
    else:  # the schedule leaves factor 1 after step 3, one step after the save at 2
        f += ["--keep_step", "3", "--decay_step", "3", "--lr_interval", "1", "--save_count", "2", "--lpips_count", "1000",
              "--tocg_checkpoint", str(tree / "tocg.pth"), "--test_dataroot", str(tree), "--test_data_list", "test_pairs.txt"]
    return f + (["--fp16"] if fp16 else []) + list(extra)


def _launch(tree, out, stage, flags, nproc=1):
    cmd = [sys.executable, os.path.abspath(__file__), str(out), stage] + flags
    if nproc > 1:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nproc-per-node", str(nproc), "--master-addr", "127.0.0.1",
               "--master-port", str(_free_port())] + cmd[1:]
    r = subprocess.run(cmd, cwd=str(tree), env=_env(tree), capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-6000:]
    return torch.load(str(out), weights_only=False)


def _free_port():
    import socket
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _final_state(ckpt):
    """Everything a run leaves: its final model files and state file, flattened to {name: tensor or value}."""
    out = {}
    for f in sorted(os.listdir(ckpt)):
        if f.endswith("final.pth"):
            sd = torch.load(os.path.join(ckpt, f), weights_only=False)
            if f == "state_final.pth":
                sd.pop("models")
            _flatten(sd, f, out)
    return out


def _flatten(obj, prefix, out):
    if isinstance(obj, dict):
        for k, v in obj.items():
            _flatten(v, "%s.%s" % (prefix, k), out)
    elif isinstance(obj, (list, tuple)):
        for i, v in enumerate(obj):
            _flatten(v, "%s.%d" % (prefix, i), out)
    else:
        out[prefix] = obj


def _assert_same(a, b):
    assert a.keys() == b.keys(), sorted(set(a) ^ set(b))[:10]
    diff = [k for k in a if not (torch.equal(a[k], b[k]) if torch.is_tensor(a[k]) else a[k] == b[k])]
    assert not diff, diff[:10]


def _check_resume(tree, stage, fp16, nproc=1):
    tag = "%s_%s_%d" % (stage, "fp16" if fp16 else "bf16", nproc)
    k = 4 if stage == "stage1" else 2
    full = _launch(tree, tree / (tag + "_full.pt"), stage, _flags(tree, stage, tag + "_full", fp16), nproc)
    state = str(tree / "ckpt" / (tag + "_full") / ("state_step_%06d.pth" % k))
    resumed = _launch(tree, tree / (tag + "_res.pt"), stage, _flags(tree, stage, tag + "_res", fp16, ["--resume", state]), nproc)
    assert sorted(full["losses"]) == list(range(1, 7)) and sorted(resumed["losses"]) == list(range(k + 1, 7))
    for s in range(k + 1, 7):
        _assert_same(full["losses"][s], resumed["losses"][s])
    a, b = (_final_state(str(tree / "ckpt" / (tag + s))) for s in ("_full", "_res"))
    assert any(".exp_avg_sq" in n for n in a) and any("running_mean" in n or "weight_u" in n for n in a)
    if fp16:
        assert any(n.endswith("scalers.G.scale") for n in a)
    if stage == "stage2":
        assert a["state_final.pth.trainer.lr_factor"] < 1.0 and full["factors"][3] == 1.0 and full["factors"][6] < full["factors"][5] < 1.0
    _assert_same(a, b)


@pytest.mark.parametrize("fp16", [False, True], ids=["bf16", "fp16"])
@pytest.mark.parametrize("stage", ["stage1", "stage2"])
def test_resume_in_a_fresh_process_is_bit_exact(tree, stage, fp16):
    _check_resume(tree, stage, fp16)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_rank_resume_is_bit_exact(tree):
    _check_resume(tree, "stage2", False, nproc=2)


# ------------------------------------------------------------------------------------------------ in-process checks

def _stage1_trainer(**kw):
    import networks
    from helpers import tocg_opt
    from hrviton_b200 import synth, train_step
    tocg = networks.ConditionGenerator(tocg_opt(True), 4, 16, 13, ngf=96, norm_layer=torch.nn.BatchNorm2d)
    sd = tocg.state_dict(); synth.fill_state_dict(sd, 11); tocg.load_state_dict(sd)
    torch.manual_seed(0)
    D = networks.define_D(input_nc=33, Ddownx2=True, Ddropout=True, n_layers_D=3, spectral=False, num_D=2)
    vgg = networks.Vgg19().cuda().eval()
    return train_step.Stage1Trainer(tocg.cuda().train(), D.cuda().train(), vgg, **kw)


def _everything(tr):
    out = {"rng.cuda": torch.cuda.get_rng_state(), "rng.cpu": torch.get_rng_state()}
    for i, m in enumerate(tr.modules()):
        out.update({"m%d.%s" % (i, k): v.detach().clone() for k, v in m.state_dict().items()})
    for name, opt in (("G", tr.opt_g), ("D", tr.opt_d)):
        for j, p in enumerate(opt.param_groups[0]["params"]):
            out.update({"%s.%d.%s" % (name, j, k): v.clone() for k, v in opt.state.get(p, {}).items()})
    for name, sc in tr.scalers.items():
        out.update({"sc.%s.%s" % (name, k): t.clone() for k, t in (("scale", sc.scale), ("tracker", sc.growth_tracker))})
    return out


def test_capture_with_rollback_leaves_state_unchanged(monkeypatch):
    from hrviton_b200 import train_step
    monkeypatch.setenv("HRV_VGG_RANDOM_INIT", "1")
    tr = _stage1_trainer(loss_scale="dynamic", tensor_lr=True)
    batch = train_step.synthetic_batch_stage1(2, 256, 192, "cuda", seed=1)
    torch.cuda.manual_seed(5)
    tr.step(batch)  # Adam state and scaler history exist before the capture
    torch.cuda.synchronize()
    before = _everything(tr)
    tr.capture(batch, rollback=True)
    torch.cuda.synchronize()
    after = _everything(tr)
    try:
        _assert_same(before, after)
        # and the first replay is the step an eager call from that state takes
        out = {k: v.clone() for k, v in tr.replay(batch).items()}
        torch.cuda.synchronize()
    finally:
        tr.release_graph()
    tr2 = _stage1_trainer(loss_scale="dynamic", tensor_lr=True)
    torch.cuda.manual_seed(5)
    tr2.step(batch)
    eager = tr2.step(batch)
    _assert_same(out, {k: v.clone() for k, v in eager.items()})


def _stage2_trainer(h, w, **kw):
    import network_generator
    import networks
    from helpers import gen_opt, tocg_opt
    from hrviton_b200 import synth, train_step
    torch.manual_seed(0)
    tocg = networks.ConditionGenerator(tocg_opt(True), 4, 16, 13, ngf=96, norm_layer=torch.nn.BatchNorm2d)
    G = network_generator.SPADEGenerator(gen_opt(h, w, True), 9)
    D = network_generator.MultiscaleDiscriminator(gen_opt(h, w, True))
    for m, seed in ((tocg, 3), (G, 4), (D, 5)):
        sd = m.state_dict()
        synth.fill_state_dict(sd, seed)
        m.load_state_dict(sd)
    return train_step.Stage2Trainer(tocg.cuda().eval(), G.cuda().train(), D.cuda().train(), networks.Vgg19().cuda().eval(), **kw)


def test_stage2_rollback_replays_equal_eager_steps(monkeypatch):
    """Stage 2 with rollback: the graph records the packing of the generator's input pyramid (which its no-grad forward in the
    discriminator update reads from a cache), so every replay uses the current weights.  Two replays equal two eager steps that
    start a new parameter generation before each call (fused Adam leaves tensor._version alone, so an eager step would otherwise
    keep the first pack too): losses, parameters, buffers, Adam state, loss scalers and generators, bit for bit."""
    from hrviton_b200 import ops, train_step
    monkeypatch.setenv("HRV_VGG_RANDOM_INIT", "1")
    h, w = SIZES["stage2"]
    batches = [train_step.synthetic_batch(2, h, w, "cuda", seed=s) for s in range(3)]
    tr = _stage2_trainer(h, w, loss_scale="dynamic", tensor_lr=True)
    torch.cuda.manual_seed(7)
    tr.capture(batches[0], h, w, rollback=True)
    try:
        graph = [{k: v.clone() for k, v in tr.replay(b).items() if torch.is_tensor(v)} for b in batches[1:]]
        torch.cuda.synchronize()
        graph_state = _everything(tr)
    finally:
        tr.release_graph()
    del tr
    tr2 = _stage2_trainer(h, w, loss_scale="dynamic", tensor_lr=True)
    torch.cuda.manual_seed(7)
    eager = []
    for b in batches[1:]:
        ops.PARAM_GEN[0] += 1
        eager.append({k: v.clone() for k, v in tr2.step(b, h, w).items() if torch.is_tensor(v)})
    torch.cuda.synchronize()
    for i, (a, b) in enumerate(zip(graph, eager)):
        assert a.keys() == b.keys()
        assert [k for k in a if not torch.equal(a[k], b[k])] == [], i
    _assert_same(graph_state, _everything(tr2))


def test_tensor_lr_at_factor_one_equals_todays_trainer(monkeypatch):
    from hrviton_b200 import train_step
    monkeypatch.setenv("HRV_VGG_RANDOM_INIT", "1")
    batches = [train_step.synthetic_batch_stage1(2, 256, 192, "cuda", seed=s) for s in range(3)]
    runs = []
    for tensor_lr in (False, True):
        tr = _stage1_trainer(tensor_lr=tensor_lr)
        if tensor_lr:
            tr.set_lr_factor(1.0)
        torch.cuda.manual_seed(9)
        tr.capture(batches[0])
        losses = [{k: v.clone() for k, v in tr.replay(b).items()} for b in batches]
        torch.cuda.synchronize()
        st = _everything(tr)
        st.update({"loss%d.%s" % (i, k): v for i, l in enumerate(losses) for k, v in l.items()})
        tr.release_graph()
        runs.append(st)
    _assert_same(*runs)


def test_driver_lpips_equals_perceptual_loss(tree, monkeypatch):
    """TrainRun.evaluate() against PerceptualLoss on the outputs it scored, accumulated as train_generator.py:578-581 does."""
    import eval_models
    from torchvision.transforms import transforms

    from hrviton_b200 import data, train_loop
    monkeypatch.setenv("HRV_VGG_RANDOM_INIT", "1")
    monkeypatch.setenv("HRV_ALEX_RANDOM_INIT", "1")
    monkeypatch.chdir(str(tree))
    h, w = SIZES["stage2"]
    tr = _stage2_trainer(h, w, tensor_lr=True)
    loader = data.VitonHDLoader(str(tree), "train", "pairs.txt", h, w, BATCH, workers=1, keys=data.STAGE2_KEYS)
    test_loader = data.VitonHDLoader(str(tree), "test", "test_pairs.txt", h, w, 1, workers=1, mode="test", keys=train_loop.EVAL_KEYS,
                                     shuffle=False, shard=False)
    model = eval_models.PerceptualLoss(model="net-lin", net="alex", use_gpu=True)
    calls = []

    class Recording:
        def forward(self, pred, target):
            calls.append((pred.clone(), target.clone()))
            return model.forward(pred, target)

    run = train_loop.TrainRun("stage2", tr, loader, str(tree / "lp"), keep_step=1, decay_step=1, lpips_count=1,
                              evaluator=(test_loader, Recording()), lpips_samples=N_TEST)
    try:
        values = [run.evaluate() for _ in range(2)]  # the second call re-reads the same samples from the start
    finally:
        if run._tryon is not None:
            run._tryon.release()
    assert len(calls) == 2 * N_TEST
    T2 = transforms.Compose([transforms.Resize((128, 128))])
    with torch.no_grad():
        avg = 0.0
        for pred, target in calls[:N_TEST]:
            avg += model.forward(pred, target)
        avg = avg / N_TEST
    assert values[0] == float(avg) and values[1] == values[0] and values[0] > 0
    assert calls[0][0].shape == (1, 3, 128, 128)
    ref = next(iter(data.VitonHDLoader(str(tree), "test", "test_pairs.txt", h, w, 1, workers=0, mode="test", keys=("image",), shuffle=False)))
    assert torch.equal(calls[0][0], T2(ref["image"]))  # pred = T2(im), the reference's argument order


# ------------------------------------------------------------------------------------------------ the subprocess side

def _worker(out, stage, argv):
    from hrviton_b200 import train_loop
    opt = train_loop.parse_args(stage, argv)
    run = train_loop.build(opt, log=lambda *a: None)
    losses, factors = {}, {}

    def on_step(step, l):
        losses[step] = {k: v.detach().clone() for k, v in l.items() if torch.is_tensor(v)}
        factors[step] = run.trainer.lr_factor if stage == "stage2" else 1.0
    run.on_step = on_step
    try:
        run.start().train()
        torch.cuda.synchronize()
    finally:
        run.trainer.release_graph()
    rank = int(os.environ.get("RANK", "0"))
    if rank == 0:
        torch.save({"losses": {s: {k: v.cpu() for k, v in l.items()} for s, l in losses.items()}, "factors": factors}, out)
    import torch.distributed as dist
    if dist.is_initialized():
        dist.destroy_process_group()


if __name__ == "__main__":
    _worker(sys.argv[1], sys.argv[2], sys.argv[3:])
    print(json.dumps({"ok": True}))
