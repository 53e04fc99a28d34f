"""CPU: the stage-2 options of train_generator.py on the command line and in the run state (hrviton_b200.train_loop): the parsed
defaults are today's trainer, the README's stage-2 command line parses, --GT refuses the flags that act on the condition generator,
a state file written before the options were recorded resumes while a mismatched option is refused, and the kernels that take the
cloth-mask composition and the class table do not spill."""
import inspect

import pytest
import torch

import hrv_env  # noqa: F401
from hrviton_b200 import train_loop, train_step


def _ckpt(tmp_path):
    ckpt = tmp_path / "tocg.pth"
    ckpt.write_bytes(b"")
    return str(ckpt)


def test_parsed_defaults_are_todays_trainer(tmp_path):
    opt = train_loop.parse_args("stage2", ["--name", "x", "--dataroot", str(tmp_path), "--tocg_checkpoint", _ckpt(tmp_path)])
    kw = train_loop.stage2_options(opt)
    assert kw == train_loop.STAGE2_OPTIONS
    sig = inspect.signature(train_step.Stage2Trainer.__init__).parameters
    assert {k: sig[k].default for k in kw if k != "no_ganFeat_loss"} == {k: v for k, v in kw.items() if k != "no_ganFeat_loss"}
    assert kw["no_ganFeat_loss"] is False  # what build() gave the discriminator before the flag existed


def test_readme_stage2_line_parses(tmp_path):
    # README: python3 train_generator.py --cuda {True} --name test -b 4 -j 8 --gpu_ids {gpu_ids} --fp16 --tocg_checkpoint {...} --occlusion
    opt = train_loop.parse_args("stage2", ["--dataroot", str(tmp_path), "--name", "test", "-b", "4", "-j", "8", "--fp16", "--tocg_checkpoint",
                                           _ckpt(tmp_path), "--occlusion"])
    assert (opt.batch_size, opt.workers, opt.fp16, opt.occlusion) == (4, 8, True, True)
    assert train_loop.stage2_options(opt) == train_loop.STAGE2_OPTIONS
    opt = train_loop.parse_args("stage2", ["--dataroot", str(tmp_path), "--name", "test", "--tocg_checkpoint", _ckpt(tmp_path),
                                           "--clothmask_composition", "detach", "--no_ganFeat_loss", "--no_vgg_loss", "--lambda_feat", "5",
                                           "--lambda_vgg", "2"])
    assert train_loop.stage2_options(opt) == {"gt": False, "clothmask_composition": "detach", "no_vgg_loss": True, "no_ganFeat_loss": True,
                                              "lambda_feat": 5.0, "lambda_vgg": 2.0}
    opt = train_loop.parse_args("stage2", ["--dataroot", str(tmp_path), "--name", "test", "--GT", "--fp16"])
    assert opt.GT and opt.tocg_checkpoint is None and train_loop.stage2_options(opt)["gt"] is True


@pytest.mark.parametrize("argv,match", [
    (["--GT", "--tocg_checkpoint", "{ckpt}"], "--tocg_checkpoint"),
    (["--GT", "--occlusion"], "--occlusion"),
    (["--GT", "--clothmask_composition", "detach"], "--clothmask_composition"),
    (["--GT", "--clothmask_composition", "no_composition"], "--clothmask_composition"),
    ([], "--tocg_checkpoint"),
    (["--tocg_checkpoint", "{ckpt}", "--clothmask_composition", "none"], "invalid choice"),
    (["--GT", "--num_D", "3"], "unrecognized"),
])
def test_cli_refuses(tmp_path, capsys, argv, match):
    ckpt = _ckpt(tmp_path)
    with pytest.raises(SystemExit) as e:
        train_loop.parse_args("stage2", ["--name", "x", "--dataroot", str(tmp_path)] + [a.format(ckpt=ckpt) for a in argv])
    assert e.value.code == 2
    assert match in capsys.readouterr().err


def test_trainer_refuses_unknown_options():
    m = torch.nn.Linear(2, 2)
    with pytest.raises(ValueError, match="clothmask_composition"):
        train_step.Stage2Trainer(m, m, m, m, clothmask_composition="none")
    with pytest.raises(ValueError, match="gt=True"):
        train_step.Stage2Trainer(None, m, m, m)
    with pytest.raises(ValueError, match="clothmask_composition"):
        train_step.make_generator_inputs(None, {}, 8, 8, clothmask_composition="none")


class _Loader:
    seed, batch_size = 7, 2

    def position(self):
        return (0, 4)

    def start_at(self, epoch, index):
        pass


class _Trainer(train_step._TrainState, train_step._LossScaling):
    """The state surface of a Stage2Trainer on CPU modules, with its options (no_ganFeat_loss on D, as build() sets it)."""
    _captured = None

    def __init__(self, **options):
        torch.manual_seed(0)
        options = dict(train_loop.STAGE2_OPTIONS, **options)
        self.G, self.D = torch.nn.Linear(4, 3), torch.nn.Linear(3, 2)
        self.D.no_ganFeat_loss = options.pop("no_ganFeat_loss")
        self.tocg = None if options["gt"] else torch.nn.Linear(4, 4)
        self._make_optimizers(self.G.parameters(), self.D.parameters(), 1e-4, 4e-4, (0.0, 0.9), True)
        self.scalers = {}
        self.occlusion = not options["gt"]
        for k, v in options.items():
            setattr(self, k, v)


def _run(tmp_path, **options):
    return train_loop.TrainRun("stage2", _Trainer(**options), _Loader(), str(tmp_path), keep_step=10, decay_step=10)


def _save(tmp_path, **options):
    run = _run(tmp_path, **options)
    run.step = 4
    return run.save()


def test_old_state_resumes_and_mismatched_options_are_refused(tmp_path, monkeypatch):
    rng = torch.zeros(16, dtype=torch.uint8)  # the CUDA generator's state, which this machine may not have
    monkeypatch.setattr(torch.cuda, "get_rng_state", lambda *a: rng.clone())
    monkeypatch.setattr(torch.cuda, "set_rng_state", lambda *a: None)
    cpu_rng = torch.get_rng_state()
    path = _save(tmp_path)
    st = torch.load(path, weights_only=False)
    assert {k: st["config"][k] for k in train_loop.STAGE2_OPTIONS} == train_loop.STAGE2_OPTIONS and "tocg_sha256" in st["config"]
    for k in train_loop.STAGE2_OPTIONS:  # the state file of a run from before the options were recorded
        del st["config"][k]
    torch.save(st, path)
    _run(tmp_path).resume(path)
    for opt in ({"clothmask_composition": "detach"}, {"no_vgg_loss": True}, {"no_ganFeat_loss": True}, {"lambda_vgg": 2.0}):
        with pytest.raises(ValueError, match=list(opt)[0]):
            _run(tmp_path, **opt).resume(path)
    with pytest.raises(ValueError, match="gt|occlusion"):
        _run(tmp_path, gt=True).resume(path)
    # a --GT run records no tocg, resumes as --GT only
    path = _save(tmp_path / "gt", gt=True, no_vgg_loss=True)
    assert "tocg_sha256" not in torch.load(path, weights_only=False)["config"]
    _run(tmp_path / "gt", gt=True, no_vgg_loss=True).resume(path)
    with pytest.raises(ValueError, match="no_vgg_loss"):
        _run(tmp_path / "gt", gt=True).resume(path)
    with pytest.raises(ValueError, match="gt|occlusion"):
        _run(tmp_path / "gt", no_vgg_loss=True).resume(path)
    torch.set_rng_state(cpu_rng)


def test_changed_kernels_do_not_spill():
    """The parse-map kernel (with its cloth-mask composition) and both one-hot kernels (identity and class table), in both library
    flavours: no stack frame, no local-memory spills."""
    import os
    import re
    import shutil
    import subprocess
    so = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "hr-viton_b200", "libhrviton_sm100.so")
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not (os.path.exists(so) and os.path.exists(tool)):
        pytest.skip("needs the built library and cuobjdump")
    usage = subprocess.run([tool, "--dump-resource-usage", so], capture_output=True, text=True, check=True).stdout
    rows = re.findall(r"Function (\S+):\s*\n\s*REG:\d+ STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", usage)
    rows = [(f, int(s), int(l)) for f, s, l in rows if "parse_blur_argmax_kernel" in f or "onehot_u8_kernel" in f]
    assert len(rows) == 6, rows  # parse_blur_argmax + two one-hot instances, two flavours
    assert all(s == 0 and l == 0 for _, s, l in rows), rows
