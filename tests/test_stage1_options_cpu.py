"""CPU: the stage-1 loss options of train_condition.py on the command line and in the run state (hrviton_b200.train_loop): the parsed
defaults are today's trainer, the README's stage-1 command line parses, --val_count refuses compositions the validation does not
implement, and a state file written before the options were recorded resumes while a mismatched option is refused."""
import inspect

import pytest
import torch

import hrv_env  # noqa: F401
from hrviton_b200 import train_loop, train_step


def test_parsed_defaults_are_todays_trainer(tmp_path):
    opt = train_loop.parse_args("stage1", ["--dataroot", str(tmp_path)])
    kw = train_loop.stage1_options(opt)
    assert kw == train_loop.STAGE1_OPTIONS
    sig = inspect.signature(train_step.Stage1Trainer.__init__).parameters
    assert {k: sig[k].default for k in kw} == kw
    assert (sig["lasttvonly"].default, sig["interflowloss"].default) == (True, True)


def test_readme_stage1_line_parses(tmp_path):
    # README: python3 train_condition.py --cuda {True} --gpu_ids {gpu_ids} --Ddownx2 --Ddropout --lasttvonly --interflowloss --occlusion
    opt = train_loop.parse_args("stage1", ["--dataroot", str(tmp_path), "--Ddownx2", "--Ddropout", "--lasttvonly", "--interflowloss",
                                           "--occlusion"])
    assert opt.occlusion and train_loop.stage1_options(opt) == train_loop.STAGE1_OPTIONS
    opt = train_loop.parse_args("stage1", ["--dataroot", str(tmp_path), "--edgeawaretv", "weighted", "--add_lasttv", "--clothmask_composition",
                                           "detach", "--no_GAN_loss", "--G_D_seperate", "--tvlambda", "3", "--CElamda", "5", "--GANlambda", "0.5"])
    assert train_loop.stage1_options(opt) == {"edgeawaretv": "weighted", "add_lasttv": True, "clothmask_composition": "detach",
                                              "no_gan_loss": True, "g_d_separate": True, "tvlambda": 3.0, "ce_lambda": 5.0, "gan_lambda": 0.5}


@pytest.mark.parametrize("argv,match", [
    (["--val_count", "10", "--clothmask_composition", "detach"], "warp_grad"),
    (["--val_count", "10", "--clothmask_composition", "no_composition"], "warp_grad"),
    (["--edgeawaretv", "edges"], "invalid choice"),
    (["--clothmask_composition", "none"], "invalid choice"),
])
def test_cli_refuses(tmp_path, capsys, argv, match):
    with pytest.raises(SystemExit) as e:
        train_loop.parse_args("stage1", ["--dataroot", str(tmp_path), "--test_dataroot", str(tmp_path)] + argv)
    assert e.value.code == 2
    assert match in capsys.readouterr().err


def test_trainer_refuses_unknown_options():
    m = torch.nn.Linear(2, 2)
    with pytest.raises(ValueError, match="edgeawaretv"):
        train_step.Stage1Trainer(m, m, m, edgeawaretv="edges")
    with pytest.raises(ValueError, match="clothmask_composition"):
        train_step.Stage1Trainer(m, m, m, clothmask_composition="none")


class _Loader:
    seed, batch_size = 7, 2

    def position(self):
        return (0, 4)

    def start_at(self, epoch, index):
        pass


class _Trainer(train_step._TrainState, train_step._LossScaling):
    """The state surface of a Stage1Trainer on CPU modules, with its loss options."""
    _captured = None

    def __init__(self, **options):
        torch.manual_seed(0)
        self.tocg, self.D = torch.nn.Linear(4, 3), torch.nn.Linear(3, 2)
        self._make_optimizers(self.tocg.parameters(), self.D.parameters(), 2e-4, 2e-4, (0.5, 0.999), False)
        self.scalers = {}
        self.occlusion = True
        for k, v in dict(train_loop.STAGE1_OPTIONS, **options).items():
            setattr(self, k, v)


def _save(tmp_path, **options):
    run = train_loop.TrainRun("stage1", _Trainer(**options), _Loader(), str(tmp_path), keep_step=10)
    run.step = 4
    return run.save()


def test_old_state_resumes_and_mismatched_options_are_refused(tmp_path, monkeypatch):
    rng = torch.zeros(16, dtype=torch.uint8)  # the CUDA generator's state, which this machine may not have
    monkeypatch.setattr(torch.cuda, "get_rng_state", lambda *a: rng.clone())
    monkeypatch.setattr(torch.cuda, "set_rng_state", lambda *a: None)
    cpu_rng = torch.get_rng_state()
    path = _save(tmp_path)
    st = torch.load(path, weights_only=False)
    assert {k: st["config"][k] for k in train_loop.STAGE1_OPTIONS} == train_loop.STAGE1_OPTIONS
    for k in train_loop.STAGE1_OPTIONS:  # the state file of a run from before the options were recorded
        del st["config"][k]
    torch.save(st, path)
    train_loop.TrainRun("stage1", _Trainer(), _Loader(), str(tmp_path), keep_step=10).resume(path)
    for opt in ({"edgeawaretv": "weighted"}, {"no_gan_loss": True}, {"tvlambda": 3.0}):
        with pytest.raises(ValueError, match=list(opt)[0]):
            train_loop.TrainRun("stage1", _Trainer(**opt), _Loader(), str(tmp_path), keep_step=10).resume(path)
    path = _save(tmp_path / "w", edgeawaretv="weighted", add_lasttv=True)
    train_loop.TrainRun("stage1", _Trainer(edgeawaretv="weighted", add_lasttv=True), _Loader(), str(tmp_path / "w"), keep_step=10).resume(path)
    with pytest.raises(ValueError, match="add_lasttv"):
        train_loop.TrainRun("stage1", _Trainer(edgeawaretv="weighted"), _Loader(), str(tmp_path / "w"), keep_step=10).resume(path)
    torch.set_rng_state(cpu_rng)


def test_tv_kernels_do_not_spill_or_use_atomics():
    """The flow TV kernels of both library flavours: no stack frame (no local-memory spills) and no atomics in the SASS."""
    import os
    import re
    import shutil
    import subprocess
    so = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "hr-viton_b200", "libhrviton_sm100.so")
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not (os.path.exists(so) and os.path.exists(tool)):
        pytest.skip("needs the built library and cuobjdump")
    usage = subprocess.run([tool, "--dump-resource-usage", so], capture_output=True, text=True, check=True).stdout
    rows = [(f, int(s)) for f, s in re.findall(r"Function (\S+):\s*\n\s*REG:\d+ STACK:(\d+)", usage) if "tv_kernels" in f]
    assert len(rows) == 10, rows  # five kernels, two flavours
    assert all(s == 0 for _, s in rows), rows
    sass = subprocess.run([tool, "-sass", so], capture_output=True, text=True, check=True).stdout
    cur, atomics = None, []
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
        elif cur and "tv_kernels" in cur and re.search(r"\b(ATOM|RED)[.A-Z0-9]*\s", line):
            atomics.append(cur)
    assert not atomics, atomics
