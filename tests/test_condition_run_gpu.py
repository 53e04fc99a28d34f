"""GPU: tools/test_condition.py and tools/norm_const.py (hrviton_b200.condition_run) end to end on a synthetic VITON-HD tree, against
the reference's own test_condition.test() and get_norm_const.get_const(), unchanged, on the drop-in modules over the same batches.

Both sides read the same tocg outputs (fp32 storage; the graph replay is bit-identical to the eager tocg the reference calls), so
every grid PNG must decode to exactly the reference's pixels.  The rejection scores differ in how the discriminator's input is built
(a fused kernel here, torch's soft-max there) and are held to test_rejection_cpu.score_bound, as the pipeline's own tests hold them."""
import contextlib
import io
import os
import sys
import types

import numpy as np
import pytest
import torch
from PIL import Image

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import hrv_env  # noqa: E402
import hrv_loader  # noqa: E402

hrv_loader.load()
from hrviton_b200 import condition_run, data, ops, synth  # noqa: E402
from test_rejection_cpu import TOL_L, reject_case, score_bound  # noqa: E402

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(hrv_env.reference_dir() is None, reason="no reference copy (oracle/_ref)")]
H, W = 256, 192


@pytest.fixture(scope="module")
def tree(tmp_path_factory):
    root = tmp_path_factory.mktemp("vitonhd")
    synth.write_vitonhd(str(root), 5, h=H, w=W, seed=31, datamode="test", pairs="test_pairs.txt")
    synth.write_vitonhd(str(root), 4, h=H, w=W, seed=32, datamode="train", pairs="train_pairs.txt")
    g, sd_t, sd_d, _, _, _ = reject_case()
    os.makedirs(root / "ckpt")
    torch.save(sd_t, str(root / "ckpt" / "tocg.pth"))
    torch.save(sd_d, str(root / "ckpt" / "D.pth"))
    return types.SimpleNamespace(root=root, M=float(g["M"]))


@pytest.fixture(autouse=True)
def _fp32():
    ops.set_precision("fp32")
    yield
    ops.set_precision("bf16")


class _CpuLoader:
    """cp_dataset.CPDataLoader's .data_loader and next_batch() over a VitonHDLoader's batches moved to the CPU."""

    def __init__(self, loader):
        self.batches = []
        for b in loader:
            self.batches.append({k: ({s: t.cpu() for s, t in v.items()} if isinstance(v, dict) and k != "c_name" else
                                     (v.cpu() if torch.is_tensor(v) else v)) for k, v in b.items()})
        loader.close()
        self.data_loader, self.i = self.batches, 0

    def next_batch(self):
        b = self.batches[self.i % len(self.batches)]
        self.i += 1
        return b


def _run_reference_test(tree, opt, tocg, D):
    keys = condition_run.GRID_KEYS + ("pose", "parse_onehot")
    cpu = _CpuLoader(data.VitonHDLoader(str(tree.root), "test", "test_pairs.txt", H, W, opt.batch_size, workers=0, mode="test", keys=keys,
                                        shuffle=False, shard=False))
    tcond = hrv_env.load_reference_script("test_condition")
    with contextlib.redirect_stdout(io.StringIO()):
        tcond.test(opt, cpu, None, tocg, D)


@pytest.mark.parametrize("composition,with_d", [("warp_grad", True), ("detach", False), ("no_composition", True)])
def test_tool_matches_reference_test_condition(tree, tmp_path, monkeypatch, composition, with_d):
    ckpt = "ckpt/tocg.pth"
    argv = ["--dataroot", str(tree.root), "--tocg_checkpoint", ckpt, "-b", "2", "-j", "0", "--clothmask_composition", composition,
            "--Ddownx2", "--Ddropout"]
    if with_d:
        argv += ["--D_checkpoint", "ckpt/D.pth", "--norm_const", repr(tree.M)]
    ours, ref = tmp_path / "ours", tmp_path / "ref"
    for d in (ours, ref):
        os.makedirs(d)
        os.symlink(tree.root / "ckpt", d / "ckpt")
    monkeypatch.chdir(ours)
    out = io.StringIO()
    with contextlib.redirect_stdout(out):
        condition_run.main(argv)
    text = out.getvalue()
    assert "1 of 5 pairs are left out" in text and "Test time" in text and "\n4\n" in text
    monkeypatch.chdir(ref)
    opt = condition_run.parse_args(argv)
    tocg, D = condition_run.build_models(opt, torch.device("cuda"), with_d)
    _run_reference_test(tree, opt, tocg, D)

    sub = os.path.join("output", "ckpt", "tocg.pth", "test", "paired", "multi-task")
    a, b = sorted(os.listdir(ours / sub)), sorted(os.listdir(ref / sub))
    assert a == b and len([f for f in a if f.endswith(".png")]) == 4
    for f in a:
        if f.endswith(".png"):
            x, y = (np.asarray(Image.open(str(d / sub / f))) for d in (ours, ref))
            assert x.shape == (3 * (H + 2) + 2, 4 * (W + 2) + 2, 3) and np.array_equal(x, y), f
    assert ("rejection_prob.txt" in a) == with_d
    if with_d:
        lines = [(ours / sub / "rejection_prob.txt").read_text().splitlines(), (ref / sub / "rejection_prob.txt").read_text().splitlines()]
        got, want = ([(n, float(s)) for n, s in (line.split() for line in ls)] for ls in lines)
        assert [s for _, s in got] == sorted((s for _, s in got), reverse=True)
        assert sorted(n for n, _ in got) == sorted(n for n, _ in want) and all(n.endswith(".png") for n, _ in got)
        want = dict(want)
        for n, s in got:
            l_ = s * tree.M / (1 + s * tree.M)
            assert abs(s - want[n]) <= score_bound(l_, tree.M), (n, s, want[n])


def test_norm_const_matches_get_const(tree, monkeypatch, tmp_path):
    monkeypatch.chdir(tmp_path)
    argv = ["--dataroot", str(tree.root), "--data_list", "train_pairs.txt", "--tocg_checkpoint", str(tree.root / "ckpt" / "tocg.pth"),
            "--D_checkpoint", str(tree.root / "ckpt" / "D.pth"), "-b", "2", "-j", "0", "--Ddownx2", "--Ddropout"]
    with contextlib.redirect_stdout(io.StringIO()) as out:
        M = condition_run.main_norm_const(argv)
    assert "M: %s" % M in out.getvalue()
    opt = condition_run.parse_norm_args(argv)
    tocg, D = condition_run.build_models(opt, torch.device("cuda"), True)
    keys = ("cloth", "cloth_mask", "parse_agnostic", "densepose", "pose", "parse_onehot", "parse", "pcm", "parse_cloth", "image")
    cpu = _CpuLoader(data.VitonHDLoader(str(tree.root), "train", "train_pairs.txt", H, W, 2, workers=0, mode="train", keys=keys, shuffle=False,
                                        shard=False))
    gnc = hrv_env.load_reference_script("get_norm_const")
    with contextlib.redirect_stdout(io.StringIO()):
        M_ref = gnc.get_const(opt, cpu, tocg, D, 4)
    print("NORM_CONST tool %.6f reference %.6f" % (M, M_ref))
    assert abs(M - M_ref) <= TOL_L * (1 + M) ** 2, (M, M_ref)
