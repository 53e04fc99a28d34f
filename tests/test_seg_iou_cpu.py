"""CPU checks of stage 1's validation IoU: the oracle (seg_iou_oracle.py) against the reference's own iou_metric bit for bit, its
tie and empty-set behaviour, the command-line flags of `train.py stage1 --val_count` and tools/eval_condition.py, and the refusal
of CPU tensors by metrics.segmentation_iou."""
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import hrv_env
import seg_iou_oracle as orc
from hrviton_b200 import metrics, train_loop

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _inputs(b, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    seg = torch.randn(b, 13, h, w, generator=g) * 3
    cm = (torch.rand(b, 1, h, w, generator=g) > 0.3).float() * torch.rand(b, 1, h, w, generator=g)
    parse = F.one_hot(torch.randint(0, 13, (b, h, w), generator=g), 13).permute(0, 3, 1, 2).float()
    return seg, cm, parse


@pytest.mark.skipif(hrv_env.reference_dir() is None, reason="no reference copy (oracle/_ref)")
@pytest.mark.parametrize("b", [1, 3, 8])
def test_oracle_equals_reference_iou_metric(b):
    tc = hrv_env.load_reference_script("train_condition")
    seg, cm, parse = _inputs(b, 37, 29, b)
    # the reference's composition and soft-max (train_condition.py:352-358)
    cloth_mask = torch.ones_like(seg)
    cloth_mask[:, 3:4, :, :] = cm
    soft = F.softmax(seg * cloth_mask, dim=1)
    ref = tc.iou_metric(soft, parse)
    ours = orc.iou_metric(soft, parse)
    assert ref.dtype == torch.float32
    assert np.float32(ref.item()).view(np.uint32) == ours.view(np.uint32), (ref.item(), ours)
    assert torch.equal(orc.probabilities(seg, cm), soft)
    # and with an empty label plane and an all-predicted plane in the batch
    parse[0] = 0
    soft[-1] = 0
    soft[-1, 5] = 1
    ref = tc.iou_metric(soft, parse)
    assert np.float32(ref.item()).view(np.uint32) == orc.iou_metric(soft, parse).view(np.uint32)


def test_oracle_counts_and_ties():
    y = torch.zeros(1, 13, 2, 2)
    y[0, 0] = 0.5                      # exactly 0.5: not predicted
    y[0, 1, 0, 0] = 0.5000001
    lab = torch.zeros(1, 13, 2, 2)
    lab[0, 1, 0, 0] = 1
    lab[0, 2, 1, 1] = 1
    assert orc.counts(y[0], lab[0]) == (1, 2, 1)
    f = np.float32
    assert orc.iou_metric(y, lab) == (f(1) + f(1e-7)) / (f(3) - f(1) + f(1e-7)) / f(1)
    # two equal top logits, the rest 200 below (their exp underflows): p = 0.5 exactly, nothing predicted
    seg = torch.full((1, 13, 1, 1), -200.0)
    seg[0, 4] = seg[0, 7] = 0.0
    p = orc.probabilities(seg, torch.ones(1, 1, 1, 1))
    assert p[0, 4, 0, 0].item() == 0.5 and orc.counts(p[0], lab[0, :, :1, :1])[0] == 0


def test_segmentation_iou_refuses_cpu_and_other_compositions():
    seg, cm, parse = _inputs(1, 8, 6, 0)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        metrics.segmentation_iou(seg, cm, parse)
    with pytest.raises(ValueError, match="warp_grad"):
        metrics.segmentation_iou(seg, cm, parse, composition="detach")


def test_stage1_cli_takes_the_validation_flags(tmp_path, capsys):
    test_root = tmp_path / "test_tree"
    test_root.mkdir()
    opt = train_loop.parse_args("stage1", ["--dataroot", str(tmp_path), "--val_count", "500", "--test_dataroot", str(test_root),
                                           "--test_data_list", "val_pairs.txt"])
    assert (opt.val_count, opt.test_dataroot, opt.test_data_list) == (500, str(test_root), "val_pairs.txt")
    opt = train_loop.parse_args("stage1", ["--dataroot", str(tmp_path)])
    assert (opt.val_count, opt.test_dataroot, opt.test_data_list) == (None, "./data/", "test_pairs.txt")  # no validation by default
    for argv, match in ((["--val_count", "0"], "val_count"), (["--val_count", "-3"], "val_count"),
                        (["--val_count", "5", "--test_dataroot", str(tmp_path / "missing")], "does not exist")):
        with pytest.raises(SystemExit) as e:
            train_loop.parse_args("stage1", ["--dataroot", str(tmp_path)] + argv)
        assert e.value.code == 2
        assert match in capsys.readouterr().err


def test_train_run_needs_a_validator_for_val_count():
    class Trainer:
        tocg = D = None
        tensor_lr = False
    with pytest.raises(ValueError, match="validator"):
        train_loop.TrainRun("stage1", Trainer(), None, "unused", keep_step=2, val_count=1)


def test_eval_condition_refuses_bad_flags(tmp_path):
    script = os.path.join(ROOT, "tools", "eval_condition.py")
    for argv, match in (([], "tocg_checkpoint"), (["--tocg_checkpoint", str(tmp_path / "none.pth")], "does not exist"),
                        (["--tocg_checkpoint", script, "--dataroot", str(tmp_path), "-b", "0"], "-b")):
        r = subprocess.run([sys.executable, script] + argv, capture_output=True, text=True, timeout=300)
        assert r.returncode == 2 and match in r.stderr, r.stderr


@pytest.mark.skipif(not os.path.exists(os.path.join(ROOT, "hr-viton_b200", "libhrviton_sm100.so")) or shutil.which("cuobjdump") is None
                    and not os.path.exists("/usr/local/cuda/bin/cuobjdump"), reason="needs the built library and cuobjdump")
def test_seg_iou_kernels_use_no_local_memory():
    so = os.path.join(ROOT, "hr-viton_b200", "libhrviton_sm100.so")
    out = subprocess.run([shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump", "--dump-resource-usage", so], capture_output=True,
                         text=True, check=True).stdout
    import re
    rows = re.findall(r"Function (\S*seg_iou\S*):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", out)
    assert len(rows) == 4, rows  # count and finish kernels, both library flavours
    assert all(int(s) == 0 and int(l) == 0 for _, _, s, l in rows), rows
