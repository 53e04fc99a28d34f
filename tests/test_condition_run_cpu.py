"""CPU: the host logic of tools/test_condition.py and tools/norm_const.py (hrviton_b200.condition_run): flags and refusals, the
output path and file names, and rejection_prob.txt's format, order and append."""
import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import hrv_loader  # noqa: E402

hrv_loader.load()
from hrviton_b200 import condition_run  # noqa: E402


@pytest.fixture
def tree(tmp_path):
    for f in ("tocg.pth", "D.pth"):
        (tmp_path / f).write_bytes(b"")
    return tmp_path


def args(tree, *extra):
    return ["--dataroot", str(tree), "--tocg_checkpoint", str(tree / "tocg.pth")] + list(extra)


def test_defaults_are_the_reference_ones(tree):
    opt = condition_run.parse_args(args(tree))
    assert (opt.batch_size, opt.datamode, opt.data_list, opt.datasetting, opt.fine_height, opt.fine_width) == (8, "test", "test_pairs.txt", "paired", 256, 192)
    assert (opt.clothmask_composition, opt.num_D, opt.norm_const, opt.D_checkpoint) == ("warp_grad", 2, None, "")
    opt = condition_run.parse_norm_args(args(tree, "--D_checkpoint", str(tree / "D.pth")))
    assert (opt.datamode, opt.data_list, opt.batch_size) == ("train", "train_pairs_zalando.txt", 8)


def test_accepts_flags_the_run_does_not_read(tree):
    opt = condition_run.parse_args(args(tree, "--occlusion", "--tensorboard_dir", "tb", "--shuffle", "--gpu_ids", "0", "--Ddownx2", "--Ddropout",
                                        "--spectral", "--num_D", "3", "-b", "2", "--fp16"))
    assert opt.occlusion and opt.Ddownx2 and opt.num_D == 3 and opt.batch_size == 2 and opt.fp16


@pytest.mark.parametrize("extra", [["--warp_feature", "encoder"], ["--out_layer", "conv"], ["--upsample", "nearest"], ["--semantic_nc", "7"],
                                   ["--output_nc", "7"], ["-b", "0"], ["--fine_height", "250"], ["--clothmask_composition", "other"],
                                   ["--D_checkpoint", "D.pth"], ["--norm_const", "0"], ["--no_such_flag"]])
def test_refusals(tree, extra, capsys):
    extra = [str(tree / e) if e == "D.pth" else e for e in extra]
    with pytest.raises(SystemExit):
        condition_run.parse_args(args(tree, *extra))


def test_refuses_missing_files(tree):
    with pytest.raises(SystemExit):
        condition_run.parse_args(["--dataroot", str(tree), "--tocg_checkpoint", str(tree / "none.pth")])
    with pytest.raises(SystemExit):
        condition_run.parse_args(args(tree, "--D_checkpoint", str(tree / "none.pth"), "--norm_const", "1.5"))
    with pytest.raises(SystemExit):
        condition_run.parse_norm_args(args(tree))  # get_norm_const needs a discriminator
    condition_run.parse_args(args(tree, "--D_checkpoint", str(tree / "D.pth"), "--norm_const", "1.5"))


def test_output_dir_and_names(tree):
    opt = condition_run.parse_args(args(tree, "--datasetting", "unpaired"))
    opt.tocg_checkpoint = "checkpoints/run1/tocg_step_1000.pth"
    assert condition_run.output_dir(opt) == os.path.join("./output", "run1", "tocg_step_1000.pth", "test", "unpaired", "multi-task")
    opt.tocg_checkpoint = "tocg.pth"
    with pytest.raises(ValueError):
        condition_run.output_dir(opt)
    c_name = {"paired": ["00001_00.jpg", "a.b.jpg"], "unpaired": ["00002_00.jpg", "c.jpg"]}
    assert [condition_run.grid_name(c_name, i) for i in range(2)] == ["00001_00_00002_00.png", "a_c.png"]


def test_rejection_file_is_sorted_descending_stable_and_appended(tmp_path):
    path = tmp_path / "rejection_prob.txt"
    scored = [("a.png", 0.5), ("b.png", 1.25), ("c.png", 0.5), ("d.png", 0.1000000014901161)]
    condition_run.write_rejection(str(path), scored)
    assert path.read_text() == "b.png 1.25\na.png 0.5\nc.png 0.5\nd.png 0.1000000014901161\n"
    condition_run.write_rejection(str(path), [("e.png", 2.0)])
    assert path.read_text().splitlines()[-1] == "e.png 2.0" and len(path.read_text().splitlines()) == 5
