"""GPU: stage-1 validation in the training driver (TrainRun.validate, `train.py stage1 --val_count`) and tools/eval_condition.py.

On a synthetic 256x192 tree, runs in fresh processes (as test_train_loop_gpu.py runs them), every one starting from a seeded tocg
checkpoint whose segmentation predicts classes, so the IoU moves with the weights (a fresh initialisation predicts no class above 0.5
and scores the same constant at every step, which no check below could tell from a stale graph or wrong batches):
- a run validating every step logs, at each step, np.mean of the oracle IoUs (seg_iou_oracle) of the eager eval tocg over the same
  test batches;
- its parameters, BatchNorm statistics, Adam state and losses equal those of a run that does not validate, bit for bit;
- a run resumed from its state file ends in the same state and logs the same IoU at every validation after the resume;
- tools/train.py stage1 --val_count 2 prints those IoUs, and tools/eval_condition.py on the final tocg prints the last one."""
import os
import re
import subprocess
import sys

import numpy as np
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
N_TRAIN, N_TEST, BATCH, STEPS = 6, 7, 2, 4  # 7 test samples: 3 full batches of 2, the last sample dropped
LOGIT_GAIN = 8.0  # the seeded out_layer's scores times this: soft-max maxima above 0.5 at most pixels, not all


def _env():
    env = dict(os.environ, HRV_VGG_RANDOM_INIT="1", CUBLAS_WORKSPACE_CONFIG=":4096:8", PYTHONPATH=os.pathsep.join([ROOT, HERE]))
    env.pop("WORLD_SIZE", None)
    return env


@pytest.fixture(scope="module")
def tree(tmp_path_factory):
    import networks
    from helpers import tocg_opt
    from hrviton_b200 import synth
    root = tmp_path_factory.mktemp("trainval")
    synth.write_vitonhd(str(root), N_TRAIN, seed=41, datamode="train")
    synth.write_vitonhd(str(root), N_TEST, seed=42, datamode="test", pairs="test_pairs.txt")
    tocg = networks.ConditionGenerator(tocg_opt(), 4, 16, 13, ngf=96, norm_layer=torch.nn.BatchNorm2d)
    sd = tocg.state_dict()
    synth.fill_state_dict(sd, 3)
    # out_layer is relu(scale(x) + bn(conv(.))): scaling the 1x1 scale conv and the last BatchNorm's affine scales every score
    for k in ("out_layer.scale.weight", "out_layer.scale.bias", "out_layer.block.4.weight", "out_layer.block.4.bias"):
        sd[k].mul_(LOGIT_GAIN)
    torch.save(sd, str(root / "tocg.pth"))
    return root


def _flags(tree, name, extra=()):
    return ["--name", name, "--dataroot", str(tree), "--data_list", "pairs.txt", "-b", str(BATCH), "-j", "1", "--checkpoint_dir",
            str(tree / "ckpt"), "--display_count", "1000", "--occlusion", "--seed", "3", "--keep_step", str(STEPS), "--save_count", "2",
            "--test_dataroot", str(tree), "--test_data_list", "test_pairs.txt", "--tocg_checkpoint", str(tree / "tocg.pth")] + list(extra)


def _launch(tree, out, flags, oracle=False):
    env = _env()
    if oracle:
        env["HRV_VAL_ORACLE"] = "1"
    r = subprocess.run([sys.executable, os.path.abspath(__file__), str(out)] + flags, cwd=str(tree), env=env, capture_output=True,
                       text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-6000:]
    return torch.load(str(out), weights_only=False)


def _final_state(ckpt):
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


def test_validation_is_the_oracle_iou_and_changes_nothing(tree):
    val = _launch(tree, tree / "val.pt", _flags(tree, "val", ["--val_count", "1"]), oracle=True)
    plain = _launch(tree, tree / "plain.pt", _flags(tree, "plain"))
    assert [s for s, _ in val["iou"]] == list(range(1, STEPS + 1)) and plain["iou"] == []
    assert [o[0] for o in val["oracle"]] == list(range(1, STEPS + 1))
    for (s, v), o in zip(val["iou"], val["oracle"]):
        assert v == o[1], (s, v, o)
    # the oracle predicted classes at every validation, on some but not all pixels, and the value moved at every step: a graph that
    # replays stale weights, other samples or another batch count would log other values
    pixels = (N_TEST // BATCH * BATCH) * 256 * 192
    assert all(0 < o[2] < pixels for o in val["oracle"]), val["oracle"]
    assert len({v for _, v in val["iou"]}) == STEPS and all(0.0 < v < 1.0 for _, v in val["iou"]), val["iou"]
    assert ["step: %8d, IoU: %.6f" % (s, v) for s, v in val["iou"]] == [l for l in val["log"] if "IoU" in l]
    assert sorted(val["losses"]) == sorted(plain["losses"]) == list(range(1, STEPS + 1))
    for s in val["losses"]:
        _assert_same(val["losses"][s], plain["losses"][s])
    a, b = (_final_state(str(tree / "ckpt" / n)) for n in ("val", "plain"))
    assert any("running_mean" in n for n in a) and any(".exp_avg_sq" in n for n in a)
    _assert_same(a, b)

    # resumed from the state file of step 2: the same IoUs at steps 3 and 4 and the same final state
    state = str(tree / "ckpt" / "val" / "state_step_000002.pth")
    res = _launch(tree, tree / "res.pt", _flags(tree, "res", ["--val_count", "1", "--resume", state]))
    assert res["iou"] == val["iou"][2:]
    _assert_same(a, _final_state(str(tree / "ckpt" / "res")))

    # the command-line tools: train.py prints the IoU every 2 steps; eval_condition.py scores the final tocg as the last validation did
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "train.py"), "stage1"] + _flags(tree, "cli", ["--val_count", "2"]),
                       cwd=str(tree), env=_env(), capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-6000:]
    printed = re.findall(r"step: +(\d+), IoU: ([0-9.]+)", r.stdout)
    assert printed == [(str(s), "%.6f" % v) for s, v in val["iou"] if s % 2 == 0], (printed, val["iou"])
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "eval_condition.py"), "--tocg_checkpoint",
                        str(tree / "ckpt" / "cli" / "tocg_final.pth"), "--dataroot", str(tree), "--data_list", "test_pairs.txt", "-b",
                        str(BATCH), "-j", "1"], cwd=str(tree), env=_env(), capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-6000:]
    assert ("IoU: %.6f  (%d samples" % (val["iou"][-1][1], N_TEST // BATCH * BATCH)) in r.stdout, r.stdout


# ------------------------------------------------------------------------------------------------ the subprocess side

def _oracle_iou(run, loader):
    """np.mean over the validation batches of seg_iou_oracle on the eager eval-mode tocg (torch's soft-max on the device), and the
    number of predicted (pixel, class) pairs over those batches."""
    import seg_iou_oracle as orc
    tocg = run.trainer.tocg
    tocg.eval()
    vals, predicted = [], 0
    loader.start_at(0, 0)
    with torch.no_grad():
        for _ in range(min(run.val_samples, len(loader.dataset)) // loader.batch_size):
            b = loader.next_batch()
            input1 = torch.cat([b["cloth"]["paired"], (b["cloth_mask"]["paired"] > 0.5).float()], 1)
            input2 = torch.cat([b["parse_agnostic"], b["densepose"]], 1)
            _, seg, _, wcm = tocg(input1, input2)
            vals.append(float(orc.segmentation_iou(seg, wcm, b["parse"])))
            predicted += int((orc.probabilities(seg, wcm) > 0.5).sum())
    tocg.train()
    return float(np.mean(vals)), predicted


def _worker(out, argv):
    from hrviton_b200 import data, train_loop
    opt = train_loop.parse_args("stage1", argv)
    log = []
    run = train_loop.build(opt, log=log.append)
    losses, oracle = {}, []
    ref_loader = None
    if os.environ.get("HRV_VAL_ORACLE") == "1":
        ref_loader = data.VitonHDLoader(opt.test_dataroot, "test", opt.test_data_list, opt.fine_height, opt.fine_width, opt.batch_size,
                                        workers=0, mode="test", keys=train_loop.VAL_KEYS, shuffle=False, shard=False)

    def on_step(step, l):  # called before the step's validation, on the same weights
        losses[step] = {k: v.detach().clone() for k, v in l.items() if torch.is_tensor(v)}
        if ref_loader is not None and run.val_count and step % run.val_count == 0:
            oracle.append((step,) + _oracle_iou(run, ref_loader))
    run.on_step = on_step
    try:
        run.start().train()
        torch.cuda.synchronize()
    finally:
        run.trainer.release_graph()
        if run._seg is not None:
            run._seg.release()
    torch.save({"losses": {s: {k: v.cpu() for k, v in l.items()} for s, l in losses.items()}, "iou": run.iou, "oracle": oracle,
                "log": log}, out)


if __name__ == "__main__":
    _worker(sys.argv[1], sys.argv[2:])
