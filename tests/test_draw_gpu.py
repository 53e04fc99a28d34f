"""GPU: the device rasteriser (hrviton_b200.draw, csrc/draw_kernels.cu) against data.agnostic_bits, the golden get_parse_agnostic
fixture and the numpy restatement; VitonHDLoader's batches with the shapes drawn on the device against ImageDraw's in the workers;
tools/parse_agnostic.py against PIL's save of the restated labels; and the refusals."""
import json
import os
import sys
from multiprocessing import Pool

import numpy as np
import pytest
import torch
from PIL import Image

from hrviton_b200 import data, draw, synth

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import draw_oracle as O  # noqa: E402

pytestmark = pytest.mark.gpu


def _cpu_bits(pose):
    with np.errstate(all="ignore"):
        return data.agnostic_bits(pose, data.ARM_CANVAS)


def test_agnostic_bits_match_imagedraw():
    rng = np.random.default_rng(21)
    poses = np.stack([O.random_pose(rng) for _ in range(2048)])
    with Pool(min(16, os.cpu_count() or 1)) as pool:
        want = np.stack(pool.map(_cpu_bits, list(poses), chunksize=16))
    got = torch.cat([draw.agnostic_bits(torch.from_numpy(poses[i:i + 256]).cuda()) for i in range(0, len(poses), 256)]).cpu().numpy()
    bad = [i for i in range(len(poses)) if not np.array_equal(got[i], want[i])]
    assert not bad, (len(bad), poses[bad[0]].tolist())


def test_parse_agnostic_matches_golden_and_restatement(golden_dir):
    g = np.load(os.path.join(golden_dir, "parse_agnostic_512x384_b6.npz"))
    got = draw.parse_agnostic(torch.from_numpy(g["labels"]).cuda(), torch.from_numpy(g["keypoints"]).cuda()).cpu().numpy()
    assert np.array_equal(got, g["result"])
    rng = np.random.default_rng(22)
    kp = np.stack([O.random_pose(rng) for _ in range(8)])
    lab = rng.choice(np.array([0, 5, 6, 7, 10, 14, 15, 3], np.uint8), (8, 1024, 768))
    got = draw.parse_agnostic(torch.from_numpy(lab).cuda(), torch.from_numpy(kp).cuda()).cpu().numpy()
    for i in range(8):
        assert np.array_equal(got[i], O.parse_agnostic(lab[i], kp[i])), i


@pytest.fixture(scope="module")
def tree(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("vitonhd_draw"))
    synth.write_vitonhd(root, 8, seed=23)
    synth.write_vitonhd(root, 8, seed=24, datamode="test", pairs="test_pairs.txt")
    return root


@pytest.mark.parametrize("mode", ["train", "test"])
def test_loader_batches_unchanged(tree, mode):
    keys = data.TRAIN_KEYS if mode == "train" else None
    pairs = "pairs.txt" if mode == "train" else "test_pairs.txt"
    batches = {}
    for flag in (False, True):
        ld = data.VitonHDLoader(tree, mode, pairs, 1024, 768, 4, workers=2, mode=mode, keys=keys, shuffle=False, device_agnostic=flag)
        batches[flag] = [b for b in ld]
        ld.close()
    assert len(batches[True]) == len(batches[False]) == 2
    for a, b in zip(batches[False], batches[True]):
        assert a.keys() == b.keys()
        for k, v in a.items():
            if isinstance(v, dict):
                for s in v:
                    assert (torch.equal(v[s], b[k][s]) if torch.is_tensor(v[s]) else v[s] == b[k][s]), (k, s)
            else:
                assert (torch.equal(v, b[k]) if torch.is_tensor(v) else v == b[k]), k


def test_tool_writes_the_reference_files(tree, tmp_path):
    sys.path.insert(0, os.path.join(os.path.dirname(HERE), "tools"))
    import parse_agnostic as tool
    base = os.path.join(tree, "train")
    names = sorted(os.listdir(os.path.join(base, "image")))
    with open(os.path.join(base, "openpose_json", names[1].replace(".jpg", "_keypoints.json")), "w") as f:
        json.dump({"people": []}, f)  # the reference skips this sample (IndexError)
    out = str(tmp_path / "out")
    written, skipped = tool.run(base, out, batch_size=3, workers=2)
    assert skipped == [names[1]] and sorted(written) == sorted(n for n in names if n != names[1])
    assert sorted(os.listdir(out)) == sorted(n.replace(".jpg", ".png") for n in written)
    for name in written:
        png = name.replace(".jpg", ".png")
        src = os.path.join(base, "image-parse-v3", png)
        with open(os.path.join(base, "openpose_json", name.replace(".jpg", "_keypoints.json"))) as f:
            pose = np.array(json.load(f)["people"][0]["pose_keypoints_2d"]).reshape((-1, 3))[:, :2]
        want = str(tmp_path / "want.png")
        tool.write_png(src, O.parse_agnostic(np.asarray(Image.open(src)), pose), want)
        with open(want, "rb") as a, open(os.path.join(out, png), "rb") as b:
            assert a.read() == b.read(), name


def test_bad_input_refused():
    kp = torch.zeros((2, 25, 2), dtype=torch.float64, device="cuda")
    lab = torch.zeros((2, 64, 48), dtype=torch.uint8, device="cuda")
    with pytest.raises(ValueError, match=r"\(N, 25, 2\)"):
        draw.agnostic_bits(torch.zeros((2, 18, 2), dtype=torch.float64, device="cuda"))
    with pytest.raises(ValueError, match="fp64"):
        draw.agnostic_bits(kp.float())
    with pytest.raises(ValueError, match="CUDA"):
        draw.agnostic_bits(kp.cpu())
    with pytest.raises(ValueError, match="3 samples"):
        draw.parse_agnostic(torch.zeros((3, 64, 48), dtype=torch.uint8, device="cuda"), kp)
    with pytest.raises(ValueError, match="CUDA uint8"):
        draw.parse_agnostic(lab.cpu(), kp)
    with pytest.raises(ValueError, match="CUDA"):
        draw.parse_agnostic(lab, kp.cpu())
