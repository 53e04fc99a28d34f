"""CPU: the host half of the VITON-HD loader (hrviton_b200.data) — Pillow's resize tables through a numpy restatement of the device's
integer passes against PIL itself, the workers' agnostic bit plane against the reference's get_agnostic, the data-parallel sharding,
and the constructor's refusals."""
import json
import os
import types

import numpy as np
import pytest
from PIL import Image

import hrv_env
from hrviton_b200 import data, synth


def _pil(a, oh, ow, resample):
    return np.asarray(Image.fromarray(a).resize((ow, oh), resample))


def test_resize_tables_match_pil_random_sizes():
    rng = np.random.default_rng(0)
    for _ in range(200):
        h, w = (int(v) for v in rng.integers(2, 120, 2))
        oh, ow = (int(v) for v in rng.integers(1, 120, 2))
        for c in (1, 3):
            a = rng.integers(0, 256, (h, w, c) if c == 3 else (h, w), dtype=np.uint8)
            if (h, w) != (oh, ow):
                assert np.array_equal(data.resize_bilinear_np(a, oh, ow), _pil(a, oh, ow, Image.BILINEAR)), (h, w, oh, ow, c)
            if c == 1:
                assert np.array_equal(data.resize_nearest_np(a, oh, ow), _pil(a, oh, ow, Image.NEAREST)), (h, w, oh, ow)


@pytest.mark.parametrize("fine_width", [384, 192])
def test_resize_tables_match_transforms_at_vitonhd_sizes(fine_width):
    import torchvision.transforms as T
    rng = np.random.default_rng(fine_width)
    oh, ow = data.resized_size(1024, 768, fine_width)
    for c in (1, 3):
        a = rng.integers(0, 256, (1024, 768, c) if c == 3 else (1024, 768), dtype=np.uint8)
        want = np.asarray(T.Resize(fine_width, interpolation=T.InterpolationMode.BILINEAR)(Image.fromarray(a)))
        assert want.shape[:2] == (oh, ow)
        assert np.array_equal(data.resize_bilinear_np(a, oh, ow), want)
        if c == 1:
            want = np.asarray(T.Resize(fine_width, interpolation=T.InterpolationMode.NEAREST)(Image.fromarray(a)))
            assert np.array_equal(data.resize_nearest_np(a, oh, ow), want)


def test_regrouping_table():
    assert sorted(l for g in data.GROUPS for l in g) == list(range(20))  # every label in exactly one group
    for g, labels in enumerate(data.GROUPS):
        assert all(data.GROUP_OF[l] == g for l in labels)


@pytest.fixture(scope="module")
def tree(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("vitonhd"))
    synth.write_vitonhd(root, 6, seed=11)
    return root


def test_agnostic_bits_match_reference(tree):
    if hrv_env.reference_dir() is None:
        pytest.skip("no reference copy (oracle/_ref)")
    cp = hrv_env.load_reference_script("cp_dataset")
    opt = types.SimpleNamespace(dataroot=tree, datamode="train", data_list="pairs.txt", fine_height=1024, fine_width=768, semantic_nc=13)
    ref = cp.CPDataset(opt)
    ds = data.VitonHDDataset(tree, "train", "pairs.txt", 1024, 768, keys=("agnostic",))
    missing = 0
    base = os.path.join(tree, "train")
    for i, name in enumerate(ref.im_names):
        im = Image.open(os.path.join(base, "image", name))
        parse = Image.open(os.path.join(base, "image-parse-v3", name.replace(".jpg", ".png")))
        with open(os.path.join(base, "openpose_json", name.replace(".jpg", "_keypoints.json"))) as f:
            pose = np.array(json.load(f)["people"][0]["pose_keypoints_2d"]).reshape((-1, 3))[:, :2]
        missing += int(any(pose[j, 0] == 0 and pose[j, 1] == 0 for j in (3, 4, 6, 7)))
        want = np.asarray(ref.get_agnostic(im, parse, pose.copy()))
        bits = ds[i]["bits"]
        assert (bits & 1).any() and (bits & 2).any() and (bits & 4).any()
        got = data.agnostic_np(np.asarray(im), np.asarray(parse), bits)
        assert np.array_equal(got, want), name
    assert missing >= 2  # the tree exercises the skipped-keypoint branches


@pytest.mark.parametrize("world", [1, 2, 3, 4])
def test_sharding(world):
    n, b = 103, 4
    for epoch in range(3):
        shards = [data.shard_indices(n, b, epoch, seed=5, rank=r, world=world) for r in range(world)]
        assert len({len(s) for s in shards}) == 1 and len(shards[0]) % b == 0  # same number of full batches
        assert len(shards[0]) == n // (world * b) * b
        union = np.concatenate(shards)
        assert len(set(union.tolist())) == len(union)  # disjoint
        perm = np.random.default_rng([5, epoch]).permutation(n)
        assert sorted(union.tolist()) == sorted(perm[:len(union)].tolist())  # the prefix of the epoch's permutation
        again = [data.shard_indices(n, b, epoch, seed=5, rank=r, world=world) for r in range(world)]
        assert all(np.array_equal(x, y) for x, y in zip(shards, again))  # every rank derives the same permutation
    e0, e1 = (data.shard_indices(n, b, e, seed=5, rank=0, world=world) for e in (0, 1))
    assert not np.array_equal(e0, e1)  # a new order every epoch
    if world == 1:
        assert np.array_equal(e0, np.random.default_rng([5, 0]).permutation(n)[:len(e0)])
    assert np.array_equal(data.shard_indices(n, b, 7, shuffle=False, rank=0, world=1), np.arange(n // b * b))


def test_constructor_refuses_uncovered_input(tree, tmp_path):
    with pytest.raises(ValueError, match="fine_height"):
        data.VitonHDDataset(tree, "train", "pairs.txt", 255, 192)
    with pytest.raises(ValueError, match="fine_height"):
        data.VitonHDDataset(tree, "train", "pairs.txt", 1000, 768)
    root = str(tmp_path)
    names = synth.write_vitonhd(root, 2, seed=1)
    Image.open(os.path.join(root, "train", "image", names[0])).convert("L").save(os.path.join(root, "train", "image", names[0]))
    with pytest.raises(ValueError, match="mode L"):
        data.VitonHDDataset(root, "train", "pairs.txt", 256, 192)
    data.VitonHDDataset(root, "train", "pairs.txt", 256, 192, keys=("cloth", "cloth_mask"))  # the image is not read for these keys
