"""GPU: png.encode against its numpy statement (byte for byte), the decoded pixels against the input, repeated calls against each
other; png.condition_grid against condition_grid_np for every cloth-mask composition."""
import io
import os
import sys

import numpy as np
import pytest
import torch
from PIL import Image

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import hrv_loader  # noqa: E402

hrv_loader.load()
from hrviton_b200 import png  # noqa: E402
from test_png_cpu import grid_fixture, grid_tensors, smooth  # noqa: E402

pytestmark = pytest.mark.gpu


def mixed(n, h, w, seed=0):
    """A batch of smooth, noisy, flat and half-noise images."""
    g = np.random.default_rng(seed)
    out = []
    for i in range(n):
        k = i % 4
        if k == 0:
            a = smooth(h, w, seed=seed + i)
        elif k == 1:
            a = g.integers(0, 256, (h, w, 3), dtype=np.uint8)
        elif k == 2:
            a = np.full((h, w, 3), g.integers(0, 256), np.uint8)
        else:
            a = smooth(h, w, seed=seed + i, noise=0)
            a[: h // 2] = g.integers(0, 256, (h // 2, w, 3), dtype=np.uint8)
        out.append(a)
    return np.stack(out)


def check(batch):
    got = png.encode(torch.from_numpy(batch).cuda())
    want = png.encode_np(batch)
    assert len(got) == len(batch)
    for i, (b, a) in enumerate(zip(got, batch)):
        assert b == want[i], (batch.shape, i, len(b), len(want[i]))
        assert np.array_equal(np.asarray(Image.open(io.BytesIO(b))), a)
    return got


@pytest.mark.parametrize("shape", [(1, 1, 1), (3, 1, 300), (3, 300, 1), (4, 7, 13), (2, 65, 333), (8, 778, 776)])
def test_encode_equals_numpy_statement(shape):
    n, h, w = shape
    batch = mixed(n, h, w, seed=h * 7 + w)
    first = check(batch)
    assert png.encode(torch.from_numpy(batch).cuda()) == first


def test_encode_grids_and_large_images():
    g = grid_fixture()
    check(np.stack([g, g[::-1].copy(), np.ascontiguousarray(g[:, ::-1])]))
    big = np.stack([np.kron(smooth(386, 386, seed=s), np.ones((8, 8, 1), np.uint8))[:3082, :3080] for s in (1, 2)])
    big[1, 1000:1100] = np.random.default_rng(0).integers(0, 256, (100, 3080, 3), dtype=np.uint8)
    check(big)


def test_encode_refuses_host_and_bad_tensors():
    with pytest.raises(ValueError):
        png.encode(torch.zeros(1, 4, 4, 3, dtype=torch.uint8))
    with pytest.raises(ValueError):
        png.encode(torch.zeros(1, 4, 4, 3, device="cuda"))


@pytest.mark.parametrize("composition", ["warp_grad", "detach", "no_composition"])
@pytest.mark.parametrize("n,h,w", [(2, 16, 12), (3, 256, 192), (1, 5, 3)])
def test_condition_grid_equals_restatement(composition, n, h, w):
    t = grid_tensors(n, h, w, seed=n + h)
    got = png.condition_grid({k: v.cuda() for k, v in t.items()}, composition).cpu().numpy()
    want = png.condition_grid_np({k: v.numpy() for k, v in t.items()}, composition)
    assert got.shape == want.shape == png.grid_shape(n, h, w)
    assert np.array_equal(got, want)


def test_condition_grid_refuses_bad_inputs():
    t = {k: v.cuda() for k, v in grid_tensors().items()}
    with pytest.raises(ValueError):
        png.condition_grid(t, "other")
    with pytest.raises(ValueError):
        png.condition_grid(dict(t, pcm=t["pcm"].double()))
    with pytest.raises(KeyError):
        png.condition_grid({k: v for k, v in t.items() if k != "image"})
