"""CPU: pytorch-fid's FID Inception weights and statistics (hrviton_b200.metrics.fid_inception_model, FeatureStats.save_npz /
load_npz), the refusals of tools/fid.py, and the float64 oracle (tests/fid_inception_oracle.py): its pooling changes are large enough
for the GPU parity bound to tell the FID network from torchvision's."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import fid_inception_oracle as fo
import inception_oracle as io_
from hrviton_b200 import metrics

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOOL = os.path.join(ROOT, "tools", "fid.py")


@pytest.fixture(scope="module")
def fid_sd():
    return fo.seeded_fid_state_dict(seed=4)


def test_fid_weights_key_set(fid_sd):
    from torchvision.models.inception import Inception3
    ref = Inception3(num_classes=1008, aux_logits=False, init_weights=False).state_dict()
    assert set(fid_sd) == {k for k in ref if not k.endswith("num_batches_tracked")}
    assert fid_sd["fc.weight"].shape == (1008, 2048)
    m = metrics.fid_inception_model(fid_sd)  # no num_batches_tracked: accepted
    assert not m.training and m.fc.out_features == 1008
    assert all(torch.equal(v, fid_sd[k]) for k, v in m.state_dict().items() if k in fid_sd)
    metrics.fid_inception_model(m.state_dict())  # with them: accepted too


def test_fid_weights_rejections(fid_sd, tmp_path):
    missing = dict(fid_sd)
    del missing["Mixed_6c.branch7x7_2.bn.running_var"]
    with pytest.raises(ValueError, match="Mixed_6c.branch7x7_2.bn.running_var"):
        metrics.fid_inception_model(missing)
    extra = dict(fid_sd, **{"AuxLogits.fc.weight": torch.zeros(1000, 768)})
    with pytest.raises(ValueError, match="AuxLogits.fc.weight"):
        metrics.fid_inception_model(extra)
    shaped = dict(fid_sd, **{"fc.bias": torch.zeros(1000)})  # torchvision's ImageNet head
    with pytest.raises(ValueError, match="fc.bias"):
        metrics.fid_inception_model(shaped)
    with pytest.raises(FileNotFoundError):
        metrics.fid_inception_model(str(tmp_path / "pt_inception-2015-12-05-6726825d.pth"))
    path = tmp_path / "w.pth"
    torch.save(fid_sd, str(path))
    assert torch.equal(metrics.fid_inception_model(str(path)).fc.bias, fid_sd["fc.bias"])
    with pytest.raises(RuntimeError):
        metrics.InceptionV3.from_fid_weights(fid_sd, device="cpu")


def _cpu_stats(feats):
    """A FeatureStats holding CPU sums (mean / cov / save_npz are plain torch arithmetic; update needs the GPU)."""
    st = object.__new__(metrics.FeatureStats)
    f = torch.from_numpy(feats)
    st.dim, st.n, st.sum, st.sum_sq = f.shape[1], f.shape[0], f.sum(0), f.T @ f
    return st


def test_npz_round_trip(tmp_path):
    rng = np.random.RandomState(3)
    fa, fb = np.abs(rng.randn(40, 16)), np.abs(rng.randn(30, 16)) * 1.1
    sa, sb = _cpu_stats(fa), _cpu_stats(fb)
    path = str(tmp_path / "a.npz")
    sa.save_npz(path)
    with np.load(path) as f:  # pytorch-fid's format
        assert sorted(f.keys()) == ["mu", "sigma"] and f["mu"].dtype == np.float64 and f["sigma"].dtype == np.float64
        assert np.abs(f["sigma"] - np.cov(fa, rowvar=False)).max() <= 1e-12 * np.abs(f["sigma"]).max()  # np.cov's N - 1
        assert np.abs(f["mu"] - fa.mean(0)).max() <= 1e-14 * np.abs(fa).max()
    mu, sigma = metrics.FeatureStats.load_npz(path)
    assert np.array_equal(mu, sa.mean().numpy()) and np.array_equal(sigma, sa.cov().numpy())
    # the FID of the loaded statistics equals the FID of the same statistics passed directly
    mm = lambda a, b: a @ b.T  # noqa: E731
    direct = metrics.fid_from_moments(sa.mean(), sa.cov(), sb.mean(), sb.cov(), mm)
    loaded = metrics.fid_from_moments(torch.from_numpy(mu), torch.from_numpy(sigma), sb.mean(), sb.cov(), mm)
    assert float(direct) == float(loaded) and float(direct) > 0
    np.savez_compressed(str(tmp_path / "bad.npz"), mean=mu)
    with pytest.raises(ValueError):
        metrics.FeatureStats.load_npz(str(tmp_path / "bad.npz"))
    with pytest.raises(RuntimeError):
        metrics.fid_of_moments((mu, sigma), (mu, sigma), device="cpu")


def _tool(*args):
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    return subprocess.run([sys.executable, TOOL] + list(args), capture_output=True, text=True, timeout=300, env=env)


def _png_folder(path, n, size=(8, 6)):
    from PIL import Image
    path.mkdir()
    rng = np.random.RandomState(n)
    for i in range(n):
        Image.fromarray(rng.randint(0, 256, (size[0], size[1], 3)).astype(np.uint8)).save(str(path / ("%03d.png" % i)))
    return str(path)


def test_tool_refusals(tmp_path):
    a = _png_folder(tmp_path / "a", 3)
    b = _png_folder(tmp_path / "b", 2)
    r = _tool(a, b, "--weights", str(tmp_path / "none.pth"))
    assert r.returncode != 0 and "weights file not found" in r.stderr, r.stderr
    weights = tmp_path / "w.pth"
    weights.write_bytes(b"")  # existence is checked first; nothing below reaches the weights
    empty = tmp_path / "empty"
    empty.mkdir()
    (empty / "notes.txt").write_text("not an image")
    (empty / "upper.PNG").write_bytes(b"")  # pytorch-fid's extensions are lower-case
    r = _tool(a, str(empty), "--weights", str(weights))
    assert r.returncode != 0 and "holds no images" in r.stderr, r.stderr
    r = _tool(a, b, "--weights", str(weights), "--kid")
    assert r.returncode != 0 and "at least 1000 images" in r.stderr, r.stderr
    np.savez_compressed(str(tmp_path / "s.npz"), mu=np.zeros(4), sigma=np.eye(4))
    r = _tool(a, str(tmp_path / "s.npz"), "--weights", str(weights), "--kid")
    assert r.returncode != 0 and "two image folders" in r.stderr, r.stderr
    r = _tool(str(tmp_path / "s.npz"), a, "--weights", str(weights), "--save-stats", str(tmp_path / "o.npz"))
    assert r.returncode != 0 and "needs A to be an image folder" in r.stderr, r.stderr
    r = _tool(a, str(tmp_path / "missing"), "--weights", str(weights))
    assert r.returncode != 0 and "neither an image folder" in r.stderr, r.stderr


def test_image_files_order(tmp_path):
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    try:
        import fid as fid_tool
    finally:
        sys.path.pop(0)
    for name in ("b.jpg", "a.png", "c.JPG", "d.webp", "e.txt", "a.jpeg"):
        (tmp_path / name).write_bytes(b"")
    (tmp_path / "sub.png").mkdir()
    assert [os.path.basename(f) for f in fid_tool.image_files(str(tmp_path))] == ["a.jpeg", "a.png", "b.jpg", "d.webp"]


def test_oracle_pooling_changes_matter(fid_sd):
    """The same weights with pytorch-fid's pooling and with torchvision's differ at Mixed_5d and Mixed_7c by far more than the GPU
    parity bound (1e-4 max|ref|): that bound tells the two networks apart."""
    g = torch.Generator().manual_seed(8)
    x = torch.rand((1, 3, 150, 120), generator=g)
    taps_f, pool_f, logits_f = fo.fp64_forward(fo.fid_network(fid_sd, pooling="fid"), x)
    taps_t, _, _ = fo.fp64_forward(fo.fid_network(fid_sd, pooling="torchvision"), x)
    assert pool_f.shape == (1, 2048) and logits_f.shape == (1, 1008)
    for name in ("Mixed_5d", "Mixed_7c"):
        assert float(taps_f[name].abs().max()) > 0.1  # alive
        r = float((taps_t[name] - taps_f[name]).abs().max() / taps_f[name].abs().max())
        print("PARITY fid_oracle[%s] torchvision pooling vs pytorch-fid pooling max|d|/max|ref| = %.3e (GPU bound 1e-4)" % (name, r))
        assert r > 100 * 1e-4, (name, r)
    assert io_.TAPS == fo.TAPS
