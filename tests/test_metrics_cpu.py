"""CPU: the evaluation metrics' boundary — the drop-in eval_models' state_dict keys and shapes against the live reference's
(tests/golden/lpips_keys.json), the float64 SSIM restatement that the GPU test holds hrv_ssim to, checked against
scipy.ndimage.gaussian_filter (skimage's own filter) and shown to be independent of the border mode, and the refusals: the skimage
shim outside evaluate.py's argument set, PerceptualLoss without alex.pth, with unsupported options or with gradients.

Parity with skimage.metrics.structural_similarity itself is not pinned: skimage is not installed here.  The restatement follows its
documented algorithm for these arguments (Gaussian moments through scipy.ndimage, cov_norm 1, crop of (win_size-1)//2 = 5)."""
import json
import os
import sys

import numpy as np
import pytest
import scipy.ndimage as ndi
import torch

from helpers import GOLDEN
import metrics_oracle as mo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _images(seed, h=61, w=47):
    rng = np.random.RandomState(seed)
    a = rng.randint(0, 256, (h, w)).astype(np.uint8)
    a[:20, :20] = 255               # saturated
    a[-15:, -10:] = 37              # flat
    b = np.clip(a.astype(np.int32) + rng.randint(-30, 31, (h, w)), 0, 255).astype(np.uint8)
    return a, b


def test_drop_in_state_dict_keys_match_reference():
    import eval_models  # noqa: F401  (the drop-in binds first: the repo root leads sys.path)
    from hrviton_b200 import metrics
    assert os.path.dirname(eval_models.__file__) == os.path.join(ROOT, "eval_models")
    ref = json.load(open(os.path.join(GOLDEN, "lpips_keys.json")))
    mine = [[k, list(v.shape)] for k, v in metrics.PNetLin(pretrained=False).state_dict().items()]
    assert mine == ref


def test_restatement_matches_scipy_gaussian_filter():
    a, b = _images(1)
    x, y = a.astype(np.float64), b.astype(np.float64)
    for t in (x, y, x * x, y * y, x * y):
        ours = mo.moments_valid(t)
        ref = ndi.gaussian_filter(t, sigma=1.5, truncate=3.5, mode="reflect")[5:-5, 5:-5]
        assert ours.shape == ref.shape
        np.testing.assert_allclose(ours, ref, rtol=0, atol=1e-10 * max(1.0, float(np.abs(ref).max())))


def test_cropped_mean_ignores_the_border_mode():
    a, b = _images(2)
    x, y = a.astype(np.float64), b.astype(np.float64)
    means = {}
    for mode in ("reflect", "constant", "nearest"):
        m = [ndi.gaussian_filter(t, sigma=1.5, truncate=3.5, mode=mode) for t in (x, y, x * x, y * y, x * y)]
        means[mode] = mo.ssim_map(*m)[5:-5, 5:-5].mean(dtype=np.float64)
    assert means["reflect"] == means["constant"] == means["nearest"]
    assert abs(means["reflect"] - mo.ssim(a, b)) < 1e-12
    assert mo.ssim(a, a) == pytest.approx(1.0, abs=1e-14)


def test_small_images_are_refused():
    from hrviton_b200 import ops
    with pytest.raises(ValueError, match="win_size"):
        ops.ssim(torch.zeros(1, 10, 40, dtype=torch.uint8), torch.zeros(1, 10, 40, dtype=torch.uint8))
    with pytest.raises(ValueError, match="win_size"):
        mo.ssim(np.zeros((40, 10)), np.zeros((40, 10)))


def test_skimage_shim_refuses_other_arguments():
    sys.path.append(os.path.join(ROOT, "shims"))
    try:
        from skimage import metrics as sk
    finally:
        sys.path.remove(os.path.join(ROOT, "shims"))
    if not sk.__file__.startswith(os.path.join(ROOT, "shims")):
        pytest.skip("a real skimage is installed")
    a, b = _images(3)
    ok = dict(data_range=255, gaussian_weights=True, use_sample_covariance=False)
    for k in (dict(ok, data_range=1.0), dict(ok, gaussian_weights=False), dict(ok, use_sample_covariance=True), {k: v for k, v in ok.items() if k != "data_range"},
              dict(ok, win_size=7), dict(ok, channel_axis=2), dict(ok, full=True)):
        with pytest.raises(NotImplementedError):
            sk.structural_similarity(a, b, **k)
    with pytest.raises(NotImplementedError):
        sk.structural_similarity(np.stack([a, a, a], -1), np.stack([b, b, b], -1), **ok)  # 3-D: not evaluate.py's grayscale call
    with pytest.raises(NotImplementedError):
        sk.structural_similarity(a, b, 255, **{k: v for k, v in ok.items() if k != "data_range"})


def test_perceptual_loss_refusals(tmp_path, monkeypatch):
    import eval_models
    from hrviton_b200 import metrics
    monkeypatch.setenv("HRV_ALEX_RANDOM_INIT", "1")
    monkeypatch.chdir(tmp_path)
    for kw in (dict(model="net"), dict(net="vgg"), dict(net="squeeze"), dict(model="L2"), dict(colorspace="Lab"), dict(spatial=True)):
        with pytest.raises(NotImplementedError):
            eval_models.PerceptualLoss(use_gpu=False, **kw)
    # neither ./eval_models/weights/v0.1/alex.pth nor one next to the package (the package root is pointed at an empty directory)
    monkeypatch.setattr(metrics, "ROOT", str(tmp_path / "empty_root"))
    assert metrics.alex_weights_path() is None
    with pytest.raises(FileNotFoundError):
        eval_models.PerceptualLoss(use_gpu=False)
    d = tmp_path / "eval_models" / "weights" / "v0.1"
    d.mkdir(parents=True)
    net = metrics.PNetLin(pretrained=False)
    torch.save({k: v for k, v in net.state_dict().items() if k.startswith("lin")}, str(d / "alex.pth"))
    assert metrics.alex_weights_path() == str(d / "alex.pth")
    with pytest.warns(UserWarning, match="randomly initialised"):  # heads only, random backbone: the number would not be LPIPS
        pl = eval_models.PerceptualLoss(use_gpu=False)
    x = torch.zeros(1, 3, 64, 64, requires_grad=True)
    with pytest.raises(NotImplementedError, match="backward"):
        pl.forward(x, torch.zeros(1, 3, 64, 64))
    with torch.no_grad(), pytest.raises(RuntimeError, match="no CPU fallback"):
        pl.forward(x, torch.zeros(1, 3, 64, 64))
