"""float64 numpy restatement of the SSIM that evaluate.py:67 asks skimage for: structural_similarity(im1, im2, data_range=255,
gaussian_weights=True, use_sample_covariance=False) = sigma 1.5, truncate 3.5 (11 taps), K1 0.01, K2 0.03, the SSIM map averaged over
the outputs 5 pixels or more from every border.  Each moment map is a separable Gaussian evaluated only where its window lies inside
the image (rows, then columns), which is what hrv_ssim computes; test_metrics_cpu.py ties it to scipy.ndimage.gaussian_filter.

reference_eval_models(alex) imports the reference's own eval_models (torch / cuDNN LPIPS) from oracle/_ref for comparisons."""
import contextlib
import importlib
import sys

import numpy as np

RADIUS = 5


def gauss_taps(sigma=1.5, truncate=3.5):
    r = int(truncate * sigma + 0.5)
    x = np.arange(-r, r + 1, dtype=np.float64)
    g = np.exp(-0.5 / (sigma * sigma) * x * x)
    return g / g.sum()


def moments_valid(a):
    """The Gaussian filter of a (H,W) float64 map at the outputs [5, H-5) x [5, W-5) (rows first, then columns)."""
    g = gauss_taps()
    h, w = a.shape
    k = len(g)
    rows = sum(g[i] * a[:, i:w - k + 1 + i] for i in range(k))
    return sum(g[i] * rows[i:h - k + 1 + i, :] for i in range(k))


def ssim_map(ux, uy, uxx, uyy, uxy, data_range=255.0):
    c1, c2 = (0.01 * data_range) ** 2, (0.03 * data_range) ** 2
    vx, vy, vxy = uxx - ux * ux, uyy - uy * uy, uxy - ux * uy
    return ((2 * ux * uy + c1) * (2 * vxy + c2)) / ((ux * ux + uy * uy + c1) * (vx + vy + c2))


def ssim(im1, im2, data_range=255.0):
    """Mean SSIM of two (H,W) images (any real dtype), float64."""
    x, y = np.asarray(im1, dtype=np.float64), np.asarray(im2, dtype=np.float64)
    if min(x.shape) < 2 * RADIUS + 1:
        raise ValueError("win_size exceeds image extent")
    m = [moments_valid(t) for t in (x, y, x * x, y * y, x * y)]
    return float(ssim_map(*m, data_range=data_range).mean(dtype=np.float64))


@contextlib.contextmanager
def reference_eval_models(alex):
    """The reference's eval_models package (oracle/_ref), imported under its own name while the drop-in is set aside in sys.modules,
    and yielded with two patches active: DistModel.initialize reads `alex` (the reference looks next to its own files, which stay
    read-only) and tv.alexnet builds the backbone without ImageNet weights (nothing is downloaded; `alex` carries the backbone).
    Construct PerceptualLoss inside the block; the patches are undone on exit."""
    import hrv_env
    import torchvision
    d = hrv_env.reference_dir()
    if d is None:
        raise FileNotFoundError("no reference copy (oracle/_ref)")
    saved = {k: sys.modules.pop(k) for k in list(sys.modules) if k == "eval_models" or k.startswith("eval_models.")}
    sys.path.insert(0, d)
    try:
        ref = importlib.import_module("eval_models")
        dm = importlib.import_module("eval_models.dist_model")
        pn = importlib.import_module("eval_models.pretrained_networks")
    finally:
        sys.path.remove(d)
        for k in [k for k in sys.modules if k == "eval_models" or k.startswith("eval_models.")]:
            del sys.modules[k]
        sys.modules.update(saved)
    assert ref.__file__.startswith(d)
    init, tv_alexnet = dm.DistModel.initialize, pn.tv.alexnet  # pn.tv is torchvision.models itself
    dm.DistModel.initialize = lambda self, **k: init(self, model_path=alex, **k)
    pn.tv.alexnet = lambda pretrained=True, **k: torchvision.models.AlexNet()
    try:
        yield ref
    finally:
        dm.DistModel.initialize = init
        pn.tv.alexnet = tv_alexnet
