"""A seeded torchvision Inception3 whose activations stay O(1) through all 94 convolutions, and float64 restatements of the Inception
metrics (FID on numpy's eigh, KID per subset on numpy), for tests/test_inception_*.py and tools/inception_bench.py.

The ImageNet weights cannot be fetched offline, and a randomly initialised Inception3 with its default BatchNorm statistics (mean 0,
var 1) lets the activations grow or die from block to block, so a comparison of its outputs tests little.  seeded_inception() draws the
BatchNorm affine parameters, then sets every running statistic to the batch statistic of one forward pass over seeded images (each
layer normalised before the next is measured), then perturbs them: every layer sees inputs of its own scale, as a trained one does.
The BatchNorm shifts keep most units in ReLU's linear part: a random network with half its units gated off amplifies any rounding
~10x every few blocks (fp32 torch itself then differs from fp64 by 3e-5 at Mixed_7c), which would measure the seed, not the kernels."""
import copy

import numpy as np
import torch
import torch.nn as nn


def seeded_inception(seed=0, transform_input=False, calib_images=4):
    """An eval-mode torchvision Inception3 (aux head included, as the ImageNet one has) on the CPU, fp32."""
    import torchvision
    torch.manual_seed(seed)
    m = torchvision.models.inception_v3(weights=None, aux_logits=True, init_weights=False, transform_input=transform_input)
    g = torch.Generator().manual_seed(seed + 1)
    bns = [mod for mod in m.modules() if isinstance(mod, nn.BatchNorm2d)]
    with torch.no_grad():
        for bn in bns:
            bn.weight.copy_(torch.rand(bn.num_features, generator=g) * 0.4 + 0.3)
            bn.bias.copy_(torch.rand(bn.num_features, generator=g) * 0.5 + 0.3)
            bn.momentum = None  # cumulative average: after one batch, the running statistics are that batch's
        m.fc.weight.mul_(4.0)  # logits spanning a few units: a soft-max far from uniform, an Inception Score well above 1
        m.train()
        m(torch.rand((calib_images, 3, 299, 299), generator=g) * 2 - 1)
        m.eval()
        for bn in bns:
            sd = bn.running_var.sqrt()
            bn.running_mean.add_(0.05 * sd * torch.randn(bn.num_features, generator=g))
            bn.running_var.mul_(torch.rand(bn.num_features, generator=g) * 0.2 + 0.9)
    return m


TAPS = ("Mixed_5d", "Mixed_6e", "Mixed_7c")


def fp64_forward(model, x):
    """({tap: fp64 NCHW}, pool fp64 (N,2048), logits fp64 (N,1000)) of a float64 CPU copy of `model` on x (cast to float64)."""
    m = copy.deepcopy(model).cpu().double().eval()
    got = {}
    hooks = [getattr(m, t).register_forward_hook(lambda mod, i, o, t=t: got.__setitem__(t, o)) for t in TAPS]
    hooks.append(m.fc.register_forward_hook(lambda mod, i, o: got.__setitem__("pool", i[0])))
    try:
        with torch.no_grad():
            logits = m(x.detach().cpu().double())
    finally:
        for h in hooks:
            h.remove()
    return {t: got[t] for t in TAPS}, got["pool"], logits


def fid_np(mu_a, sig_a, mu_b, sig_b):
    """FID in float64 numpy through the eigendecompositions of sig_a and of sqrt(sig_a) sig_b sqrt(sig_a)."""
    ea, va = np.linalg.eigh(sig_a)
    root = (va * np.sqrt(np.clip(ea, 0, None))) @ va.T
    m = root @ sig_b @ root
    em = np.clip(np.linalg.eigvalsh((m + m.T) / 2), 0, None)
    d = mu_a - mu_b
    return float(d @ d + np.trace(sig_a) + np.trace(sig_b) - 2 * np.sqrt(em).sum())


def mmd2_np(x, y):
    """Unbiased MMD^2 of two float64 feature sets with the kernel (x.y/d + 1)^3, as the KID implementations state it."""
    d = x.shape[1]
    kxx, kyy, kxy = (x @ x.T / d + 1) ** 3, (y @ y.T / d + 1) ** 3, (x @ y.T / d + 1) ** 3
    m = x.shape[0]
    sxx = kxx.sum() - np.diag(kxx).sum()
    syy = kyy.sum() - np.diag(kyy).sum()
    return (sxx + syy) / (m * (m - 1)) - 2 * kxy.sum() / (m * m)


def kid_np(fa, fb, ix, iy):
    """(mean, std) over the subsets given by the index rows ix, iy (kid_subsets) of mmd2_np, float64."""
    fa, fb = np.asarray(fa, np.float64), np.asarray(fb, np.float64)
    v = np.array([mmd2_np(fa[a], fb[b]) for a, b in zip(ix, iy)])
    return float(v.mean()), float(v.std())
