"""CPU: the host arithmetic of the Inception metrics (hrviton_b200.metrics) — the FID formula against scipy.linalg.sqrtm, KID's subset
draw and MMD^2 against a numpy restatement, the BatchNorm / average-pool / input-affine folds and the stride-2 space-to-depth rewrite
against torch in fp64 — and the refusals that need no GPU."""
import numpy as np
import pytest
import scipy.linalg
import torch
import torch.nn.functional as F

import inception_oracle as io_
from hrviton_b200 import metrics, ops


def _cov(d, eigs, seed):
    q, _ = np.linalg.qr(np.random.RandomState(seed).randn(d, d))
    return (q * eigs) @ q.T


def _fid_sqrtm(mu_a, sig_a, mu_b, sig_b):
    covmean = scipy.linalg.sqrtm(sig_a @ sig_b)
    covmean = np.real(covmean)
    d = mu_a - mu_b
    return float(d @ d + np.trace(sig_a) + np.trace(sig_b) - 2 * np.trace(covmean))


@pytest.mark.parametrize("cond", ["well", "bad"])
def test_fid_formula_matches_sqrtm(cond):
    d = 64
    rng = np.random.RandomState(1)
    if cond == "well":
        ea, eb = rng.uniform(0.5, 2.0, d), rng.uniform(0.5, 2.0, d)
    else:  # condition numbers of 1e10 and 1e8
        ea, eb = np.logspace(0, -10, d), np.logspace(1, -7, d)
    sa, sb = _cov(d, ea, 2), _cov(d, eb, 3)
    mu_a, mu_b = rng.randn(d), rng.randn(d)
    ref = _fid_sqrtm(mu_a, sa, mu_b, sb)
    T = lambda a: torch.from_numpy(a)  # noqa: E731
    got = float(metrics.fid_from_moments(T(mu_a), T(sa), T(mu_b), T(sb), lambda a, b: a @ b.T))
    rel = abs(got - ref) / abs(ref)
    print("PARITY fid_formula[%s] |fid - sqrtm fid| / fid = %.3e (bound %.0e)" % (cond, rel, 1e-10 if cond == "well" else 1e-7))
    assert rel <= (1e-10 if cond == "well" else 1e-7), (got, ref)
    assert abs(got - io_.fid_np(mu_a, sa, mu_b, sb)) <= 1e-10 * abs(ref)
    # identical statistics: 0 up to rounding (the square roots of eigenvalues near 0 amplify it for the badly conditioned one)
    same = float(metrics.fid_from_moments(T(mu_a), T(sa), T(mu_a), T(sa), lambda a, b: a @ b.T))
    assert abs(same) <= (1e-12 if cond == "well" else 1e-7) * np.trace(sa), same


def test_kid_subsets_and_mmd_match_numpy():
    rng = np.random.RandomState(4)
    fa, fb = np.abs(rng.randn(60, 16)), np.abs(rng.randn(50, 16)) * 1.2
    ix, iy = metrics.kid_subsets(60, 50, 5, 20, seed=7)
    assert ix.shape == iy.shape == (5, 20) and ix.dtype == np.int32
    assert all(len(set(r)) == 20 for r in ix) and all(len(set(r)) == 20 for r in iy)  # without replacement
    assert ix.max() < 60 and iy.max() < 50
    ix2, iy2 = metrics.kid_subsets(60, 50, 5, 20, seed=7)
    assert np.array_equal(ix, ix2) and np.array_equal(iy, iy2)
    assert not np.array_equal(ix, metrics.kid_subsets(60, 50, 5, 20, seed=8)[0])
    # the three sums the kernel forms, here in numpy, through the package's MMD^2 -> the numpy restatement
    d = fa.shape[1]
    sums = []
    for a, b in zip(ix, iy):
        kxx, kyy, kxy = (fa[a] @ fa[a].T / d + 1) ** 3, (fb[b] @ fb[b].T / d + 1) ** 3, (fa[a] @ fb[b].T / d + 1) ** 3
        sums.append([kxx.sum() - np.trace(kxx), kyy.sum() - np.trace(kyy), kxy.sum()])
    mmd = metrics.mmd2_from_sums(torch.tensor(sums, dtype=torch.float64), 20)
    mean, std = io_.kid_np(fa, fb, ix, iy)
    assert abs(float(mmd.mean()) - mean) <= 1e-12 * abs(mean) and abs(float(mmd.std(unbiased=False)) - std) <= 1e-10 * abs(std)


def _basic_conv(cin, cout, k, pad, stride=1, seed=0):
    from torchvision.models.inception import BasicConv2d
    torch.manual_seed(seed)
    bc = BasicConv2d(cin, cout, kernel_size=k, padding=pad, stride=stride).double().eval()
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        bc.bn.weight.copy_(torch.rand(cout, generator=g, dtype=torch.float64) + 0.5)
        bc.bn.bias.copy_(torch.randn(cout, generator=g, dtype=torch.float64))
        bc.bn.running_mean.copy_(torch.randn(cout, generator=g, dtype=torch.float64))
        bc.bn.running_var.copy_(torch.rand(cout, generator=g, dtype=torch.float64) + 0.1)
    assert bc.bn.eps == 0.001
    return bc


def _apply(w, s, t, x, pad, stride=1):
    return torch.relu(F.conv2d(x, w, padding=pad, stride=stride) * s.view(1, -1, 1, 1) + t.view(1, -1, 1, 1))


def test_batchnorm_fold():
    x = torch.randn(2, 8, 13, 11, dtype=torch.float64)
    for k, pad in (((1, 7), (0, 3)), ((3, 3), (0, 0)), ((5, 5), (2, 2))):
        bc = _basic_conv(8, 16, k, pad)
        w, s, t = metrics.fold_basic_conv(bc)
        with torch.no_grad():
            ref = bc(x)
        assert (_apply(w, s, t, x, pad) - ref).abs().max() <= 1e-12 * ref.abs().max()


def test_avgpool_fold():
    x = torch.randn(2, 8, 9, 10, dtype=torch.float64)
    bc = _basic_conv(8, 16, 1, 0, seed=1)
    w, s, t = metrics.fold_basic_conv(bc, pool=True)
    assert w.shape == (16, 8, 3, 3)
    with torch.no_grad():
        ref = bc(F.avg_pool2d(x, kernel_size=3, stride=1, padding=1))  # InceptionA/C/E branch_pool
    assert (_apply(w, s, t, x, 1) - ref).abs().max() <= 1e-12 * ref.abs().max()


def test_transform_input_fold_and_s2d():
    """transform_input folded into Conv2d_1a_3x3 (3x3, stride 2, no padding), and that convolution as a 2x2 one over the
    space-to-depth input (ops.s2d_weight(w, 0), offset 0)."""
    import torchvision
    m = torchvision.models.inception_v3(weights=None, aux_logits=False, init_weights=False, transform_input=True).double().eval()
    x = torch.rand(2, 3, 17, 16, dtype=torch.float64)
    bc = _basic_conv(3, 32, 3, 0, stride=2, seed=2)
    w, s, t = metrics.fold_basic_conv(bc, affine=metrics._TRANSFORM)
    with torch.no_grad():
        ref = bc(m._transform_input(x))
    got = _apply(w, s, t, x, 0, stride=2)
    assert (got - ref).abs().max() <= 1e-12 * ref.abs().max()
    # space-to-depth: channel (py*2+px)*8 + ci of pixel (Y, X) holds x[2Y+py, 2X+px, ci] (channels padded to 8, odd edges zero)
    xp = F.pad(x, (0, 0, 0, 1))  # 17 rows -> 18
    xs = torch.zeros(2, 32, 9, 8, dtype=torch.float64)
    for py in range(2):
        for px in range(2):
            xs[:, (py * 2 + px) * 8:(py * 2 + px) * 8 + 3] = xp[:, :, py::2, px::2]
    ws = ops.s2d_weight(w, 0)
    got2 = torch.relu(F.conv2d(xs, ws) * s.view(1, -1, 1, 1) + t.view(1, -1, 1, 1))
    assert got2.shape == ref.shape and (got2 - ref).abs().max() <= 1e-12 * ref.abs().max()


def test_refusals_without_gpu():
    import torchvision
    m = torchvision.models.inception_v3(weights=None, aux_logits=False, init_weights=False)
    with pytest.raises(ValueError):
        metrics.InceptionV3.from_torchvision(m)  # train mode
    with pytest.raises(RuntimeError):
        metrics.InceptionV3.from_torchvision(m.eval())  # weights on the CPU
    with pytest.raises(TypeError):
        metrics.InceptionV3.from_torchvision(torch.nn.Conv2d(3, 3, 1).eval())
    with pytest.raises(RuntimeError):
        metrics.inception_score(torch.rand(4, 1000))
    with pytest.raises(RuntimeError):
        metrics.kid(torch.rand(8, 16), torch.rand(8, 16), subsets=1, subset_size=4)
    with pytest.raises(RuntimeError):
        metrics.FeatureStats(16, device="cpu")
    with pytest.raises(TypeError):
        metrics.fid(None, None)
