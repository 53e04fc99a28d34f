"""GPU: Inception-v3 on the kernels (hrviton_b200.metrics.InceptionV3) against torchvision's own Inception3 in float64, the new metric
kernels against exact or float64 references, the Inception Score against the reference's evaluate.Evaluation, FID / KID against their
float64 CPU restatements (tests/inception_oracle.py), and reproducibility.

- Blocks Mixed_5d / 6e / 7c, pool features and logits: max|delta| <= 1e-4 * max|ref| against the float64 CPU model (seeded weights whose
  activations stay O(1) through all 94 convolutions), with and without transform_input, 299x299 and resized inputs.
- hrv_resize_bilinear_nhwc: bit-exact against F.interpolate on the GPU, every written value checked against a NaN sentinel.
- hrv_gram_f64: within 1e-12 * (|A| |B|^T) per element of a numpy float64 product; hrv_global_avgpool: exact.  Every new entry point
  writes its whole destination and nothing in a NaN guard band around it.
- unit_range on a transform_input model: [0, 1] images give what the model gives their ImageNet-normalised form.
- IS: within 1e-4 relative of evaluate.Evaluation; FID within 1e-6, KID within 1e-9 relative of the float64 restatements."""
import contextlib
import copy
import ctypes
import io
import os
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import inception_oracle as io_
from hrviton_b200 import capi, metrics, ops

pytestmark = pytest.mark.gpu
IMAGENET_MEAN, IMAGENET_STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)


@pytest.fixture(scope="module")
def seeded():
    return {ti: io_.seeded_inception(seed=3, transform_input=ti) for ti in (False, True)}


def _ratio(got, ref):
    return float((got.double().cpu() - ref).abs().max() / ref.abs().max())


def _nchw(a):
    return a.buf[..., a.c0:a.c0 + a.c].permute(0, 3, 1, 2)


@pytest.mark.parametrize("transform_input", [False, True])
def test_inception_matches_fp64_torchvision(seeded, transform_input):
    model = seeded[transform_input]
    net = metrics.InceptionV3.from_torchvision(model.cuda())
    g = torch.Generator(device="cuda").manual_seed(11)
    cases = [("299", torch.rand((2, 3, 299, 299), generator=g, device="cuda") * 2 - 1, False),
             ("341x256 unit", torch.rand((2, 3, 341, 256), generator=g, device="cuda"), True)]
    for label, x, unit in cases:
        with torch.no_grad():
            pool, logits, kept = net.run(x, unit_range=unit, keep=io_.TAPS)
        xin = F.interpolate(2 * x - 1 if unit else x, (299, 299), mode="bilinear", align_corners=False) if x.shape[2] != 299 else x
        if unit and transform_input:
            # [0, 1] images for a transform_input model: what torchvision's pipeline feeds it, ImageNet-normalised (the model's own
            # transform then maps them to 2x - 1); applying the transform to 2x - 1 instead would distort them
            xin = F.interpolate(x, (299, 299), mode="bilinear", align_corners=False).double()
            xin = (xin - torch.tensor(IMAGENET_MEAN, device="cuda").view(1, 3, 1, 1)) / torch.tensor(IMAGENET_STD, device="cuda").view(1, 3, 1, 1)
        taps, ref_pool, ref_logits = io_.fp64_forward(model, xin)
        for name in io_.TAPS:
            assert float(taps[name].abs().max()) > 0.1  # the seeded network keeps its activations alive
        for name, got, ref in [(t, _nchw(kept[t]), taps[t]) for t in io_.TAPS] + [("pool", pool, ref_pool), ("logits", logits, ref_logits)]:
            r = _ratio(got, ref)
            print("PARITY inception[transform_input=%s %s] %s max|d|/max|ref| = %.3e (bound 1e-4)" % (transform_input, label, name, r))
            assert got.shape == ref.shape and r <= 1e-4, (name, r)
        p2, l2 = net(x, unit_range=unit)
        assert torch.equal(p2, pool) and torch.equal(l2, logits)
        if unit and transform_input:  # unit_range skips the folded transform: the same bits as the model without it
            plain = copy.deepcopy(model)
            plain.transform_input = False
            p3, l3 = metrics.InceptionV3.from_torchvision(plain)(x, unit_range=True)
            assert torch.equal(p3, pool) and torch.equal(l3, logits)
            d = (net(x * 2 - 1)[1] - logits).abs().max() / logits.abs().max()  # without unit_range the transform does apply
            assert float(d) > 1e-2, float(d)
    model.cpu()


def test_resize_bilinear_bit_exact():
    g = torch.Generator(device="cuda").manual_seed(5)
    for (n, c, h, w), (oh, ow), pitch in (((2, 3, 1024, 768), (299, 299), 8), ((1, 3, 37, 53), (299, 299), 8), ((2, 5, 300, 301), (299, 299), 8),
                                          ((1, 9, 5, 7), (13, 4), 16), ((1, 3, 299, 299), (299, 299), 8), ((1, 3, 200, 150), (311, 97), 8)):
        x = torch.rand((n, c, h, w), generator=g, device="cuda")
        for unit in (False, True):
            dst = ops.Act(torch.full((n, oh, ow, pitch), float("nan"), device="cuda"), c=c)
            t = dst.ct()
            capi.check(capi.lib().hrv_resize_bilinear_nhwc(x.data_ptr(), n, c, h, w, int(unit), ctypes.byref(t), ops._stream()), "resize")
            ref = F.interpolate(2 * x - 1 if unit else x, (oh, ow), mode="bilinear", align_corners=False).permute(0, 2, 3, 1)
            c8 = (c + 7) // 8 * 8
            assert torch.equal(dst.buf[..., :c], ref), ((h, w), (oh, ow), unit, float((dst.buf[..., :c] - ref).abs().max()))
            assert bool((dst.buf[..., c:c8] == 0).all())             # the pad channels of the last 8-channel group are zeros
            assert bool(torch.isnan(dst.buf[..., c8:]).all())        # nothing past them is written
            assert torch.equal(ops.resize_bilinear_nhwc(x, (oh, ow), unit_range=unit).buf[..., :c], ref)


def test_global_avgpool_exact():
    g = torch.Generator(device="cuda").manual_seed(6)
    x = torch.randn((3, 8, 8, 2056), generator=g, device="cuda")
    xa = ops.Act(x, c=2048)
    y = ops.Act(torch.full((3, 1, 1, 2048), float("nan"), device="cuda"))
    ops.global_avgpool(xa, out=y)
    # 64 fp32 terms of these magnitudes sum exactly in fp64, and /64 is exact: one rounding, to fp32
    assert torch.equal(y.buf.view(3, 2048), x[..., :2048].double().mean((1, 2)).float())


def _gram_check(a, b, out, k_major):
    an, bn = a.double().cpu().numpy(), b.double().cpu().numpy()
    if k_major:
        an, bn = an.T, bn.T
    ref = an @ bn.T
    bound = np.abs(an) @ np.abs(bn).T
    r = float((np.abs(out.cpu().numpy() - ref) / np.maximum(bound, 1e-300)).max())
    return r, ref


def test_gram_f64_within_fp64_product():
    g = torch.Generator(device="cuda").manual_seed(7)
    worst = 0.0
    cases = [((300, 2048), (200, 2048), False, torch.float32, True),    # KID-like: K = 2048 contiguous, 20 tiles: split
             ((50, 2048), (50, 2048), True, torch.float32, False),      # FID moments: X^T X over a batch of samples
             ((5000, 40), (5000, 24), True, torch.float32, True),       # one tile, long K: split into slabs
             ((37, 4099), (29, 4099), False, torch.float64, True),      # fp64 operands, split, ragged edges
             ((70, 70), (70, 70), False, torch.float64, False)]
    for sa, sb, k_major, dt, split in cases:
        a = torch.randn(sa, generator=g, device="cuda", dtype=dt)
        b = torch.randn(sb, generator=g, device="cuda", dtype=dt)
        m, n = (sa[1], sb[1]) if k_major else (sa[0], sb[0])
        k = sa[0] if k_major else sa[1]
        nws = int(capi.lib().hrv_gram_f64_workspace_bytes(m, n, k))
        assert (nws > 0) == split
        out = torch.full((m, n), float("nan"), dtype=torch.float64, device="cuda")
        ops.gram_f64(a, b, out=out, k_major=k_major)
        assert bool(torch.isfinite(out).all())  # every element written
        r, ref = _gram_check(a, b, out, k_major)
        worst = max(worst, r)
        assert r <= 1e-12, (sa, sb, r)
        again = ops.gram_f64(a, b, k_major=k_major)
        assert torch.equal(again, out)  # fixed summation order
        ops.gram_f64(a, b, out=again, k_major=k_major, accumulate=True)
        assert torch.equal(again, out + out)
    # a transposed (column-major) fp64 operand, as eigh returns its eigenvectors
    v = torch.randn((64, 96), generator=g, device="cuda", dtype=torch.float64).mT
    r, _ = _gram_check(v, v, ops.gram_f64(v, v), False)
    worst = max(worst, r)
    assert r <= 1e-12
    print("PARITY gram_f64 max |C - C_fp64| / (|A||B|^T) = %.3e (bound 1e-12)" % worst)


def test_new_entry_points_write_only_their_outputs():
    """Each new entry point on small shapes, its destination inside a NaN-filled guard band (padded rows, columns past ldc / the
    pitch, an extra output row): every output element is written and nothing around it."""
    g = torch.Generator(device="cuda").manual_seed(13)
    L, st = capi.lib(), ops._stream()
    # global average pool: y's pitch 24 > c 16, one image more in the buffer than the call covers
    x = ops.Act(torch.randn((2, 3, 5, 16), generator=g, device="cuda"))
    yb = torch.full((3, 1, 1, 24), float("nan"), device="cuda")
    y = ops.Act(yb[:2].contiguous(), c=16)
    tx, ty = x.ct(), y.ct()
    capi.check(L.hrv_global_avgpool(ctypes.byref(tx), ctypes.byref(ty), st), "global_avgpool")
    assert bool(torch.isfinite(y.buf[..., :16]).all()) and bool(torch.isnan(y.buf[..., 16:]).all()) and bool(torch.isnan(yb[2]).all())
    # gram: C inside a (m + 2) x (ldc) NaN block, ldc > n, split and unsplit, fp32 and fp64, transposed strides
    for (m, n, k, dt, k_major) in ((5, 3, 7, torch.float32, False), (6, 4, 3000, torch.float32, True), (3, 9, 2100, torch.float64, False),
                                   (65, 66, 17, torch.float64, True)):
        a = torch.randn((k, m) if k_major else (m, k), generator=g, device="cuda", dtype=dt)
        b = torch.randn((k, n) if k_major else (n, k), generator=g, device="cuda", dtype=dt)
        ldc = n + 5
        cb = torch.full((m + 2, ldc), float("nan"), dtype=torch.float64, device="cuda")
        ops.gram_f64(a, b, out=cb[1:m + 1, :n], k_major=k_major)
        assert bool(torch.isfinite(cb[1:m + 1, :n]).all()), (m, n, k)
        assert bool(torch.isnan(cb[0]).all()) and bool(torch.isnan(cb[m + 1]).all()) and bool(torch.isnan(cb[:, n:]).all()), (m, n, k)
    # kid_sums: out with one row more than the subsets
    f = torch.rand((9, 16), generator=g, device="cuda", dtype=torch.float64)
    gm = ops.gram_f64(f, f)
    ix = torch.tensor([[0, 3, 8], [1, 2, 5]], dtype=torch.int32, device="cuda")
    out = torch.full((3, 3), float("nan"), dtype=torch.float64, device="cuda")
    capi.check(L.hrv_kid_sums(gm.data_ptr(), gm.data_ptr(), gm.data_ptr(), 9, 9, ix.data_ptr(), ix.data_ptr(), 2, 3, 1.0 / 16, out.data_ptr(), st),
               "kid_sums")
    assert bool(torch.isfinite(out[:2]).all()) and bool(torch.isnan(out[2]).all())
    kk = (gm / 16 + 1) ** 3
    for s_, r in enumerate(ix.long()):
        sub = kk[r][:, r]
        ref = float(sub.sum() - sub.diagonal().sum())
        assert abs(float(out[s_, 0]) - ref) <= 1e-13 * ref and float(out[s_, 2]) == pytest.approx(float(sub.sum()), rel=1e-13)


def test_inception_score_matches_reference_evaluate(seeded, tmp_path, monkeypatch):
    """evaluate.Evaluation (the reference copy, unmodified, with the seeded Inception3 in place of the ImageNet one and cuDNN in fp32)
    against inception_score on the package's probabilities of the same T3 inputs."""
    import hrv_env
    from PIL import Image
    if hrv_env.reference_dir() is None:
        pytest.skip("no reference copy (oracle/_ref)")
    import torchvision.transforms as Tr
    from test_metrics_gpu import _weights_dir
    monkeypatch.setenv("HRV_ALEX_RANDOM_INIT", "1")
    monkeypatch.chdir(tmp_path)
    _weights_dir(tmp_path)
    gt_dir, pred_dir = tmp_path / "gt", tmp_path / "pred"
    gt_dir.mkdir()
    pred_dir.mkdir()
    rng = np.random.RandomState(9)
    for i in range(6):
        base = np.kron(rng.randint(0, 256, (32, 24, 3)), np.ones((8, 8, 1)))
        Image.fromarray(np.clip(base + rng.randint(-10, 11, base.shape), 0, 255).astype(np.uint8)).save(str(gt_dir / ("%05d_00.jpg" % i)), quality=90)
        Image.fromarray(np.clip(base + rng.randint(-40, 41, base.shape), 0, 255).astype(np.uint8)).save(str(pred_dir / ("%05d_00.jpg" % i)), quality=90)
    names = sorted(os.listdir(str(gt_dir)))
    model = seeded[False]
    opt = types.SimpleNamespace(predict_dir=str(pred_dir), ground_truth_dir=str(gt_dir), resolution=1024)
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)  # the reference arm in fp32, as the package computes
    ev = hrv_env.load_reference_script("evaluate", alias="ref_evaluate_is")
    ev.inception_v3 = lambda pretrained=True, transform_input=False: io_.seeded_inception(seed=3, transform_input=transform_input)
    with contextlib.redirect_stdout(io.StringIO()):
        _, _, _, is_ref, isd_ref = ev.Evaluation(opt, list(names), list(names))
    T3 = Tr.Compose([Tr.Resize((299, 299)), Tr.ToTensor(), Tr.Normalize(mean=(0.5, 0.5, 0.5), std=(0.5, 0.5, 0.5))])
    x = torch.stack([T3(Image.open(str(pred_dir / nm))) for nm in names]).cuda()
    net = metrics.InceptionV3.from_torchvision(model.cuda())
    with torch.no_grad():
        probs = torch.softmax(net(x)[1], 1)
        is_mean, is_std = metrics.inception_score(probs)
        is_img, _ = metrics.inception_score(x, model=net, batch_size=4)
    model.cpu()
    rel = abs(float(is_mean) - is_ref) / is_ref
    print("PARITY inception_score |IS - evaluate.py IS| / IS = %.3e (bound 1e-4; IS = %.6f)" % (rel, is_ref))
    assert rel <= 1e-4 and float(is_mean) > 1.0 and float(is_std) == isd_ref == 0.0
    assert torch.equal(is_img, is_mean)


def _features(n, seed, shift):
    g = torch.Generator(device="cuda").manual_seed(seed)
    z = torch.randn((n, 64), generator=g, device="cuda")
    mix = torch.randn((64, 2048), generator=g, device="cuda") / 8
    return (z @ mix + 0.3 * torch.randn((n, 2048), generator=g, device="cuda") + shift).relu()  # correlated, non-negative, like pool features


def test_fid_kid_match_cpu_restatements():
    fa, fb = _features(2500, 1, 0.2), _features(2300, 2, 0.25)
    sa, sb = metrics.FeatureStats(), metrics.FeatureStats()
    for i in range(0, 2500, 333):  # ragged batches
        sa.update(fa[i:i + 333])
    for i in range(0, 2300, 500):
        sb.update(fb[i:i + 500])
    na, nb = fa.double().cpu().numpy(), fb.double().cpu().numpy()
    mu_a, mu_b, ca, cb = na.mean(0), nb.mean(0), np.cov(na, rowvar=False), np.cov(nb, rowvar=False)
    assert np.abs(sa.mean().cpu().numpy() - mu_a).max() <= 1e-12 * np.abs(mu_a).max()
    assert np.abs(sa.cov().cpu().numpy() - ca).max() <= 1e-10 * np.abs(ca).max()
    ref = io_.fid_np(mu_a, ca, mu_b, cb)
    got = metrics.fid(sa, sb)
    assert got.dtype == torch.float64 and got.is_cuda
    rel = abs(float(got) - ref) / ref
    print("PARITY fid |FID - fp64 CPU| / FID = %.3e (bound 1e-6; FID = %.6f)" % (rel, ref))
    assert rel <= 1e-6
    ix, iy = metrics.kid_subsets(1200, 1100, 20, 500, seed=3)
    km, ks = metrics.kid(fa[:1200], fb[:1100], subsets=20, subset_size=500, seed=3)
    rm, rs = io_.kid_np(na[:1200], nb[:1100], ix, iy)
    rel_m, rel_s = abs(float(km) - rm) / abs(rm), abs(float(ks) - rs) / abs(rs)
    print("PARITY kid |KID - fp64 CPU| / KID = %.3e, std %.3e (bound 1e-9; KID = %.6e +- %.2e)" % (rel_m, rel_s, rm, rs))
    assert rel_m <= 1e-9 and rel_s <= 1e-9
    # bit-identical on a second run, and under the bf16 training precision
    prec = ops.get_precision()
    try:
        for p in ("fp32", "bf16"):
            ops.set_precision(p)
            sa2, sb2 = metrics.FeatureStats(), metrics.FeatureStats()
            for i in range(0, 2500, 333):
                sa2.update(fa[i:i + 333])
            for i in range(0, 2300, 500):
                sb2.update(fb[i:i + 500])
            assert torch.equal(metrics.fid(sa2, sb2), got)
            km2, ks2 = metrics.kid(fa[:1200], fb[:1100], subsets=20, subset_size=500, seed=3)
            assert torch.equal(km2, km) and torch.equal(ks2, ks)
    finally:
        ops.set_precision(prec)


def test_features_reproducible(seeded):
    model = seeded[False]
    net = metrics.InceptionV3.from_torchvision(model.cuda())
    g = torch.Generator(device="cuda").manual_seed(12)
    x = torch.rand((7, 3, 299, 299), generator=g, device="cuda") * 2 - 1
    prec = ops.get_precision()
    try:
        ops.set_precision("bf16")
        with torch.no_grad():
            pool7, logits7 = net(x)
            pool1, logits1 = net(x[3:4].clone())
            again = net(x)
        ops.set_precision("fp32")
        with torch.no_grad():
            p32, l32 = net(x)
    finally:
        ops.set_precision(prec)
        model.cpu()
    assert torch.equal(pool1, pool7[3:4]) and torch.equal(logits1, logits7[3:4])  # one image alone = the same image in a batch of 7
    assert torch.equal(again[0], pool7) and torch.equal(again[1], logits7)
    assert torch.equal(p32, pool7) and torch.equal(l32, logits7)  # the training precision does not reach the metric


def test_refusals(seeded):
    model = seeded[False]
    net = metrics.InceptionV3.from_torchvision(model.cuda())
    x = torch.rand((1, 3, 299, 299), device="cuda")
    before = ops.LAUNCHES[0]
    with pytest.raises(NotImplementedError):
        net(x.clone().requires_grad_(True))
    with pytest.raises(ValueError):
        net(x[:, :2])
    with pytest.raises(ValueError):
        net(x.double())
    with pytest.raises(RuntimeError):
        net(x.cpu())
    with pytest.raises(ValueError):
        metrics.inception_score(torch.rand(3, 10, device="cuda"), splits=4)
    with pytest.raises(ValueError):
        metrics.inception_score(x)  # images without a model
    f = torch.rand(10, 2048, device="cuda")
    with pytest.raises(ValueError):
        metrics.kid(f, f, subsets=2, subset_size=11)
    with pytest.raises(ValueError):
        metrics.kid(f, f[:, :100], subsets=2, subset_size=5)
    with pytest.raises(NotImplementedError):
        metrics.kid(f.clone().requires_grad_(True), f, subsets=2, subset_size=5)
    with pytest.raises(ValueError):
        metrics.FeatureStats().update(f[:, :100])
    with pytest.raises(ValueError):
        metrics.FeatureStats().cov()
    assert ops.LAUNCHES[0] == before  # refused before any launch
    model.cpu()
