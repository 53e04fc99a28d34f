"""GPU: pytorch-fid's FID Inception on the kernels (metrics.InceptionV3.from_fid_weights) against its float64 CPU restatement
(tests/fid_inception_oracle.py), its two new kernels against torch bit for bit, and tools/fid.py end to end.

- hrv_pool3x3s1: bit-exact against F.avg_pool2d(count_include_pad=False) and F.max_pool2d on the device, NaNs and ties included,
  channel-slice sources and destinations inside a sentinel guard band.
- hrv_resize_bilinear_fid: bit-exact against F.interpolate(TF.to_tensor(img)) * 2 - 1 from uint8 and fp32 sources.
- Mixed_5d / 6e / 7c, pool features and logits within 1e-4 * max|ref| of float64, from uint8 and fp32 images; the same weights through
  from_torchvision (count_include_pad=True pooling) miss that bound, so the test sees which network ran.
- One image alone equals the same image in a batch of 7; FID and KID repeat bit for bit, also under set_precision('bf16').
- tools/fid.py on two PNG folders: its features equal the network's on the same tensors, its FID is within 1e-3 of the float64
  oracle's, and --save-stats then an npz-vs-folder run gives the same FID."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import fid_inception_oracle as fo
import inception_oracle as io_
from hrviton_b200 import capi, metrics, ops

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SENTINEL = 3.0e38  # guard value no pool of the finite test inputs can produce


@pytest.fixture(scope="module")
def fid_sd():
    return fo.seeded_fid_state_dict(seed=4)


@pytest.fixture(scope="module")
def fid_net(fid_sd):
    return metrics.InceptionV3.from_fid_weights(fid_sd)


def _same_bits(got, ref):
    """Bit-identical, NaNs in the same places (NaN payloads aside)."""
    nan = torch.isnan(ref)
    return torch.equal(torch.isnan(got), nan) and torch.equal(got[~nan].view(torch.int32), ref[~nan].view(torch.int32))


def _ratio(got, ref):
    return float((got.double().cpu() - ref).abs().max() / ref.abs().max())


def _nchw(a):
    return a.buf[..., a.c0:a.c0 + a.c].permute(0, 3, 1, 2)


@pytest.mark.parametrize("mode", ["avg", "max"])
def test_pool3x3s1_bit_exact(mode):
    g = torch.Generator(device="cuda").manual_seed(21)
    # (n, h, w, c, source channel offset / pitch, destination offset / pitch): 16-byte and scalar paths, slices, tiny extents
    cases = [((2, 35, 35, 192), (0, 192), (0, 192)), ((2, 17, 17, 64), (8, 80), (4, 72)), ((3, 8, 8, 40), (0, 40), (16, 64)),
             ((1, 7, 9, 6), (1, 9), (3, 11)), ((2, 1, 1, 8), (0, 8), (0, 8)), ((1, 2, 2, 4), (0, 4), (4, 12)), ((1, 2, 3, 3), (2, 7), (1, 5)),
             ((1, 5, 3, 4), (4, 12), (0, 4))]
    for (n, h, w, c), (xc0, xp), (yc0, yp) in cases:
        for values in ("randn", "ties", "nan"):
            if values == "ties":  # few distinct values: equal maxima everywhere, exact sums
                x = torch.randint(-2, 3, (n, h, w, xp), generator=g, device="cuda").float()
            else:
                x = torch.randn((n, h, w, xp), generator=g, device="cuda")
            if values == "nan":
                x[torch.rand((n, h, w, xp), generator=g, device="cuda") < 0.05] = float("nan")
            xa = ops.Act(x, c=c, c0=xc0)
            yb = torch.full((n + 1, h, w, yp), SENTINEL, device="cuda")  # one image more than the call covers
            ya = ops.Act(yb[:n], c=c, c0=yc0)
            ops.pool3x3s1(xa, mode, out=ya)
            xs = _nchw(xa).contiguous()
            ref = F.avg_pool2d(xs, 3, 1, 1, count_include_pad=False) if mode == "avg" else F.max_pool2d(xs, 3, 1, 1)
            got = _nchw(ya)
            assert _same_bits(got, ref), ((n, h, w, c), values, float((got - ref).abs().nan_to_num().max()))
            guard = torch.ones_like(yb, dtype=torch.bool)
            guard[:n, ..., yc0:yc0 + c] = False
            assert bool((yb[guard] == SENTINEL).all()), ((n, h, w, c), values)  # nothing written outside the destination
    x = ops.Act(torch.randn((1, 4, 4, 8), device="cuda"))
    with pytest.raises(RuntimeError):
        ops.pool3x3s1(x, mode, out=ops.Act(torch.empty((1, 4, 3, 8), device="cuda")))  # not x's extent
    print("PARITY pool3x3s1[%s] bit-exact against torch on %d cases" % (mode, len(cases) * 3))


def _to_tensor_ref(imgs, size):
    """pytorch-fid's input from uint8 (N,H,W,3) numpy images: F.interpolate(TF.to_tensor(img)[None].cuda(), size) * 2 - 1."""
    import torchvision.transforms.functional as TF
    return torch.cat([F.interpolate(TF.to_tensor(im)[None].cuda(), size, mode="bilinear", align_corners=False) * 2 - 1 for im in imgs])


def test_resize_bilinear_fid_bit_exact():
    import torchvision.transforms.functional as TF
    rng = np.random.RandomState(5)
    L, st = capi.lib(), ops._stream()
    for (h, w), (oh, ow) in (((1024, 768), (299, 299)), ((341, 256), (299, 299)), ((299, 299), (299, 299)), ((150, 120), (299, 299)),
                             ((37, 53), (299, 299)), ((20, 30), (47, 33))):
        imgs = rng.randint(0, 256, (2, h, w, 3)).astype(np.uint8)
        ref = _to_tensor_ref(imgs, (oh, ow)).permute(0, 2, 3, 1)
        u8 = torch.from_numpy(imgs).cuda()
        f32 = torch.stack([TF.to_tensor(im) for im in imgs]).cuda()  # the same [0, 1] values as fp32 NCHW
        for src, x in ((capi.FID_SRC_U8_NHWC, u8), (capi.FID_SRC_F32_NCHW, f32)):
            buf = torch.full((3, oh, ow, 16), float("nan"), device="cuda")  # pitch 16, one image more than the call covers
            dst = ops.Act(buf[:2], c=3)
            t = dst.ct()
            capi.check(L.hrv_resize_bilinear_fid(x.data_ptr(), src, 2, 3, h, w, ctypes.byref(t), st), "resize_bilinear_fid")
            assert torch.equal(buf[:2, ..., :3], ref), ((h, w), src, float((buf[:2, ..., :3] - ref).abs().max()))
            assert bool((buf[:2, ..., 3:8] == 0).all())          # the pad channels of the 8-channel group are zeros
            assert bool(torch.isnan(buf[:2, ..., 8:]).all()) and bool(torch.isnan(buf[2]).all())  # nothing past them
            assert torch.equal(ops.resize_bilinear_fid(x, (oh, ow)).buf[..., :3], ref)
    # an fp32 source that is not a uint8 image
    g = torch.Generator(device="cuda").manual_seed(6)
    x = torch.rand((2, 3, 341, 256), generator=g, device="cuda")
    ref = (F.interpolate(x, (299, 299), mode="bilinear", align_corners=False) * 2 - 1).permute(0, 2, 3, 1)
    assert torch.equal(ops.resize_bilinear_fid(x).buf[..., :3], ref)


def _images(n, h, w, seed):
    """Smooth uint8 RGB images with noise, (n, h, w, 3) numpy."""
    rng = np.random.RandomState(seed)
    base = np.kron(rng.randint(0, 256, (n, h // 32 + 1, w // 32 + 1, 3)), np.ones((1, 32, 32, 1)))[:, :h, :w]
    return np.clip(base + rng.randint(-30, 31, base.shape), 0, 255).astype(np.uint8)


def test_fid_inception_matches_fp64_oracle(fid_sd, fid_net):
    oracle = fo.fid_network(fid_sd, pooling="fid")
    u8 = torch.from_numpy(_images(2, 341, 256, 7)).cuda()
    f32 = (u8.cpu().permute(0, 3, 1, 2).float() / 255).cuda()  # the same values as fp32 NCHW (a CPU division rounds as TF.to_tensor)
    for label, x in (("uint8 341x256", u8), ("fp32 341x256", f32)):
        with torch.no_grad():
            pool, logits, kept = fid_net.run(x, keep=io_.TAPS)
        taps, ref_pool, ref_logits = fo.fp64_forward(oracle, x)
        for name, got, ref in [(t, _nchw(kept[t]), taps[t]) for t in io_.TAPS] + [("pool", pool, ref_pool), ("logits", logits, ref_logits)]:
            assert float(ref.abs().max()) > 0.1
            r = _ratio(got, ref)
            print("PARITY fid_inception[%s] %s max|d|/max|ref| = %.3e (bound 1e-4)" % (label, name, r))
            assert got.shape == ref.shape and r <= 1e-4, (label, name, r)
        p2, l2 = fid_net(x)
        assert torch.equal(p2, pool) and torch.equal(l2, logits)
    # the same weights through from_torchvision (count_include_pad=True averages, max-free Mixed_7c) miss the bound at Mixed_5d
    tv = metrics.InceptionV3.from_torchvision(metrics.fid_inception_model(fid_sd).cuda())
    with torch.no_grad():
        _, _, kept_tv = tv.run(f32, unit_range=True, keep=io_.TAPS)
    taps, _, _ = fo.fp64_forward(oracle, f32)
    r = _ratio(_nchw(kept_tv["Mixed_5d"]), taps["Mixed_5d"])
    print("PARITY fid_inception[from_torchvision, same weights] Mixed_5d max|d|/max|ref| = %.3e (misses 1e-4)" % r)
    assert r > 1e-2, r


def test_fid_inception_reproducible(fid_net):
    a = torch.from_numpy(_images(7, 256, 192, 8)).cuda()
    b = torch.from_numpy(_images(7, 256, 192, 9)).cuda()
    prec = ops.get_precision()
    runs = []
    try:
        for p in ("fp32", "bf16", "fp32"):
            ops.set_precision(p)
            with torch.no_grad():
                fa, la = fid_net(a)
                fb, _ = fid_net(b)
                one, l1 = fid_net(a[3:4].clone())
                sa, sb = metrics.FeatureStats().update(fa), metrics.FeatureStats().update(fb)
                runs.append((fa, la, one, l1, metrics.fid(sa, sb), metrics.kid(fa, fb, subsets=5, subset_size=4)))
    finally:
        ops.set_precision(prec)
    fa, la, one, l1, f, (km, ks) = runs[0]
    assert torch.equal(one, fa[3:4]) and torch.equal(l1, la[3:4])  # one image alone = the same image in a batch of 7
    assert float(f) > 0 and bool(torch.isfinite(km))
    for fa2, la2, _, _, f2, (km2, ks2) in runs[1:]:
        assert torch.equal(fa2, fa) and torch.equal(la2, la)
        assert torch.equal(f2, f) and torch.equal(km2, km) and torch.equal(ks2, ks)


def test_fid_inception_refusals(fid_net):
    before = ops.LAUNCHES[0]
    u8 = torch.zeros((1, 64, 64, 3), dtype=torch.uint8, device="cuda")
    with pytest.raises(ValueError):
        fid_net(u8.permute(0, 3, 1, 2).contiguous())  # uint8 must be (N,H,W,3)
    with pytest.raises(ValueError):
        fid_net(u8.float())  # fp32 must be (N,3,H,W)
    with pytest.raises(ValueError):
        fid_net(u8, unit_range=True)
    with pytest.raises(RuntimeError):
        fid_net(u8.cpu())
    assert ops.LAUNCHES[0] == before


def _write_folder(path, imgs):
    from PIL import Image
    path.mkdir()
    for i, im in enumerate(imgs):
        Image.fromarray(im).save(str(path / ("%05d_00.png" % i)))
    return str(path)


def test_fid_tool_on_folders(fid_sd, fid_net, tmp_path, capsys):
    from PIL import Image
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    try:
        import fid as fid_tool
    finally:
        sys.path.pop(0)
    a = _write_folder(tmp_path / "a", _images(64, 1024, 768, 10))
    b = _write_folder(tmp_path / "b", np.clip(_images(64, 1024, 768, 11).astype(np.int32) * 9 // 10 + 20, 0, 255).astype(np.uint8))
    weights = str(tmp_path / "pt_inception.pth")
    torch.save(fid_sd, weights)
    feats, oracle_feats = [], []
    oracle = fo.fid_network(fid_sd, pooling="fid")
    for folder in (a, b):
        files = fid_tool.image_files(folder)
        assert len(files) == 64
        decoded = torch.from_numpy(np.stack([np.asarray(Image.open(f).convert("RGB")) for f in files]))
        with torch.no_grad():
            got = fid_tool.folder_features(files, fid_net, batch_size=50, workers=2)
            direct = torch.cat([fid_net(decoded[i:i + 16].cuda())[0] for i in range(0, 64, 16)])
        assert torch.equal(got, direct)  # the tool's decode and batching change nothing
        feats.append(got)
        oracle_feats.append(torch.cat([fo.fp64_forward(oracle, decoded[i:i + 8])[1] for i in range(0, 64, 8)]).numpy())
    res = fid_tool.main([a, b, "--weights", weights, "--workers", "2", "--save-stats", str(tmp_path / "a.npz")])
    assert "FID:" in capsys.readouterr().out
    mom = [(f.mean(0), np.cov(f, rowvar=False)) for f in oracle_feats]
    ref = io_.fid_np(mom[0][0], mom[0][1], mom[1][0], mom[1][1])
    rel = abs(res["fid"] - ref) / ref
    print("PARITY fid_tool |FID - fp64 oracle FID| / FID = %.3e (bound 1e-3; FID = %.6f, %s)" % (rel, ref, res))
    assert rel <= 1e-3, (res["fid"], ref)
    res2 = fid_tool.main([str(tmp_path / "a.npz"), b, "--weights", weights, "--workers", "2"])
    assert res2["fid"] == res["fid"]
    sa, sb = metrics.FeatureStats().update(feats[0]), metrics.FeatureStats().update(feats[1])
    assert float(metrics.fid(sa, sb)) == res["fid"]  # fid_of_moments on the same moments: the same bits
