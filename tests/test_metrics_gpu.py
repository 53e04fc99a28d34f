"""GPU: the evaluation-metric kernels against exact references, the drop-in LPIPS against the live reference's numbers
(tests/golden/lpips_alex.npz), and the reference's own evaluate.Evaluation run unchanged on the package.

- hrv_maxpool3s2: bit-exact against torch; hrv_lpips_input: bit-exact against torch's scaling + unfold; hrv_lpips_dist: within
  64*2^-24*S of an fp64 computation on the same fp32 features (S = the pixel mean of sum_c w_c (|f0_c| + |f1_c|)^2, the magnitude the
  result is formed from; the per-element rule of test_forward_kernels_gpu.py).  Every written value is checked against a NaN sentinel.
- hrv_ssim: within 1e-10 absolute of the float64 restatement (tests/metrics_oracle.py) on uint8 and fp32 images with flat, textured
  and saturated regions, at 1024x768, odd sizes and in a batch.
- PerceptualLoss: |delta| < 1e-4 on every per-layer distance and the total, exactly 0 for an identical pair, with ops precision bf16
  (the metric runs in fp32 storage whatever the training precision)."""
import contextlib
import ctypes
import io
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from helpers import GOLDEN
import metrics_oracle as mo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import make_golden_lpips as mgl  # noqa: E402  (seeded weights and inputs of the fixture)

from hrviton_b200 import capi, metrics, ops  # noqa: E402

pytestmark = pytest.mark.gpu
U = 2.0 ** -24


def _nan_act(n, h, w, c, pitch):
    return ops.Act(torch.full((n, h, w, pitch), float("nan"), device="cuda"), c=c)


def test_maxpool3s2_bit_exact():
    g = torch.Generator(device="cuda").manual_seed(1)
    for n, h, w, c, pitch in ((2, 31, 31, 64, 64), (3, 14, 21, 192, 200), (1, 7, 3, 8, 8)):
        x = torch.randn((n, h, w, pitch), generator=g, device="cuda").relu()
        x[..., : c // 2] = torch.round(x[..., : c // 2] * 2) / 2  # ties
        xa = ops.Act(x, c=c)
        ho, wo = (h - 3) // 2 + 1, (w - 3) // 2 + 1
        y = _nan_act(n, ho, wo, c, pitch)
        tx, ty = xa.ct(), y.ct()
        capi.check(capi.lib().hrv_maxpool3s2(ctypes.byref(tx), ctypes.byref(ty), ops._stream()), "maxpool3s2")
        ref = F.max_pool2d(x[..., :c].permute(0, 3, 1, 2), 3, 2).permute(0, 2, 3, 1)
        assert torch.equal(y.buf[..., :c], ref)
        assert bool(torch.isnan(y.buf[..., c:]).all())  # the pitch's pad channels are not written
        assert torch.equal(ops.maxpool3s2(xa).buf[..., :c], ref)
    # a NaN wins its windows, as in torch (a comparison `v > m` alone would drop it)
    x = torch.rand((1, 9, 9, 8), generator=g, device="cuda")
    x[0, 4, 4, 3] = float("nan")
    x[0, 0, 8, 5] = float("nan")
    y = ops.maxpool3s2(ops.Act(x)).buf
    ref = F.max_pool2d(x.permute(0, 3, 1, 2), 3, 2).permute(0, 2, 3, 1)
    assert int(torch.isnan(ref).sum()) == 5 and torch.equal(torch.isnan(y), torch.isnan(ref))
    assert torch.equal(y.nan_to_num(-1.0), ref.nan_to_num(-1.0))


def test_lpips_input_bit_exact():
    g = torch.Generator(device="cuda").manual_seed(2)
    shift = torch.tensor([-.030, -.088, -.188], device="cuda")
    scale = torch.tensor([.458, .448, .450], device="cuda")
    for n, h, w in ((2, 128, 128), (3, 96, 161), (1, 7, 9)):
        x = torch.rand((n, 3, h, w), generator=g, device="cuda") * 2 - 1
        ho, wo = (h - 7) // 4 + 1, (w - 7) // 4 + 1
        dst = _nan_act(n, ho, wo, ops.LPIPS_K, 368)
        t = dst.ct()
        capi.check(capi.lib().hrv_lpips_input(x.data_ptr(), n, h, w, shift.data_ptr(), scale.data_ptr(), ctypes.byref(t), ops._stream()), "lpips_input")
        scaled = (x - shift.view(1, 3, 1, 1)) / scale.view(1, 3, 1, 1)
        cols = F.unfold(scaled, 11, padding=2, stride=4)  # (n, 3*121 in (ci, ky, kx) order, L)
        ref = cols.view(n, 3, 121, ho, wo).permute(0, 3, 4, 2, 1).reshape(n, ho, wo, 363)
        assert torch.equal(dst.buf[..., :363], ref)
        assert bool((dst.buf[..., 363:] == 0).all())  # pad channels written as zeros


def test_lpips_dist_within_fp64_bound():
    g = torch.Generator(device="cuda").manual_seed(3)
    for npair, h, w, c in ((4, 31, 31, 64), (2, 14, 14, 192), (3, 6, 6, 384), (1, 6, 7, 256)):
        f = torch.randn((2 * npair, h, w, c), generator=g, device="cuda").relu()
        f[0, 0, 0] = 0.0  # an all-zero pixel: norm 0, normalised to 0
        wl = torch.rand(c, generator=g, device="cuda") * 0.1
        out = torch.full((npair,), float("nan"), device="cuda")
        t = ops.Act(f).ct()
        capi.check(capi.lib().hrv_lpips_dist(ctypes.byref(t), wl.data_ptr(), out.data_ptr(), ops._stream()), "lpips_dist")
        fd, wd = f.double(), wl.double()
        nrm = fd / (fd.pow(2).sum(-1, keepdim=True).sqrt() + 1e-10)
        f0, f1 = nrm[:npair], nrm[npair:]
        ref = ((f0 - f1) ** 2 * wd).sum(-1).mean((1, 2))
        S = ((f0.abs() + f1.abs()) ** 2 * wd).sum(-1).mean((1, 2))
        assert bool(torch.isfinite(out).all())
        assert bool(((out.double() - ref).abs() <= 64 * U * S).all()), ((out.double() - ref).abs() / S / U).max()


def _gray(h, w, seed):
    rng = np.random.RandomState(seed)
    a = rng.randint(0, 256, (h, w)).astype(np.uint8)  # textured
    a[: h // 4, : w // 4] = 255                        # saturated
    a[h // 2:, w // 2:] = 90                           # flat
    b = np.clip(a.astype(np.int32) + rng.randint(-25, 26, (h, w)), 0, 255).astype(np.uint8)
    b[h // 2:, w // 2:] = 90                           # flat in both
    b[: h // 8, : w // 8] = 0
    return a, b


def test_ssim_matches_float64_restatement():
    for (h, w) in ((1024, 768), (37, 53), (11, 11), (129, 200)):
        a, b = _gray(h, w, h + w)
        ref = mo.ssim(a, b)
        got = metrics.ssim(a, b)
        assert isinstance(got, np.ndarray) and got.dtype == np.float64
        assert abs(float(got) - ref) < 1e-10, (h, w, float(got), ref)
        got32 = metrics.ssim(torch.from_numpy(a).float().cuda(), torch.from_numpy(b).float().cuda())
        assert got32.dtype == torch.float64 and abs(float(got32) - ref) < 1e-10
        assert abs(float(metrics.ssim(a, a)) - 1.0) < 1e-12
    pairs = [_gray(61, 47, s) for s in range(5)]
    A = torch.from_numpy(np.stack([p[0] for p in pairs])).cuda()
    B = torch.from_numpy(np.stack([p[1] for p in pairs])).cuda()
    got = metrics.ssim(A, B)
    assert got.shape == (5,)
    for i, (a, b) in enumerate(pairs):
        assert abs(float(got[i]) - mo.ssim(a, b)) < 1e-10
    with pytest.raises(ValueError):
        metrics.ssim(A[:, :10], B[:, :10])
    # every written value against a NaN sentinel, at the C-ABI
    n, h, w = A.shape
    out = torch.full((n + 1,), float("nan"), dtype=torch.float64, device="cuda")
    nws = int(capi.lib().hrv_ssim_workspace_bytes(n, h, w))
    ws = torch.full((nws // 8,), float("nan"), dtype=torch.float64, device="cuda")
    capi.check(capi.lib().hrv_ssim(A.data_ptr(), B.data_ptr(), capi.SSIM_U8, n, h, w, 255.0, out.data_ptr(), ws.data_ptr(), nws,
                                   ops._stream()), "ssim")
    assert bool(torch.isfinite(out[:n]).all()) and bool(torch.isnan(out[n]))  # exactly the n outputs are written
    assert torch.equal(out[:n], got)


def _weights_dir(tmp_path):
    net = metrics.PNetLin(pretrained=False)
    sd = mgl.seeded_state_dict(net.state_dict())
    d = tmp_path / "eval_models" / "weights" / "v0.1"
    d.mkdir(parents=True)
    torch.save(sd, str(d / "alex.pth"))
    return sd, str(d / "alex.pth")


def test_perceptual_loss_matches_reference_fixture(tmp_path, monkeypatch):
    import eval_models
    gold = np.load(os.path.join(GOLDEN, "lpips_alex.npz"))
    sd, _ = _weights_dir(tmp_path)
    sums = np.array([float(v.double().sum()) for v in sd.values()])
    # the fixture's weights, rebuilt (the fp64 sums themselves may differ in the last bits with the host's summation order)
    assert list(sd.keys()) == list(gold["sd_keys"]) and np.allclose(sums, gold["sd_sums"], rtol=1e-12, atol=1e-12 * gold["sd_abs_sums"])
    monkeypatch.setenv("HRV_ALEX_RANDOM_INIT", "1")
    monkeypatch.chdir(tmp_path)
    with contextlib.redirect_stdout(io.StringIO()):
        pl = eval_models.PerceptualLoss(model="net-lin", net="alex", use_gpu=True)
    prec = ops.get_precision()
    ops.set_precision("bf16")
    try:
        with torch.no_grad():
            for name in mgl.CASES:
                in0 = mgl.to_input(gold[name + "_in0"]).cuda()
                in1 = mgl.to_input(gold[name + "_in1"]).cuda()
                val, res = pl.net(in0, in1, retPerLayer=True)
                tot = pl.forward(in1, in0)  # PerceptualLoss.forward(pred, target) runs net(target, pred)
                assert tot.shape == (in0.shape[0], 1, 1, 1) and tot.dtype == torch.float32
                assert torch.equal(tot, val)
                got_res = torch.stack([r.reshape(-1) for r in res]).cpu().numpy()
                if name.startswith("same"):
                    assert float(np.abs(got_res).max()) == 0.0 and float(tot.abs().max()) == 0.0
                assert np.abs(got_res - gold[name + "_res"]).max() < 1e-4, name
                assert np.abs(tot.reshape(-1).cpu().numpy() - gold[name + "_val"]).max() < 1e-4, name
                with torch.enable_grad(), pytest.raises(NotImplementedError):
                    pl.forward(in1.clone().requires_grad_(True), in0)
    finally:
        ops.set_precision(prec)


def test_reference_evaluate_runs_unchanged(tmp_path, monkeypatch):
    """evaluate.Evaluation from the reference copy, unmodified, on synthetic JPEG pairs: `eval_models` and skimage's SSIM bind to this
    package.  The same call with the reference's own eval_models on torch and the float64 SSIM restatement is the comparison.  The
    Inception and AlexNet ImageNet weights are replaced by seeded ones and alex.pth by the seeded fixture weights: nothing is downloaded."""
    import hrv_env
    from PIL import Image
    if hrv_env.reference_dir() is None:
        pytest.skip("no reference copy (oracle/_ref)")
    import torchvision
    monkeypatch.setenv("HRV_ALEX_RANDOM_INIT", "1")
    monkeypatch.chdir(tmp_path)
    _, alex = _weights_dir(tmp_path)
    gt_dir, pred_dir = tmp_path / "gt", tmp_path / "pred"
    gt_dir.mkdir()
    pred_dir.mkdir()
    rng = np.random.RandomState(5)
    for i in range(3):
        base = np.kron(rng.randint(0, 256, (32, 24, 3)), np.ones((8, 8, 1)))
        Image.fromarray(np.clip(base + rng.randint(-10, 11, base.shape), 0, 255).astype(np.uint8)).save(str(gt_dir / ("%05d_00.jpg" % i)), quality=90)
        Image.fromarray(np.clip(base + rng.randint(-40, 41, base.shape), 0, 255).astype(np.uint8)).save(str(pred_dir / ("%05d_00.jpg" % i)), quality=90)
    names = sorted(os.listdir(str(gt_dir)))

    def inception(pretrained=True, transform_input=False):
        torch.manual_seed(0)
        return torchvision.models.inception_v3(weights=None, aux_logits=True, init_weights=True, transform_input=transform_input)

    import types
    opt = types.SimpleNamespace(predict_dir=str(pred_dir), ground_truth_dir=str(gt_dir), resolution=1024)
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    ev = hrv_env.load_reference_script("evaluate", alias="ref_evaluate_pkg")
    import eval_models
    assert ev.models is eval_models and ev.ssim.__module__ == "skimage.metrics"
    ev.inception_v3 = inception
    with contextlib.redirect_stdout(io.StringIO()):
        ours = ev.Evaluation(opt, list(names), list(names))

    # the same call on the reference's own eval_models (torch / cuDNN) and the float64 SSIM restatement
    ev2 = hrv_env.load_reference_script("evaluate", alias="ref_evaluate_torch")
    ev2.inception_v3 = inception
    ev2.ssim = lambda a, b, data_range, gaussian_weights, use_sample_covariance: mo.ssim(a, b, data_range)
    with mo.reference_eval_models(alex) as ref_models, contextlib.redirect_stdout(io.StringIO()):
        ev2.models = ref_models
        ref = ev2.Evaluation(opt, list(names), list(names))
    ssim_o, mse_o, lp_o, is_o, isd_o = ours
    ssim_r, mse_r, lp_r, is_r, isd_r = ref
    assert abs(ssim_o - ssim_r) < 1e-10
    assert abs(float(lp_o) - float(lp_r)) < 1e-4 and float(lp_o) > 0
    assert float(mse_o) == float(mse_r)
    assert is_o == is_r and isd_o == isd_r


def test_reference_train_generator_lpips_branch(tmp_path, monkeypatch):
    """The reference's train_generator.train(), unmodified, runs its LPIPS branch (train_generator.py:480-584: --lpips_count hit once
    after one step, 500 test try-ons, each scored by model.forward(T2(im), T2(output))) with the drop-in PerceptualLoss in place of the
    _Lpips stand-in of test_reference_scripts_gpu.py.  The value it prints is finite and equals PerceptualLoss on the same outputs,
    accumulated as the script does."""
    import hrv_env
    if hrv_env.reference_dir() is None:
        pytest.skip("no reference copy (oracle/_ref)")
    import eval_models
    import network_generator
    import networks
    from test_reference_scripts_gpu import _Loader, _opt
    monkeypatch.setenv("HRV_ALEX_RANDOM_INIT", "1")
    monkeypatch.chdir(tmp_path)
    _weights_dir(tmp_path)
    tg = hrv_env.load_reference_script("train_generator")
    assert tg.models is eval_models
    h, w = 512, 384
    opt = _opt(tg, ["--name", "t", "--cuda", "True", "--gpu_ids", "0", "-b", "1", "--fine_height", str(h), "--fine_width", str(w), "--keep_step", "1",
                    "--decay_step", "0", "--display_count", "1000", "--save_count", "1000", "--tensorboard_count", "1000", "--lpips_count", "1",
                    "--occlusion"])
    torch.manual_seed(0)
    tocg = networks.ConditionGenerator(opt, input1_nc=4, input2_nc=opt.semantic_nc + 3, output_nc=13, ngf=96, norm_layer=torch.nn.BatchNorm2d)
    generator = network_generator.SPADEGenerator(opt, 9)
    generator.cuda()
    generator.init_weights(opt.init_type, opt.init_variance)
    out = io.StringIO()
    with contextlib.redirect_stdout(out):
        discriminator = tg.create_network(network_generator.MultiscaleDiscriminator, opt)
        model = eval_models.PerceptualLoss(model="net-lin", net="alex", use_gpu=True)  # as train_generator.py:651 builds it
    calls = []
    forward = model.forward

    def recording_forward(pred, target, normalize=False):
        calls.append((pred.clone(), target.clone()))
        return forward(pred, target, normalize)

    model.forward = recording_forward
    scalars = {}

    class Board(tg.SummaryWriter):  # the script's writer, recording what it logs: the exact value behind the print
        def add_scalar(self, tag, value, step=None, *a, **k):
            scalars[tag] = value

    loader = _Loader(1, h, w)
    with contextlib.redirect_stdout(out):
        tg.train(opt, loader, loader, None, Board(log_dir="unused"), tocg, generator, discriminator, model)
    torch.cuda.synchronize()
    lines = [l for l in out.getvalue().splitlines() if l.startswith("LPIPS") and l != "LPIPS"]
    assert len(lines) == 1 and len(calls) == 500, (lines, len(calls))
    logged = scalars["test/LPIPS"]
    assert bool(torch.isfinite(logged).all()) and float(logged) > 0
    with torch.no_grad():  # PerceptualLoss on the same outputs, accumulated as train_generator.py:578-580 does
        avg = 0.0
        for pred, target in calls:
            avg += forward(pred, target)
        avg = avg / 500
    assert torch.equal(logged, avg)
    assert lines[0] == f"LPIPS{avg}"
