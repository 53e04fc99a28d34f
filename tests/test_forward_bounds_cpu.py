"""The per-element bound of tests/test_forward_kernels_gpu.py must be tight enough to matter: at the shapes those tests use, it accepts
the correctly rounded fp64 reference and rejects the realistic mistakes a forward kernel makes, each of which the max-norm
rel_err < 1e-2 of the older tests accepts.  CPU only (fp64 references)."""
import pytest
import torch
import torch.nn.functional as F

import test_forward_kernels_gpu as fk
from hrviton_b200 import ops
from hrviton_b200.ops import ACT_LRELU


@pytest.fixture(params=["bf16", "fp16"])
def precision(request):
    ops.set_precision(request.param)
    yield request.param
    ops.set_precision("bf16")


def accepted(got, ref, S, u):
    return fk.excess(got, ref, S, u) <= 1.0


def store(ref, out):
    """The correctly rounded output a kernel would store: the storage type for 16-bit outputs, fp32 otherwise."""
    return fk.q(ref) if out == "slice" else ref.float().double()


def caught(wrong, ref, S, u):
    """The per-element bound rejects `wrong`, and the max-norm of the older tests lets it through."""
    return not accepted(wrong, ref, S, u) and fk.rel_err(wrong, ref) < 1e-2


# ------------------------------------------------------------------------------------------------ convolution, LINEAR


@pytest.mark.parametrize("case", fk.CONV_CASES, ids=lambda c: c[0])
def test_correctly_rounded_conv_output_passes(case, precision):
    out = case[9]
    ref, S = fk.conv_ref(case, fk.conv_inputs(case))
    assert accepted(store(ref, out), ref, S, fk.U16[precision] if out == "slice" else 0.0)


WIDE_CASES = [c for c in fk.CONV_CASES if c[3] >= 32 and c[9] == "slice"]


@pytest.mark.parametrize("case", WIDE_CASES, ids=lambda c: c[0])
def test_bound_rejects_a_zeroed_or_stale_low_magnitude_group(case, precision):
    """One 8-channel group of the smallest channels zeroed, or holding another image's (another row's) values: under 1 % of the
    tensor's largest value, so only a per-element bound sees it."""
    u = fk.U16[precision]
    ref, S = fk.conv_ref(case, fk.conv_inputs(case))
    c = ref.shape[1]
    g0 = (c // 8 - 1) * 8  # the last full group: the smallest channels
    good = fk.q(ref)
    assert accepted(good, ref, S, u)
    wrong = good.clone()
    wrong[:, g0:g0 + 8] = 0
    assert caught(wrong, ref, S, u), "zeroed group"
    wrong = good.clone()
    wrong[:, g0:g0 + 8] = good[:, g0:g0 + 8].roll(1, 0) if ref.shape[0] > 1 else good[:, g0:g0 + 8].roll(1, 2)
    assert caught(wrong, ref, S, u), "stale group"


LRELU_SHIFT_CASES = [c for c in fk.CONV_CASES if c[7] == ACT_LRELU and c[8] in ("shift", "scale") and c[9] == "slice"]


@pytest.mark.parametrize("case", LRELU_SHIFT_CASES, ids=lambda c: c[0])
def test_bound_rejects_the_shift_after_the_activation(case, precision):
    """act(v) + shift instead of act(v + shift), with a bias small enough (2 % of the test's) that the max-norm accepts it."""
    u = fk.U16[precision]
    d = fk.conv_inputs(case)
    d["shift"] = d["shift"] * 0.02
    ref, S = fk.conv_ref(case, d)
    no_shift, _ = fk.conv_ref(case, dict(d, shift=None))  # act(conv * scale)
    wrong = fk.q(no_shift + d["shift"][None, :, None, None])
    assert accepted(fk.q(ref), ref, S, u)
    assert caught(wrong, ref, S, u)


# ------------------------------------------------------------------------------------------------ convolution, SPADE


def spade_stats(case, d):
    """fp32 InstanceNorm statistics of cat(up2^shift(x0), x1) + noise * noise_scale, from fp64 sums (what the kernel returns)."""
    name, n, cin, c0, c1, H, W, shift, nsc, act = case
    xs = fk.nearest_up(d["x0"], shift)
    if d["x1"] is not None:
        xs = torch.cat([xs, d["x1"]], 1)
    z = xs + d["noise"][:, None] * d["ns"][None, :, None, None] if d["noise"] is not None else xs
    return z.mean((2, 3)).float().double(), (z.var((2, 3), unbiased=False) + fk.EPS_NORM).rsqrt().float().double()


@pytest.mark.parametrize("case", fk.SPADE_CASES, ids=lambda c: c[0])
def test_bound_rejects_gamma_rounded_before_the_modulation(case, precision):
    """gamma rounded to 16 bits (as if read back from gamma_out) before xn * (1 + gamma): a second rounding the output must not carry."""
    u = fk.U16[precision]
    d = fk.spade_inputs(case)
    mean, rstd = spade_stats(case, d)
    ref = fk.spade_ref(case, d, mean, rstd)
    out, So = ref["out"]
    gamma, Sg = ref["gamma"]
    assert accepted(fk.q(out), out, So, u) and accepted(fk.q(gamma), gamma, Sg, u)
    m, r = mean[:, :, None, None], rstd[:, :, None, None]
    xs = fk.nearest_up(d["x0"], case[7])
    if d["x1"] is not None:
        xs = torch.cat([xs, d["x1"]], 1)
    nz = d["noise"][:, None] * d["ns"][None, :, None, None] if d["noise"] is not None else 0.0
    beta = F.conv2d(d["actv"], d["wb"], d["bb"], padding=1)
    wrong = fk.q(fk.act_fwd((xs + nz - m) * r * (1 + fk.q(gamma)) + beta, case[9]))
    assert caught(wrong, out, So, u)


NOISY = [c for c in fk.SPADE_CASES if c[8] is not None and c[8] <= 1e-2]


@pytest.mark.parametrize("case", NOISY, ids=lambda c: c[0])
def test_bound_rejects_a_dropped_noise_term(case, precision):
    """The SPADE noise term left out of the modulation at noise_scale = 1e-2 on unit-variance features (the statistics still include
    it).  Without the magnitude spread: in a channel of std 1e-3 the same term would be the whole signal and the max-norm sees it too."""
    u = fk.U16[precision]
    d = fk.spade_inputs(case)
    g = fk.gen(51)
    d["x0"] = fk.q(torch.randn(d["x0"].shape, generator=g))
    d["x1"] = fk.q(torch.randn(d["x1"].shape, generator=g))
    d["ns"] = torch.full_like(d["ns"], 1e-2)
    mean, rstd = spade_stats(case, d)
    out, So = fk.spade_ref(case, d, mean, rstd)["out"]
    wrong = fk.q(fk.spade_ref(case, dict(d, noise=None, ns=None), mean, rstd)["out"][0])
    assert caught(wrong, out, So, u)


def test_bound_rejects_the_previous_images_statistics(precision):
    """A tile over three 4x4 images that keeps image 0's mean / rstd for image 1.  Image 1 is image 0 shifted by 1e-3 of each
    channel's spread, so the two sets of statistics differ only slightly and the max-norm accepts the mix-up."""
    u = fk.U16[precision]
    case = next(c for c in fk.SPADE_CASES if c[0] == "c80_half_x1_3img")
    d = fk.spade_inputs(case)
    for k in ("x0", "x1"):
        x = d[k].clone()
        x[1] = x[0] + 1e-3 * x[0].std((1, 2), keepdim=True)
        d[k] = x
    mean, rstd = spade_stats(case, d)
    out, So = fk.spade_ref(case, d, mean, rstd)["out"]
    assert accepted(fk.q(out), out, So, u)
    m2, r2 = mean.clone(), rstd.clone()
    m2[1], r2[1] = mean[0], rstd[0]
    wrong = fk.q(fk.spade_ref(case, d, m2, r2)["out"][0])
    assert caught(wrong, out, So, u)
