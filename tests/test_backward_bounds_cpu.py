"""The per-element bound of tests/test_backward_kernels_gpu.py must be tight enough to matter: at the shapes those tests use, it
accepts the correctly rounded result and rejects the realistic mistakes a backward kernel makes.  CPU only (fp64 references)."""
import pytest
import torch
import torch.nn.functional as F

import test_backward_kernels_gpu as bk
from hrviton_b200 import ops


@pytest.fixture(params=["bf16", "fp16"])
def precision(request):
    ops.set_precision(request.param)
    yield request.param
    ops.set_precision("bf16")


def accepted(got, ref, S, u=0.0, extra=None):
    return bk.excess(got, ref, S, u, extra) <= 1.0


@pytest.mark.parametrize("shape", bk.UP2_SHAPES, ids=lambda s: "n%d_c%d_%dx%d" % s)
def test_bound_rejects_a_wrong_border_weight(shape, precision):
    """bilinear x2 backward: the first low-res row folds the clamped high-res row 0 in with weight 1.0; 0.75 (the interior weight)
    there must fail."""
    n, c, h, w = shape
    u = bk.U16[precision]
    dout = bk.q(bk.rnd(bk.gen(18), n, c, 2 * h, 2 * w))
    ref, S = bk.up2_bwd_ref(dout)
    assert accepted(bk.q(ref), ref, S, u)
    a = torch.zeros((n, c, 1, w), dtype=torch.float64, requires_grad=True)
    row0, = torch.autograd.grad(F.interpolate(a, scale_factor=(1, 2), mode="bilinear", align_corners=False), a, dout[:, :, 0:1])
    wrong = ref.clone()
    wrong[:, :, 0:1] -= 0.25 * row0  # high-res row 0 taken with weight 0.75 instead of 1.0
    assert not accepted(bk.q(wrong), ref, S, u)
    wrong = ref.clone()
    wrong[..., -1:] = ref[..., -1:] * 0.75  # or the last column scaled by the interior weight
    assert not accepted(bk.q(wrong), ref, S, u)


def cpu_norm_case(case):
    n, c0, c1, H, W, shift, act, with_noise, _ = case
    u = bk.U16[ops.get_precision()]
    d = bk.spade_norm_inputs(11, n, c0, c1, H, W, shift, act, with_noise)
    xs = bk.nearest_up(d["x0"], shift)
    if d["x1"] is not None:
        xs = torch.cat([xs, d["x1"]], 1)
    z = xs + d["noise"][:, None] * d["ns"][None, :, None, None] if with_noise else xs
    mean = z.mean((2, 3)).float().double()
    rstd = (z.var((2, 3), unbiased=False) + bk.EPS_NORM).rsqrt().float().double()
    h = bk.spade_forward_h(d, shift, mean, rstd, act)
    return bk.norm_bwd_ref(d["dh"], h, d["gamma"], d["x0"], shift, d["x1"], d["noise"], d["ns"], mean, rstd, act, u), u


def dx0_varies(case):
    n, c0, c1, H, W, shift = case[:6]
    return (H >> shift) * (W >> shift) > 1


@pytest.mark.parametrize("case", bk.NORM_CASES,ids=lambda c: "n%d_c%d+%d_%dx%d_s%d_a%d_nz%d_p%s" % c)
def test_bound_rejects_norm_bwd_mistakes(case, precision):
    """SPADE norm backward: gamma and beta swapped in the interleaved d(gamma|beta), the x1 slice of d noise_scale dropped, one
    8-channel group of dx0 zeroed."""
    ref, u = cpu_norm_case(case)
    c0 = case[1]
    (dg, Sg, _), (db, Sb, _) = ref["dgamma"], ref["dbeta"]
    assert accepted(bk.q(dg), dg, Sg, u) and accepted(bk.q(db), db, Sb, u)
    assert not (accepted(bk.q(db), dg, Sg, u) and accepted(bk.q(dg), db, Sb, u))  # swapped interleave
    # a 1x1 x0 under a 2x2 map gathers every pixel: its InstanceNorm gradient sums to zero, so look at dx1 there
    dx, S0, e0 = ref["dx0"] if dx0_varies(case) else ref["dx1"]
    assert accepted(bk.q(dx), dx, S0, u, e0)
    wrong = bk.q(dx)
    grp = 8 if dx.shape[1] > 8 else 0
    wrong[:, grp:grp + 8] = 0
    assert not accepted(wrong, dx, S0, u, e0)
    if "dns" in ref:
        dns, Sn, en = ref["dns"]
        assert accepted(dns.float(), dns, Sn, 0.0, en)
        if "dx1" in ref:
            wrong = dns.clone()
            wrong[c0:] = 0
            assert not accepted(wrong.float(), dns, Sn, 0.0, en)


@pytest.mark.parametrize("case", bk.DGRAD_CASES, ids=lambda c: c[0])
def test_bound_rejects_a_zeroed_channel_group(case, precision):
    """Data-gradient convolution: one 8-channel group of the output zeroed must fail."""
    name, n, cin, cout, H, W, k, pad, crop, pitch, gate, form = case
    u = bk.U16[precision]
    g = bk.gen(15)
    oh, ow = (H + 2 * pad - k + 1, W + 2 * pad - k + 1) if crop is None else crop
    kc = 2 * cout if form == "interleave" else cout
    kk = 1 if form == "im2col" else k
    w = bk.q(bk.rnd(g, kc, cin, kk, kk, scale=(1.0 / (kc * kk * kk)) ** 0.5))
    dy = bk.q(bk.rnd(g, n, kc, oh, ow))
    ref, S = bk.dgrad_ref((n, cin, H, W), w, dy, pad)
    assert accepted(bk.q(ref), ref, S, u)
    wrong = bk.q(ref)
    grp = 8 if cin > 8 else 0
    wrong[:, grp:grp + 8] = 0
    assert not accepted(wrong, ref, S, u)
