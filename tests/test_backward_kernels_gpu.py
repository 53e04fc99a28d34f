"""Every training backward entry point, one at a time, against torch autograd in float64 on the CPU, in both 16-bit storage flavours.

Each reference differentiates the forward op the kernel differentiates, applied to the exact 16-bit values the kernel read: stored
activations, gamma and saved outputs are read back from the device, mean/rstd are the kernel's own statistics (the backward kernels
take them as inputs), and the activation derivative is evaluated at the stored output h, as the kernels do.

The bound is per element and derived from the accumulation, not tuned.  With S the same fp64 linear map applied to absolute values
(for a convolution conv(|x|, |w|), the sum |x||w| of the fp32 tests):
  16-bit outputs             |got - ref| <= u*|ref| + K_ACC * 2^-24 * S     u = 2^-8 (bf16), 2^-11 (fp16): one rounding of the result
                                               (+ 2^-24 in fp16, one subnormal step: below 2^-14 its rounding is absolute)
  fp32 / fp64 outputs        |got - ref| <= K_ACC * 2^-24 * S
Where a kernel stores an intermediate in 16 bits between two passes (dxn between the two InstanceNorm backward passes), the same
linear map applied to that intermediate's absolute value, times u, is added: it is the rounding the output inherits.

K_ACC: every kernel sums in fp32 per thread (or in the fp32 wgmma accumulators) and combines threads, blocks and split-K slabs in
fp64 or in a fixed fp32 order.  The longest fp32 chain below has fewer than 64^2 = 4096 additions (the 18720-deep K loop of the
1040-channel gamma|beta data gradient is 1170 wgmma steps, the 18200-pixel weight gradient 1138), each rounded to nearest or, in the
tensor cores, truncated.  Such a chain over terms of mixed sign drifts by about sqrt(m) units of 2^-24 * S, at most 64 here; the fp64
combination adds nothing visible at this scale.  tests/test_backward_bounds_cpu.py shows that the bound still rejects the realistic
mistakes (a border weight, a gamma/beta swap, a dropped channel slice, a zeroed 8-channel group) at these shapes."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "..", "oracle"))
import hrviton_oracle as orc  # noqa: E402
from hrviton_b200 import capi, ops  # noqa: E402
from hrviton_b200.ops import ACT_LRELU, ACT_NONE, ACT_RELU, ACT_TANH, Act  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
EPS32 = 2.0 ** -24
K_ACC = 64  # see the module docstring
U16 = {"bf16": 2.0 ** -8, "fp16": 2.0 ** -11}
FP16_SUBNORMAL = 2.0 ** -24  # the spacing of fp16 subnormals
EPS_NORM = 1e-5
WORST = {}  # (entry point, flavour) -> worst |got - ref| / bound seen


@pytest.fixture(params=["bf16", "fp16"])
def precision(request):
    """Both 16-bit storage flavours of the library (hrv_<op> and hrv_<op>_f16)."""
    ops.set_precision(request.param)
    yield request.param
    ops.set_precision("bf16")


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    for (what, flav), r in sorted(WORST.items()):
        print("BWDBOUND %-28s %-4s worst error = %.3f of its bound" % (what, flav, r))


# ------------------------------------------------------------------------------------------------ comparison


def excess(got, ref, S, u=0.0, extra=None):
    """Largest |got - ref| / (u*|ref| + K_ACC*2^-24*S [+ extra]) over all elements (inf where the bound is 0 and got != ref)."""
    got, ref, S = (t.detach().double().cpu() for t in (got, ref, S))
    assert got.shape == ref.shape == S.shape, (got.shape, ref.shape, S.shape)
    bound = u * ref.abs() + K_ACC * EPS32 * S + (FP16_SUBNORMAL if u == U16["fp16"] else 0.0)
    if extra is not None:
        bound = bound + extra.detach().double().cpu()
    err = (got - ref).abs()
    if not bool(torch.isfinite(got).all()):
        return float("inf")
    ratio = torch.where(bound > 0, err / bound.clamp_min(1e-300), torch.where(err > 0, float("inf"), 0.0))
    return float(ratio.max())


def check(what, got, ref, S, u=0.0, extra=None):
    r = excess(got, ref, S, u, extra)
    key = (what, ops.get_precision())
    WORST[key] = max(WORST.get(key, 0.0), r)
    assert r <= 1.0, "%s (%s): error is %.3g x its bound" % (what, ops.get_precision(), r)


# ------------------------------------------------------------------------------------------------ data


def gen(seed):
    return torch.Generator().manual_seed(seed)


def rnd(g, *shape, scale=1.0, mean=0.0):
    """fp32 normal values (rounded to the storage type later with q())."""
    return torch.randn(*shape, generator=g) * scale + mean


def q(x):
    """x rounded to the storage type of the current flavour, as fp64."""
    return x.float().to(ops.STORAGE[0]).double()


def upload(x, pitch=None, fill=0.0):
    """fp64/fp32 NCHW (CPU) -> NHWC Act in the storage type; channels past c hold `fill`."""
    n, c, h, w = x.shape
    buf = torch.full((n, h, w, ops.round_up(c, 8) if pitch is None else pitch), fill, dtype=ops.STORAGE[0], device=DEV)
    buf[..., :c] = x.permute(0, 2, 3, 1).float().to(ops.STORAGE[0]).to(DEV)
    return Act(buf, c=c)


def nchw(a):
    """Act -> fp64 NCHW on the CPU."""
    return a.buf[..., a.c0:a.c0 + a.c].permute(0, 3, 1, 2).double().cpu()


def act_fwd(v, act):
    return {ACT_NONE: lambda t: t, ACT_RELU: torch.relu, ACT_LRELU: lambda t: F.leaky_relu(t, 0.2), ACT_TANH: torch.tanh}[act](v)


def act_slope(h, act):
    """act'(v) evaluated at the stored output h = act(v), as the kernels evaluate it."""
    if act == ACT_NONE:
        return torch.ones_like(h)
    if act == ACT_RELU:
        return (h > 0).double()
    if act == ACT_LRELU:
        return torch.where(h > 0, 1.0, 0.2).double()
    return 1.0 - h * h


def slope_abs(h, act):
    """|act'| as the kernel forms it (for tanh 1 - h*h is two roundings of 1 + h^2)."""
    return 1.0 + h * h if act == ACT_TANH else act_slope(h, act).abs()


# ------------------------------------------------------------------------------------------------ 1. norm_bwd


def nearest_up(x, shift):
    return x.repeat_interleave(2, 2).repeat_interleave(2, 3) if shift else x


def sum_kids(t, shift):
    if not shift:
        return t
    n, c, h, w = t.shape
    return t.reshape(n, c, h // 2, 2, w // 2, 2).sum((3, 5))


def norm_bwd_ref(dh, h, gamma, x0, shift, x1, noise, ns, mean, rstd, act, u):
    """fp64 autograd of h = act(xn*(1 + gamma) + beta), xn = InstanceNorm(cat(up2^shift(x0), x1) + noise*ns), with the
    activation linearised at the stored h and the statistics' VALUES pinned to the kernel's mean/rstd (their derivatives are those
    of the fp64 statistics).  gamma None = the InstanceNorm + activation form.  Returns {output: (ref, S, extra)}."""
    c0 = x0.shape[1]
    x0l = x0.clone().requires_grad_(True)
    x1l = x1.clone().requires_grad_(True) if x1 is not None else None
    nsl = ns.clone().requires_grad_(True) if ns is not None else None
    gam = gamma if gamma is not None else torch.zeros_like(dh)
    gl = gam.clone().requires_grad_(True)
    beta = torch.zeros_like(dh, requires_grad=True)
    xs = nearest_up(x0l, shift)
    if x1l is not None:
        xs = torch.cat([xs, x1l], 1)
    z = xs + noise[:, None] * nsl[None, :, None, None] if noise is not None else xs
    m64 = z.mean((2, 3), keepdim=True)
    r64 = (z.var((2, 3), unbiased=False, keepdim=True) + EPS_NORM).rsqrt()
    mk, rk = mean[:, :, None, None], rstd[:, :, None, None]
    xn = (z - (mk + (m64 - m64.detach()))) * (rk + (r64 - r64.detach()))
    v = xn * (1 + gl) + beta
    (v * act_slope(h, act)).backward(dh)
    # absolute-value maps
    sdv = dh.abs() * slope_abs(h, act)
    za = xs.detach().abs() + (noise.abs()[:, None] * ns.abs()[None, :, None, None] if noise is not None else 0.0)
    X = (za + mk.abs()) * rk
    sdxn = sdv * (1 + gam.abs())
    mp = lambda t: t.mean((2, 3), keepdim=True)
    sdxs = rk * (sdxn + mp(sdxn) + X * mp(sdxn * X))
    ext = u * rk * (dh * act_slope(h, act) * (1 + gam)).abs()  # dxn is stored in 16 bits between the passes
    out = {"dgamma": (gl.grad, sdv * X, None), "dbeta": (beta.grad, sdv, None),
           "dx0": (x0l.grad, sum_kids(sdxs[:, :c0], shift), sum_kids(ext[:, :c0], shift)),
           "sum_dgamma": (gl.grad.sum((0, 2, 3)), (sdv * X).sum((0, 2, 3)), None),
           "sum_dbeta": (beta.grad.sum((0, 2, 3)), sdv.sum((0, 2, 3)), None)}
    if x1l is not None:
        out["dx1"] = (x1l.grad, sdxs[:, c0:], ext[:, c0:])
    if nsl is not None:
        out["dns"] = (nsl.grad, (sdxs * noise.abs()[:, None]).sum((0, 2, 3)), (ext * noise.abs()[:, None]).sum((0, 2, 3)))
    return out


def spade_norm_inputs(seed, n, c0, c1, H, W, shift, act, with_noise):
    """CPU inputs of one SPADE norm backward, already rounded to the storage type where the kernel stores them."""
    g = gen(seed)
    C = c0 + c1
    x0 = q(rnd(g, n, c0, H >> shift, W >> shift, mean=0.3))
    x1 = q(rnd(g, n, c1, H, W, mean=-0.2)) if c1 else None
    noise = rnd(g, n, H, W).double() if with_noise else None
    ns = (rnd(g, C) * 0.3).double() if with_noise else None
    gamma = q(rnd(g, n, C, H, W, scale=0.5))
    dh = q(rnd(g, n, C, H, W))
    beta = rnd(g, n, C, H, W, scale=0.5).double()
    return dict(x0=x0, x1=x1, noise=noise, ns=ns, gamma=gamma, dh=dh, beta=beta)


def spade_forward_h(d, shift, mean, rstd, act):
    """The stored forward output h = act(xn*(1+gamma)+beta) the backward reads (only its sign matters for LReLU)."""
    xs = nearest_up(d["x0"], shift)
    if d["x1"] is not None:
        xs = torch.cat([xs, d["x1"]], 1)
    z = xs + d["noise"][:, None] * d["ns"][None, :, None, None] if d["noise"] is not None else xs
    xn = (z - mean[:, :, None, None]) * rstd[:, :, None, None]
    return q(act_fwd(xn * (1 + d["gamma"]) + d["beta"], act))


NORM_CASES = [  # n, c0, c1, H, W, x0_shift, act, noise, x0 pitch
    (2, 64, 0, 37, 29, 0, ACT_LRELU, True, None),    # 5 pixel blocks per image, the last one partial (49 of 256 pixels)
    (2, 64, 16, 38, 30, 1, ACT_NONE, True, 72),      # x0 nearest-up-sampled, 16-channel x1, x0 read at pitch 72 > 64
    (2, 64, 16, 38, 30, 1, ACT_LRELU, False, None),
    (1, 1024, 16, 10, 14, 1, ACT_LRELU, True, None), # C = 1040 (SPADE 1024 + 16): 18 blocks of 8 pixels, the last of 4
    (1, 2040, 0, 5, 3, 0, ACT_LRELU, True, None),    # 255 channel groups: next to the 2048-channel limit
    (2, 8, 0, 1, 7, 0, ACT_LRELU, True, None),       # 1-wide map
    (1, 24, 8, 2, 2, 1, ACT_NONE, True, None),       # 2x2 map from a 1x1 x0
]


@pytest.mark.parametrize("case", NORM_CASES, ids=lambda c: "n%d_c%d+%d_%dx%d_s%d_a%d_nz%d_p%s" % c)
def test_norm_bwd_spade(case, precision):
    """ops.norm_bwd with gamma (hrv_norm_bwd_reduce + hrv_norm_bwd_apply): d(gamma|beta) interleaved, dx0, dx1, d noise_scale and the
    summed dgamma / dbeta against fp64 autograd of the SPADE modulation + InstanceNorm."""
    n, c0, c1, H, W, shift, act, with_noise, p0 = case
    u = U16[precision]
    d = spade_norm_inputs(11, n, c0, c1, H, W, shift, act, with_noise)
    C = c0 + c1
    a_x0 = upload(d["x0"], pitch=p0)
    a_x1 = upload(d["x1"]) if c1 else None
    noise = d["noise"].float().to(DEV).contiguous() if with_noise else None
    ns = d["ns"].float().to(DEV) if with_noise else None
    mean, rstd = ops.instnorm_stats(a_x0, shift, a_x1, H, W, noise, ns)
    mean, rstd = mean.double().cpu(), rstd.double().cpu()
    h = spade_forward_h(d, shift, mean, rstd, act)
    dgb, dx0, dx1, dns, sdg, sdb = ops.norm_bwd(upload(d["dh"]), upload(h), upload(d["gamma"]), a_x0, shift, a_x1, noise, ns,
                                                mean.float().to(DEV), rstd.float().to(DEV), act, want_dgb=True)
    torch.cuda.synchronize()
    ref = norm_bwd_ref(d["dh"], h, d["gamma"], d["x0"], shift, d["x1"], d["noise"], d["ns"], mean, rstd, act, u)
    gb = nchw(dgb)
    assert gb.shape[1] == 2 * C
    got = {"dgamma": gb[:, 0::2], "dbeta": gb[:, 1::2], "dx0": nchw(dx0), "sum_dgamma": sdg, "sum_dbeta": sdb}
    if c1:
        got["dx1"] = nchw(dx1)
    if with_noise:
        got["dns"] = dns
    assert set(got) == set(ref)
    for k, (r, S, ext) in ref.items():
        check("norm_bwd " + k, got[k], r, S, u if k in ("dgamma", "dbeta", "dx0", "dx1") else 0.0, ext)


@pytest.mark.parametrize("shape", [(2, 24, 13, 11), (1, 64, 37, 29), (2, 16, 1, 5)])
def test_norm_bwd_instnorm_act(shape, precision):
    """InstNormActFn (gamma None: InstanceNorm + LeakyReLU) through autograd against fp64 autograd of F.instance_norm-style
    normalisation with the kernel's statistics."""
    from hrviton_b200.autograd_g import InstNormActFn
    n, c, H, W = shape
    u = U16[precision]
    g = gen(12)
    x = q(rnd(g, n, c, H, W, mean=0.4, scale=1.5))
    dh = q(rnd(g, n, c, H, W))
    xa = upload(x)
    xb = xa.buf.clone().requires_grad_(True)
    y = InstNormActFn.apply(xb, ACT_LRELU)
    y.backward(upload(dh).buf)
    torch.cuda.synchronize()
    mean, rstd = ops.instnorm_stats(xa, 0, None, H, W, None, None)
    h = nchw(Act(y.detach(), c=c))
    ref = norm_bwd_ref(dh, h, None, x, 0, None, None, None, mean.double().cpu(), rstd.double().cpu(), ACT_LRELU, u)
    r, S, ext = ref["dx0"]
    check("norm_bwd dx (instnorm)", nchw(Act(xb.grad, c=c)), r, S, u, ext)


@pytest.mark.parametrize("act", [ACT_RELU, ACT_NONE])
@pytest.mark.parametrize("shape", [(3, 20, 9, 7), (2, 64, 17, 15)])
def test_norm_bwd_batchnorm(shape, act, precision):
    """autograd_tocg.BatchNormActFn (norm_bwd with chan_scale and batch statistics) against fp64 autograd of
    F.batch_norm(training=True) with affine weight and bias: dx, dweight, dbias."""
    from hrviton_b200.autograd_tocg import BatchNormActFn
    n, c, H, W = shape
    u = U16[precision]
    g = gen(13)
    x = q(rnd(g, n, c, H, W, mean=0.3))
    dh = q(rnd(g, n, c, H, W))
    wt, bs = (rnd(g, c, scale=0.5, mean=1.0)), rnd(g, c, scale=0.3)
    bn = torch.nn.BatchNorm2d(c).to(DEV)
    xb = upload(x).buf.clone().requires_grad_(True)
    wl, bl = wt.to(DEV).requires_grad_(True), bs.to(DEV).requires_grad_(True)
    y = BatchNormActFn.apply(xb, wl, bl, None, bn, act)
    y.backward(upload(dh).buf)
    torch.cuda.synchronize()
    h = nchw(Act(y.detach(), c=c))
    xl, w64, b64 = x.clone().requires_grad_(True), wt.double().requires_grad_(True), bs.double().requires_grad_(True)
    (F.batch_norm(xl, None, None, w64, b64, training=True, eps=EPS_NORM) * act_slope(h, act)).backward(dh)
    mean = x.mean((0, 2, 3), keepdim=True)
    rstd = (x.var((0, 2, 3), unbiased=False, keepdim=True) + EPS_NORM).rsqrt()
    sdv = dh.abs() * slope_abs(h, act)
    X = (x.abs() + mean.abs()) * rstd
    sdxn = sdv * w64.detach().abs()[None, :, None, None]
    mp = lambda t: t.mean((0, 2, 3), keepdim=True)
    sdx = rstd * (sdxn + mp(sdxn) + X * mp(sdxn * X))
    ext = u * rstd * (dh * act_slope(h, act) * w64.detach()[None, :, None, None]).abs()
    check("norm_bwd dx (batchnorm)", nchw(Act(xb.grad, c=c)), xl.grad, sdx, u, ext)
    check("norm_bwd dweight (batchnorm)", wl.grad, w64.grad, (sdv * X).sum((0, 2, 3)))
    check("norm_bwd dbias (batchnorm)", bl.grad, b64.grad, sdv.sum((0, 2, 3)))


# ------------------------------------------------------------------------------------------------ 2. act_bwd_bias


def act_bwd_bias_raw(dy, y, act, want_dv):
    """hrv_act_bwd_bias through the C-ABI: (dv Act | None, fp64 bias sums over roundup8(c) channels)."""
    dv = Act(torch.full_like(dy.buf, 7.0), c=dy.c) if want_dv else None
    bsum = torch.full((ops.round_up(dy.c, 8),), 5.0, dtype=torch.float64, device=DEV)
    tdy = dy.ct()
    ty = y.ct() if y is not None else ops._NULL
    tdv = dv.ct() if dv is not None else ops._NULL
    capi.check(ops._L(dy).hrv_act_bwd_bias(ctypes.byref(tdy), ctypes.byref(ty), act, ctypes.byref(tdv), bsum.data_ptr(), ops._stream()),
               "act_bwd_bias")
    torch.cuda.synchronize()
    return dv, bsum.cpu()


@pytest.mark.parametrize("want_dv", [True, False])
@pytest.mark.parametrize("act", [ACT_NONE, ACT_RELU, ACT_LRELU, ACT_TANH])
@pytest.mark.parametrize("shape", [(2, 20, 37, 29, 32), (1, 64, 45, 31, None), (1, 1040, 9, 7, None), (1, 2044, 3, 5, None)])
def test_act_bwd_bias(shape, act, want_dv, precision):
    """dv = dy * act'(y) and the bias gradient sum(dv).  Pixel counts give full chunks (4-way unrolled loop only) and a partial last
    chunk (remainder loop); c = 20 at pitch 32 checks that dv's pad channels are written as zero.  dy is dyadic (multiples of 2^-6),
    so for NONE / RELU every partial sum is exact and the fp64 bias sums must equal the reference exactly."""
    n, c, H, W, pitch = shape
    u = U16[precision]
    g = gen(14)
    dy = (rnd(g, n, c, H, W) * 64).round().clamp(-255, 255).double() / 64
    v = rnd(g, n, c, H, W)
    h = q(act_fwd(v.double(), act))
    dya = upload(dy, pitch=pitch)
    dv, bsum = act_bwd_bias_raw(dya, upload(h, pitch=pitch) if act != ACT_NONE else None, act, want_dv)
    sl = act_slope(h, act)
    ref_dv = dy * sl
    S_dv = dy.abs() * slope_abs(h, act)
    c8 = ops.round_up(c, 8)
    if act in (ACT_NONE, ACT_RELU):
        assert torch.equal(bsum[:c], ref_dv.sum((0, 2, 3))), "bias sums must be exact on dyadic data"
    check("act_bwd_bias bias", bsum[:c], ref_dv.sum((0, 2, 3)), S_dv.sum((0, 2, 3)))
    if c8 > c:
        assert float(bsum[c:c8].abs().max()) == 0.0
    if want_dv:
        check("act_bwd_bias dv", nchw(dv), ref_dv, S_dv, u)
        if c8 > c:
            assert float(dv.buf[..., c:c8].float().abs().max()) == 0.0, "dv pad channels must be zero where dy's are"


# ------------------------------------------------------------------------------------------------ 3. data-gradient convolution


def dgrad_ref(x_shape, w, dy, pad):
    """fp64 torch.nn.grad.conv2d_input of a stride-1 convolution with a possibly cropped (top-left aligned) output gradient, and its
    absolute-value map.  The rows / columns the cropped forward never computed carry zero gradient."""
    oh, ow = x_shape[2] + 2 * pad - w.shape[2] + 1, x_shape[3] + 2 * pad - w.shape[3] + 1
    dyf = F.pad(dy, (0, ow - dy.shape[3], 0, oh - dy.shape[2]))
    ref = torch.nn.grad.conv2d_input(x_shape, w, dyf, padding=pad)
    S = torch.nn.grad.conv2d_input(x_shape, w.abs(), dyf.abs(), padding=pad)
    return ref, S


DGRAD_CASES = [  # name, n, cin (dgrad output channels), cout (dgrad K), H, W, k, pad, dy crop, dx pitch, gate, form
    ("3x3p1_pitch", 2, 20, 64, 17, 13, 3, 1, None, 32, None, "plain"),
    ("1x1p0", 2, 96, 384, 9, 7, 1, 0, None, None, None, "plain"),
    ("4x4p2", 2, 40, 36, 11, 9, 4, 2, None, None, None, "plain"),          # forward output H+1, K = 36 (not a multiple of 8)
    ("s2d_2x2p1_crop", 2, 64, 96, 9, 7, 2, 1, (9, 7), None, None, "plain"),  # k3/s2/p1 on 17x13: natural 10x8, cropped to 9x7
    ("s2d_2x2p1_crop_k4", 1, 32, 48, 10, 6, 2, 1, (10, 6), None, None, "plain"),  # k4/s2/p2 on 19x11: 10x6 of 11x7
    ("im2col_1x1", 2, 64, 128, 12, 9, 1, 0, None, None, None, "im2col"),
    ("1wide", 1, 32, 64, 1, 9, 3, 1, None, None, None, "plain"),
    ("2wide", 2, 16, 24, 2, 2, 3, 1, None, None, None, "plain"),
    ("gate_relu", 2, 64, 64, 12, 10, 3, 1, None, None, ACT_RELU, "plain"),
    ("gate_lrelu", 1, 48, 96, 9, 11, 3, 1, None, 56, ACT_LRELU, "plain"),
    ("gamma_beta_80", 2, 128, 80, 12, 9, 3, 1, None, None, None, "interleave"),
    ("gamma_beta_1040", 1, 128, 1040, 6, 5, 3, 1, None, None, None, "interleave"),  # K = 2080 interleaved columns
]


@pytest.mark.parametrize("case", DGRAD_CASES, ids=lambda c: c[0])
def test_conv_dgrad(case, precision):
    """hrv_conv2d_fwd on pack_weight(..., dgrad=True) against torch.nn.grad.conv2d_input in fp64, in each form training uses, with the
    RES_GATE_RELU / RES_GATE_LRELU epilogues (dx * act'(x_saved)) and output into a wider-pitch buffer whose pad channels stay zero."""
    name, n, cin, cout, H, W, k, pad, crop, pitch, gate, form = case
    u = U16[precision]
    g = gen(15)
    oh, ow = (H + 2 * pad - k + 1, W + 2 * pad - k + 1) if crop is None else crop
    if form == "interleave":  # the gamma|beta GEMM: cout = C channels, K = 2C interleaved (gamma_c, beta_c) columns
        wg, wb = rnd(g, cout, cin, 3, 3, scale=0.03), rnd(g, cout, cin, 3, 3, scale=0.03)
        pw = ops.pack_weight(wg.to(DEV), (k - 1 - pad, k - 1 - pad), interleave=wb.to(DEV), dgrad=True)
        w = q(torch.stack([wg, wb], 1).reshape(2 * cout, cin, 3, 3))
        kc = 2 * cout
    elif form == "im2col":  # the tap-major column form of a 3x3 convolution over 7 channels
        from hrviton_b200.autograd_g import im2col_weight
        w3 = rnd(g, cout, 7, 3, 3, scale=0.2)
        wf = im2col_weight(w3, cin)
        pw = ops.pack_weight(wf.to(DEV), (0, 0), dgrad=True)
        w = q(wf)
        kc = cout
    else:
        wf = rnd(g, cout, cin, k, k, scale=(1.0 / (cout * k * k)) ** 0.5)
        pw = ops.pack_weight(wf.to(DEV), (k - 1 - pad, k - 1 - pad), dgrad=True)
        w = q(wf)
        kc = cout
    dy = q(rnd(g, n, kc, oh, ow))
    dxa = Act(torch.zeros((n, H, W, pitch or ops.round_up(cin, 8)), dtype=ops.STORAGE[0], device=DEV), c=cin)
    ref, S = dgrad_ref((n, cin, H, W), w, dy, pad)
    if gate is not None:
        xs = q(act_fwd(rnd(g, n, cin, H, W).double(), gate))
        ops.conv2d(upload(dy), pw, dxa, res=upload(xs, pitch=dxa.pitch), res_mode={ACT_RELU: capi.RES_GATE_RELU, ACT_LRELU: capi.RES_GATE_LRELU}[gate])
        ref, S = ref * act_slope(xs, gate), S * act_slope(xs, gate).abs()
    else:
        ops.conv2d(upload(dy), pw, dxa)
    torch.cuda.synchronize()
    check("conv dgrad", nchw(dxa), ref, S, u)
    if dxa.pitch > cin:
        assert float(dxa.buf[..., cin:].float().abs().max()) == 0.0, "pad channels of the output buffer must stay zero"


# ------------------------------------------------------------------------------------------------ 4. weight gradient


def wgrad_case(n, cin, cout, H, W, k, pad, crop, seed=16):
    g = gen(seed)
    x = q(rnd(g, n, cin, H, W))
    oh, ow = (H + 2 * pad - k + 1, W + 2 * pad - k + 1) if crop is None else crop
    dy = q(rnd(g, n, cout, oh, ow))
    dyf = F.pad(dy, (0, W + 2 * pad - k + 1 - ow, 0, H + 2 * pad - k + 1 - oh))
    ref = torch.nn.grad.conv2d_weight(x, (cout, cin, k, k), dyf, padding=pad)
    S = torch.nn.grad.conv2d_weight(x.abs(), (cout, cin, k, k), dyf.abs(), padding=pad)
    return x, dy, ref, S


def wgrad_splits(xa, dya, k):
    tx, tdy = xa.ct(), dya.ct()
    return int(ops._L(xa).hrv_conv2d_wgrad_workspace_bytes(ctypes.byref(tx), ctypes.byref(tdy), k, k)) > 0


WGRAD_CROP_CASES = [  # n, cin, cout, H, W, k, pad, cropped dy extent
    (2, 64, 96, 9, 7, 2, 1, (9, 7)),        # space-to-depth form of k3/s2/p1 on 17x13 (natural 10x8)
    (1, 128, 64, 10, 6, 2, 1, (10, 6)),     # space-to-depth form of k4/s2/p2 on 19x11 (natural 11x7)
    (2, 40, 72, 11, 9, 4, 2, (10, 8)),      # 4x4/p2 with a cropped output (natural 12x10)
    (2, 32, 24, 70, 58, 2, 1, (70, 58)),    # many pixels, few tiles: split-K
    (1, 128, 64, 3, 40, 2, 1, (1, 40)),     # one 64-pixel chunk (natural 4x41): one CTA per tile, no split
]


@pytest.mark.parametrize("case", WGRAD_CROP_CASES, ids=lambda c: "n%d_%dto%d_%dx%d_k%dp%d_crop%dx%d" % (c[:7] + c[7]))
def test_conv_wgrad_cropped(case, precision):
    """hrv_conv2d_wgrad with a cropped dy (dy extent < h + 2*pad - k + 1: the stride-2 layers' out_hw) against fp64
    torch.nn.grad.conv2d_weight of the zero-extended dy, per element."""
    n, cin, cout, H, W, k, pad, crop = case
    x, dy, ref, S = wgrad_case(n, cin, cout, H, W, k, pad, crop)
    xa, dya = upload(x), upload(dy)
    got = ops.conv2d_wgrad(xa, dya, k, k, pad)
    torch.cuda.synchronize()
    check("conv wgrad", got, ref, S)


def test_conv_wgrad_geometries_covered():
    """The cropped cases above run both the split-K path (workspace slabs + fixed-order reduction) and the single-CTA path."""
    splits = set()
    for n, cin, cout, H, W, k, pad, crop in WGRAD_CROP_CASES:
        x = torch.zeros((n, H, W, ops.round_up(cin, 8)), dtype=torch.bfloat16, device=DEV)
        dy = torch.zeros((n, crop[0], crop[1], ops.round_up(cout, 8)), dtype=torch.bfloat16, device=DEV)
        splits.add(wgrad_splits(Act(x, c=cin), Act(dy, c=cout), k))
    assert splits == {True, False}


WGRAD_CASES = [(2, 64, 128, 24, 16, 3, 1), (1, 128, 160, 32, 24, 3, 1), (2, 80, 32, 64, 48, 3, 1), (1, 7, 128, 32, 24, 3, 1),
               (1, 1040, 512, 16, 12, 3, 1), (2, 96, 384, 16, 12, 1, 0), (2, 64, 24, 17, 13, 2, 1), (1, 256, 1, 17, 13, 4, 2),
               (1, 32, 3, 128, 96, 3, 1), (2, 128, 288, 130, 70, 3, 1)]  # the shapes of test_kernels_gpu.test_conv_wgrad


@pytest.mark.parametrize("case", WGRAD_CASES, ids=lambda c: "n%d_%dto%d_%dx%d_k%dp%d" % c)
def test_conv_wgrad_per_element(case, precision):
    n, cin, cout, H, W, k, pad = case
    x, dy, ref, S = wgrad_case(n, cin, cout, H, W, k, pad, None)
    got = ops.conv2d_wgrad(upload(x), upload(dy), k, k, pad)
    torch.cuda.synchronize()
    check("conv wgrad", got, ref, S)


# ------------------------------------------------------------------------------------------------ 5. stride-2 chain


@pytest.mark.parametrize("k,pad,act,shape", [(3, 1, ACT_NONE, (2, 12, 40, 17, 13)), (4, 2, ACT_LRELU, (1, 20, 32, 19, 11)),
                                             (3, 1, ACT_NONE, (1, 64, 64, 9, 7))])
def test_stride2_chain_through_autograd(k, pad, act, shape, precision):
    """space_to_depth_t + _s2d_weight_t + conv(..., pad=1, out_hw=...) (autograd_tocg._resblock k3/p1, the discriminators k4/p2)
    against fp64 autograd of F.conv2d(stride=2) at odd H and W: dx, dW, db."""
    from hrviton_b200.autograd_g import _s2d_weight_t, conv, space_to_depth_t
    n, cin, cout, H, W = shape
    u = U16[precision]
    g = gen(17)
    x = q(rnd(g, n, cin, H, W))
    wf = rnd(g, cout, cin, k, k, scale=(1.0 / (cin * k * k)) ** 0.5)
    bf = rnd(g, cout, scale=0.1)
    oh, ow = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    if k == 4:
        oh, ow = H // 2 + 1, W // 2 + 1
    xb = upload(x).buf.clone().requires_grad_(True)
    wl, bl = wf.to(DEV).requires_grad_(True), bf.to(DEV).requires_grad_(True)
    y = conv(space_to_depth_t(xb, cin), _s2d_weight_t(wl), bl, act=act, pad=1, out_hw=(oh, ow))
    assert y.shape[1:3] == (oh, ow)
    dy = q(rnd(g, n, cout, oh, ow))
    y.backward(upload(dy).buf)
    torch.cuda.synchronize()
    h = nchw(Act(y.detach(), c=cout))
    w = q(wf)
    xl, w64, b64 = x.clone().requires_grad_(True), w.clone().requires_grad_(True), bf.double().requires_grad_(True)
    ref_y = F.conv2d(xl, w64, b64, stride=2, padding=pad)
    assert ref_y.shape[2:] == (oh, ow)
    (ref_y * act_slope(h, act)).backward(dy)
    sdv = dy.abs() * slope_abs(h, act)
    S_dx = torch.nn.grad.conv2d_input(x.shape, w.abs(), sdv, stride=2, padding=pad)
    S_dw = torch.nn.grad.conv2d_weight(x.abs(), w.shape, sdv, stride=2, padding=pad)
    # dv = dy * act'(h) is stored in 16 bits before both GEMMs: the rounding they inherit
    ext_dx = u * torch.nn.grad.conv2d_input(x.shape, w.abs(), (dy * act_slope(h, act)).abs(), stride=2, padding=pad) if act != ACT_NONE else None
    ext_dw = u * S_dw if act != ACT_NONE else None
    check("stride2 chain dx", nchw(Act(xb.grad, c=cin)), xl.grad, S_dx, u, ext_dx)
    check("stride2 chain dW", wl.grad, w64.grad, S_dw, 0.0, ext_dw)
    check("stride2 chain db", bl.grad, b64.grad, sdv.sum((0, 2, 3)))


# ------------------------------------------------------------------------------------------------ 6. bilinear x2 backward


def up2_bwd_ref(dout):
    """fp64 autograd of F.interpolate(scale_factor=2, bilinear, align_corners=False): (da, S)."""
    n, c, H, W = dout.shape
    a = torch.zeros((n, c, H // 2, W // 2), dtype=torch.float64, requires_grad=True)
    up = F.interpolate(a, scale_factor=2, mode="bilinear", align_corners=False)
    ref, = torch.autograd.grad(up, a, dout)
    S, = torch.autograd.grad(up, a, dout.abs())
    return ref, S


UP2_SHAPES = [(2, 20, 1, 1), (1, 8, 1, 6), (2, 24, 2, 3), (1, 64, 7, 2), (2, 20, 9, 13)]  # low-res n, c, h, w


@pytest.mark.parametrize("shape", UP2_SHAPES, ids=lambda s: "n%d_c%d_%dx%d" % s)
def test_bilinear_up2_bwd(shape, precision):
    """hrv_bilinear_up2_bwd against fp64 autograd of F.interpolate(x2, bilinear), including 1- and 2-wide maps; Up2Fn passes the
    lateral gradient through unchanged."""
    from hrviton_b200.autograd_tocg import Up2Fn
    n, c, h, w = shape
    u = U16[precision]
    dout = q(rnd(gen(18), n, c, 2 * h, 2 * w))
    ref, S = up2_bwd_ref(dout)
    da = ops.bilinear_up2_bwd(upload(dout))
    torch.cuda.synchronize()
    check("bilinear_up2_bwd", nchw(da), ref, S, u)
    a_buf = upload(q(rnd(gen(19), n, c, h, w))).buf.clone().requires_grad_(True)
    b_buf = torch.zeros((n, 2 * h, 2 * w, a_buf.shape[3]), dtype=ops.STORAGE[0], device=DEV, requires_grad=True)
    out = Up2Fn.apply(a_buf, b_buf)
    g_buf = upload(dout).buf
    out.backward(g_buf)
    torch.cuda.synchronize()
    assert torch.equal(b_buf.grad, g_buf)
    assert torch.equal(a_buf.grad, da.buf)


# ------------------------------------------------------------------------------------------------ 7. flow warp backward


def flow_warp_bwd_raw(flow, src, ddst, dfu_in):
    """hrv_flow_warp_bwd through the C-ABI: (dsrc32 before rounding, dflow_up accumulated onto dfu_in, dflow_lo)."""
    n, hl, wl, _ = flow.shape
    H, W = 2 * hl, 2 * wl
    dsrc32 = torch.zeros((n, src.h, src.w, ops.round_up(src.c, 8)), dtype=torch.float32, device=DEV)
    dfu = dfu_in.float().to(DEV).contiguous().clone()
    dflo = torch.empty((n, hl, wl, 2), dtype=torch.float32, device=DEV)
    fl = flow.float().to(DEV).contiguous()
    ts, td = src.ct(), ddst.ct()
    capi.check(ops._L(src).hrv_flow_warp_bwd(fl.data_ptr(), ops.linspace_table(W, DEV).data_ptr(), ops.linspace_table(H, DEV).data_ptr(),
                                             ctypes.byref(ts), ctypes.byref(td), dsrc32.data_ptr(), dfu.data_ptr(), dflo.data_ptr(),
                                             ops._stream()), "flow_warp_bwd")
    torch.cuda.synchronize()
    return dsrc32.cpu().double(), dfu.cpu().double(), dflo.cpu().double()


def flow_warp_bwd_ref(flow, src, ddst, dfu_in):
    """fp64 autograd of orc.flow_warp's chain (x2 bilinear flow up-sampling, normalise, base grid, grid_sample(border)) plus
    <dfu_in, flow_up>.  The sampling grid's VALUES are pinned to the kernel's fp32 coordinates (np_flow_warp_coords, bit-exact with
    the kernel; extents are powers of two so (2*ix+1)/W - 1 maps back to ix exactly); its derivative is the fp64 chain's.  Returns
    {output: (ref, S)}."""
    n, c, H, W = src.shape
    x0, y0, tx, ty = orc.np_flow_warp_coords(flow.float().numpy(), H, W, H, W)
    ix = torch.from_numpy(x0).double() + torch.from_numpy(tx).double()  # clamped to [0, W-1]: on the border = clamped (torch)
    iy = torch.from_numpy(y0).double() + torch.from_numpy(ty).double()
    gval = torch.stack([(2 * ix + 1) / W - 1, (2 * iy + 1) / H - 1], 3)
    fl = flow.double().clone().requires_grad_(True)
    fu = orc._up2(fl.permute(0, 3, 1, 2)).permute(0, 2, 3, 1)
    fu.retain_grad()
    g64 = torch.cat([fu[..., 0:1] / ((W / 2 - 1.0) / 2.0), fu[..., 1:2] / ((H / 2 - 1.0) / 2.0)], 3) + orc.make_base_grid(n, H, W).double()
    grid = gval + (g64 - g64.detach())
    sl = src.clone().requires_grad_(True)
    out = F.grid_sample(sl, grid, mode="bilinear", padding_mode="border", align_corners=False)
    ((out * ddst).sum() + (fu * dfu_in).sum()).backward()
    # absolute-value maps: the scatter of |d| for dsrc; for d flow_up, |d| times the four taps' |src| times d ix / d flow_up
    s2 = torch.zeros_like(src, requires_grad=True)
    S_src, = torch.autograd.grad(F.grid_sample(s2, gval, mode="bilinear", padding_mode="border", align_corners=False), s2, ddst.abs())
    xi0, yi0 = torch.from_numpy(x0).long(), torch.from_numpy(y0).long()
    xi1, yi1 = (xi0 + 1).clamp(max=W - 1), (yi0 + 1).clamp(max=H - 1)
    bidx = torch.arange(n)[:, None, None]
    sa = src.abs().permute(0, 2, 3, 1)
    taps = sa[bidx, yi0, xi0] + sa[bidx, yi0, xi1] + sa[bidx, yi1, xi0] + sa[bidx, yi1, xi1]  # (n, H, W, c)
    dabs = (ddst.abs().permute(0, 2, 3, 1) * taps).sum(3)
    S_up = torch.stack([dabs * (W / 2) / ((W / 2 - 1.0) / 2.0), dabs * (H / 2) / ((H / 2 - 1.0) / 2.0)], 3) + dfu_in.abs()
    a = torch.zeros_like(fl, requires_grad=True)
    S_lo, = torch.autograd.grad(orc._up2(a.permute(0, 3, 1, 2)).permute(0, 2, 3, 1), a, S_up)
    return {"dsrc32": (sl.grad, S_src), "dflow_up": (fu.grad, S_up), "dflow_lo": (fl.grad, S_lo)}


def run_flow_case(flow, c, seed):
    n, hl, wl, _ = flow.shape
    H, W = 2 * hl, 2 * wl
    g = gen(seed)
    src = q(rnd(g, n, c, H, W))
    ddst = q(rnd(g, n, c, H, W))
    dfu_in = rnd(g, n, H, W, 2, scale=0.5).double()
    dsrc32, dfu, dflo = flow_warp_bwd_raw(flow, upload(src), upload(ddst), dfu_in)
    ref = flow_warp_bwd_ref(flow, src, ddst, dfu_in)
    got = {"dsrc32": dsrc32[..., :c].permute(0, 3, 1, 2), "dflow_up": dfu, "dflow_lo": dflo}
    for k, (r, S) in ref.items():
        check("flow_warp_bwd " + k, got[k], r, S)
    if dsrc32.shape[3] > c:
        assert float(dsrc32[..., c:].abs().max()) == 0.0
    return got, dfu_in


@pytest.mark.parametrize("c,hl,wl,scale", [(4, 16, 16, 1.0), (8, 16, 16, 12.0), (384, 8, 16, 1.0), (384, 16, 16, 12.0)])
def test_flow_warp_bwd(c, hl, wl, scale, precision):
    """dsrc32 (before it is rounded), dflow_up (accumulated onto a nonzero incoming gradient) and dflow_lo against fp64 autograd of
    orc.flow_warp.  scale 1: interior sampling points; scale 12: many coordinates clamped on both sides."""
    flow = (rnd(gen(20), 2, hl, wl, 2) * scale).double()
    run_flow_case(flow, c, 21)


def test_flow_warp_bwd_exact_border(precision):
    """Sampling points exactly ON the border: a constant flow field up-samples exactly, and with W = H = 32,
    flow = +0.234375 puts column / row 0 at ix = 0.0 exactly, flow = -0.234375 puts column / row 31 at 31.0 exactly.  torch's
    grid_sample treats the border as clamped, so the coordinate gradient there is zero on that axis."""
    a = 0.234375
    signs = [(1, 1), (1, -1), (-1, 1), (-1, -1)]
    flow = torch.zeros(4, 16, 16, 2, dtype=torch.float64)
    for i, (sx, sy) in enumerate(signs):
        flow[i, ..., 0], flow[i, ..., 1] = sx * a, sy * a
    # the unclamped fp32 coordinates of the kernel's chain (np_flow_warp_coords before its clamp)
    up = orc.np_bilinear_up2(np.moveaxis(flow.float().numpy(), -1, 1))
    s = np.float32((32 / 2 - 1.0) / 2.0)
    lin = orc.np_linspace_grid(32)
    ix = (((up[:, 0] / s + lin[None, None, :]).astype(np.float32) + np.float32(1)) * np.float32(32) - np.float32(1)) / np.float32(2)
    iy = (((up[:, 1] / s + lin[None, :, None]).astype(np.float32) + np.float32(1)) * np.float32(32) - np.float32(1)) / np.float32(2)
    x0, y0, tx, ty = orc.np_flow_warp_coords(flow.float().numpy(), 32, 32, 32, 32)
    for i, (sx, sy) in enumerate(signs):
        col, row = (0 if sx > 0 else 31), (0 if sy > 0 else 31)
        assert np.all(ix[i, :, col] == col) and np.all(x0[i, :, col] == col) and np.all(tx[i, :, col] == 0)
        assert np.all(iy[i, row, :] == row) and np.all(y0[i, row, :] == row) and np.all(ty[i, row, :] == 0)
    got, dfu_in = run_flow_case(flow, 8, 22)
    for i, (sx, sy) in enumerate(signs):
        col, row = (0 if sx > 0 else 31), (0 if sy > 0 else 31)
        # nothing is added on the clamped axis: the incoming gradient comes back unchanged
        assert torch.equal(got["dflow_up"][i, :, col, 0], dfu_in[i, :, col, 0].float().double())
        assert torch.equal(got["dflow_up"][i, row, :, 1], dfu_in[i, row, :, 1].float().double())


# ------------------------------------------------------------------------------------------------ 8. pooling, L1, affine norm apply


@pytest.mark.parametrize("shape", [(2, 20, 9, 7), (1, 64, 6, 5), (2, 8, 3, 3)])
def test_maxpool2_bwd_relu_gate(shape, precision):
    """hrv_maxpool2_bwd with relu_gate=1 against fp64 autograd of F.max_pool2d times (x > 0): odd extents (the unread row / column
    gets zero) and constructed ties (the first maximum in row-major order wins, as in torch); all-zero windows route nothing."""
    n, c, H, W = shape
    g = gen(23)
    x = q(torch.relu(rnd(g, n, c, H, W)))
    x[:, :, 0:2, 0:2] = 0.5                          # a four-way positive tie
    if H >= 4 and W >= 4:
        x[:, :, 2, 2], x[:, :, 3, 3], x[:, :, 2, 3], x[:, :, 3, 2] = 0.25, 0.75, 0.75, -0.0  # a two-way tie, second in row-major order
    dy = q(rnd(g, n, c, H // 2, W // 2))
    xl = x.clone().requires_grad_(True)
    F.max_pool2d(xl, 2).backward(dy)
    ref = xl.grad * (x > 0).double()
    dx = ops.maxpool2_bwd(upload(x), upload(dy), relu_gate=True)
    torch.cuda.synchronize()
    assert torch.equal(nchw(dx), ref)


@pytest.mark.parametrize("shape", [(2, 20, 9, 7, 32), (1, 64, 5, 3, None)])
def test_l1_bwd_relu_gate_and_l1_sum_pad(shape, precision):
    """hrv_l1_bwd with relu_gate=1 (sign(a - b) * g * (a > 0), exact) and hrv_l1_sum with nonzero garbage in the pad channels, which it
    must not count."""
    n, c, H, W, pitch = shape
    g = gen(24)
    a = q(rnd(g, n, c, H, W))
    b = q(rnd(g, n, c, H, W))
    b[:, :, 0] = a[:, :, 0]  # equal elements: zero gradient
    A, B = upload(a, pitch=pitch, fill=100.0), upload(b, pitch=pitch, fill=-100.0)
    gs = torch.full((1,), 0.75 / a.numel(), device=DEV)
    da = ops.l1_bwd(A, B, gs, relu_gate=True)
    s = ops.l1_sum(A, B)
    torch.cuda.synchronize()
    want = q(torch.sign(a - b) * float(gs)) * (a > 0).double()
    assert torch.equal(nchw(da), want)
    if da.pitch > c:
        assert float(da.buf[..., c:ops.round_up(c, 8)].float().abs().max()) == 0.0
    d = (a - b).abs()
    check("l1_sum", s.cpu(), d.sum().reshape(1), d.sum().reshape(1))


@pytest.mark.parametrize("act", [ACT_NONE, ACT_RELU, ACT_LRELU, ACT_TANH])
@pytest.mark.parametrize("with_res", [False, True])
def test_norm_apply_affine(act, with_res, precision):
    """hrv_norm_apply_affine (the train-mode BatchNorm forward: (x - mean) * rstd * gamma + beta (+ res), activation) in fp64."""
    n, c, H, W = 2, 20, 9, 7
    u = U16[precision]
    g = gen(25)
    x = q(rnd(g, n, c, H, W, mean=0.3))
    res = q(rnd(g, n, c, H, W)) if with_res else None
    c8 = ops.round_up(c, 8)
    mean = F.pad(rnd(g, c, scale=0.2), (0, c8 - c)).double()
    rstd = F.pad(torch.rand(c, generator=g) + 0.5, (0, c8 - c)).double()
    gam = F.pad(rnd(g, c, scale=0.5, mean=1.0), (0, c8 - c)).double()
    bet = F.pad(rnd(g, c, scale=0.3), (0, c8 - c)).double()
    to = lambda t: t.float()[None].expand(n, c8).contiguous().to(DEV)
    wide = lambda t: Act(upload(t).buf, c=c8)  # as BatchNormActFn calls it: all c8 channels, [N][c8] statistics, zero pad weights
    y = ops.norm_apply_affine(wide(x), to(mean), to(rstd), gam.float().to(DEV), bet.float().to(DEV), wide(res) if with_res else None, act)
    torch.cuda.synchronize()
    assert float(y.buf[..., c:].float().abs().max()) == 0.0
    y = Act(y.buf, c=c)
    bc = lambda t: t[:c][None, :, None, None]
    v = (x - bc(mean)) * bc(rstd) * bc(gam) + bc(bet) + (res if with_res else 0.0)
    ref = act_fwd(v, act)
    Sv = (x.abs() + bc(mean).abs()) * bc(rstd) * bc(gam).abs() + bc(bet).abs() + (res.abs() if with_res else 0.0)
    # every activation has |act'| <= 1, so S of v bounds S of the output; tanhf's few ulp of |tanh v| <= |v| <= S fit in K_ACC
    check("norm_apply_affine", nchw(y), ref, Sv, u)


# ------------------------------------------------------------------------------------------------ 9. SpadeFn routing


def test_spadefn_gradient_routing(precision):
    """One SpadeFn call at C = 80 (64 x0 channels at half resolution + 16 in x1): all eight gradients against fp64 autograd of
    orc.spade_norm's expression on the same 16-bit operands.  Relative L2 within 4 u per gradient: enough to catch slicing and
    interleave mistakes (dwcat[0::2], sum_dg -> bg)."""
    from hrviton_b200.autograd_g import SpadeFn
    u = U16[precision]
    n, H, W, c0, c1, ca = 2, 16, 12, 64, 16, 128
    C = c0 + c1
    g = gen(26)
    actv = q(torch.relu(rnd(g, n, ca, H, W)))
    wg, wb = rnd(g, C, ca, 3, 3, scale=0.03), rnd(g, C, ca, 3, 3, scale=0.03)
    bg, bb = rnd(g, C, scale=0.1), rnd(g, C, scale=0.1)
    x0 = q(rnd(g, n, c0, H // 2, W // 2, mean=0.3))
    x1 = q(rnd(g, n, c1, H, W))
    noise = rnd(g, n, H, W)
    ns = rnd(g, C, scale=0.3)
    dout = q(rnd(g, n, C, H, W))
    leaves = dict(actv=upload(actv).buf, wg=wg.to(DEV), wb=wb.to(DEV), bg=bg.to(DEV), bb=bb.to(DEV), x0=upload(x0).buf,
                  x1=upload(x1).buf, ns=ns.to(DEV))
    for t in leaves.values():
        t.requires_grad_(True)
    out = SpadeFn.apply(leaves["actv"], leaves["wg"], leaves["wb"], leaves["bg"], leaves["bb"], leaves["x0"], leaves["x1"],
                        noise.to(DEV).contiguous(), leaves["ns"], 1, ACT_LRELU)
    out.backward(upload(dout).buf)
    torch.cuda.synchronize()
    got = {k: (nchw(Act(t.grad, c=t.shape[3])) if t.dim() == 4 and t.dtype != torch.float32 else t.grad.double().cpu())
           for k, t in leaves.items()}
    r = dict(actv=actv, wg=q(wg), wb=q(wb), bg=bg.double(), bb=bb.double(), x0=x0, x1=x1, ns=ns.double())
    for t in r.values():
        t.requires_grad_(True)
    xs = torch.cat([F.interpolate(r["x0"], scale_factor=2, mode="nearest"), r["x1"]], 1)
    z = xs + noise.double()[:, None] * r["ns"][None, :, None, None]
    normalized = (z - z.mean((2, 3), keepdim=True)) / (z.var((2, 3), unbiased=False, keepdim=True) + EPS_NORM).sqrt()
    gamma = F.conv2d(r["actv"], r["wg"], r["bg"], padding=1)
    beta = F.conv2d(r["actv"], r["wb"], r["bb"], padding=1)
    F.leaky_relu(normalized * (1 + gamma) + beta, 0.2).backward(dout)
    for k in leaves:
        ref = r[k].grad
        rel = float((got[k] - ref).norm() / ref.norm())
        key = ("SpadeFn d" + k + " (rel L2 / 4u)", precision)
        WORST[key] = max(WORST.get(key, 0.0), rel / (4 * u))
        assert rel <= 4 * u, (k, rel, 4 * u)
