"""Every 16-bit forward entry point, one at a time, against a float64 reference on the CPU, in both 16-bit storage flavours.

Each reference is computed in fp64 from the exact 16-bit values the kernel read (activations and packed weights are rounded to the
flavour's storage type first, or read back from the device).  Kernels that take statistics as inputs get the kernel's own mean/rstd
(or, for instnorm_apply, fp32 statistics restated on the host), and the reference uses those same fp32 values.

The bound is per element and derived from the accumulation, not tuned.  With S the same fp64 map applied to absolute values (for a
convolution conv(|x|, |w|) * |scale| + |shift| + |residual|):
  16-bit outputs             |got - ref| <= u*|ref| + K_ACC * 2^-24 * S     u = 2^-8 (bf16), 2^-11 (fp16): one rounding of the result
                                               (+ 2^-24 in fp16, one subnormal step: below 2^-14 its rounding is absolute)
  fp32 outputs               |got - ref| <= K_ACC * 2^-24 * S
Pure copies and index gathers (max-pool, space-to-depth, im2col, layout changes, one-hot, weight packing, nearest resampling, the flow
warp's indices and up-sampled flow) must be bit-exact instead.

The statistics kernels are bounded by their single-pass formula var = E[t^2] - m^2 over fp32 per-thread sums combined in fp64.  With
|t| <= T = |x| + |noise * noise_scale| per element:
  mean  |dm| <= K_ACC * 2^-24 * E[T]  (+ 2^-24 |m|, the fp32 result)
  var   |dv| <= K_ACC * 2^-24 * (E[T^2] + 2 |m| E[T])  (+ 2^-24 var)
  rstd  |dr| / r <= dv / (2 (var + eps)) + 2^-24
The var term carries the cancellation of a large mean: at mean / std = 64 the bound is 4097 times the variance's own scale, so the
measured ratio, not the bound, tells how much of it a kernel uses (DESIGN.md §4 records it).

K_ACC: every kernel sums in fp32 per thread (or in the fp32 wgmma accumulators) and combines threads, blocks and slabs in fp64 or in a
fixed fp32 order.  The longest fp32 chain below is the 2080-channel 3x3 convolution: K = 18720 products in 1170 wgmma k16 steps; the
statistics kernels' per-thread chains are at most a few dozen pixels at these shapes, and the elementwise kernels chain at most nine
terms.  A chain of m < 64^2 = 4096 steps over terms of mixed sign drifts by about sqrt(m) units of 2^-24 * S, at most 64 here.
tests/test_forward_bounds_cpu.py shows that the bound still rejects the realistic mistakes (a zeroed or stale channel group of a
low-magnitude channel, a dropped noise term, a double-rounded gamma, another image's statistics, a shift added after the activation)
at these shapes, where the max-norm rel_err < 1e-2 accepts them.

Test data is built to be hard: per-channel magnitudes spread over three decades, odd extents and partial pixel tiles, tiles that span
several images (h*w < 128), channel counts that leave a narrow last N tile, channel-slice views (c0 > 0, pitch > c) with garbage in the
channels around the view, and outputs inside NaN-sentinel buffers whose untouched elements must stay bit-for-bit unchanged."""
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
GARBAGE = 3.0  # channels around a view hold this: a kernel that reads them shows it
SENTINEL = {torch.bfloat16: (torch.int16, 0x7FC1), torch.float16: (torch.int16, 0x7E01), torch.float32: (torch.int32, 0x7FC00123)}
WORST = {}  # (op, flavour) -> worst |got - ref| / bound seen (0 for bit-exact ops)


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
        print("FWDBOUND %-32s %-4s worst = %.3f of its bound" % (what, flav, r))


# ------------------------------------------------------------------------------------------------ comparison


def ratio(got, ref, bound):
    """Largest |got - ref| / bound over all elements (inf where got is not finite, or where the bound is 0 and got != ref)."""
    got, ref, bound = (torch.as_tensor(t).detach().double().cpu() for t in (got, ref, bound))
    assert got.shape == ref.shape == bound.shape, (got.shape, ref.shape, bound.shape)
    if not bool(torch.isfinite(got).all()):
        return float("inf")
    err = (got - ref).abs()
    r = torch.where(bound > 0, err / bound.clamp_min(1e-300), torch.where(err > 0, float("inf"), 0.0))
    return float(r.max()) if r.numel() else 0.0


def bound16(ref, S, u):
    """u*|ref| + K_ACC*2^-24*S (+ one fp16 subnormal step); u = 0 for fp32 outputs."""
    ref, S = ref.detach().double().cpu(), S.detach().double().cpu()
    return u * ref.abs() + K_ACC * EPS32 * S + (FP16_SUBNORMAL if u == U16["fp16"] else 0.0)


def excess(got, ref, S, u=0.0):
    return ratio(got, ref, bound16(ref, S, u))


def record(what, r):
    key = (what, ops.get_precision())
    WORST[key] = max(WORST.get(key, 0.0), r)
    assert r <= 1.0, "%s (%s): error is %.3g x its bound" % (what, ops.get_precision(), r)


def check(what, got, ref, S, u=0.0):
    record(what, excess(got, ref, S, u))


def check_exact(what, got, want):
    got, want = got.detach().cpu(), want.detach().cpu()
    assert got.shape == want.shape, (what, got.shape, want.shape)
    bad = got != want
    assert not bool(bad.any()), "%s (%s): %d of %d elements differ, first at %s" % (
        what, ops.get_precision(), int(bad.sum()), bad.numel(), bad.nonzero()[:4].tolist())
    record(what, 0.0)


def rel_err(got, ref):
    """The max-norm of the older tests: max|got - ref| / max|ref|."""
    got, ref = got.double().cpu(), ref.double().cpu()
    return float((got - ref).abs().max() / ref.abs().max())


# ------------------------------------------------------------------------------------------------ data


def gen(seed):
    return torch.Generator().manual_seed(seed)


def rnd(g, *shape, scale=1.0, mean=0.0):
    return torch.randn(*shape, generator=g) * scale + mean


def spread(c):
    """Per-channel magnitudes 1 ... 1e-3, log-spaced in channel order: the last 8-channel groups are the smallest, so an error
    confined to one of them stays under 1 % of the tensor's largest value."""
    return 10.0 ** torch.linspace(0.0, -3.0, c)


def q(x):
    """x rounded to the storage type of the current flavour, as fp64."""
    return x.float().to(ops.STORAGE[0]).double()


def upload(x, c0=0, pitch=None, fill=GARBAGE):
    """fp64 NCHW (CPU) -> NHWC Act in the storage type, viewing channels [c0, c0 + c) of a buffer whose other channels hold `fill`."""
    n, c, h, w = x.shape
    P = c0 + ops.round_up(c, 8) if pitch is None else pitch
    buf = torch.full((n, h, w, P), fill, dtype=ops.STORAGE[0], device=DEV)
    buf[..., c0:c0 + c] = x.permute(0, 2, 3, 1).float().to(ops.STORAGE[0]).to(DEV)
    return Act(buf, c=c, c0=c0)


def nchw(a):
    """Act -> fp64 NCHW on the CPU (the view's channels)."""
    return a.buf[..., a.c0:a.c0 + a.c].permute(0, 3, 1, 2).double().cpu()


def sentinel_buf(shape, dtype):
    idt, bits = SENTINEL[dtype]
    b = torch.empty(shape, dtype=dtype, device=DEV)
    b.view(idt).fill_(bits)
    return b


def untouched(buf):
    idt, bits = SENTINEL[buf.dtype]
    return (buf.view(idt) == bits).cpu()


def assert_written_set(buf, region, what):
    """Exactly the elements of `region` (an index tuple) were written."""
    keep = torch.ones(buf.shape, dtype=torch.bool)
    keep[region] = False
    got = untouched(buf)
    bad = got != keep
    assert not bool(bad.any()), "%s (%s): written set differs at %d elements, first %s" % (
        what, ops.get_precision(), int(bad.sum()), bad.nonzero()[:4].tolist())


def act_fwd(v, act):
    return {ACT_NONE: lambda t: t, ACT_RELU: torch.relu, ACT_LRELU: lambda t: F.leaky_relu(t, 0.2), ACT_TANH: torch.tanh}[act](v)


def nearest_up(x, shift):
    return x.repeat_interleave(2, 2).repeat_interleave(2, 3) if shift else x


def flavour_lib():
    """The C-ABI handle of the current flavour (for the fp32-only entry points, which exist in both)."""
    return capi.lib(ops.STORAGE[0])


# ------------------------------------------------------------------------------------------------ 1. conv2d, LINEAR epilogue

CONV_CASES = [  # name, n, cin, cout, H, W, form, act, epilogue, output
    ("3x3_n13", 2, 64, 13, 17, 13, "3x3", ACT_LRELU, "shift", "slice"),          # BNT 64, one partial 8-channel group
    ("3x3_n160_scale", 1, 128, 160, 9, 11, "3x3", ACT_RELU, "scale", "slice"),   # BNT 128: second N tile 32 columns wide
    ("3x3_n288_tanh", 1, 64, 288, 7, 9, "3x3", ACT_TANH, "shift", "slice"),      # three N tiles, the last 32 wide
    ("1x1_n384", 2, 96, 384, 9, 7, "1x1", ACT_NONE, "shift", "slice"),
    ("3x3_n20_res16_3img", 3, 24, 20, 4, 4, "3x3", ACT_RELU, "res16", "slice"),  # one tile over 3 images, residual pad channels
    ("3x3_n96_res16_lrelu", 1, 32, 96, 11, 13, "3x3", ACT_LRELU, "res16", "slice"),
    ("3x3_n13_res32", 1, 40, 13, 9, 7, "3x3", ACT_TANH, "res32", "slice"),      # fp32 residual (res_c = 13)
    ("4x4p2_n64", 2, 40, 64, 11, 9, "4x4p2", ACT_LRELU, "shift", "slice"),       # output (H+1) x (W+1)
    ("4x4p2_n1_nchw", 1, 256, 1, 17, 13, "4x4p2", ACT_NONE, "shift", "nchw"),    # discriminator logit
    ("s2d_k3_n96", 1, 16, 96, 17, 13, "s2d_k3", ACT_NONE, "none", "slice"),      # stride 2 as 2x2/p1 on space-to-depth
    ("s2d_k4_c9_n32", 2, 9, 32, 19, 11, "s2d_k4", ACT_LRELU, "shift", "slice"),  # thin input, k4/s2/p2
    ("im2col_c7_n64", 2, 7, 64, 12, 9, "im2col", ACT_RELU, "shift", "slice"),    # the 1x1 form over the 7-channel label map
    ("3x3_c7_n128", 2, 7, 128, 13, 11, "3x3", ACT_LRELU, "shift", "slice"),
    ("3x3_c2080_n64", 1, 2080, 64, 6, 5, "3x3", ACT_NONE, "shift", "slice"),     # K = 18720: 1170 wgmma steps
    ("3x3_c1040_n384", 1, 1040, 384, 5, 7, "3x3", ACT_LRELU, "scale", "slice"),
    ("3x3_n1_f32p1", 2, 32, 1, 20, 12, "3x3", ACT_TANH, "shift", "f32p1"),       # fp32 NHWC, pitch 1
    ("3x3_n2_f32p2_3img", 3, 48, 2, 4, 4, "3x3", ACT_NONE, "shift", "f32p2"),    # fp32 NHWC, pitch 2
    ("3x3_n3_f32p4", 1, 32, 3, 33, 63, "3x3", ACT_NONE, "shift", "f32p4"),       # fp32 NHWC, 3 channels of a 4-wide pitch
    ("3x3_n3_nchw_3img", 3, 40, 3, 4, 4, "3x3", ACT_TANH, "shift", "nchw"),      # fp32 NCHW (image head)
]
FORMS = {"3x3": (3, 1, 1), "1x1": (1, 0, 1), "4x4p2": (4, 2, 1), "s2d_k3": (3, 1, 2), "s2d_k4": (4, 2, 2), "im2col": (3, 1, 1)}


def conv_out_hw(H, W, form):
    k, pad, stride = FORMS[form]
    return (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1


def conv_inputs(case, seed=31):
    """CPU operands of one LINEAR case, already rounded to the storage type where the kernel reads them in 16 bits."""
    name, n, cin, cout, H, W, form, act, epi, out = case
    k = FORMS[form][0]
    g = gen(seed)
    oh, ow = conv_out_hw(H, W, form)
    mag = spread(cout)
    x = q(rnd(g, n, cin, H, W) * spread(cin)[None, :, None, None])
    w = q(rnd(g, cout, cin, k, k, scale=(1.0 / (cin * k * k)) ** 0.5) * mag[:, None, None, None])
    d = dict(x=x, w=w, scale=None, shift=None, res=None, res_pad=None)
    if epi in ("shift", "scale", "res16", "res32"):
        d["shift"] = (rnd(g, cout, scale=0.1) * mag).float().double()
    if epi == "scale":
        d["scale"] = (torch.rand(cout, generator=g) + 0.5).float().double()
    if epi in ("res16", "res32"):
        r = rnd(g, n, ops.round_up(cout, 8), oh, ow) * F.pad(mag, (0, ops.round_up(cout, 8) - cout), value=1.0)[None, :, None, None]
        r = q(r) if epi == "res16" else r.float().double()
        d["res"], d["res_pad"] = r[:, :cout], r[:, cout:]
    return d


def conv_ref(case, d):
    """fp64 act(conv(x, w) * scale + shift + res) and its absolute-value map."""
    name, n, cin, cout, H, W, form, act, epi, out = case
    k, pad, stride = FORMS[form]
    v = F.conv2d(d["x"], d["w"], stride=stride, padding=pad)
    S = F.conv2d(d["x"].abs(), d["w"].abs(), stride=stride, padding=pad)
    bc = lambda t: t[None, :, None, None]
    if d["scale"] is not None:
        v, S = v * bc(d["scale"]), S * bc(d["scale"].abs())
    if d["shift"] is not None:
        v, S = v + bc(d["shift"]), S + bc(d["shift"].abs())
    if d["res"] is not None:
        v, S = v + d["res"], S + d["res"].abs()
    return act_fwd(v, act), S


@pytest.mark.parametrize("case", CONV_CASES, ids=lambda c: c[0])
def test_conv2d_linear(case, precision):
    """hrv_conv2d_fwd, LINEAR epilogue: input read through a channel slice with garbage around it, output inside a NaN-sentinel buffer
    with an extra image.  16-bit outputs are written on [c0, c0 + roundup8(c)) (pad channels = act(0 + residual pad)); fp32 outputs on
    exactly their view.  Values against fp64 torch per element."""
    name, n, cin, cout, H, W, form, act, epi, out = case
    u = U16[precision]
    d = conv_inputs(case)
    oh, ow = conv_out_hw(H, W, form)
    k, pad, stride = FORMS[form]
    xa = upload(d["x"], c0=8, pitch=8 + ops.round_up(cin, 8) + 8)
    if form.startswith("s2d"):
        xa = ops.space_to_depth(xa)
        pw = ops.pack_weight(ops.s2d_weight(d["w"].float().to(DEV), pad), (1, 1), cin_total=xa.c)
    elif form == "im2col":
        from hrviton_b200.autograd_g import im2col_weight
        xa = ops.im2col(xa, 3, 3, 1)
        pw = ops.pack_weight(im2col_weight(d["w"].float().to(DEV), xa.c), (0, 0))
    else:
        pw = ops.pack_weight(d["w"].float().to(DEV), (pad, pad))
    c8 = ops.round_up(cout, 8)
    res = None
    if epi == "res16":
        res = upload(torch.cat([d["res"], d["res_pad"]], 1), pitch=c8)
        res = Act(res.buf, c=cout)
    elif epi == "res32":
        res = Act(d["res"].permute(0, 2, 3, 1).float().contiguous().to(DEV), c=cout)
    sc = d["scale"].float().to(DEV) if d["scale"] is not None else None
    sh = d["shift"].float().to(DEV) if d["shift"] is not None else None
    if out == "slice":
        big = sentinel_buf((n + 1, oh, ow, 8 + c8 + 8), ops.STORAGE[0])
        ops.conv2d(xa, pw, Act(big[:n], c=cout, c0=8), act=act, scale=sc, shift=sh, res=res)
        region, got = (slice(0, n), slice(None), slice(None), slice(8, 8 + c8)), big[:n, ..., 8:8 + cout].permute(0, 3, 1, 2)
    elif out == "nchw":
        big = sentinel_buf((n + 1, cout, oh, ow), torch.float32)
        ops.conv2d(xa, pw, big[:n], act=act, scale=sc, shift=sh, res=res, out_layout=capi.NCHW)
        region, got = (slice(0, n),), big[:n]
    else:
        P, c0 = {"f32p1": (1, 0), "f32p2": (2, 0), "f32p4": (4, 1)}[out]
        big = sentinel_buf((n + 1, oh, ow, P), torch.float32)
        ops.conv2d(xa, pw, Act(big[:n], c=cout, c0=c0), act=act, scale=sc, shift=sh, res=res)
        region, got = (slice(0, n), slice(None), slice(None), slice(c0, c0 + cout)), big[:n, ..., c0:c0 + cout].permute(0, 3, 1, 2)
    torch.cuda.synchronize()
    assert_written_set(big, region, "conv2d " + name)
    ref, S = conv_ref(case, d)
    check("conv2d LINEAR" + (" fp32 out" if out != "slice" else ""), got, ref, S, u if out == "slice" else 0.0)
    if out == "slice" and c8 > cout:  # pad channels: act(0 + the residual's pad channels)
        rp = d["res_pad"] if epi == "res16" else torch.zeros(n, c8 - cout, oh, ow, dtype=torch.float64)
        check("conv2d LINEAR pad channels", big[:n, ..., 8 + cout:8 + c8].permute(0, 3, 1, 2), act_fwd(rp, act), rp.abs(), u)


def test_conv_cases_cover_the_gemm_widths():
    ng = {c[3] for c in CONV_CASES}
    assert {1, 2, 3, 13, 20, 32, 64, 96, 160, 288, 384} <= ng
    assert min(ng) <= 64 < max(ng)  # both N-tile widths (64 / 128 columns)


# ------------------------------------------------------------------------------------------------ 2. conv2d, SPADE epilogue

SPADE_CASES = [  # name, n, cin (of the gamma|beta conv), x0 channels, x1 channels, H, W, x0_shift, noise_scale (None: no noise), act
    ("c80_half_x1_ns0.01", 2, 48, 64, 16, 18, 14, 1, 1e-2, ACT_LRELU),
    ("c80_full_ns1", 1, 32, 80, 0, 17, 13, 0, 1.0, ACT_LRELU),
    ("c80_half_x1_3img", 3, 48, 64, 16, 4, 4, 1, None, ACT_NONE),
    ("c80_full_x1_ns0.01", 2, 40, 64, 16, 9, 11, 0, 1e-2, ACT_NONE),
    ("c1040_half_x1_ns0.3", 1, 64, 1024, 16, 6, 8, 1, 0.3, ACT_LRELU),
    ("c1040_full", 1, 32, 1040, 0, 5, 7, 0, None, ACT_LRELU),
]


def spade_inputs(case, seed=32):
    name, n, cin, c0, c1, H, W, shift, nsc, act = case
    g = gen(seed)
    C = c0 + c1
    actv = q(torch.relu(rnd(g, n, cin, H, W)))
    ws = (1.0 / (cin * 9)) ** 0.5
    d = dict(actv=actv, wg=q(rnd(g, C, cin, 3, 3, scale=ws)), wb=q(rnd(g, C, cin, 3, 3, scale=ws)),
             bg=rnd(g, C, scale=0.1).float().double(), bb=rnd(g, C, scale=0.1).float().double(),
             x0=q(rnd(g, n, c0, H >> shift, W >> shift) * spread(c0)[None, :, None, None] + 0.5),
             x1=q(rnd(g, n, c1, H, W, mean=-0.3)) if c1 else None,
             noise=rnd(g, n, H, W).float().double() if nsc is not None else None,
             ns=(rnd(g, C) * nsc).float().double() if nsc is not None else None)
    return d


def spade_ref(case, d, mean, rstd):
    """fp64 SPADE modulation with the given (fp32) statistics: {output: (ref, S)} for out and gamma."""
    name, n, cin, c0, c1, H, W, shift, nsc, act = case
    gamma = F.conv2d(d["actv"], d["wg"], d["bg"], padding=1)
    beta = F.conv2d(d["actv"], d["wb"], d["bb"], padding=1)
    Sg = F.conv2d(d["actv"].abs(), d["wg"].abs(), d["bg"].abs(), padding=1)
    Sb = F.conv2d(d["actv"].abs(), d["wb"].abs(), d["bb"].abs(), padding=1)
    xs = nearest_up(d["x0"], shift)
    if d["x1"] is not None:
        xs = torch.cat([xs, d["x1"]], 1)
    nz = d["noise"][:, None] * d["ns"][None, :, None, None] if d["noise"] is not None else torch.zeros_like(xs)
    m, r = mean[:, :, None, None], rstd[:, :, None, None]
    xn = (xs + nz - m) * r
    Sxn = (xs.abs() + nz.abs() + m.abs()) * r
    return {"out": (act_fwd(xn * (1 + gamma) + beta, act), Sxn * (1 + Sg) + Sb), "gamma": (gamma, Sg)}


@pytest.mark.parametrize("case", SPADE_CASES, ids=lambda c: c[0])
def test_conv2d_spade(case, precision):
    """hrv_conv2d_fwd, SPADE epilogue with the kernel's own statistics (hrv_instnorm_stats): out and gamma_out as channel slices of
    NaN-sentinel buffers, x0 at full or half resolution, with and without x1 and noise.  C = 80 leaves the second N tile 32 columns
    wide; C = 1040 runs 9 N tiles."""
    name, n, cin, c0, c1, H, W, shift, nsc, act = case
    u = U16[precision]
    d = spade_inputs(case)
    C = c0 + c1
    a_actv = upload(d["actv"], c0=8, pitch=8 + ops.round_up(cin, 8) + 8)
    a_x0 = upload(d["x0"], c0=8, pitch=8 + c0 + 8)
    a_x1 = upload(d["x1"], c0=8, pitch=8 + c1 + 16) if c1 else None
    noise = d["noise"].float().to(DEV).contiguous() if nsc is not None else None
    ns = d["ns"].float().to(DEV) if nsc is not None else None
    mean, rstd = ops.instnorm_stats(a_x0, shift, a_x1, H, W, noise, ns)
    pw = ops.pack_weight(d["wg"].float().to(DEV), (1, 1), interleave=d["wb"].float().to(DEV))
    sh = torch.stack([d["bg"], d["bb"]], 1).reshape(-1).float().to(DEV)
    out_big = sentinel_buf((n + 1, H, W, C + 24), ops.STORAGE[0])
    gam_big = sentinel_buf((n + 1, H, W, C + 16), ops.STORAGE[0])
    ops.conv2d_spade(a_actv, pw, Act(out_big[:n], c=C, c0=16), a_x0, shift, a_x1, mean, rstd, noise, ns, sh, act,
                     gamma_out=Act(gam_big[:n], c=C, c0=8))
    torch.cuda.synchronize()
    assert_written_set(out_big, (slice(0, n), slice(None), slice(None), slice(16, 16 + C)), "spade out")
    assert_written_set(gam_big, (slice(0, n), slice(None), slice(None), slice(8, 8 + C)), "spade gamma_out")
    ref = spade_ref(case, d, mean.double().cpu(), rstd.double().cpu())
    check("conv2d SPADE out", out_big[:n, ..., 16:16 + C].permute(0, 3, 1, 2), *ref["out"], u)
    check("conv2d SPADE gamma_out", gam_big[:n, ..., 8:8 + C].permute(0, 3, 1, 2), *ref["gamma"], u)


# ------------------------------------------------------------------------------------------------ 3. statistics

OFFSETS = (0.0, 8.0, 64.0)  # mean / std per channel, cycling over the channels of one tensor


def offset_data(g, n, c, h, w):
    """Channels of std 1 ... 1e-3 (spread) with mean / std cycling through OFFSETS."""
    sig = spread(c)
    off = torch.tensor(OFFSETS)[torch.arange(c) % len(OFFSETS)] * sig
    return q(rnd(g, n, c, h, w) * sig[None, :, None, None] + off[None, :, None, None])


def stats_ref(z, T, dims):
    """fp64 mean / biased var of z over `dims` and the bounds of the single-pass formula (T >= |z| elementwise)."""
    m, v = z.mean(dims), z.var(dims, unbiased=False)
    ET, ET2 = T.mean(dims), (T * T).mean(dims)
    dm = K_ACC * EPS32 * ET + EPS32 * m.abs()
    dv = K_ACC * EPS32 * (ET2 + 2 * m.abs() * ET)
    return m, v, dm, dv


def check_stats(what, mean, rstd, z, T, dims=(2, 3)):
    m, v, dm, dv = stats_ref(z, T, dims)
    r = (v + EPS_NORM).rsqrt()
    record(what + " mean", ratio(mean, m, dm))
    record(what + " rstd", ratio(rstd, r, r * (0.5 * dv / (v + EPS_NORM) + 2 * EPS32)))


STATS_CASES = [  # n, x0 channels, x1 channels, H, W, x0_shift, noise
    (2, 64, 16, 38, 30, 1, True),
    (3, 24, 0, 37, 29, 0, True),
    (1, 1024, 16, 10, 14, 1, True),
    (2, 48, 8, 13, 11, 0, False),
    (4, 16, 0, 3, 5, 0, True),
]


def stats_inputs(case, seed=33):
    n, c0, c1, H, W, shift, with_noise = case
    g = gen(seed)
    x0 = offset_data(g, n, c0, H >> shift, W >> shift)
    x1 = offset_data(g, n, c1, H, W) if c1 else None
    xs = nearest_up(x0, shift)
    if x1 is not None:
        xs = torch.cat([xs, x1], 1)
    noises = [rnd(g, n, H, W).float().double() for _ in range(2)] if with_noise else [None, None]
    nss = [(rnd(g, c0 + c1) * s).float().double() for s in (0.3, 1e-2)] if with_noise else [None, None]
    return x0, x1, xs, noises, nss


def with_noise(xs, noise, ns):
    if noise is None:
        return xs, xs.abs()
    t = noise[:, None] * ns[None, :, None, None]
    return xs + t, xs.abs() + t.abs()


@pytest.mark.parametrize("case", STATS_CASES, ids=lambda c: "n%d_c%d+%d_%dx%d_s%d_nz%d" % c)
def test_instnorm_stats(case, precision):
    """hrv_instnorm_stats (x0 possibly at half resolution, x1, noise) against fp64 statistics of the stored values, with channel means
    of 0, 8 and 64 standard deviations in the same tensor."""
    n, c0, c1, H, W, shift, wn = case
    x0, x1, xs, noises, nss = stats_inputs(case)
    dev = lambda t: t.float().to(DEV).contiguous() if t is not None else None
    mean, rstd = ops.instnorm_stats(upload(x0, c0=8, pitch=8 + c0 + 8), shift, upload(x1) if x1 is not None else None, H, W,
                                    dev(noises[0]), dev(nss[0]))
    torch.cuda.synchronize()
    z, T = with_noise(xs, noises[0], nss[0])
    check_stats("instnorm_stats", mean, rstd, z, T)


@pytest.mark.parametrize("norms", [1, 2])
@pytest.mark.parametrize("case", STATS_CASES, ids=lambda c: "n%d_c%d+%d_%dx%d_s%d_nz%d" % c)
def test_instnorm_stats2(case, norms, precision):
    """hrv_instnorm_stats2: one or two norms over the same source, each with its own noise (the second with noise_scale ~ 1e-2)."""
    n, c0, c1, H, W, shift, wn = case
    x0, x1, xs, noises, nss = stats_inputs(case)
    dev = lambda t: t.float().to(DEV).contiguous() if t is not None else None
    outs = ops.instnorm_stats2(upload(x0, c0=8, pitch=8 + c0 + 8), shift, upload(x1) if x1 is not None else None, H, W,
                               [dev(t) for t in noises[:norms]], [dev(t) for t in nss[:norms]])
    torch.cuda.synchronize()
    for j in range(norms):
        z, T = with_noise(xs, noises[j], nss[j])
        check_stats("instnorm_stats2", outs[j][0], outs[j][1], z, T)


@pytest.mark.parametrize("shape", [(3, 24, 17, 15), (2, 64, 9, 7), (8, 16, 4, 4)])
def test_batchnorm_stats(shape, precision):
    """ops.batchnorm_stats (the statistics kernel's per-image sums combined over N*H*W): mean and biased variance."""
    n, c, H, W = shape
    x = offset_data(gen(34), n, c, H, W)
    mean, var = ops.batchnorm_stats(upload(x))
    torch.cuda.synchronize()
    m, v, dm, dv = stats_ref(x, x.abs(), (0, 2, 3))
    record("batchnorm_stats mean", ratio(mean, m, dm))
    record("batchnorm_stats var", ratio(var, v, dv + EPS32 * v))


# ------------------------------------------------------------------------------------------------ 4. elementwise and resampling


@pytest.mark.parametrize("act", [ACT_NONE, ACT_RELU, ACT_LRELU, ACT_TANH])
@pytest.mark.parametrize("shape", [(2, 20, 9, 7), (3, 64, 4, 5)])
def test_instnorm_apply(shape, act, precision):
    """hrv_instnorm_apply: act((x - mean) * rstd) from a channel slice into a slice of a sentinel buffer; the pad channels up to the
    next multiple of 8 are written as 0."""
    n, c, H, W = shape
    u = U16[precision]
    g = gen(35)
    x = offset_data(g, n, c, H, W)
    mean32 = x.mean((2, 3)).float()
    rstd32 = (x.var((2, 3), unbiased=False) + EPS_NORM).rsqrt().float()
    c8 = ops.round_up(c, 8)
    big = sentinel_buf((n + 1, H, W, 8 + c8 + 8), ops.STORAGE[0])
    ops.instnorm_apply(upload(x, c0=8, pitch=8 + c8 + 8), mean32.to(DEV), rstd32.to(DEV), act, out=Act(big[:n], c=c, c0=8))
    torch.cuda.synchronize()
    assert_written_set(big, (slice(0, n), slice(None), slice(None), slice(8, 8 + c8)), "instnorm_apply")
    m, r = mean32.double()[:, :, None, None], rstd32.double()[:, :, None, None]
    check("instnorm_apply", big[:n, ..., 8:8 + c].permute(0, 3, 1, 2), act_fwd((x - m) * r, act), (x.abs() + m.abs()) * r, u)
    if c8 > c:
        check_exact("instnorm_apply pad channels", big[:n, ..., 8 + c:8 + c8].float().cpu(), torch.zeros(n, H, W, c8 - c))


@pytest.mark.parametrize("shape", [(2, 20, 9, 7), (1, 64, 17, 13), (3, 8, 1, 5), (1, 24, 2, 3)])
def test_avgpool3s2(shape, precision):
    """hrv_avgpool3s2 (3x3, stride 2, pad 1, count_include_pad=False) at odd extents, from a channel slice."""
    n, c, H, W = shape
    x = q(rnd(gen(36), n, c, H, W) * spread(c)[None, :, None, None])
    y = ops.avgpool3s2(upload(x, c0=8, pitch=8 + ops.round_up(c, 8) + 8))
    torch.cuda.synchronize()
    pool = lambda t: F.avg_pool2d(t, 3, stride=2, padding=1, count_include_pad=False)
    check("avgpool3s2", nchw(y), pool(x), pool(x.abs()), U16[precision])


@pytest.mark.parametrize("with_b", [False, True])
@pytest.mark.parametrize("shape", [(2, 24, 7, 5), (1, 16, 1, 3), (2, 40, 9, 1), (1, 20, 4, 6)])
def test_bilinear_up2_add(shape, with_b, precision):
    """hrv_bilinear_up2_add: F.interpolate(a, x2, bilinear) (+ b) at odd low-resolution extents, including 1-wide maps."""
    n, c, h, w = shape
    g = gen(38)
    a = q(rnd(g, n, c, h, w) * spread(c)[None, :, None, None])
    b = q(rnd(g, n, c, 2 * h, 2 * w, scale=0.1)) if with_b else None
    out = Act.empty(n, 2 * h, 2 * w, c)
    ops.bilinear_up2_add(upload(a, c0=8, pitch=8 + ops.round_up(c, 8) + 8), upload(b) if with_b else None, out)
    torch.cuda.synchronize()
    up = lambda t: F.interpolate(t, scale_factor=2, mode="bilinear", align_corners=False)
    ref, S = up(a), up(a.abs())
    if with_b:
        ref, S = ref + b, S + b.abs()
    check("bilinear_up2_add", nchw(out), ref, S, U16[precision])


# ------------------------------------------------------------------------------------------------ 5. flow warps and blur


def gather_ref(src, x0, y0, tx, ty):
    """fp64 bilinear gather at the kernel's fp32 taps (border: the second tap clamps onto the first with weight tx = 0 there)."""
    n, c, H, W = src.shape
    x0, y0 = torch.from_numpy(x0).long(), torch.from_numpy(y0).long()
    tx, ty = torch.from_numpy(tx).double(), torch.from_numpy(ty).double()
    x1, y1 = (x0 + 1).clamp(max=W - 1), (y0 + 1).clamp(max=H - 1)
    b = torch.arange(n)[:, None, None]
    s = src.permute(0, 2, 3, 1)
    ref = torch.zeros(x0.shape + (c,), dtype=torch.float64)
    S = torch.zeros_like(ref)
    for yy, wy in ((y0, 1 - ty), (y1, ty)):
        for xx, wx in ((x0, 1 - tx), (x1, tx)):
            v, w = s[b, yy, xx], (wy * wx)[..., None]
            ref, S = ref + v * w, S + v.abs() * w.abs()
    return ref.permute(0, 3, 1, 2), S.permute(0, 3, 1, 2)


@pytest.mark.parametrize("c,hl,wl,scale,dst32", [(20, 16, 12, 3.0, False), (20, 16, 12, 12.0, True), (384, 8, 16, 1.0, False),
                                                 (4, 16, 16, 12.0, True)])
def test_flow_warp(c, hl, wl, scale, dst32, precision):
    """hrv_flow_warp from a 16-bit source (channel slice) into a 16-bit or fp32 destination: gather indices and the up-sampled flow
    bit-exact with the oracle's fp32 chain, values per element.  scale 12 clamps many coordinates on both sides."""
    n, H, W = 2, 2 * hl, 2 * wl
    g = gen(39)
    flow = rnd(g, n, hl, wl, 2, scale=scale).float()
    src = q(rnd(g, n, c, H, W) * spread(c)[None, :, None, None])
    if dst32:
        big = sentinel_buf((n, H, W, c + 3), torch.float32)
        dst = Act(big, c=c)
    else:
        dst = Act.empty(n, H, W, c)
    flow_up, idx = ops.flow_warp(flow.to(DEV).contiguous(), upload(src, c0=8, pitch=8 + ops.round_up(c, 8) + 8), dst, want_idx=True)
    torch.cuda.synchronize()
    x0, y0, tx, ty = orc.np_flow_warp_coords(flow.numpy(), H, W, H, W)
    idx = idx.cpu()
    check_exact("flow_warp indices", idx, torch.from_numpy(np.stack([x0, y0], -1).astype(np.int32)))
    check_exact("flow_warp flow_up", flow_up.cpu(), torch.from_numpy(np.moveaxis(orc.np_bilinear_up2(np.moveaxis(flow.numpy(), -1, 1)), 1, -1)))
    ref, S = gather_ref(src, x0, y0, tx, ty)
    if dst32:
        assert_written_set(big, (slice(None), slice(None), slice(None), slice(0, c)), "flow_warp fp32 dst")
        check("flow_warp fp32 dst", nchw(dst), ref, S)
    else:
        check("flow_warp", nchw(dst), ref, S, U16[precision])


def np_flow_nchw_coords(flow, H, W, Hs, Ws, div):
    """The fp32 chain of flow_warp_nchw_kernel restated in numpy (every operation rounded to fp32, no contraction): the grid
    (gx, gy) and the taps (sx0, sy0, tx, ty) of each output pixel."""
    f32 = np.float32
    n, hl, wl, _ = flow.shape

    def axis(n_out, n_lo):
        f = np.maximum((f32(n_lo) / f32(n_out)) * (np.arange(n_out, dtype=f32) + f32(0.5)) - f32(0.5), f32(0))
        i0 = f.astype(np.int64)
        lo = f - i0.astype(f32)
        return i0, np.minimum(i0 + 1, n_lo - 1), lo, f32(1) - lo

    y0, y1, ly, hy = axis(H, hl)
    x0, x1, lx, hx = axis(W, wl)
    ly, hy, lx, hx = ly[:, None], hy[:, None], lx[None, :], hx[None, :]
    fl = flow.astype(f32)
    f00, f01 = fl[:, y0][:, :, x0], fl[:, y0][:, :, x1]
    f10, f11 = fl[:, y1][:, :, x0], fl[:, y1][:, :, x1]
    u = [hy * (hx * f00[..., k] + lx * f01[..., k]) + ly * (hx * f10[..., k] + lx * f11[..., k]) for k in range(2)]
    gx = u[0] / f32(div[0]) + torch.linspace(-1.0, 1.0, W).numpy()[None, None, :]
    gy = u[1] / f32(div[1]) + torch.linspace(-1.0, 1.0, H).numpy()[None, :, None]
    ix = np.clip(((gx + f32(1)) * f32(Ws) - f32(1)) / f32(2), f32(0), f32(Ws - 1))
    iy = np.clip(((gy + f32(1)) * f32(Hs) - f32(1)) / f32(2), f32(0), f32(Hs - 1))
    bx, by = np.floor(ix), np.floor(iy)
    return np.stack([gx, gy], -1), bx.astype(np.int64), by.astype(np.int64), ix - bx, iy - by


@pytest.mark.parametrize("shape", [((2, 16, 12), (50, 37), 3), ((1, 16, 12), (64, 48), 4)])
def test_flow_warp_nchw(shape, precision):
    """hrv_flow_warp_nchw through the flavour's own handle (hrv_flow_warp_nchw / _f16): the grid bit-exact with the restated fp32
    chain, the warped cloth and mask per element at its taps."""
    (n, hl, wl), (H, W), c = shape
    g = gen(40)
    flow = rnd(g, n, hl, wl, 2, scale=6.0).float()
    src = rnd(g, n, c, H, W).float()
    mask = (torch.rand(n, 1, H, W, generator=g) > 0.3).float()
    div = ((wl - 1.0) / 2.0, (hl - 1.0) / 2.0)
    out = torch.empty((n, c, H, W), device=DEV)
    grid = torch.empty((n, H, W, 2), device=DEV)
    mout = torch.empty((n, 1, H, W), device=DEV)
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    fd, sd, md = flow.to(DEV), src.to(DEV), mask.to(DEV)
    capi.check(flavour_lib().hrv_flow_warp_nchw(p(fd), n, hl, wl, p(ops.linspace_table(W, DEV)), p(ops.linspace_table(H, DEV)), p(sd), c, H,
                                                W, p(out), H, W, float(div[0]), float(div[1]), p(grid), p(md), None, p(mout), 0,
                                                ops._stream()), "flow_warp_nchw")
    torch.cuda.synchronize()
    gref, x0, y0, tx, ty = np_flow_nchw_coords(flow.numpy(), H, W, H, W, div)
    check_exact("flow_warp_nchw grid", grid.cpu(), torch.from_numpy(gref))
    ref, S = gather_ref(src.double(), x0, y0, tx, ty)
    check("flow_warp_nchw", out.cpu(), ref, S)
    mref, mS = gather_ref(mask.double(), x0, y0, tx, ty)
    check("flow_warp_nchw mask", mout.cpu(), mref, mS)


@pytest.mark.parametrize("ksize,sigma", [(15, 3.0), (7, 1.5)])
def test_gaussian_blur(ksize, sigma, precision):
    """hrv_gaussian_blur through the flavour's own handle against the fp64 separable Gaussian (zero padding) on odd extents."""
    x = rnd(gen(41), 2, 5, 70, 45).float()
    out = torch.empty((2, 5, 70, 45), device=DEV)
    xd = x.to(DEV)
    capi.check(flavour_lib().hrv_gaussian_blur(ctypes.c_void_p(xd.data_ptr()), 10, 70, 45, ksize, float(sigma), ctypes.c_void_p(out.data_ptr()),
                                               ops._stream()), "gaussian_blur")
    torch.cuda.synchronize()
    r = ksize // 2
    k = torch.arange(ksize, dtype=torch.float64) - r
    gk = torch.exp(-k * k / (2 * sigma * sigma))
    gk = gk / gk.sum()
    blur = lambda t: F.conv2d(F.conv2d(t.reshape(10, 1, 70, 45), gk.view(1, 1, 1, ksize), padding=(0, r)), gk.view(1, 1, ksize, 1),
                              padding=(r, 0)).reshape(2, 5, 70, 45)
    xd64 = x.double()
    check("gaussian_blur", out.cpu(), blur(xd64), blur(xd64.abs()))


def parse_blur_argmax(seg, size, group_of, groups):
    n, c, h, w = seg.shape
    H, W = size
    idx = torch.empty((n, 1, H, W), dtype=torch.int64, device=DEV)
    onehot = torch.empty((n, groups, H, W), dtype=torch.float32, device=DEV) if group_of is not None else None
    garr = (ctypes.c_int32 * c)(*group_of) if group_of is not None else None
    capi.check(flavour_lib().hrv_parse_blur_argmax(ctypes.c_void_p(seg.data_ptr()), n, c, h, w, H, W, garr, groups, ctypes.c_void_p(idx.data_ptr()),
                                                   ctypes.c_void_p(onehot.data_ptr()) if onehot is not None else None, 0, None, ops._stream()),
               "parse_blur_argmax")
    return idx, onehot


def test_parse_blur_argmax(precision):
    """hrv_parse_blur_argmax through the flavour's own handle: the arg-max of the fp32 resize -> blur pipeline, except where the two
    best blurred scores are within 1e-5; the one-hot planes exactly the regrouped arg-max."""
    from hrviton_b200 import synth, train_step
    n, H, W = 2, 160, 96
    seg = synth.normalish((n, 13, 40, 24), 7, "seg").to(DEV)
    for size in [(H, W), (50, 45)]:
        idx, onehot = parse_blur_argmax(seg, size, train_step.GROUP_OF_13, 7)
        torch.cuda.synchronize()
        gauss = train_step.gaussian_blur_15_3(F.interpolate(seg, size=size, mode="bilinear"))
        diff = idx != gauss.argmax(1, keepdim=True)
        if bool(diff.any()):
            top2 = gauss.topk(2, dim=1).values
            assert float((top2[:, 0] - top2[:, 1])[diff[:, 0]].max()) < 1e-5
        assert float(diff.float().mean()) < 2e-3
        m = torch.zeros(7, 13, device=DEV)
        for i, grp in enumerate(train_step.LABELS7):
            m[i, grp] = 1.0
        check_exact("parse_blur_argmax onehot", onehot, torch.einsum("ij,njhw->nihw", m,
                                                                     torch.zeros(n, 13, *size, device=DEV).scatter_(1, idx, 1.0)))


# ------------------------------------------------------------------------------------------------ 6. bit-exact ops


@pytest.mark.parametrize("shape", [(2, 20, 9, 7), (1, 64, 5, 3), (3, 8, 2, 2)])
def test_maxpool2(shape, precision):
    """hrv_maxpool2_fwd from a channel slice at odd extents (the last row / column is not read)."""
    n, c, H, W = shape
    x = q(rnd(gen(42), n, c, H, W))
    y = ops.maxpool2(upload(x, c0=8, pitch=8 + ops.round_up(c, 8) + 8))
    torch.cuda.synchronize()
    check_exact("maxpool2", nchw(y), F.max_pool2d(x, 2))


@pytest.mark.parametrize("shape", [(2, 13, 9, 7), (1, 64, 1, 5), (3, 8, 4, 4)])
def test_space_to_depth(shape, precision):
    """hrv_space_to_depth at odd extents: sub-image (py, px) of the zero-extended input in channels [sub * c8, sub * c8 + c)."""
    n, c, H, W = shape
    x = q(rnd(gen(43), n, c, H, W))
    s = ops.space_to_depth(upload(x, c0=8, pitch=8 + ops.round_up(c, 8) + 8))
    torch.cuda.synchronize()
    c8 = ops.round_up(c, 8)
    got = nchw(s)
    xp = F.pad(x, (0, W & 1, 0, H & 1))
    for sub in range(4):
        check_exact("space_to_depth", got[:, sub * c8:sub * c8 + c], xp[:, :, sub >> 1::2, sub & 1::2])


@pytest.mark.parametrize("shape", [(2, 5, 12, 9, 3, 1), (1, 3, 8, 8, 3, 1), (1, 12, 5, 7, 2, 1), (2, 7, 12, 9, 3, 1)])
def test_im2col(shape, precision):
    """hrv_im2col: dst[..., tap * c + ci] = x at the tap offset (zero outside), zero past kh*kw*c.  c = 7 with 3x3 / pad 1 runs the
    specialised kernel."""
    n, c, H, W, k, pad = shape
    x = q(rnd(gen(44), n, c, H, W))
    cols = ops.im2col(upload(x, c0=8, pitch=8 + ops.round_up(c, 8) + 8), k, k, pad)
    torch.cuda.synchronize()
    xp = F.pad(x, (pad, k, pad, k))
    want = torch.zeros((n, cols.c, H, W), dtype=torch.float64)
    for ky in range(k):
        for kx in range(k):
            t = ky * k + kx
            want[:, t * c:(t + 1) * c] = xp[:, :, ky:ky + H, kx:kx + W]
    check_exact("im2col", nchw(cols), want)


def test_nhwc_to_nchw(precision):
    """hrv_nhwc_to_nchw of a channel slice: exact widening to fp32."""
    x = q(rnd(gen(45), 2, 13, 9, 7))
    got = upload(x, c0=8, pitch=8 + 16 + 8).to_nchw()
    torch.cuda.synchronize()
    check_exact("nhwc_to_nchw", got.double().cpu(), x)


def test_onehot_u8(precision):
    lab = torch.randint(0, 13, (3, 1, 37, 29), dtype=torch.uint8, generator=gen(46))
    out = torch.empty((3, 13, 37, 29), device=DEV)
    ld = lab.to(DEV)
    capi.check(flavour_lib().hrv_onehot_u8(ctypes.c_void_p(ld.data_ptr()), 3, 13, 37, 29, ctypes.c_void_p(out.data_ptr()), ops._stream()),
               "onehot_u8")
    torch.cuda.synchronize()
    check_exact("onehot_u8", out.cpu(), torch.zeros(3, 13, 37, 29).scatter_(1, lab.long(), 1.0))


def special_weights(cout, cin, k, seed=47):
    """fp32 weights mixing normal values with the hard cases of a 16-bit conversion: fp16 subnormals and their ties, fp16 / bf16 ties
    between neighbours, values past the fp16 maximum (65504) and fp32 subnormals."""
    g = gen(seed)
    w = rnd(g, cout * cin * k * k)
    m = w.numel() // 8
    sub = torch.randint(1, 1024, (m,), generator=g).double()
    w[0:m] = (sub * 2.0 ** -24).float()                        # fp16 subnormals
    w[m:2 * m] = ((sub + 0.5) * 2.0 ** -24).float()            # ties between fp16 subnormals
    a16 = rnd(g, m).to(torch.float16)
    b16 = (a16.view(torch.int16) + 1).view(torch.float16)
    w[2 * m:3 * m] = (a16.float() + b16.float()) / 2             # ties between fp16 neighbours
    bits = rnd(g, m).view(torch.int32)
    w[3 * m:4 * m] = ((bits & ~0xFFFF) | 0x8000).view(torch.float32)  # ties between bf16 neighbours
    big = torch.tensor([65504.0, 65519.99, 65520.0, -65520.0, 7e4, -1e5, 3.4e38, 2.0 ** -25, -(2.0 ** -25), 1e-40, -3e-39, 2.0 ** -26])
    w[4 * m:4 * m + big.numel()] = big
    return w[torch.randperm(w.numel(), generator=g)].reshape(cout, cin, k, k).contiguous()


@pytest.mark.parametrize("k", [3, 1])
def test_pack_conv_weight(k, precision):
    """hrv_pack_conv_weight rounds each fp32 weight exactly as torch.Tensor.to(float16 / bfloat16) does (round to nearest even,
    subnormals, overflow to inf), in the [taps][n_pad][cin_k] layout with zero padding."""
    cout, cin = 20, 13
    w = special_weights(cout, cin, k)
    pw = ops.pack_weight(w.to(DEV), (k // 2, k // 2))
    torch.cuda.synchronize()
    want = torch.zeros(pw.w.shape, dtype=torch.float32)
    want[:, :cout, :cin] = w.permute(2, 3, 0, 1).reshape(k * k, cout, cin)
    check_exact("pack_conv_weight", pw.w.cpu().view(torch.int16), want.to(ops.STORAGE[0]).view(torch.int16))


NEAREST_CASES = [  # (c, in_h, in_w) -> (out_h, out_w)
    ((9, 32, 24), (32, 24)), ((9, 32, 24), (16, 12)), ((9, 32, 24), (8, 6)), ((9, 32, 24), (64, 48)), ((9, 32, 24), (2, 1)),
    ((3, 200, 336), (24, 80)),   # torch picks row 124 for dst 15 (the exact floor: 125); 7 of 80 column indices differ
    ((3, 336, 200), (80, 24)),
    ((3, 24, 80), (200, 336)),
]


@pytest.mark.parametrize("case", NEAREST_CASES, ids=lambda c: "%dx%d_to_%dx%d" % (c[0][1:] + c[1]))
def test_nchw_to_nhwc_nearest(case, precision):
    """hrv_nchw_to_nhwc with nearest resampling: bit-exact against F.interpolate(mode='nearest') rounded to the storage type, at
    dyadic and non-dyadic ratios; channels past c are written as zero."""
    (c, h, w), (oh, ow) = case
    x = rnd(gen(48), 2, c, h, w).float()
    a = ops.from_nchw(x.to(DEV), size=(oh, ow))
    torch.cuda.synchronize()
    want = F.interpolate(x, size=(oh, ow), mode="nearest").to(ops.STORAGE[0]).double()
    check_exact("nchw_to_nhwc nearest", nchw(a), want)
    check_exact("nchw_to_nhwc pad channels", a.buf[..., c:].float().cpu(), torch.zeros(2, oh, ow, a.pitch - c))
