"""Every forward entry point that takes fp32 activation storage, one at a time, against a float64 reference on the CPU: the 3xTF32
convolution in every form the fp32 networks run (LPIPS, Inception-v3 and pytorch-fid's variant, reference-precision try-on), its
hi/lo weight split, and the fp32 element paths of the HBM-bound kernels.  The fp32-storage counterpart of
tests/test_forward_kernels_gpu.py, whose data builders, sentinel buffers and checkers it reuses (fk.q is the fp32 rounding here).

The convolution bound is per element and derived from the kernel's arithmetic (conv_f32.cu), not tuned.  S is the fp64 map applied
to absolute values, conv(|x|, |w|) * |scale| + |shift| + |residual|, as in the 16-bit file.
  Split.  hi = rna_tf32(v) keeps 11 significant bits, so |v - hi| <= 2^-11 |v|; v - hi is exact in fp32 and lo = rna_tf32(v - hi)
          leaves |v - hi - lo| <= 2^-11 |v - hi| <= 2^-22 |v|, for activations (split in shared memory) and weights (split when
          packed) alike.  Each TF32 x TF32 product is exact in fp32.  lo*Bhi + hi*Blo + hi*Bhi = x*w - lo*Blo - e_x*w - hi_lo*e_w with
          every dropped term at most 2^-22 |x||w|: 3 * 2^-22 = K_SPLIT = 12 units of 2^-24 * S.
  Accumulation.  Each stage (one tap, one 32-channel K block) is 12 wgmma k8 instructions into a fresh partial, which the tensor
          core accumulates with truncation: at most about one ulp of the partial per instruction, so 12 * 2^-23 of that stage's own
          share of S, 24 * 2^-24 * S summed over the stages.  The partials are promoted with round-to-nearest fp32 adds; the longest
          chain here is KT = 9 * ceil(2080 / 32) = 585 stages, which drifts by about sqrt(585) = 24 units over terms of mixed sign.
          The epilogue adds a few roundings of the result (fmaf with scale and shift, the residual, the activation).  K_ACC = 64 of
          the 16-bit file covers the sum with room to spare, by the same sqrt(m) argument.
  fp32 outputs       |got - ref| <= (K_ACC + K_SPLIT) * 2^-24 * S
There is no storage-rounding term u*|ref|: the output is fp32.  The truncation model is conv_f32.cu's own; nobody has measured how the
H100 accumulates TF32 wgmma internally, so the worst ratios of the FWDBOUND lines are the evidence for it.  SPADE carries the GEMM bound
through the modulation as the 16-bit file does: (|x_hat| * S_gamma + S_beta) with x_hat the normalised input.

The HBM-bound kernels keep the 16-bit file's bounds with u = 0 (fp32 outputs); copies and gathers (space-to-depth, im2col, layout
changes with the nearest resize, the flow warp's indices and up-sampled flow, the weight split) must be bit-exact.
tests/test_forward_bounds_fp32_cpu.py shows that the convolution bound rejects the realistic mistakes at these shapes.

Every convolution case reads its input through a channel slice (c0 = 4 or 8, garbage around it) and writes into a NaN-sentinel buffer
with an extra image whose untouched elements must keep their bits; pad channels of NHWC outputs are checked as act(0 + residual pad)."""
import ctypes
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import test_forward_kernels_gpu as fk
from test_fp32_cpu import rna_tf32
from hrviton_b200 import capi, metrics, ops
from hrviton_b200.autograd_g import im2col_weight
from hrviton_b200.ops import ACT_LRELU, ACT_NONE, ACT_RELU, ACT_TANH, Act

orc = fk.orc
pytestmark = pytest.mark.gpu
DEV = "cuda"
EPS32 = fk.EPS32
K_SPLIT = 12  # the three-product split: see the module docstring
K_CONV = fk.K_ACC + K_SPLIT
F32 = torch.float32
REL64 = {}  # statistics op -> worst relative rstd error in the channels whose mean is 64 standard deviations


@pytest.fixture
def fp32():
    """fp32 activation storage (ops.set_precision("fp32")): the 3xTF32 convolution and the fp32 element paths."""
    ops.set_precision("fp32")
    yield
    ops.set_precision("bf16")


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    for key in sorted(k for k in fk.WORST if k[1] == "fp32"):
        extra = ("  (rstd rel err at mean/std 64: %.2e)" % REL64[key[0]]) if key[0] in REL64 else ""
        print("FWDBOUND %-40s fp32 worst = %.3f of its bound%s" % (key[0], fk.WORST.pop(key), extra))


def check_conv(what, got, ref, S):
    fk.record(what, fk.ratio(got, ref, K_CONV * EPS32 * S.double()))


# ------------------------------------------------------------------------------------------------ 1. conv2d, LINEAR epilogue

# kh, kw, pad_y, pad_x, stride, how the kernel runs it
FORMS = {"3x3": (3, 3, 1, 1, 1, "plain"), "1x1": (1, 1, 0, 0, 1, "plain"), "4x4p2": (4, 4, 2, 2, 1, "plain"),
         "5x5p2": (5, 5, 2, 2, 1, "plain"), "1x7": (1, 7, 0, 3, 1, "plain"), "7x1": (7, 1, 3, 0, 1, "plain"),
         "1x3": (1, 3, 0, 1, 1, "plain"), "3x1": (3, 1, 1, 0, 1, "plain"),
         "pool3x3": (3, 3, 1, 1, 1, "pool"),       # avg_pool2d(3, 1, 1) + 1x1 BasicConv2d folded into one 3x3 with taps w / 9
         "s2d_k3": (3, 3, 1, 1, 2, "s2d"), "s2d_k4": (4, 4, 2, 2, 2, "s2d"),
         "s2d_k3v": (3, 3, 0, 0, 2, "s2d"),        # Inception's stride-2 3x3 valid: 2x2 valid over space-to-depth
         "im2col": (3, 3, 1, 1, 1, "im2col")}

# name, n, cin, cout, H, W, form, act, epilogue, output.  The names carry the K chunking of the 32-channel K blocks: "t11" = a last K
# chunk 11 channels wide (TMA zero-fills it against the garbage channels), "t16" = 16 wide.
FP32_CASES = [
    ("1x1_c363t11_n64_lpips1", 2, 363, 64, 9, 7, "1x1", ACT_RELU, "shift", "slice"),       # LPIPS conv1 (11x11/s4 as a K = 363 GEMM)
    ("5x5p2_c64_n192_lpips2", 1, 64, 192, 9, 11, "5x5p2", ACT_RELU, "shift", "slice"),     # AlexNet conv2
    ("5x5p2_c48t16_n64_mixed5", 2, 48, 64, 7, 9, "5x5p2", ACT_RELU, "scale", "slice"),     # Inception Mixed_5 branch5x5_2
    ("1x7_c128_n192_mixed6", 1, 128, 192, 9, 11, "1x7", ACT_RELU, "scale", "slice"),       # off_x = 3, off_y = 0
    ("7x1_c160_n192_mixed6", 1, 160, 192, 11, 9, "7x1", ACT_RELU, "scale", "slice"),       # off_y = 3, off_x = 0
    ("1x7_c192_n192_mixed6", 2, 192, 192, 5, 7, "1x7", ACT_RELU, "scale", "slice"),
    ("1x3_c384_n384_cat320_mixed7", 1, 384, 384, 5, 7, "1x3", ACT_RELU, "scale", "cat320"),  # into channels 320.. of a 2048-wide concat
    ("3x1_c384_n384_cat704_mixed7", 2, 384, 384, 3, 5, "3x1", ACT_RELU, "scale", "cat704"),
    ("s2dv_c48t16_n64_35to17", 1, 48, 64, 35, 35, "s2d_k3v", ACT_RELU, "scale", "slice"),  # Inception reductions, odd extents
    ("s2dv_c192_n320_17to8_mixed7a", 1, 192, 320, 17, 17, "s2d_k3v", ACT_RELU, "scale", "slice"),
    ("pool3x3_c192_n32_branchpool", 2, 192, 32, 9, 7, "pool3x3", ACT_RELU, "scale", "slice"),
    ("1x1_c2048_n1008_fc_3img", 3, 2048, 1008, 1, 1, "1x1", ACT_NONE, "shift", "slice"),  # one tile of 128 image slots, 125 invalid
    ("3x3_c1040t16_n64_lrelu", 1, 1040, 64, 5, 6, "3x3", ACT_LRELU, "scale", "slice"),
    ("3x3_c44t12_n13_res32_lrelu", 2, 44, 13, 9, 7, "3x3", ACT_LRELU, "res32", "slice"),   # fp32 residual, res_c = 13 < store_c = 16
    ("3x3_c36t4_n24_res_tanh", 1, 36, 24, 7, 5, "3x3", ACT_TANH, "res16", "slice"),        # residual over the pad channels too
]
# The 16-bit file's LINEAR cases run unchanged on fp32 storage: both N-tile widths, the 2080- and 1040-channel K chains, the s2d_k3,
# s2d_k4 and im2col forms, fp32 NHWC outputs at pitch 1 / 2 / 4 and NCHW heads (the per-element epilogue, out_vec = 0).
CASES = [("fk_" + c[0],) + tuple(c[1:]) for c in fk.CONV_CASES] + FP32_CASES
OUT_C0 = {"slice": 8, "cat320": 320, "cat704": 704}  # NHWC outputs in the storage type: 8-channel vector stores (out_vec = 1)


def conv_out_hw(H, W, form):
    kh, kw, py, px, stride, _ = FORMS[form]
    return (H + 2 * py - kh) // stride + 1, (W + 2 * px - kw) // stride + 1


def pooled_weights(g, cin, cout, mag):
    """An eval-mode BasicConv2d (1x1 conv, BatchNorm with running statistics) folded by metrics.fold_basic_conv(pool=True)."""
    conv = torch.nn.Conv2d(cin, cout, 1, bias=False)
    bn = torch.nn.BatchNorm2d(cout, eps=1e-3)
    with torch.no_grad():
        conv.weight.copy_(fk.rnd(g, cout, cin, 1, 1, scale=(1.0 / cin) ** 0.5) * mag[:, None, None, None])
        bn.weight.copy_(torch.rand(cout, generator=g) + 0.5)
        bn.bias.copy_(fk.rnd(g, cout, scale=0.1) * mag)
        bn.running_mean.copy_(fk.rnd(g, cout, scale=0.1) * mag)
        bn.running_var.copy_(torch.rand(cout, generator=g) + 0.5)
    return metrics.fold_basic_conv(types.SimpleNamespace(conv=conv, bn=bn.eval()), pool=True)


def conv_inputs(case, seed=31):
    """CPU operands of one LINEAR case in fp64, rounded to fp32 where the kernel reads fp32 (the 16-bit file's draws for its cases)."""
    name, n, cin, cout, H, W, form, act, epi, out = case
    kh, kw, py, px, stride, kind = FORMS[form]
    g = fk.gen(seed)
    oh, ow = conv_out_hw(H, W, form)
    mag = fk.spread(cout)
    x = fk.q(fk.rnd(g, n, cin, H, W) * fk.spread(cin)[None, :, None, None])
    if kind == "pool":
        w, s, t = pooled_weights(g, cin, cout, mag)
        return dict(x=x, w=fk.q(w), scale=fk.q(s), shift=fk.q(t), res=None, res_pad=None)
    w = fk.q(fk.rnd(g, cout, cin, kh, kw, scale=(1.0 / (cin * kh * kw)) ** 0.5) * mag[:, None, None, None])
    d = dict(x=x, w=w, scale=None, shift=None, res=None, res_pad=None)
    if epi in ("shift", "scale", "res16", "res32"):
        d["shift"] = fk.q(fk.rnd(g, cout, scale=0.1) * mag)
    if epi == "scale":
        d["scale"] = fk.q(torch.rand(cout, generator=g) + 0.5)
    if epi in ("res16", "res32"):
        c8 = ops.round_up(cout, 8)
        r = fk.q(fk.rnd(g, n, c8, oh, ow) * F.pad(mag, (0, c8 - cout), value=1.0)[None, :, None, None])
        d["res"], d["res_pad"] = r[:, :cout], r[:, cout:]
    return d


def conv_ref(case, d):
    """fp64 act(conv(x, w) * scale + shift + res) and its absolute-value map S (fk.conv_ref for any kernel shape and stride)."""
    name, n, cin, cout, H, W, form, act, epi, out = case
    kh, kw, py, px, stride, kind = FORMS[form]
    conv = lambda a, b: F.conv2d(a, b, stride=stride, padding=(py, px))
    v, S = conv(d["x"], d["w"]), conv(d["x"].abs(), d["w"].abs())
    bc = lambda t: t[None, :, None, None]
    if d["scale"] is not None:
        v, S = v * bc(d["scale"]), S * bc(d["scale"].abs())
    if d["shift"] is not None:
        v, S = v + bc(d["shift"]), S + bc(d["shift"].abs())
    if d["res"] is not None:
        v, S = v + d["res"], S + d["res"].abs()
    return fk.act_fwd(v, act), S


def run_conv(case, d):
    """Runs one LINEAR case on the kernel.  Returns (sentinel buffer, written region, output view as NCHW, out_vec)."""
    name, n, cin, cout, H, W, form, act, epi, out = case
    kh, kw, py, px, stride, kind = FORMS[form]
    oh, ow = conv_out_hw(H, W, form)
    c0 = 8 if name.startswith("fk_") else 4  # fp32 TMA needs 16-byte aligned views: c0 a multiple of 4, pitch of 8
    xa = fk.upload(d["x"], c0=c0, pitch=ops.round_up(c0 + cin, 8) + 8)
    wd = d["w"].float().to(DEV)
    if kind == "s2d":
        xa = ops.space_to_depth(xa, dtype=F32)
        pw = ops.pack_weight(ops.s2d_weight(wd, py), (1, 1) if py else (0, 0), cin_total=xa.c)
    elif kind == "im2col":
        xa = ops.im2col(xa, 3, 3, 1)
        pw = ops.pack_weight(im2col_weight(wd, xa.c), (0, 0))
    else:
        pw = ops.pack_weight(wd, (py, px))
    assert pw.w.dtype == F32 and pw.w.shape[0] == 2
    c8 = ops.round_up(cout, 8)
    res = None
    if epi == "res16":  # a storage-type residual as wide as the output's pad channels
        res = Act(fk.upload(torch.cat([d["res"], d["res_pad"]], 1), pitch=c8).buf, c=cout)
    elif epi == "res32":  # pitch = cout: only channels [0, cout) carry a residual
        res = Act(d["res"].permute(0, 2, 3, 1).float().contiguous().to(DEV), c=cout)
    sc = d["scale"].float().to(DEV) if d["scale"] is not None else None
    sh = d["shift"].float().to(DEV) if d["shift"] is not None else None
    if out in OUT_C0:
        oc0 = OUT_C0[out]
        P = 2048 if out.startswith("cat") else oc0 + c8 + 8
        big = fk.sentinel_buf((n + 1, oh, ow, P), F32)
        ops.conv2d(xa, pw, Act(big[:n], c=cout, c0=oc0), act=act, scale=sc, shift=sh, res=res)
        region, got = (slice(0, n), slice(None), slice(None), slice(oc0, oc0 + c8)), big[:n, ..., oc0:oc0 + cout].permute(0, 3, 1, 2)
        return big, region, got, True
    if out == "nchw":
        big = fk.sentinel_buf((n + 1, cout, oh, ow), F32)
        ops.conv2d(xa, pw, big[:n], act=act, scale=sc, shift=sh, res=res, out_layout=capi.NCHW)
        return big, (slice(0, n),), big[:n], False
    P, oc0 = {"f32p1": (1, 0), "f32p2": (2, 0), "f32p4": (4, 1)}[out]
    big = fk.sentinel_buf((n + 1, oh, ow, P), F32)
    ops.conv2d(xa, pw, Act(big[:n], c=cout, c0=oc0), act=act, scale=sc, shift=sh, res=res)
    return big, (slice(0, n), slice(None), slice(None), slice(oc0, oc0 + cout)), big[:n, ..., oc0:oc0 + cout].permute(0, 3, 1, 2), False


@pytest.mark.parametrize("case", CASES, ids=lambda c: c[0])
def test_conv2d_linear_fp32(case, fp32):
    """hrv_conv2d_fwd on fp32 storage (3xTF32), LINEAR epilogue: written set, values per element against fp64 torch, and the pad
    channels [c, roundup8(c)) of NHWC outputs as act(0 + residual pad)."""
    name, n, cin, cout, H, W, form, act, epi, out = case
    d = conv_inputs(case)
    big, region, got, vec = run_conv(case, d)
    torch.cuda.synchronize()
    fk.assert_written_set(big, region, "conv2d " + name)
    ref, S = conv_ref(case, d)
    check_conv("conv2d LINEAR, " + ("NHWC 8-channel stores" if vec else "per-element stores"), got, ref, S)
    c8 = ops.round_up(cout, 8)
    if vec and c8 > cout:
        oc0 = OUT_C0[out]
        oh, ow = conv_out_hw(H, W, form)
        rp = d["res_pad"] if epi == "res16" else torch.zeros(n, c8 - cout, oh, ow, dtype=torch.float64)
        fk.check("conv2d LINEAR pad channels", big[:n, ..., oc0 + cout:oc0 + c8].permute(0, 3, 1, 2), fk.act_fwd(rp, act), rp.abs())


def test_fp32_cases_cover_the_kernel_forms():
    """What the case ids promise: every form, both N-tile widths, both epilogue store paths, tail K chunks of 11 and 16 channels."""
    assert {c[6] for c in CASES} == set(FORMS)
    ng = [c[3] for c in CASES]
    assert min(ng) <= 64 < max(ng)
    assert {c[9] for c in CASES} >= {"slice", "cat320", "cat704", "nchw", "f32p1", "f32p2", "f32p4"}
    tails = {c[2] % 32 for c in CASES if FORMS[c[6]][5] in ("plain", "pool")}
    assert {11, 16} <= tails
    assert {c[7] for c in CASES} == {ACT_NONE, ACT_RELU, ACT_LRELU, ACT_TANH}
    assert {c[8] for c in CASES} >= {"shift", "scale", "res16", "res32", "none"}


# ------------------------------------------------------------------------------------------------ 2. conv2d, SPADE epilogue


def run_spade(case, d, mean, rstd):
    name, n, cin, c0, c1, H, W, shift, nsc, act = case
    C = c0 + c1
    a_actv = fk.upload(d["actv"], c0=8, pitch=8 + ops.round_up(cin, 8) + 8)
    a_x0 = fk.upload(d["x0"], c0=8, pitch=8 + c0 + 8)
    a_x1 = fk.upload(d["x1"], c0=8, pitch=8 + c1 + 16) if c1 else None
    noise = d["noise"].float().to(DEV).contiguous() if nsc is not None else None
    ns = d["ns"].float().to(DEV) if nsc is not None else None
    pw = ops.pack_weight(d["wg"].float().to(DEV), (1, 1), interleave=d["wb"].float().to(DEV))
    sh = torch.stack([d["bg"], d["bb"]], 1).reshape(-1).float().to(DEV)
    out_big = fk.sentinel_buf((n + 1, H, W, C + 24), F32)
    args = (a_actv, pw, Act(out_big[:n], c=C, c0=16), a_x0, shift, a_x1, mean, rstd, noise, ns, sh, act)
    return out_big, args


def spade_stats(case, d):
    """The kernel's own statistics (hrv_instnorm_stats on the same fp32 views)."""
    name, n, cin, c0, c1, H, W, shift, nsc, act = case
    a_x0 = fk.upload(d["x0"], c0=8, pitch=8 + c0 + 8)
    a_x1 = fk.upload(d["x1"], c0=8, pitch=8 + c1 + 16) if c1 else None
    noise = d["noise"].float().to(DEV).contiguous() if nsc is not None else None
    ns = d["ns"].float().to(DEV) if nsc is not None else None
    return ops.instnorm_stats(a_x0, shift, a_x1, H, W, noise, ns)


@pytest.mark.parametrize("case", fk.SPADE_CASES, ids=lambda c: c[0])
def test_conv2d_spade_fp32(case, fp32):
    """hrv_conv2d_fwd on fp32 storage, SPADE epilogue with the kernel's own statistics: out as a channel slice (c0 = 16) of a
    NaN-sentinel buffer, x0 at full or half resolution, with and without x1 and noise.  C = 80 leaves the second N tile 32 columns
    wide; C = 1040 runs 9 N tiles.  gamma_out (a backward-pass output) is refused on fp32 storage before anything is written."""
    name, n, cin, c0, c1, H, W, shift, nsc, act = case
    d = fk.spade_inputs(case)
    C = c0 + c1
    mean, rstd = spade_stats(case, d)
    out_big, args = run_spade(case, d, mean, rstd)
    gam_big = fk.sentinel_buf((n + 1, H, W, C + 16), F32)
    with pytest.raises(RuntimeError, match="gamma_out belongs to the backward pass"):
        ops.conv2d_spade(*args, gamma_out=Act(gam_big[:n], c=C, c0=8))
    torch.cuda.synchronize()
    fk.assert_written_set(out_big, (slice(0, 0),), "spade out after the refused call")
    fk.assert_written_set(gam_big, (slice(0, 0),), "spade gamma_out after the refused call")
    ops.conv2d_spade(*args)
    torch.cuda.synchronize()
    fk.assert_written_set(out_big, (slice(0, n), slice(None), slice(None), slice(16, 16 + C)), "spade out")
    out, So = fk.spade_ref(case, d, mean.double().cpu(), rstd.double().cpu())["out"]
    check_conv("conv2d SPADE out", out_big[:n, ..., 16:16 + C].permute(0, 3, 1, 2), out, So)


# ------------------------------------------------------------------------------------------------ 3. both library handles


@pytest.mark.parametrize("which", ["linear", "spade"])
def test_both_library_handles_run_the_same_fp32_kernel(which, fp32, monkeypatch):
    """hrv_conv2d_fwd of the bf16 and the fp16 flavour both hand fp32 inputs to the one 3xTF32 kernel: bit-identical outputs,
    sentinels included."""
    outs = []
    if which == "linear":
        case = next(c for c in CASES if c[0] == "1x1_c363t11_n64_lpips1")
        d = conv_inputs(case)
    else:
        case = next(c for c in fk.SPADE_CASES if c[0] == "c80_half_x1_ns0.01")
        d = fk.spade_inputs(case)
        mean, rstd = spade_stats(case, d)
    for dt in (torch.bfloat16, torch.float16):
        L = capi.lib(dt)
        with monkeypatch.context() as m:
            m.setattr(ops, "_L", lambda *things, L=L: L)
            if which == "linear":
                big = run_conv(case, d)[0]
            else:
                big, args = run_spade(case, d, mean, rstd)
                ops.conv2d_spade(*args)
        torch.cuda.synchronize()
        outs.append(big.view(torch.int32).cpu())
    assert not bool(fk.untouched(big)[0].all()), "nothing was written"
    assert torch.equal(outs[0], outs[1])


# ------------------------------------------------------------------------------------------------ 4. the weight split


def split_weights(shape, seed=61):
    """fp32 weights mixing normal values with the edges of the split: ties of the hi rounding (1 + 2^-11, away from zero), a tie of
    the lo rounding, mantissas that carry into the next binade (2 - 2^-20), fp32 subnormals, -0 and +0."""
    g = fk.gen(seed)
    w = fk.rnd(g, int(np.prod(shape)), scale=0.05).float()
    edges = [1 + 2 ** -11, -(1 + 2 ** -11), 1 + 3 * 2 ** -11, (1 + 2 ** -11) * 2 ** -60, -(1 + 2 ** -11) * 2 ** 40,
             2 - 2 ** -20, -(2 - 2 ** -20), (2 - 2 ** -20) * 2 ** -9, 1 + 2 ** -12 + 2 ** -23, -(1 + 2 ** -12 + 2 ** -23),
             1 + 2 ** -11 + 2 ** -23, 2 ** -126, 1.5 * 2 ** -126, 2 ** -149, -(2 ** -149), 3 * 2 ** -140, -(1 + 2 ** -11) * 2 ** -130,
             1e-40, -3e-39, -0.0, 0.0, 65504.0, 3.0e38]
    e = torch.tensor(edges, dtype=F32)
    assert w.numel() >= e.numel()
    w[:e.numel()] = e
    return w[torch.randperm(w.numel(), generator=g)].reshape(shape).contiguous()


def want_planes(w0, w1, n_pad, cin_k, cin_total=None):
    """[2][taps][n_pad][cin_k]: rna_tf32(w) and rna_tf32(w - hi), rows (interleaved gamma/beta pairs) and columns zero past the weight."""
    cout, cin, kh, kw = w0.shape
    rows = w0 if w1 is None else torch.stack([w0, w1], 1).reshape(2 * cout, cin, kh, kw)
    full = torch.zeros(kh * kw, n_pad, cin_k, dtype=F32)
    full[:, :rows.shape[0], :cin] = rows.permute(2, 3, 0, 1).reshape(kh * kw, rows.shape[0], cin)
    hi = rna_tf32(full)
    return torch.stack([hi, rna_tf32(full - hi)])


SPLIT_CASES = [  # name, cout, cin, kh, kw, interleave, cin_total, s2d pad (None: not an s2d weight)
    ("3x3", 20, 13, 3, 3, False, None, None),
    ("1x1_n70", 70, 40, 1, 1, False, None, None),
    ("1x7", 24, 36, 1, 7, False, None, None),
    ("5x5", 12, 48, 5, 5, False, None, None),
    ("3x3_interleave", 20, 13, 3, 3, True, None, None),
    ("3x3_cin_total45", 16, 13, 3, 3, False, 45, None),
    ("s2d_k3v", 24, 13, 3, 3, False, None, 0),
    ("s2d_k4p2", 16, 9, 4, 4, False, None, 2),
]


@pytest.mark.parametrize("case", SPLIT_CASES, ids=lambda c: c[0])
def test_pack_conv_weight_tf32x2(case, fp32):
    """hrv_pack_conv_weight_tf32x2 (ops.pack_weight on fp32 storage): plane 0 = rna_tf32(w), plane 1 = rna_tf32(w - hi) bit for bit
    (cvt.rna.tf32.f32 restated on the host), in the [2][taps][n_pad][cin_k] layout with rows past n_gemm and columns past cin zero."""
    name, cout, cin, kh, kw, inter, cin_total, s2d = case
    w0 = split_weights((cout, cin, kh, kw))
    w1 = split_weights((cout, cin, kh, kw), seed=62) if inter else None
    if s2d is not None:
        w0 = ops.s2d_weight(w0, s2d)
        kh = kw = 2
    pw = ops.pack_weight(w0.to(DEV), (kh // 2, kw // 2), cin_total=cin_total, storage=F32,
                         interleave=w1.to(DEV) if inter else None)
    torch.cuda.synchronize()
    _, taps, n_pad, cin_k = pw.w.shape
    assert taps == kh * kw and pw.bk == 32 and cin_k % 32 == 0 and cin_k >= (cin_total or w0.shape[1]) and n_pad >= pw.n_gemm
    fk.check_exact("pack_conv_weight_tf32x2", pw.w.cpu().view(torch.int32), want_planes(w0, w1, n_pad, cin_k).view(torch.int32))


# ------------------------------------------------------------------------------------------------ 5. statistics


def offset64_mask(c0, c1):
    """Channels whose mean is 64 standard deviations (fk.offset_data cycles OFFSETS over each source's channels)."""
    k = len(fk.OFFSETS) - 1
    return torch.cat([torch.arange(c0) % len(fk.OFFSETS) == k, torch.arange(c1) % len(fk.OFFSETS) == k])


def rel_rstd_at_64(what, rstd, z, c0, c1):
    v = z.var((2, 3), unbiased=False)
    r = (v + fk.EPS_NORM).rsqrt()
    m = offset64_mask(c0, c1)
    rel = float(((rstd.double().cpu() - r).abs() / r)[:, m].max())
    REL64[what] = max(REL64.get(what, 0.0), rel)
    print("STATS fp32 %s: relative rstd error at mean/std = 64: %.2e" % (what, rel))


@pytest.mark.parametrize("case", fk.STATS_CASES, ids=lambda c: "n%d_c%d+%d_%dx%d_s%d_nz%d" % c)
def test_instnorm_stats_fp32(case, fp32):
    """hrv_instnorm_stats on fp32 views (x0 possibly at half resolution, x1, noise) against fp64 statistics, with channel means of 0,
    8 and 64 standard deviations in one tensor: where the single-pass E[t^2] - m^2 cancels."""
    n, c0, c1, H, W, shift, wn = case
    x0, x1, xs, noises, nss = fk.stats_inputs(case)
    dev = lambda t: t.float().to(DEV).contiguous() if t is not None else None
    mean, rstd = ops.instnorm_stats(fk.upload(x0, c0=8, pitch=8 + c0 + 8), shift, fk.upload(x1) if x1 is not None else None, H, W,
                                    dev(noises[0]), dev(nss[0]))
    torch.cuda.synchronize()
    z, T = fk.with_noise(xs, noises[0], nss[0])
    fk.check_stats("instnorm_stats", mean, rstd, z, T)
    rel_rstd_at_64("instnorm_stats rstd", rstd, z, c0, c1)


@pytest.mark.parametrize("norms", [1, 2])
@pytest.mark.parametrize("case", fk.STATS_CASES, ids=lambda c: "n%d_c%d+%d_%dx%d_s%d_nz%d" % c)
def test_instnorm_stats2_fp32(case, norms, fp32):
    """hrv_instnorm_stats2 on fp32 views: one or two norms over the same source, each with its own noise."""
    n, c0, c1, H, W, shift, wn = case
    x0, x1, xs, noises, nss = fk.stats_inputs(case)
    dev = lambda t: t.float().to(DEV).contiguous() if t is not None else None
    outs = ops.instnorm_stats2(fk.upload(x0, c0=8, pitch=8 + c0 + 8), shift, fk.upload(x1) if x1 is not None else None, H, W,
                               [dev(t) for t in noises[:norms]], [dev(t) for t in nss[:norms]])
    torch.cuda.synchronize()
    for j in range(norms):
        z, T = fk.with_noise(xs, noises[j], nss[j])
        fk.check_stats("instnorm_stats2", outs[j][0], outs[j][1], z, T)
        rel_rstd_at_64("instnorm_stats2 rstd", outs[j][1], z, c0, c1)


# ------------------------------------------------------------------------------------------------ 6. elementwise and resampling


@pytest.mark.parametrize("act", [ACT_NONE, ACT_RELU, ACT_LRELU, ACT_TANH])
@pytest.mark.parametrize("shape", [(2, 20, 9, 7), (3, 64, 4, 5)])
def test_instnorm_apply_fp32(shape, act, fp32):
    """hrv_instnorm_apply on fp32 storage: act((x - mean) * rstd) from a channel slice into a slice of a sentinel buffer; the pad
    channels up to the next multiple of 8 are written as 0."""
    n, c, H, W = shape
    x = fk.offset_data(fk.gen(35), n, c, H, W)
    mean32 = x.mean((2, 3)).float()
    rstd32 = (x.var((2, 3), unbiased=False) + fk.EPS_NORM).rsqrt().float()
    c8 = ops.round_up(c, 8)
    big = fk.sentinel_buf((n + 1, H, W, 8 + c8 + 8), F32)
    ops.instnorm_apply(fk.upload(x, c0=8, pitch=8 + c8 + 8), mean32.to(DEV), rstd32.to(DEV), act, out=Act(big[:n], c=c, c0=8))
    torch.cuda.synchronize()
    fk.assert_written_set(big, (slice(0, n), slice(None), slice(None), slice(8, 8 + c8)), "instnorm_apply")
    m, r = mean32.double()[:, :, None, None], rstd32.double()[:, :, None, None]
    fk.check("instnorm_apply", big[:n, ..., 8:8 + c].permute(0, 3, 1, 2), fk.act_fwd((x - m) * r, act), (x.abs() + m.abs()) * r)
    if c8 > c:
        fk.check_exact("instnorm_apply pad channels", big[:n, ..., 8 + c:8 + c8].cpu(), torch.zeros(n, H, W, c8 - c))


@pytest.mark.parametrize("shape", [(2, 20, 9, 7), (1, 64, 17, 13), (3, 8, 1, 5), (1, 24, 2, 3), (2, 16, 1, 1), (1, 8, 17, 2),
                                   (1, 40, 16, 17)])
def test_avgpool3s2_fp32(shape, fp32):
    """hrv_avgpool3s2 on fp32 storage (3x3, stride 2, pad 1, count_include_pad=False) at extents 1-17, from a channel slice."""
    n, c, H, W = shape
    x = fk.q(fk.rnd(fk.gen(36), n, c, H, W) * fk.spread(c)[None, :, None, None])
    y = ops.avgpool3s2(fk.upload(x, c0=8, pitch=8 + ops.round_up(c, 8) + 8))
    torch.cuda.synchronize()
    assert y.buf.dtype == F32
    pool = lambda t: F.avg_pool2d(t, 3, stride=2, padding=1, count_include_pad=False)
    fk.check("avgpool3s2", fk.nchw(y), pool(x), pool(x.abs()))


@pytest.mark.parametrize("with_b", [False, True])
@pytest.mark.parametrize("shape", [(2, 24, 7, 5), (1, 16, 1, 3), (2, 40, 9, 1), (1, 20, 4, 6)])
def test_bilinear_up2_add_fp32(shape, with_b, fp32):
    """hrv_bilinear_up2_add on fp32 storage: F.interpolate(a, x2, bilinear) (+ b) at odd low-resolution extents, a and b channel
    slices, the output a slice of a sentinel buffer (written in whole 8-channel groups)."""
    n, c, h, w = shape
    g = fk.gen(38)
    a = fk.q(fk.rnd(g, n, c, h, w) * fk.spread(c)[None, :, None, None])
    b = fk.q(fk.rnd(g, n, c, 2 * h, 2 * w, scale=0.1)) if with_b else None
    c8 = ops.round_up(c, 8)
    big = fk.sentinel_buf((n + 1, 2 * h, 2 * w, 8 + c8 + 8), F32)
    ops.bilinear_up2_add(fk.upload(a, c0=8, pitch=8 + c8 + 8), fk.upload(b, c0=8, pitch=8 + c8 + 8) if with_b else None,
                         Act(big[:n], c=c, c0=8))
    torch.cuda.synchronize()
    fk.assert_written_set(big, (slice(0, n), slice(None), slice(None), slice(8, 8 + c8)), "bilinear_up2_add")
    up = lambda t: F.interpolate(t, scale_factor=2, mode="bilinear", align_corners=False)
    ref, S = up(a), up(a.abs())
    if with_b:
        ref, S = ref + b, S + b.abs()
    fk.check("bilinear_up2_add", big[:n, ..., 8:8 + c].permute(0, 3, 1, 2), ref, S)


@pytest.mark.parametrize("c,hl,wl,scale", [(20, 16, 12, 12.0), (384, 8, 16, 1.0), (4, 16, 16, 12.0)])
def test_flow_warp_fp32(c, hl, wl, scale, fp32):
    """hrv_flow_warp with an fp32 source (channel slice) and an fp32 destination: gather indices and the up-sampled flow bit-exact
    with the oracle's fp32 chain, values per element at its taps, channels past c untouched.  Scale 12 clamps many coordinates."""
    n, H, W = 2, 2 * hl, 2 * wl
    g = fk.gen(39)
    flow = fk.rnd(g, n, hl, wl, 2, scale=scale).float()
    src = fk.q(fk.rnd(g, n, c, H, W) * fk.spread(c)[None, :, None, None])
    big = fk.sentinel_buf((n, H, W, c + 3), F32)
    dst = Act(big, c=c)
    flow_up, idx = ops.flow_warp(flow.to(DEV).contiguous(), fk.upload(src, c0=8, pitch=8 + ops.round_up(c, 8) + 8), dst, want_idx=True)
    torch.cuda.synchronize()
    x0, y0, tx, ty = orc.np_flow_warp_coords(flow.numpy(), H, W, H, W)
    fk.check_exact("flow_warp indices", idx.cpu(), torch.from_numpy(np.stack([x0, y0], -1).astype(np.int32)))
    fk.check_exact("flow_warp flow_up", flow_up.cpu(),
                   torch.from_numpy(np.moveaxis(orc.np_bilinear_up2(np.moveaxis(flow.numpy(), -1, 1)), 1, -1)))
    fk.assert_written_set(big, (slice(None), slice(None), slice(None), slice(0, c)), "flow_warp fp32 dst")
    ref, S = fk.gather_ref(src, x0, y0, tx, ty)
    fk.check("flow_warp", fk.nchw(dst), ref, S)


# ------------------------------------------------------------------------------------------------ 7. copies and gathers, bit-exact


@pytest.mark.parametrize("shape", [(2, 13, 9, 7), (1, 64, 1, 5), (3, 8, 4, 4), (1, 20, 35, 35), (2, 5, 17, 1)])
def test_space_to_depth_fp32(shape, fp32):
    """hrv_space_to_depth on fp32 storage at odd extents: sub-image (py, px) of the zero-extended input in channels
    [sub * c8, sub * c8 + c), the channels between the sub-images zero."""
    n, c, H, W = shape
    x = fk.q(fk.rnd(fk.gen(43), n, c, H, W))
    s = ops.space_to_depth(fk.upload(x, c0=8, pitch=8 + ops.round_up(c, 8) + 8), dtype=F32)
    torch.cuda.synchronize()
    c8 = ops.round_up(c, 8)
    xp = F.pad(x, (0, W & 1, 0, H & 1))
    want = torch.zeros((n, 4 * c8, (H + 1) // 2, (W + 1) // 2), dtype=torch.float64)
    for sub in range(4):
        want[:, sub * c8:sub * c8 + c] = xp[:, :, sub >> 1::2, sub & 1::2]
    fk.check_exact("space_to_depth", fk.nchw(s), want)


@pytest.mark.parametrize("shape", [(2, 5, 12, 9, 3, 1, None), (1, 3, 8, 8, 3, 1, 64), (1, 12, 5, 7, 2, 1, None),
                                   (2, 7, 12, 9, 3, 1, 64), (1, 7, 5, 4, 3, 1, 96), (1, 4, 3, 5, 5, 2, 104)])
def test_im2col_fp32(shape, fp32):
    """hrv_im2col on fp32 storage: dst[..., tap * c + ci] = x at the tap offset (zero outside), zero from kh*kw*c up to k_pad."""
    n, c, H, W, k, pad, k_pad = shape
    x = fk.q(fk.rnd(fk.gen(44), n, c, H, W))
    cols = ops.im2col(fk.upload(x, c0=8, pitch=8 + ops.round_up(c, 8) + 8), k, k, pad, k_pad=k_pad)
    torch.cuda.synchronize()
    assert cols.buf.dtype == F32 and (k_pad is None or cols.c == k_pad)
    xp = F.pad(x, (pad, k, pad, k))
    want = torch.zeros((n, cols.c, H, W), dtype=torch.float64)
    for ky in range(k):
        for kx in range(k):
            t = ky * k + kx
            want[:, t * c:(t + 1) * c] = xp[:, :, ky:ky + H, kx:kx + W]
    fk.check_exact("im2col", fk.nchw(cols), want)


@pytest.mark.parametrize("case", fk.NEAREST_CASES, ids=lambda c: "%dx%d_to_%dx%d" % (c[0][1:] + c[1]))
def test_nchw_to_nhwc_nearest_fp32(case, fp32):
    """hrv_nchw_to_nhwc into fp32 storage with nearest resampling: bit-exact against F.interpolate(mode='nearest') at dyadic and
    non-dyadic ratios; channels past c are written as zero; to_nchw of the result gives the same values back."""
    (c, h, w), (oh, ow) = case
    x = fk.rnd(fk.gen(48), 2, c, h, w).float()
    a = ops.from_nchw(x.to(DEV), size=(oh, ow))
    torch.cuda.synchronize()
    assert a.buf.dtype == F32
    want = F.interpolate(x, size=(oh, ow), mode="nearest")
    fk.check_exact("nchw_to_nhwc nearest", a.buf[..., :c].permute(0, 3, 1, 2).cpu(), want)
    fk.check_exact("nchw_to_nhwc pad channels", a.buf[..., c:].cpu(), torch.zeros(2, oh, ow, a.pitch - c))
    fk.check_exact("nhwc_to_nchw", a.to_nchw().cpu(), want)


def test_nhwc_to_nchw_fp32_slice(fp32):
    """hrv_nhwc_to_nchw of an fp32 channel slice with garbage around it: an exact copy of the view."""
    x = fk.q(fk.rnd(fk.gen(45), 2, 13, 9, 7))
    got = fk.upload(x, c0=4, pitch=4 + 16 + 4).to_nchw()
    torch.cuda.synchronize()
    fk.check_exact("nhwc_to_nchw", got.double().cpu(), x)


# ------------------------------------------------------------------------------------------------ 8. one storage type per call


def test_entry_points_refuse_mixed_storage_fp32(fp32):
    """An fp32 source with a 16-bit destination or second source is refused, and nothing is written (the entry points
    test_fp32_gpu.py's refusal test does not cover)."""
    a32 = fk.upload(fk.q(fk.rnd(fk.gen(63), 1, 16, 8, 8)))
    x1_16 = Act(torch.zeros((1, 8, 8, 16), dtype=torch.bfloat16, device=DEV))
    s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    L = capi.lib()
    for what, dst, call in [
            ("space_to_depth", (1, 4, 4, 64), lambda t, d: L.hrv_space_to_depth(ctypes.byref(t), ctypes.byref(d), s)),
            ("avgpool3s2", (1, 4, 4, 16), lambda t, d: L.hrv_avgpool3s2(ctypes.byref(t), ctypes.byref(d), s)),
            ("im2col", (1, 8, 8, 144), lambda t, d: L.hrv_im2col(ctypes.byref(t), ctypes.byref(d), 3, 3, 1, s))]:
        d16 = Act(fk.sentinel_buf(dst, torch.bfloat16))
        with pytest.raises(RuntimeError, match="one storage type per call"):
            capi.check(call(a32.ct(), d16.ct()), what)
        torch.cuda.synchronize()
        fk.assert_written_set(d16.buf, (slice(0, 0),), what + " refused")
    with pytest.raises(RuntimeError, match="one storage type per call"):
        ops.instnorm_stats2(a32, 0, x1_16, 8, 8, [None], [None])
    with pytest.raises(RuntimeError, match="one storage type per call"):
        ops.space_to_depth(a32, dtype=torch.bfloat16)
