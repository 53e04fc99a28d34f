"""The per-element bound of tests/test_forward_kernels_fp32_gpu.py, (K_ACC + K_SPLIT) * 2^-24 * S, must be tight enough to matter.  At
the shapes of that file it accepts the correctly rounded fp64 result and a CPU emulation of the 3xTF32 kernel's arithmetic, and
rejects the realistic mistakes of an fp32-storage convolution.  The max-norms the fp32 metrics path is held to elsewhere
(max|d| <= 1e-4 max|ref| in test_inception_gpu.py, rel_err < 1e-2) are reported beside each verdict; the docstring of each test says
where they accept the mistake.  CPU only: fp64 references and fp32 emulations."""
import pytest
import torch
import torch.nn.functional as F

import test_forward_kernels_fp32_gpu as f32k
import test_forward_kernels_gpu as fk
from test_fp32_cpu import rna_tf32
from hrviton_b200 import ops
from hrviton_b200.ops import ACT_LRELU

EPS32 = fk.EPS32
KB = 32  # the fp32 kernel's K block: 32 channels per stage


@pytest.fixture
def fp32():
    ops.set_precision("fp32")
    yield
    ops.set_precision("bf16")


def bound(S):
    return f32k.K_CONV * EPS32 * S


def accepted(got, ref, S):
    return fk.ratio(got, ref, bound(S)) <= 1.0


def maxnorm_accepts(got, ref):
    """The older max-norms: test_inception_gpu.py's max|d| <= 1e-4 max|ref| (which implies rel_err < 1e-2)."""
    return fk.rel_err(got, ref) <= 1e-4


# ------------------------------------------------------------------------------------------------ the kernel's arithmetic on the CPU


def taps(x, kh, kw, off_y, off_x, stride, oh, ow):
    """Per tap (ky, kx): the input pixels it reads for every output pixel, (n, c, oh, ow), zero outside the image."""
    n, c, H, W = x.shape
    P = max(kh, kw) + max(off_y, off_x) + 1
    xp = F.pad(x, (P, P + stride * ow, P, P + stride * oh))
    out = {}
    for ky in range(kh):
        for kx in range(kw):
            y0, x0 = P + ky - off_y, P + kx - off_x
            out[ky, kx] = xp[:, :, y0:y0 + stride * oh:stride, x0:x0 + stride * ow:stride]
    return out


def linear_tail(v, d, act):
    bc = lambda t: t[None, :, None, None]
    if d["scale"] is not None:
        v = v * bc(d["scale"])
    if d["shift"] is not None:
        v = v + bc(d["shift"])
    if d["res"] is not None:
        v = v + d["res"]
    return fk.act_fwd(v, act)


def gemm(case, d, mode="tf32x3", off=None, dtype=torch.float32):
    """The convolution of one case computed tap by tap in stages of KB input channels.
      tf32x3     the kernel: x and w split into rna_tf32 hi / lo, each stage's lo*Bhi + hi*Blo + hi*Bhi summed in fp32, the stage
                 partials added to the accumulator in fp32 round-to-nearest (dtype=float64: the same products summed exactly)
      tf32x1     one TF32 pass (hi*Bhi only)
      no_loBhi   the lo*Bhi chain dropped;  no_hiBlo: the hi*Blo chain dropped (= a zero lo weight plane)
      drop_tail  the last K chunk of every tap skipped (cin % 32 != 0)
      garbage_tail  the last K chunk reads the garbage around the view (fk.GARBAGE) in place of its channels
    off: (off_y, off_x) read offsets (default: the form's padding)."""
    name, n, cin, cout, H, W, form, act, epi, out = case
    kh, kw, py, px, stride, kind = f32k.FORMS[form]
    oh, ow = f32k.conv_out_hw(H, W, form)
    off_y, off_x = (py, px) if off is None else off
    x, w = d["x"].float(), d["w"].float()
    xh, wh = rna_tf32(x), rna_tf32(w)
    xl, wl = rna_tf32(x - xh), rna_tf32(w - wh)
    if mode == "garbage_tail":
        t0 = (cin - 1) // KB * KB
        x = x.clone()
        x[:, t0:] = fk.GARBAGE
        xh, xl = rna_tf32(x), rna_tf32(x - rna_tf32(x))
    chains = {"tf32x3": [(xl, wh), (xh, wl), (xh, wh)], "tf32x1": [(xh, wh)], "no_loBhi": [(xh, wl), (xh, wh)],
              "no_hiBlo": [(xl, wh), (xh, wh)], "drop_tail": [(xl, wh), (xh, wl), (xh, wh)],
              "garbage_tail": [(xl, wh), (xh, wl), (xh, wh)]}[mode]
    tx = [taps(a.to(dtype), kh, kw, off_y, off_x, stride, oh, ow) for a, _ in chains]
    acc = torch.zeros(n, cout, oh, ow, dtype=dtype)
    nblk = (cin + KB - 1) // KB
    for ky in range(kh):
        for kx in range(kw):
            for b in range(nblk - 1 if mode == "drop_tail" and cin % KB else nblk):
                c = slice(b * KB, min(cin, (b + 1) * KB))
                part = torch.zeros_like(acc)
                for t, (_, wb) in zip(tx, chains):
                    part = part + torch.einsum("nchw,oc->nohw", t[ky, kx][:, c], wb[:, c, ky, kx].to(dtype))
                acc = acc + part
    return acc.double()


def emulate(case, d, mode="tf32x3", off=None):
    """The LINEAR output of a kernel with `gemm(mode)` arithmetic and an fp32 epilogue."""
    v = gemm(case, d, mode, off)
    return linear_tail(v, d, case[7]).float().double()


def correctly_rounded(ref):
    return ref.float().double()


CASES = f32k.CASES
ids = lambda c: c[0]


@pytest.mark.parametrize("case", CASES, ids=ids)
def test_correctly_rounded_and_emulated_kernel_pass(case, fp32):
    """The fp64 result rounded once to fp32, and the emulated 3xTF32 arithmetic (truncation aside: the emulation rounds to nearest),
    sit inside the bound; the emulation uses a small part of it."""
    d = f32k.conv_inputs(case)
    ref, S = f32k.conv_ref(case, d)
    assert accepted(correctly_rounded(ref), ref, S)
    r = fk.ratio(emulate(case, d), ref, bound(S))
    print("EMULATED %-36s 3xTF32 ratio %.3f" % (case[0], r))
    assert r <= 0.5


# ------------------------------------------------------------------------------------------------ the mistakes


def test_split_bound_is_what_the_products_lose(fp32):
    """K_SPLIT: over random fp32 pairs, |x*w - (lo*Bhi + hi*Blo + hi*Bhi)| stays within 3 * 2^-22 |x||w|, and dropping one chain
    does not."""
    g = fk.gen(70)
    x, w = torch.randn(100000, generator=g), torch.randn(100000, generator=g)
    xh, wh = rna_tf32(x), rna_tf32(w)
    xl, wl = rna_tf32(x - xh), rna_tf32(w - wh)
    d = lambda *terms: (x.double() * w.double() - sum(a.double() * b.double() for a, b in terms)).abs() / (x * w).double().abs()
    assert float(d((xl, wh), (xh, wl), (xh, wh)).max()) <= f32k.K_SPLIT * EPS32
    assert float(d((xh, wl), (xh, wh)).max()) > 100 * f32k.K_SPLIT * EPS32
    assert float(d((xl, wh), (xh, wh)).max()) > 100 * f32k.K_SPLIT * EPS32


def caught(wrong, ref, S):
    """The per-element bound rejects `wrong`, and the max-norm rel_err < 1e-2 lets it through."""
    return not accepted(wrong, ref, S) and fk.rel_err(wrong, ref) < 1e-2


@pytest.mark.parametrize("mode", ["tf32x1", "no_loBhi", "no_hiBlo"])
@pytest.mark.parametrize("case", CASES, ids=ids)
def test_bound_rejects_a_missing_split_term(case, mode, fp32):
    """One TF32 pass, or the 3xTF32 kernel with its lo*Bhi or hi*Blo chain dropped (the latter is also what a zero lo weight plane
    computes), each with the kernel's fp32 stage sums.  Rejected in every case, the 18720-long K of the 2080-channel layer included
    (4-6x its bound there); rel_err < 1e-2 accepts all of them, and max|d| <= 1e-4 max|ref| accepts some (printed)."""
    d = f32k.conv_inputs(case)
    ref, S = f32k.conv_ref(case, d)
    wrong = emulate(case, d, mode)
    print("MISTAKE %-36s %-9s ratio %7.2f  max-norm 1e-4 %s" % (case[0], mode, fk.ratio(wrong, ref, bound(S)),
                                                                "accepts" if maxnorm_accepts(wrong, ref) else "rejects"))
    assert caught(wrong, ref, S)


TAIL_CASES = [c for c in CASES if c[2] % KB and f32k.FORMS[c[6]][5] in ("plain", "pool")]


@pytest.mark.parametrize("mode", ["drop_tail", "garbage_tail"])
@pytest.mark.parametrize("case", TAIL_CASES, ids=ids)
def test_bound_rejects_a_wrong_tail_chunk(case, mode, fp32):
    """cin % 32 != 0: the last K chunk of every tap skipped, or filled with the garbage channels around the view instead of its own.
    Rejected by the bound.  The dropped chunk holds the smallest input channels: rel_err < 1e-2 accepts it in most cases, while
    max|d| <= 1e-4 max|ref| rejects it.  Both max-norms reject the garbage chunk."""
    d = f32k.conv_inputs(case)
    ref, S = f32k.conv_ref(case, d)
    assert not accepted(emulate(case, d, mode), ref, S)


ASYM_CASES = [c for c in CASES if c[6] in ("1x7", "7x1", "1x3", "3x1")]


@pytest.mark.parametrize("case", ASYM_CASES, ids=ids)
def test_bound_rejects_swapped_tap_offsets(case, fp32):
    """An asymmetric kernel read with off_x and off_y swapped (1x7 with its (0, 3) offsets applied as (3, 0))."""
    d = f32k.conv_inputs(case)
    ref, S = f32k.conv_ref(case, d)
    py, px = f32k.FORMS[case[6]][2:4]
    assert not accepted(emulate(case, d, off=(px, py)), ref, S)


WIDE_CASES = [c for c in CASES if c[3] >= 32 and c[9] in f32k.OUT_C0]


@pytest.mark.parametrize("case", WIDE_CASES, ids=ids)
def test_bound_rejects_a_zeroed_or_stale_low_magnitude_group(case, fp32):
    """One 8-channel group of the smallest output channels zeroed, or holding another image's (another row's) values: about 1e-3 of
    the tensor's largest value, which rel_err < 1e-2 accepts."""
    ref, S = f32k.conv_ref(case, f32k.conv_inputs(case))
    c = ref.shape[1]
    g0 = (c // 8 - 1) * 8
    good = correctly_rounded(ref)
    assert accepted(good, ref, S)
    wrong = good.clone()
    wrong[:, g0:g0 + 8] = 0
    assert caught(wrong, ref, S), "zeroed group"
    wrong = good.clone()
    wrong[:, g0:g0 + 8] = good[:, g0:g0 + 8].roll(1, 0) if ref.shape[0] > 1 else good[:, g0:g0 + 8].roll(1, 2)
    assert caught(wrong, ref, S), "stale group"


LRELU_SHIFT_CASES = [c for c in CASES if c[7] == ACT_LRELU and c[8] in ("shift", "scale") and c[9] in f32k.OUT_C0]


@pytest.mark.parametrize("case", LRELU_SHIFT_CASES, ids=ids)
def test_bound_rejects_the_shift_after_the_activation(case, fp32):
    """act(v) + shift instead of act(v + shift), with a bias small enough (2 % of the test's) that rel_err < 1e-2 accepts it."""
    d = f32k.conv_inputs(case)
    d["shift"] = d["shift"] * 0.02
    ref, S = f32k.conv_ref(case, d)
    no_shift, _ = f32k.conv_ref(case, dict(d, shift=None))
    assert accepted(correctly_rounded(ref), ref, S)
    assert caught(correctly_rounded(no_shift + d["shift"][None, :, None, None]), ref, S)


def spade_stats(case, d):
    """fp32 InstanceNorm statistics of cat(up2^shift(x0), x1) + noise * noise_scale from fp64 sums."""
    name, n, cin, c0, c1, H, W, shift, nsc, act = case
    xs = fk.nearest_up(d["x0"], shift)
    if d["x1"] is not None:
        xs = torch.cat([xs, d["x1"]], 1)
    z = xs + d["noise"][:, None] * d["ns"][None, :, None, None] if d["noise"] is not None else xs
    return z.mean((2, 3)).float().double(), (z.var((2, 3), unbiased=False) + fk.EPS_NORM).rsqrt().float().double()


def test_bound_rejects_the_previous_images_statistics(fp32):
    """A tile over three 4x4 images that keeps image 0's mean / rstd for image 1, where image 1 is image 0 shifted by 1e-3 of each
    channel's spread: the two sets of statistics differ so little that rel_err < 1e-2 accepts the mix-up."""
    case = next(c for c in fk.SPADE_CASES if c[0] == "c80_half_x1_3img")
    d = fk.spade_inputs(case)
    for k in ("x0", "x1"):
        x = d[k].clone()
        x[1] = fk.q(x[0] + 1e-3 * x[0].std((1, 2), keepdim=True))
        d[k] = x
    mean, rstd = spade_stats(case, d)
    out, So = fk.spade_ref(case, d, mean, rstd)["out"]
    assert accepted(correctly_rounded(out), out, So)
    m2, r2 = mean.clone(), rstd.clone()
    m2[1], r2[1] = mean[0], rstd[0]
    assert caught(correctly_rounded(fk.spade_ref(case, d, m2, r2)["out"][0]), out, So)
