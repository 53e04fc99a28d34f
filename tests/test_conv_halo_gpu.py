"""The halo main loop of the 16-bit convolution against the tap-by-tap loop, bit for bit.

conv_fwd picks the loop from the shape: output rows of a multiple of 64 pixels take the halo loop (for kernels with more than one tap
whose halo fits).  Each case runs once at width W (halo loop) and once embedded in tensors W + 8 pixels wide (tap loop), whose pixels
past W are zeros, as TMA's out-of-range fill is.  Every output element gets the same wgmma sequence over the same data in both, so
the cropped results must be identical.  Outputs live in NaN-sentinel buffers; comparing whole buffers also checks that both loops
write the same set of elements."""
import os
import sys

import pytest
import torch

from hrviton_b200 import capi, ops, synth
from hrviton_b200.ops import Act

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
import conv_staging  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
PAD = 8  # extra pixels of the tap-loop twin: W + 8 is never a multiple of 64
SENTINEL = {torch.bfloat16: 0x7FC1, torch.float16: 0x7E01}


@pytest.fixture(params=["bf16", "fp16"])
def storage(request):
    prev = ops.get_precision()
    ops.set_precision(request.param)
    yield ops.STORAGE[0]
    ops.set_precision(prev)


def widen(t, dim):
    """t with PAD zero pixels appended along `dim` (the width)."""
    shape = list(t.shape)
    shape[dim] = PAD
    return torch.cat([t, torch.zeros(shape, dtype=t.dtype, device=t.device)], dim).contiguous()


def nhwc(shape, seed, tag, dtype, scale=1.0):
    return (synth.normalish(shape, seed, tag, scale)).to(dtype).to(DEV)


def sentinel(shape, dtype):
    b = torch.empty(shape, dtype=dtype, device=DEV)
    if dtype == torch.float32:
        b.view(torch.int32).fill_(0x7FC00123)
    else:
        b.view(torch.int16).fill_(SENTINEL[dtype])
    return b


def same_bits(halo_buf, tap_buf, wdim):
    """halo_buf equals tap_buf cropped to halo_buf's width, bit for bit (sentinels included), and the halo loop wrote something."""
    crop = tap_buf.narrow(wdim, 0, halo_buf.shape[wdim])
    idt = torch.int32 if halo_buf.dtype == torch.float32 else torch.int16
    a, b = halo_buf.contiguous().view(idt), crop.contiguous().view(idt)
    assert not torch.equal(a, sentinel(halo_buf.shape, halo_buf.dtype).view(idt)), "nothing written"
    diff = (a != b).sum().item()
    assert diff == 0, "%d of %d elements differ between the halo and the tap loop" % (diff, a.numel())


def run_linear(x, pw, out_shape, out_dtype, c0, cout, layout, **kw):
    """conv2d of x into a sentinel buffer of out_shape (NHWC channel slice at c0, or a raw fp32 NCHW tensor)."""
    buf = sentinel(out_shape, out_dtype)
    n = x.n
    out = buf[:n] if layout == capi.NCHW else Act(buf[:n], c=cout, c0=c0)
    ops.conv2d(x, pw, out, out_layout=layout, **kw)
    return buf


# (cin, n_gemm): 3x3, K chunks 1..2, N tiles of 64 and 128 columns with a partial last tile
LINEAR = [(cin, ng) for cin in (8, 64, 128) for ng in (16, 64, 160, 288)]
SHAPES = [(2, 5, 64), (1, 4, 768)]  # batch > 1 with an odd height (a half-empty tile row); the full training width


@pytest.mark.parametrize("n,h,w", SHAPES)
@pytest.mark.parametrize("cin,n_gemm", LINEAR)
def test_linear_3x3(storage, n, h, w, cin, n_gemm):
    assert conv_staging.halo_eligible(cin, n_gemm, 3, 3, w) and not conv_staging.halo_eligible(cin, n_gemm, 3, 3, w + PAD)
    seed = 21
    x = nhwc((n, h, w, cin), seed, "x", storage)
    wt = synth.normalish((n_gemm, cin, 3, 3), seed, "w", 0.1).to(DEV)
    pw = ops.pack_weight(wt, (1, 1))
    b = synth.normalish((n_gemm,), seed, "b", 0.1).to(DEV)
    P = ops.round_up(n_gemm, 8) + 16
    bufs = [run_linear(Act(xx), pw, (n + 1, h, ww, P), storage, 8, n_gemm, capi.NHWC, act=ops.ACT_LRELU, shift=b)
            for xx, ww in ((x, w), (widen(x, 2), w + PAD))]
    torch.cuda.synchronize()
    same_bits(bufs[0], bufs[1], 2)


@pytest.mark.parametrize("cin,cout", [(32, 64), (48, 160)])
def test_space_to_depth_2x2(storage, cin, cout):
    """A stride-2 4x4 convolution as the 2x2 convolution over the space-to-depth input (128 and 192 channels: 2 and 3 K chunks)."""
    seed = 22
    n, h, w = 2, 3, 64
    cs = 4 * ops.round_up(cin, 8)
    assert conv_staging.halo_eligible(cs, cout, 2, 2, w)
    x = nhwc((n, h, w, cs), seed, "x", storage)
    pw = ops.pack_s2d(synth.normalish((cout, cin, 4, 4), seed, "w", 0.1).to(DEV), 2)
    sc = synth.uniform((cout,), seed, "s", 0.5, 1.5).to(DEV)
    bufs = [run_linear(Act(xx), pw, (n + 1, h, ww, cout), storage, 0, cout, capi.NHWC, act=ops.ACT_RELU, scale=sc)
            for xx, ww in ((x, w), (widen(x, 2), w + PAD))]
    torch.cuda.synchronize()
    same_bits(bufs[0], bufs[1], 2)


@pytest.mark.parametrize("mode", ["res16", "res32", "gate_relu", "gate_lrelu", "f32_nhwc", "f32_nchw"])
@pytest.mark.parametrize("n_gemm", [64, 160])
def test_linear_epilogues(storage, mode, n_gemm):
    """Scale and shift with a 16-bit or fp32 residual, the two gate modes, fp32 NHWC and fp32 NCHW outputs."""
    seed = 23
    n, h, w, cin = 2, 4, 128, 64
    x = nhwc((n, h, w, cin), seed, "x", storage)
    pw = ops.pack_weight(synth.normalish((n_gemm, cin, 3, 3), seed, "w", 0.1).to(DEV), (1, 1))
    sc = synth.uniform((n_gemm,), seed, "s", 0.5, 1.5).to(DEV)
    sh = synth.normalish((n_gemm,), seed, "b", 0.1).to(DEV)
    kw = dict(scale=sc, shift=sh)
    out_dtype, layout, c0, P = storage, capi.NHWC, 0, n_gemm
    res = None
    if mode in ("res16", "gate_relu", "gate_lrelu"):
        res = nhwc((n, h, w, n_gemm), seed, "r", storage)
        kw["res_mode"] = {"res16": capi.RES_ADD, "gate_relu": 1, "gate_lrelu": 2}[mode]
    elif mode == "res32":
        res = nhwc((n, h, w, n_gemm), seed, "r", torch.float32)
        kw["act"] = ops.ACT_TANH
    elif mode == "f32_nhwc":
        out_dtype, c0, P = torch.float32, 4, n_gemm + 12
    else:
        out_dtype, layout = torch.float32, capi.NCHW
    bufs = []
    for xx, rr, ww in ((x, res, w), (widen(x, 2), widen(res, 2) if res is not None else None, w + PAD)):
        shape = (n + 1, n_gemm, h, ww) if layout == capi.NCHW else (n + 1, h, ww, P)
        if rr is not None:
            kw["res"] = Act(rr)
        bufs.append(run_linear(Act(xx), pw, shape, out_dtype, c0, n_gemm, layout, **kw))
    torch.cuda.synchronize()
    same_bits(bufs[0], bufs[1], 3 if layout == capi.NCHW else 2)


@pytest.mark.parametrize("w", [64, 768])
@pytest.mark.parametrize("with_x1", [False, True])
def test_spade(storage, w, with_x1):
    """SPADE gamma/beta convolution (cin 128) with x0 at half resolution, an x1 part, noise and gamma_out."""
    seed = 24
    n, h, cin = 2, 4, 128
    cx0, cx1 = (64, 16) if with_x1 else (80, 0)
    C = cx0 + cx1
    actv = nhwc((n, h, w, cin), seed, "a", storage)
    pw = ops.pack_weight(synth.normalish((C, cin, 3, 3), seed, "wg", 0.05).to(DEV), (1, 1),
                         interleave=synth.normalish((C, cin, 3, 3), seed, "wb", 0.05).to(DEV))
    assert conv_staging.halo_eligible(cin, 2 * C, 3, 3, w)
    sh = synth.normalish((2 * C,), seed, "gb", 0.1).to(DEV)
    x0 = nhwc((n, h // 2, w // 2, cx0), seed, "x0", storage)
    x1 = nhwc((n, h, w, cx1), seed, "x1", storage) if cx1 else None
    noise = synth.spade_noise(n, h, w, seed, 0).to(DEV)
    ns = synth.normalish((C,), seed, "ns", 0.1).to(DEV)
    mean = synth.normalish((n, C), seed, "m", 0.2).to(DEV)
    rstd = synth.uniform((n, C), seed, "r", 0.5, 1.5).to(DEV)
    outs, gams = [], []
    for wide in (False, True):
        ww = w + PAD if wide else w
        f = (lambda t, d: widen(t, d)) if wide else (lambda t, d: t)
        out_b = sentinel((n + 1, h, ww, C + 24), storage)
        gam_b = sentinel((n + 1, h, ww, C + 16), storage)
        ops.conv2d_spade(Act(f(actv, 2)), pw, Act(out_b[:n], c=C, c0=16), Act(widen_half(x0) if wide else x0), 1,
                         Act(f(x1, 2)) if x1 is not None else None, mean, rstd, f(noise, 2), ns, sh, ops.ACT_LRELU,
                         gamma_out=Act(gam_b[:n], c=C, c0=8))
        outs.append(out_b)
        gams.append(gam_b)
    torch.cuda.synchronize()
    same_bits(outs[0], outs[1], 2)
    same_bits(gams[0], gams[1], 2)


def widen_half(x0):
    """x0 at half resolution of the widened output: PAD / 2 zero pixels."""
    return torch.cat([x0, torch.zeros(x0.shape[:2] + (PAD // 2,) + x0.shape[3:], dtype=x0.dtype, device=x0.device)], 2).contiguous()
