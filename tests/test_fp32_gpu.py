"""GPU: the fp32 reference-precision inference mode (ops.set_precision("fp32"): fp32 activation storage, 3xTF32 convolutions).

Parity with the goldens of the UNMODIFIED reference is asserted at the fp32 tolerance AS WRITTEN: max|delta| < 1e-3 per element, for
every stored golden.  The convolution kernel is checked against an fp64 convolution with a per-output bound of 1e-5 * sum|x||w| that
one TF32 pass does not meet; every HBM-bound entry point that takes fp32 storage is checked against torch."""
import contextlib
import io
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "..", "oracle"))
import hrviton_oracle as orc  # noqa: E402
import floors  # noqa: E402
from helpers import gen_opt, load_golden, synth_state_dict, tocg_opt  # noqa: E402
from hrviton_b200 import ops, pipeline, synth, train_step  # noqa: E402
from hrviton_b200.ops import Act  # noqa: E402

pytestmark = pytest.mark.gpu

DEV = "cuda"
TOL_F32 = 1e-3  # BASELINE.json north star: |delta| < 1e-3 for fp32


@pytest.fixture
def fp32():
    ops.set_precision("fp32")
    yield
    ops.set_precision("bf16")


def parity(name, got, ref, tol=TOL_F32):
    s = floors.stats(got, ref)
    print("PARITY fp32 %-34s n=%-8d max %.3e (<= %.1e)  mean %.3e  ref absmax %.3g" % (name, s["n"], s["max"], tol, s["mean"], s["absmax"]))
    assert s["max"] < tol, (name, s)
    return s


def _gen_module(h, w, sd, seed):
    import network_generator
    m = network_generator.SPADEGenerator(gen_opt(h, w, True), 9)
    m.load_state_dict(sd)
    m = m.cuda().eval()
    cnt = [0]

    def noise(b, hh, ww):
        t = synth.spade_noise(b, hh, ww, seed, cnt[0]).cuda()
        cnt[0] += 1
        return t

    m.noise_source = noise
    return m, cnt


def _tocg_module(sd):
    import networks
    m = networks.ConditionGenerator(tocg_opt(True), 4, 16, 13, ngf=96, norm_layer=torch.nn.BatchNorm2d)
    m.load_state_dict(sd)
    return m.cuda().eval()


# ------------------------------------------------------------------------------------------------ modules vs the goldens at 1e-3

@pytest.mark.parametrize("name", ["tocg_256x192_b1", "tocg_128x96_b2"])
def test_tocg_forward_fp32(name, fp32):
    g = load_golden(name)
    n, h, w = [int(v) for v in g["shape"]]
    seed = int(g["seed"])
    m = _tocg_module(synth_state_dict("tocg", seed))
    i1, i2 = synth.tocg_inputs(n, h, w, seed)
    with torch.no_grad():
        flows, seg, wc, wcm = m(i1.cuda(), i2.cuda())
    torch.cuda.synchronize()
    for i, f in enumerate(flows):
        parity("%s flow%d" % (name[:8], i), f, g["flow%d" % i])
    parity("%s seg" % name[:8], seg, g["seg"])
    parity("%s warped_c" % name[:8], wc, g["warped_c"])
    parity("%s warped_cm" % name[:8], wcm, g["warped_cm"])
    # the gather indices of the final warp, from the kernel's own last flow: bit-exact against the oracle's index arithmetic
    fl = flows[-1].contiguous()
    src = Act.empty(n, h, w, 8)
    dst = Act.empty(n, h, w, 8)
    src.buf.zero_()
    _, idx = ops.flow_warp(fl, src, dst, want_flow_up=False, want_idx=True)
    x0, y0, _, _ = orc.np_flow_warp_coords(fl.cpu().numpy(), h, w, h, w)
    idx = idx.cpu().numpy()
    assert np.array_equal(idx[..., 0], x0) and np.array_equal(idx[..., 1], y0)


@pytest.mark.parametrize("name", ["gen_512x384_b1", "gen_256x256_b2"])
def test_generator_forward_fp32(name, fp32):
    g = load_golden(name)
    n, h, w = [int(v) for v in g["shape"]]
    seed = int(g["seed"])
    m, cnt = _gen_module(h, w, synth_state_dict("gen", seed), seed)
    x, seg = synth.gen_inputs(n, h, w, seed)
    with torch.no_grad():
        out = m(x.cuda(), seg.cuda())
    torch.cuda.synchronize()
    assert cnt[0] == 23
    parity("%s out" % name, out, g["out"].astype(np.float32))


def test_gen_discriminator_forward_fp32(fp32):
    import network_generator
    name = "gend_128x96_b2"
    g = load_golden(name)
    n, h, w = [int(v) for v in g["shape"]]
    seed = int(g["seed"])
    m = network_generator.MultiscaleDiscriminator(gen_opt(h, w, True))
    m.load_state_dict(synth_state_dict("gend", seed))
    m = m.cuda().eval()
    x, seg = synth.gen_inputs(n, h, w, seed, input_nc=3)
    with torch.no_grad():
        res = m(torch.cat([seg, x], 1).cuda())
    for i, fs in enumerate(res):
        for j, f in enumerate(fs):
            key = "d%d_f%d" % (i, j)
            parity("gend %s" % key, f, g[key])


def test_tocg_discriminator_forward_fp32(fp32):
    import networks
    name = "tocgd_256x192_b1"
    g = load_golden(name)
    seed = int(g["seed"])
    with contextlib.redirect_stdout(io.StringIO()):
        m = networks.define_D(input_nc=33, Ddownx2=True, Ddropout=True, n_layers_D=3, spectral=False, num_D=2)
    m.load_state_dict(synth_state_dict("tocgd", seed))
    m = m.cuda().eval()
    i1, i2 = synth.tocg_inputs(1, 256, 192, seed)
    segs = synth.one_hot(synth.labels((1, 256, 192), 13, seed, "dseg"), 13)
    with torch.no_grad():
        res = m(torch.cat([i1, i2, segs], 1).cuda())
    for i, r in enumerate(res):
        parity("tocgd d%d" % i, r[0], g["d%d" % i])


def test_generator_1024x768_b8_fp32(fp32):
    g = load_golden("gen_1024x768_b8")
    n, h, w = [int(v) for v in g["shape"]]
    seed = int(g["seed"])
    m, _ = _gen_module(h, w, synth_state_dict("gen", seed), seed)
    x, seg = synth.gen_inputs(n, h, w, seed)
    with torch.no_grad():
        out = m(x.cuda(), seg.cuda())
    torch.cuda.synchronize()
    outc = out.cpu()
    del out
    crops = torch.stack([outc[:, :, y:y + 64, x0:x0 + 64] for y, x0 in g["crop_yx"]], 1)
    parity("gen 1024x768 sub8", outc[:, :, ::8, ::8], g["sub8"].astype(np.float32))
    parity("gen 1024x768 crops", crops, g["crops"].astype(np.float32))
    dmean = np.abs(outc.double().sum((2, 3)).numpy() - g["chan_sums"]) / float(h * w)
    print("PARITY fp32 gen 1024x768 per-image channel-mean error max %.3e" % dmean.max())
    assert dmean.max() < 1e-4  # signed mean of a whole 786k-pixel plane: far below the per-element bound


def test_tocg_1024x768_b4_fp32(fp32):
    g = load_golden("tocg_1024x768_b4")
    n, h, w = [int(v) for v in g["shape"]]
    seed = int(g["seed"])
    m = _tocg_module(synth_state_dict("tocg", seed))
    i1, i2 = synth.tocg_inputs(n, h, w, seed)
    with torch.no_grad():
        flows, seg, wc, wcm = m(i1.cuda(), i2.cuda())
    torch.cuda.synchronize()
    step = lambda i: 1 if i < 3 else 4
    segc, wcc, wcmc = seg.cpu(), wc.cpu(), wcm.cpu()
    parity("tocg 1024x768 seg_sub8", segc[:, :, ::8, ::8], g["seg_sub8"])
    parity("tocg 1024x768 seg_crop", segc[:, :, h - 64:, w - 64:], g["seg_crop"])
    parity("tocg 1024x768 warped_c_sub8", wcc[:, :, ::8, ::8], g["warped_c_sub8"])
    parity("tocg 1024x768 warped_cm_sub8", wcmc[:, :, ::8, ::8], g["warped_cm_sub8"])
    for i, f in enumerate(flows):
        parity("tocg 1024x768 flow%d_sub" % i, f.cpu()[:, ::step(i), ::step(i)], g["flow%d_sub" % i])
    dmean = np.abs(segc.double().sum((2, 3)).numpy() - g["seg_sums"]) / float(h * w)
    print("PARITY fp32 tocg 1024x768 per-plane mean error max %.3e" % dmean.max())
    assert dmean.max() < 1e-4


# ------------------------------------------------------------------------------------------------ the 3xTF32 convolution vs fp64

WIDE_CASES = [  # spade, cin, n_gemm, h, w, batch, x0_shift, c1 (x1 channels) — the shapes of test_kernels_gpu.test_conv_tiles_match_torch
    (True, 128, 160, 64, 48, 2, 0, 0), (True, 128, 160, 64, 48, 2, 1, 16), (True, 128, 288, 48, 32, 3, 1, 16),
    (True, 128, 544, 64, 48, 2, 1, 16), (True, 128, 2080, 16, 12, 2, 1, 16), (True, 128, 144, 30, 22, 1, 0, 0),
    (False, 160, 160, 50, 37, 3, 0, 0), (False, 256, 256, 64, 48, 2, 0, 0), (False, 80, 192, 128, 96, 1, 0, 0),
    (True, 128, 64, 64, 48, 2, 1, 16), (True, 128, 128, 48, 32, 2, 0, 0), (False, 80, 32, 64, 48, 2, 0, 0), (False, 144, 64, 50, 37, 2, 0, 0),
    (False, 160, 128, 64, 48, 1, 0, 0), (False, 2080, 128, 16, 12, 2, 0, 0)]

REL = 1e-5  # |delta| <= REL * sum|x||w| per output: fp32-class accuracy, independent of cancellation in the sum


def rna_tf32(t):
    """Round fp32 to TF32 (10 mantissa bits), to nearest with ties away from zero — cvt.rna.tf32.f32."""
    b = t.float().contiguous().view(torch.int32)
    mag = (b & 0x7FFFFFFF) + 0x1000
    return ((mag & ~0x1FFF) | (b & ~0x7FFFFFFF)).view(torch.float32)


def _conv64(x, w):
    return F.conv2d(x.double(), w.double(), padding=1)


@pytest.mark.parametrize("case", WIDE_CASES)
def test_conv_tf32x3_matches_fp64(case, fp32):
    spade, cin, ng, h, w, B, shift, c1 = case
    g = torch.Generator().manual_seed(1)
    rnd = lambda *s: torch.randn(*s, generator=g)
    xh = rnd(B, h, w, ops.round_up(cin, 8))
    x = Act(xh.to(DEV), c=cin)
    xn = xh[..., :cin].permute(0, 3, 1, 2)
    lrelu = lambda t: F.leaky_relu(t, 0.2)
    if spade:
        C = ng // 2
        wg, wb = rnd(C, cin, 3, 3) * 0.05, rnd(C, cin, 3, 3) * 0.05
        pw = ops.pack_weight(wg.to(DEV), (1, 1), interleave=wb.to(DEV))
        x0h, x1h = rnd(B, h >> shift, w >> shift, C - c1), (rnd(B, h, w, c1) if c1 else None)
        x0, x1 = Act(x0h.to(DEV)), (Act(x1h.to(DEV)) if c1 else None)
        mean, rstd = rnd(B, C) * 0.1, torch.rand(B, C, generator=g) + 0.5
        noise, ns, sh = rnd(B, h, w), rnd(C) * 0.1, rnd(2 * C) * 0.1
        out = Act.empty(B, h, w, C, zero=True)
        ops.conv2d_spade(x, pw, out, x0, shift, x1, mean.to(DEV), rstd.to(DEV), noise.to(DEV), ns.to(DEV), sh.to(DEV), 2)
        torch.cuda.synchronize()
        gamma, beta = _conv64(xn, wg) + sh[0::2, None, None].double(), _conv64(xn, wb) + sh[1::2, None, None].double()
        sg, sb = _conv64(xn.abs(), wg.abs()), _conv64(xn.abs(), wb.abs())
        xs = x0h.permute(0, 3, 1, 2)
        if shift:
            xs = F.interpolate(xs, scale_factor=2, mode="nearest")
        if c1:
            xs = torch.cat([xs, x1h.permute(0, 3, 1, 2)], 1)
        v = (xs.double() + noise[:, None].double() * ns[None, :, None, None].double() - mean[:, :, None, None].double()) * rstd[:, :, None, None].double()
        ref = lrelu(v * (1 + gamma) + beta)
        # LeakyReLU is 1-Lipschitz: the GEMM bound carries through the modulation; plus fp32 rounding of the epilogue itself
        bound = REL * (v.abs() * sg + sb) + 1e-6 * ref.abs() + 1e-7
        tf1 = lrelu(v * (1 + _conv64(rna_tf32(xn), rna_tf32(wg)) + sh[0::2, None, None].double())
                    + _conv64(rna_tf32(xn), rna_tf32(wb)) + sh[1::2, None, None].double())
    else:
        wt, bias = rnd(ng, cin, 3, 3) * 0.05, rnd(ng)
        pw = ops.pack_weight(wt.to(DEV), (1, 1))
        out = Act.empty(B, h, w, ng, zero=True)
        ops.conv2d(x, pw, out, act=2, shift=bias.to(DEV))
        torch.cuda.synchronize()
        ref = lrelu(_conv64(xn, wt) + bias[:, None, None].double())
        bound = REL * _conv64(xn.abs(), wt.abs()) + 1e-6 * ref.abs() + 1e-7
        tf1 = lrelu(_conv64(rna_tf32(xn), rna_tf32(wt)) + bias[:, None, None].double())
    got = out.buf[..., :ref.shape[1]].permute(0, 3, 1, 2).cpu().double()
    ratio = float(((got - ref).abs() / bound).max())
    ratio1 = float(((tf1 - ref).abs() / bound).max())
    print("CONV fp32 %s: max |d| / bound %.3f (one TF32 pass: %.1f)" % (case, ratio, ratio1))
    assert ratio <= 1.0
    assert ratio1 > 1.0  # a single TF32 pass does not meet the bound: the split is what delivers fp32-class accuracy


@pytest.mark.parametrize("layout", ["nhwc_res", "nchw"])
def test_conv_tf32x3_residual_and_nchw(layout, fp32):
    """LINEAR epilogue with folded scale/shift and an fp32 residual (NHWC, pad channels written) and with an fp32 NCHW output."""
    g = torch.Generator().manual_seed(2)
    rnd = lambda *s: torch.randn(*s, generator=g)
    B, h, w, cin, cout = 2, 40, 28, 96, 20
    xh = rnd(B, h, w, cin)
    x = Act(xh.to(DEV))
    xn = xh.permute(0, 3, 1, 2)
    wt, sc, shf = rnd(cout, cin, 3, 3) * 0.05, rnd(cout) * 0.5 + 1.0, rnd(cout)
    pw = ops.pack_weight(wt.to(DEV), (1, 1))
    conv = _conv64(xn, wt) * sc[:, None, None].double() + shf[:, None, None].double()
    bound = REL * _conv64(xn.abs(), wt.abs()) * sc.abs()[:, None, None].double() + 1e-6 * conv.abs() + 1e-7
    if layout == "nhwc_res":
        resh = rnd(B, h, w, ops.round_up(cout, 8))
        resh[..., cout:] = 0.0
        res = Act(resh.to(DEV), c=cout)
        out = Act.empty(B, h, w, cout)
        out.buf.fill_(7.0)
        ops.conv2d(x, pw, out, act=ops.ACT_RELU, scale=sc.to(DEV), shift=shf.to(DEV), res=res)
        torch.cuda.synchronize()
        ref = torch.relu(conv + resh[..., :cout].permute(0, 3, 1, 2).double())
        got = out.buf[..., :cout].permute(0, 3, 1, 2).cpu().double()
        assert float(out.buf[..., cout:].abs().max()) == 0.0  # pad channels: act(0) + zero residual pad
    else:
        out = torch.empty((B, cout, h, w), dtype=torch.float32, device=DEV)
        ops.conv2d(x, pw, out, act=ops.ACT_TANH, scale=sc.to(DEV), shift=shf.to(DEV), out_layout=ops.capi.NCHW)
        torch.cuda.synchronize()
        ref, got = torch.tanh(conv), out.cpu().double()
    assert float(((got - ref).abs() / bound).max()) <= 1.0


def test_conv_tf32x3_bit_reproducible(fp32):
    g = torch.Generator().manual_seed(4)
    x = Act(torch.randn(2, 64, 48, 128, generator=g).to(DEV))
    pw = ops.pack_weight((torch.randn(256, 128, 3, 3, generator=g) * 0.05).to(DEV), (1, 1))
    a = ops.conv2d(x, pw, Act.empty(2, 64, 48, 256)).buf.clone()
    b = ops.conv2d(x, pw, Act.empty(2, 64, 48, 256)).buf
    assert torch.equal(a, b)


def test_conv_fp32_refuses_mixed_storage(fp32):
    g = torch.Generator().manual_seed(5)
    x = Act(torch.randn(1, 16, 16, 32, generator=g).to(DEV))
    pw = ops.pack_weight((torch.randn(32, 32, 3, 3, generator=g) * 0.05).to(DEV), (1, 1))
    with pytest.raises(RuntimeError, match="fp32"):
        ops.conv2d(x, pw, Act.empty(1, 16, 16, 32, dtype=torch.bfloat16))
    with pytest.raises(RuntimeError, match="fp32"):
        ops.conv2d(x, pw, Act.empty(1, 16, 16, 32), res=Act.empty(1, 16, 16, 32, dtype=torch.bfloat16, zero=True))
    with pytest.raises(RuntimeError):
        ops.conv2d(x, pw, Act.empty(1, 16, 16, 32), res=Act.empty(1, 16, 16, 32, zero=True), res_mode=ops.capi.RES_GATE_RELU)


# ------------------------------------------------------------------------------------------------ HBM-bound entry points on fp32 storage

def _nhwc(t, pitch=None):
    """fp32 NCHW (CPU) -> fp32 Act on the GPU with the given channel pitch (pad channels zero)."""
    n, c, h, w = t.shape
    buf = torch.zeros((n, h, w, pitch or ops.round_up(c, 8)), dtype=torch.float32)
    buf[..., :c] = t.permute(0, 2, 3, 1)
    return Act(buf.to(DEV), c=c)


def _nchw(a):
    return a.buf[..., :a.c].permute(0, 3, 1, 2).cpu()


def test_hbm_entry_points_fp32(fp32):
    g = torch.Generator().manual_seed(6)
    rnd = lambda *s: torch.randn(*s, generator=g)
    x = rnd(2, 20, 17, 13)
    # layout converters (nearest resize on the way in)
    a = ops.from_nchw(x.to(DEV), size=(34, 26))
    assert a.buf.dtype == torch.float32
    assert torch.equal(_nchw(a), F.interpolate(x, size=(34, 26), mode="nearest"))
    assert float(a.buf[..., 20:].abs().max()) == 0.0
    assert torch.equal(a.to_nchw().cpu(), F.interpolate(x, size=(34, 26), mode="nearest"))
    xa = _nhwc(x)
    # space-to-depth (odd edges zero-filled)
    s = ops.space_to_depth(xa)
    xp = F.pad(x, (0, 1, 0, 1))
    for sub in range(4):
        py, px = divmod(sub, 2)
        assert torch.equal(s.buf[..., sub * 24:sub * 24 + 20].permute(0, 3, 1, 2).cpu(), xp[:, :, py::2, px::2])
    # 3x3/s2 average pool
    assert float((_nchw(ops.avgpool3s2(xa)) - F.avg_pool2d(x, 3, 2, 1, count_include_pad=False)).abs().max()) < 1e-6
    # bilinear x2 (+ add)
    lo = rnd(2, 24, 9, 7)
    b = rnd(2, 24, 18, 14)
    up = ops.bilinear_up2_add(_nhwc(lo), _nhwc(b), Act.empty(2, 18, 14, 24))
    assert float((_nchw(up) - (F.interpolate(lo, scale_factor=2, mode="bilinear", align_corners=False) + b)).abs().max()) < 1e-5
    # InstanceNorm statistics (one and two norms, half-resolution x0 + x1 concat, noise) and apply
    x0, x1 = rnd(2, 16, 9, 7) * 2 + 0.5, rnd(2, 8, 18, 14)
    noise, ns = rnd(2, 18, 14), rnd(24) * 0.3
    full = torch.cat([F.interpolate(x0, scale_factor=2, mode="nearest"), x1], 1) + noise[:, None] * ns[None, :, None, None]
    m_ref = full.double().mean((2, 3))
    r_ref = 1.0 / torch.sqrt(full.double().var((2, 3), unbiased=False) + 1e-5)
    m, r = ops.instnorm_stats(_nhwc(x0), 1, _nhwc(x1), 18, 14, noise.to(DEV), ns.to(DEV))
    assert float((m.cpu().double() - m_ref).abs().max()) < 2e-6 and float(((r.cpu().double() - r_ref) / r_ref).abs().max()) < 2e-6
    (m2, r2), = ops.instnorm_stats2(_nhwc(x0), 1, _nhwc(x1), 18, 14, [noise.to(DEV)], [ns.to(DEV)])
    assert float((m2.cpu().double() - m_ref).abs().max()) < 2e-6 and float(((r2.cpu().double() - r_ref) / r_ref).abs().max()) < 2e-6
    y = rnd(2, 24, 18, 14)
    ya = _nhwc(y)
    my, ry = ops.instnorm_stats(ya, 0, None, 18, 14, None, None)
    ops.instnorm_apply(ya, my, ry, ops.ACT_LRELU)
    assert float((_nchw(ya) - F.leaky_relu(F.instance_norm(y, eps=1e-5), 0.2)).abs().max()) < 1e-5
    # im2col (3x3 over a 7-channel map, the SPADE label-map form)
    sm = rnd(2, 7, 11, 9)
    cols = ops.im2col(_nhwc(sm), 3, 3, 1, k_pad=64)
    unf = F.unfold(sm, 3, padding=1).view(2, 7, 9, 11, 9).permute(0, 2, 1, 3, 4).reshape(2, 63, 11, 9)  # tap-major
    assert torch.equal(cols.buf[..., :63].permute(0, 3, 1, 2).cpu(), unf) and float(cols.buf[..., 63:].abs().max()) == 0.0
    # flow warp, fp32 source and destination
    fl = rnd(2, 9, 7, 2) * 3
    src = rnd(2, 24, 18, 14)
    dst = Act.empty(2, 18, 14, 24)
    ops.flow_warp(fl.to(DEV), _nhwc(src), dst)
    assert float((_nchw(dst) - orc.flow_warp(src, fl)).abs().max()) < 1e-5


def test_hbm_entry_points_refuse_mixed_storage(fp32):
    a32 = Act.empty(1, 8, 8, 16, zero=True)
    a16 = Act.empty(1, 8, 8, 16, dtype=torch.bfloat16, zero=True)
    with pytest.raises(RuntimeError, match="storage type"):
        ops.bilinear_up2_add(a32, None, Act.empty(1, 16, 16, 16, dtype=torch.bfloat16))
    with pytest.raises(RuntimeError, match="storage type"):
        ops.bilinear_up2_add(a32, Act.empty(1, 16, 16, 16, dtype=torch.bfloat16, zero=True), Act.empty(1, 16, 16, 16))
    with pytest.raises(RuntimeError, match="storage type"):
        ops.instnorm_stats(a32, 0, a16, 8, 8, None, None)
    m16, r16 = ops.instnorm_stats(a16, 0, None, 8, 8, None, None)
    with pytest.raises(RuntimeError, match="bf16"):
        ops.instnorm_apply(a16, m16, r16, ops.ACT_NONE, out=a32)


# ------------------------------------------------------------------------------------------------ whole networks: determinism, pipeline

def test_generator_fp32_bit_reproducible(fp32):
    g = load_golden("gen_256x256_b2")
    n, h, w = [int(v) for v in g["shape"]]
    seed = int(g["seed"])
    m, cnt = _gen_module(h, w, synth_state_dict("gen", seed), seed)
    x, seg = synth.gen_inputs(n, h, w, seed)
    with torch.no_grad():
        a = m(x.cuda(), seg.cuda()).clone()
        cnt[0] = 0
        b = m(x.cuda(), seg.cuda())
    assert torch.equal(a, b)


def _oracle_pipeline(sdt, sdg, batch, h, w, seed):
    cnt = [0]

    def noise(b, hh, ww):
        t = synth.spade_noise(b, hh, ww, seed, cnt[0])
        cnt[0] += 1
        return t

    class _Tocg:
        def __call__(self, i1, i2):
            return orc.tocg_forward(sdt, i1, i2)

    b = dict(batch)
    b["cloth_mask"] = (b["cloth_mask"] > 0.5).float()
    with torch.no_grad():
        g_in, parse = train_step.make_generator_inputs(_Tocg(), b, h, w, occlusion=True, unfused_parse=True)
        out = orc.spade_generator_forward(sdg, g_in, parse, noise)
    return out, g_in[:, 6:], parse


def test_tryon_pipeline_fp32_matches_oracle_pipeline(fp32):
    n, h, w, seed = 2, 512, 384, 19
    sdt, sdg = synth_state_dict("tocg", seed), synth_state_dict("gen", seed + 1)
    batch = train_step.synthetic_batch(n, h, w, "cpu", seed=seed)
    out_r, wc_r, parse_r = _oracle_pipeline(sdt, sdg, batch, h, w, seed)
    tocg = _tocg_module(sdt)
    G, _ = _gen_module(h, w, sdg, seed)
    out, wc, parse = pipeline.tryon_forward(tocg, G, {k: v.cuda() for k, v in batch.items()}, occlusion=True)
    torch.cuda.synchronize()
    out, wc, parse = out.cpu(), wc.cpu(), parse.cpu()
    agree = float((parse == parse_r).float().mean())
    same = (parse == parse_r).all(1, keepdim=True).float()
    d = (out - out_r).abs()
    mean_same = float((d * same).sum() / same.sum() / 3)
    dwc = float((wc - wc_r).abs().max())
    print("PIPELINE fp32: PSNR %.2f dB  max|d| %.3e  mean|d| over agreeing pixels %.3e  parse agreement %.6f  warped cloth max|d| %.3e"
          % (pipeline.psnr(out, out_r), float(d.max()), mean_same, agree, dwc))
    assert dwc < 1e-3
    assert agree >= 0.9999
    assert mean_same <= 1e-4


# ------------------------------------------------------------------------------------------------ training is refused; bf16 unchanged

def test_training_refused_in_fp32_and_bf16_unchanged():
    import network_generator
    import networks
    g = load_golden("gen_256x256_b2")
    n, h, w = [int(v) for v in g["shape"]]
    seed = int(g["seed"])
    sd = synth_state_dict("gen", seed)
    m, cnt = _gen_module(h, w, sd, seed)
    x, seg = synth.gen_inputs(n, h, w, seed)
    x, seg = x.cuda(), seg.cuda()
    with torch.no_grad():
        before = m(x, seg).clone()
    ops.set_precision("fp32")
    try:
        with pytest.raises(NotImplementedError, match="fp32 storage is inference-only"):
            m(x, seg)  # grad enabled, parameters require grad: the training path
        d = network_generator.MultiscaleDiscriminator(gen_opt(h, w, True)).cuda()
        with pytest.raises(NotImplementedError, match="fp32 storage is inference-only"):
            d(torch.cat([seg, x[:, :3]], 1))
        t = networks.ConditionGenerator(tocg_opt(True), 4, 16, 13, ngf=96, norm_layer=torch.nn.BatchNorm2d).cuda().train()
        i1, i2 = synth.tocg_inputs(1, 256, 192, seed)
        with pytest.raises(NotImplementedError, match="fp32 storage is inference-only"):
            t(i1.cuda(), i2.cuda())
        with contextlib.redirect_stdout(io.StringIO()):
            td = networks.define_D(input_nc=33, Ddownx2=True, Ddropout=True, n_layers_D=3, spectral=False, num_D=2).cuda()
        with pytest.raises(NotImplementedError, match="fp32 storage is inference-only"):
            td(torch.zeros(1, 33, 64, 48, device=DEV, requires_grad=True))
        with torch.no_grad():
            cnt[0] = 0
            m(x, seg)  # inference still runs
    finally:
        ops.set_precision("bf16")
    with torch.no_grad():
        cnt[0] = 0
        after = m(x, seg)
    assert torch.equal(before, after)
