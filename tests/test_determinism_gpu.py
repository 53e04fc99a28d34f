"""Run-to-run reproducibility on the GPU.

- The ordered flow-warp backward (hrv_flow_warp_bwd_ordered): dsrc32 equals, bit for bit, the sequential fp32 sum of d_dst * weight
  over each source pixel's (destination pixel, tap) pairs in ascending order; d flow_up / d flow_lo meet the fp64 bound of
  test_backward_kernels_gpu; three launches agree bit for bit.  Collision-heavy flows (every pixel pulled onto a few source pixels,
  or onto the border) are where the legacy atomic kernel's order shows.
- The fixed-order reductions meet their fp64 bounds and give identical bits across launches.
- hrv_flow_warp_nchw_bwd against fp64 autograd of F.interpolate(size, bilinear) + grid_sample(border), factors 2-32.
- Whole stage-1 and stage-2 training steps (eager, then CUDA-graph replays) under torch.use_deterministic_algorithms(True), twice
  from the same seed and state: every loss, parameter, optimizer state and running statistic is bit-identical."""
import ctypes
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "..", "oracle"))
import hrviton_oracle as orc  # noqa: E402
from hrviton_b200 import capi, ops  # noqa: E402
from hrviton_b200.ops import Act  # noqa: E402
from test_backward_kernels_gpu import EPS32, K_ACC, check, flow_warp_bwd_raw, flow_warp_bwd_ref, gen, precision, q, rnd, upload  # noqa: E402,F401

pytestmark = pytest.mark.gpu
DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def ordered_raw(flow, src, ddst, dfu_in):
    """hrv_flow_warp_bwd_ordered through the C-ABI; dsrc32 starts as NaN (the call overwrites it)."""
    n, hl, wl, _ = flow.shape
    H, W = 2 * hl, 2 * wl
    dsrc32 = torch.full((n, src.h, src.w, ops.round_up(src.c, 8)), float("nan"), dtype=torch.float32, device=DEV)
    dfu = dfu_in.float().to(DEV).contiguous().clone()
    dflo = torch.empty((n, hl, wl, 2), dtype=torch.float32, device=DEV)
    fl = flow.float().to(DEV).contiguous()
    ts, td = src.ct(), ddst.ct()
    L = ops._L(src)
    nws = int(L.hrv_flow_warp_bwd_ordered_workspace_bytes(ctypes.byref(ts), ctypes.byref(td)))
    ws = torch.empty(nws, dtype=torch.uint8, device=DEV)
    capi.check(L.hrv_flow_warp_bwd_ordered(fl.data_ptr(), ops.linspace_table(W, DEV).data_ptr(), ops.linspace_table(H, DEV).data_ptr(),
                                           ctypes.byref(ts), ctypes.byref(td), dsrc32.data_ptr(), dfu.data_ptr(), dflo.data_ptr(),
                                           ws.data_ptr(), nws, ops._stream()), "flow_warp_bwd_ordered")
    torch.cuda.synchronize()
    return dsrc32.cpu(), dfu.cpu(), dflo.cpu()


def sequential_dsrc(flow, ddst16, H, W):
    """The exact oracle: per source pixel, acc = fp32(acc + fp32(d * w)) over its (dst pixel, tap) pairs in ascending order, with
    the kernel's fp32 taps (np_flow_warp_coords) and weights fp32(wy * wx); zero-weight taps contribute nothing."""
    x0, y0, tx, ty = orc.np_flow_warp_coords(flow.float().numpy(), H, W, H, W)
    n = x0.shape[0]
    one = np.float32(1)
    vx, vy = x0 + 1 <= W - 1, y0 + 1 <= H - 1
    x1, y1 = np.where(vx, x0 + 1, x0), np.where(vy, y0 + 1, y0)
    wx1, wy1 = np.where(vx, tx, np.float32(0)), np.where(vy, ty, np.float32(0))
    wx0, wy0 = one - tx, one - ty
    b = np.arange(n)[:, None, None]
    keys = np.stack([(b * H + y0) * W + x0, (b * H + y0) * W + x1, (b * H + y1) * W + x0, (b * H + y1) * W + x1], -1).reshape(-1)
    wts = np.stack([wy0 * wx0, wy0 * wx1, wy1 * wx0, wy1 * wx1], -1).astype(np.float32).reshape(-1)
    d = ddst16.permute(0, 2, 3, 1).reshape(n * H * W, -1).float().numpy()  # (dst pixel, c), exact 16-bit values
    ent = np.nonzero(wts != 0)[0]
    order = ent[np.argsort(keys[ent], kind="stable")]
    k_sorted = keys[order]
    first = np.r_[True, k_sorted[1:] != k_sorted[:-1]]
    start = np.maximum.accumulate(np.where(first, np.arange(len(order)), 0))
    rank = np.arange(len(order)) - start
    acc = np.zeros((n * H * W, d.shape[1]), np.float32)
    for r in range(int(rank.max()) + 1 if len(rank) else 0):
        sel = order[rank == r]
        acc[keys[sel]] = acc[keys[sel]] + d[sel // 4] * wts[sel][:, None]
    return torch.from_numpy(acc.reshape(n, H, W, -1))


def collision_flow(n, hl, wl, seed):
    """Image 0: every destination pixel pulled to within a pixel of one interior point; image 1: far outside, onto the border."""
    H, W = 2 * hl, 2 * wl
    sx, sy = (W / 2 - 1.0) / 2.0, (H / 2 - 1.0) / 2.0
    X = torch.arange(wl, dtype=torch.float64)
    Y = torch.arange(hl, dtype=torch.float64)
    linx = -1 + 2 * (2 * X + 0.5) / (W - 1)
    liny = -1 + 2 * (2 * Y + 0.5) / (H - 1)
    flow = torch.zeros(n, hl, wl, 2, dtype=torch.float64)
    flow[0, ..., 0] = (-linx[None, :] + 0.13) * sx
    flow[0, ..., 1] = (-liny[:, None] - 0.21) * sy
    flow[0] += rnd(gen(seed), hl, wl, 2, scale=0.05).double()
    for i in range(1, n):
        flow[i] = rnd(gen(seed + i), hl, wl, 2, scale=40.0).double()
    return flow


@pytest.mark.parametrize("kind,c", [("smooth", 8), ("smooth", 384), ("collide", 8), ("collide", 64)])
def test_flow_warp_bwd_ordered(kind, c, precision):
    hl = wl = 16
    H, W = 2 * hl, 2 * wl
    flow = (rnd(gen(30), 2, hl, wl, 2) * 2.0).double() if kind == "smooth" else collision_flow(2, hl, wl, 31)
    g = gen(32)
    src, ddst = q(rnd(g, 2, c, H, W)), q(rnd(g, 2, c, H, W))
    dfu_in = rnd(g, 2, H, W, 2, scale=0.5).double()
    runs = [ordered_raw(flow, upload(src), upload(ddst), dfu_in) for _ in range(3)]
    for r in runs[1:]:
        for a, b in zip(runs[0], r):
            assert torch.equal(a.view(torch.int32), b.view(torch.int32)), "launches differ"
    dsrc32, dfu, dflo = runs[0]
    exact = sequential_dsrc(flow, ddst, H, W)
    assert torch.equal(dsrc32[..., :c].contiguous().view(torch.int32), exact[..., :c].contiguous().view(torch.int32)), \
        "dsrc32 differs from the ordered sequential fp32 sum"
    assert float(dsrc32[..., c:].abs().max()) == 0.0 if dsrc32.shape[3] > c else True
    ref = flow_warp_bwd_ref(flow, src, ddst, dfu_in)
    check("flow_warp_bwd_ordered dsrc32", dsrc32[..., :c].permute(0, 3, 1, 2), *ref["dsrc32"])
    check("flow_warp_bwd_ordered dflow_up", dfu, *ref["dflow_up"])
    check("flow_warp_bwd_ordered dflow_lo", dflo, *ref["dflow_lo"])
    if kind == "collide":  # reported, not asserted: the atomic kernel's order depends on timing
        legacy = flow_warp_bwd_raw(flow, upload(src), upload(ddst), dfu_in)[0].float()
        same = torch.equal(legacy[..., :c].contiguous().view(torch.int32), exact[..., :c].contiguous().view(torch.int32))
        print("LEGACY flow_warp_bwd %s c%d %s: bit-exact to the ordered sum: %s (%d differing elements)"
              % (kind, c, precision, same, int((legacy[..., :c] != exact[..., :c]).sum())))


def _same_bits(xs):
    return all(torch.equal(xs[0].cpu().contiguous().view(torch.uint8), x.cpu().contiguous().view(torch.uint8)) for x in xs[1:])


def test_act_bwd_bias_ordered(precision):
    g = gen(40)
    dy = q(rnd(g, 3, 72, 40, 33, scale=3.0))
    a = upload(dy)
    outs = [ops.act_bwd_bias(a, None, ops.ACT_NONE)[1] for _ in range(3)]
    assert _same_bits(outs)
    ref = dy.sum((0, 2, 3))
    S = dy.abs().sum((0, 2, 3))
    check("act_bwd_bias_ordered", outs[0].double().cpu(), ref, S, u=2.0 ** -24)


def test_l1_sum_ordered(precision):
    g = gen(41)
    x, y = q(rnd(g, 2, 64, 48, 40)), q(rnd(g, 2, 64, 48, 40))
    outs = [ops.l1_sum(upload(x), upload(y)) for _ in range(3)]
    assert _same_bits(outs)
    ref = (x - y).abs().sum().reshape(1)
    check("l1_sum", outs[0].cpu(), ref, ref)


def test_instnorm_stats_and_norm_bwd_ordered(precision):
    g = gen(42)
    n, c, h, w = 2, 64, 48, 40
    x = q(rnd(g, n, c, h, w, scale=2.0, mean=0.5))
    xa = upload(x)
    stats = [ops.instnorm_stats(xa, 0, None, h, w, None, None) for _ in range(3)]
    assert _same_bits([m for m, _ in stats]) and _same_bits([r for _, r in stats])
    check("instnorm_stats mean", stats[0][0].double().cpu(), x.mean((2, 3)), x.abs().mean((2, 3)))
    bn = [ops.batchnorm_stats(xa) for _ in range(3)]
    assert _same_bits([m for m, _ in bn]) and _same_bits([v for _, v in bn])
    mean, rstd = stats[0]
    noise = torch.randn(n, h, w, generator=g).to(DEV)
    ns = torch.randn(c, generator=g).to(DEV)
    mean2, rstd2 = ops.instnorm_stats(xa, 0, None, h, w, noise, ns)
    dh = upload(q(rnd(g, n, c, h, w)))
    outs = [ops.norm_bwd(dh, None, None, xa, 0, None, noise, ns, mean2, rstd2, ops.ACT_NONE, False) for _ in range(3)]
    for k in (1, 3, 4, 5):
        vals = [o[k].buf if isinstance(o[k], Act) else o[k] for o in outs]
        assert _same_bits(vals), k
    two = ops.instnorm_stats2(xa, 0, None, h, w, [noise, None], [ns, None])
    again = ops.instnorm_stats2(xa, 0, None, h, w, [noise, None], [ns, None])
    assert _same_bits([two[0][0], again[0][0]]) and _same_bits([two[0][1], again[0][1]])


@pytest.mark.parametrize("factor", [2, 4, 8, 16, 32])
def test_flow_warp_nchw_bwd(factor):
    """d flow_lo of hrv_flow_warp_nchw at 64x64 from a (64/f)x(64/f) flow against fp64 autograd of F.interpolate(size, bilinear) +
    grid_sample(border), with the sampling points pinned to the kernel's own fp32 grid (power-of-two extents map back exactly); the
    second image's constant flow puts whole rows and columns exactly on the border."""
    H = W = 64
    hl = wl = H // factor
    n, c = 2, 3
    g = gen(50 + factor)
    flow = rnd(g, n, hl, wl, 2, scale=3.0)
    src = rnd(g, n, c, H, W)
    mask = (rnd(g, n, 1, H, W) > 0).float()
    d_out, d_mask = rnd(g, n, c, H, W), rnd(g, n, 1, H, W)
    div = ((wl - 1.0) / 2.0, (hl - 1.0) / 2.0)
    flow[1, ..., 0] = div[0] / W  # g.x = lin_x + 1/W: column 0 lands exactly on ix = 0
    flow[1, ..., 1] = -div[1] / H  # g.y = lin_y - 1/H: the last row lands exactly on iy = H - 1
    fl_d = flow.to(DEV)
    outs = [ops.flow_warp_nchw_bwd(fl_d, src.to(DEV), (H, W), div, d_out.to(DEV), mask=mask.to(DEV), d_mask=d_mask.to(DEV)) for _ in range(3)]
    assert _same_bits(outs)
    _, grid = ops.flow_warp_nchw(fl_d, src.to(DEV), (H, W), div, want_grid=True)
    gk = grid.cpu()
    ix = ((gk[..., 0] + 1) * W - 1) / 2
    iy = ((gk[..., 1] + 1) * H - 1) / 2
    ix, iy = ix.clamp(0, W - 1).double(), iy.clamp(0, H - 1).double()
    gval = torch.stack([(2 * ix + 1) / W - 1, (2 * iy + 1) / H - 1], 3)
    fl = flow.double().clone().requires_grad_(True)
    up = F.interpolate(fl.permute(0, 3, 1, 2), size=(H, W), mode="bilinear", align_corners=False).permute(0, 2, 3, 1)
    base = torch.stack([torch.linspace(-1, 1, W).double().view(1, 1, W).expand(n, H, W), torch.linspace(-1, 1, H).double().view(1, H, 1).expand(n, H, W)], 3)
    g64 = torch.cat([up[..., 0:1] / div[0], up[..., 1:2] / div[1]], 3) + base
    grid64 = gval + (g64 - g64.detach())
    sm = torch.cat([src.double(), mask.double()], 1)
    out = F.grid_sample(sm, grid64, mode="bilinear", padding_mode="border", align_corners=False)
    (out * torch.cat([d_out, d_mask], 1).double()).sum().backward()
    # |.| map: |d| times the four taps' |value| times d ix / d flow, carried through the same resize adjoint
    x0, y0 = ix.floor().long(), iy.floor().long()
    x1, y1 = (x0 + 1).clamp(max=W - 1), (y0 + 1).clamp(max=H - 1)
    b = torch.arange(n)[:, None, None]
    sa = sm.abs().permute(0, 2, 3, 1)
    taps = sa[b, y0, x0] + sa[b, y0, x1] + sa[b, y1, x0] + sa[b, y1, x1]
    dabs = (torch.cat([d_out, d_mask], 1).double().abs().permute(0, 2, 3, 1) * taps).sum(3)
    S_hi = torch.stack([dabs * (W / 2) / div[0], dabs * (H / 2) / div[1]], 3)
    a = torch.zeros_like(fl, requires_grad=True)
    S_lo, = torch.autograd.grad(F.interpolate(a.permute(0, 3, 1, 2), size=(H, W), mode="bilinear", align_corners=False).permute(0, 2, 3, 1), a, S_hi)
    check("flow_warp_nchw_bwd", outs[0].cpu(), fl.grad, S_lo)


STEP_SCRIPT = textwrap.dedent(r'''
    import contextlib, io, os, sys, types
    import torch
    torch.use_deterministic_algorithms(True)
    torch.utils.deterministic.fill_uninitialized_memory = False
    sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
    import hrv_loader; hrv_loader.load()
    from hrviton_b200 import capi, synth, train_step
    L = capi.lib()
    def _refuse(*a, **k):
        raise RuntimeError("legacy non-reproducible entry point called")
    for name in ("hrv_flow_warp_bwd", "hrv_act_bwd_bias"):
        setattr(L, name, _refuse)
        setattr(L, name + "_f16", _refuse)
    import networks, network_generator
    from helpers import gen_opt, tocg_opt
    os.environ["HRV_VGG_RANDOM_INIT"] = "1"

    def state(mods, opts, outs):
        t = {}
        for mn, m in mods.items():
            for k, v in m.state_dict().items():
                t[mn + "." + k] = v.detach().clone()
        for on, o in opts.items():
            for i, s in enumerate(o.state.values()):
                for k, v in s.items():
                    if torch.is_tensor(v):
                        t["%s.%d.%s" % (on, i, k)] = v.detach().clone()
        for i, out in enumerate(outs):
            for k, v in out.items():
                t["loss%d.%s" % (i, k)] = v.detach().clone()
        return {k: v.cpu() for k, v in t.items()}

    def stage1():
        torch.manual_seed(0)
        tocg = networks.ConditionGenerator(tocg_opt(True), 4, 16, 13, ngf=96, norm_layer=torch.nn.BatchNorm2d)
        sdt = tocg.state_dict(); synth.fill_state_dict(sdt, 3); tocg.load_state_dict(sdt)
        tocg = tocg.cuda().train()
        with contextlib.redirect_stdout(io.StringIO()):
            D = networks.define_D(input_nc=33, Ddownx2=True, Ddropout=True, n_layers_D=3, spectral=False, num_D=2)
        D = D.cuda().train()
        vgg = networks.Vgg19().cuda().eval()
        tr = train_step.Stage1Trainer(tocg, D, vgg)
        batch = train_step.synthetic_batch_stage1(4, 256, 192, "cuda", seed=9)
        outs = [tr.step(batch) for _ in range(3)]
        tr.capture(batch)
        outs += [tr.replay(batch) for _ in range(3)]
        torch.cuda.synchronize()
        return state({"tocg": tocg, "D": D}, {"opt_g": tr.opt_g, "opt_d": tr.opt_d}, outs)

    def stage2():
        torch.manual_seed(0)
        h, w = 512, 384
        topt = types.SimpleNamespace(warp_feature="T1", out_layer="relu", cuda=True)
        tocg = networks.ConditionGenerator(topt, 4, 16, 13, ngf=96, norm_layer=torch.nn.BatchNorm2d)
        sdt = tocg.state_dict(); synth.fill_state_dict(sdt, 3); tocg.load_state_dict(sdt)
        tocg = tocg.cuda().eval()
        G = network_generator.SPADEGenerator(gen_opt(h, w, True), 9)
        sdg = G.state_dict(); synth.fill_state_dict(sdg, 4); G.load_state_dict(sdg)
        G = G.cuda().train()
        D = network_generator.MultiscaleDiscriminator(gen_opt(h, w, True))
        sdd = D.state_dict(); synth.fill_state_dict(sdd, 5); D.load_state_dict(sdd)
        D = D.cuda().train()
        vgg = networks.Vgg19().cuda().eval()
        tr = train_step.Stage2Trainer(tocg, G, D, vgg)
        batch = train_step.synthetic_batch(1, h, w, "cuda", seed=7)
        outs = [tr.step(batch, h, w) for _ in range(3)]
        tr.capture(batch, h, w)
        outs += [tr.replay(batch) for _ in range(3)]
        torch.cuda.synchronize()
        return state({"G": G, "D": D}, {"opt_g": tr.opt_g, "opt_d": tr.opt_d}, outs)

    fn = stage1 if sys.argv[1] == "stage1" else stage2
    a, b = fn(), fn()
    assert a.keys() == b.keys()
    bits = lambda t: t if t.dtype == torch.bool else t.reshape(-1).view(torch.uint8)
    diff = [k for k in a if not torch.equal(bits(a[k]), bits(b[k]))]
    print("DETERMINISM %s: %d tensors compared, %d differ %s" % (sys.argv[1], len(a), len(diff), diff[:10]))
    sys.exit(1 if diff else 0)
''')


@pytest.mark.parametrize("stage", ["stage1", "stage2"])
def test_training_steps_bit_identical(stage, tmp_path):
    script = tmp_path / "steps.py"
    script.write_text("ROOT = %r\n" % ROOT + STEP_SCRIPT)
    env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8")
    r = subprocess.run([sys.executable, "-s", str(script), stage], capture_output=True, text=True, env=env, timeout=1500)
    print(r.stdout[-3000:])
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-6000:]
