"""Dynamic loss scaling on the GPU: hrv_grad_unscale_check against torch, the fp16 underflow of the VGG and feature-matching
gradients that scaling removes, the skip of an overflowing step, bit-identical scaled training under CUDA-graph replay (stage 1 and 2),
and the reference's own --fp16 loop through the apex shim."""
import contextlib
import io
import os
import subprocess
import sys
import textwrap

import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import hrv_env  # noqa: E402
import hrviton_oracle as orc  # noqa: E402
from floors import check, stats  # noqa: E402
from helpers import gen_opt  # noqa: E402
from hrviton_b200 import autograd_g, ops, train_step  # noqa: E402
from hrviton_b200.ops import Act  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
S16 = 2.0 ** 16


@contextlib.contextmanager
def precision(name):
    old = ops.get_precision()
    ops.set_precision(name)
    try:
        yield
    finally:
        ops.set_precision(old)


def _bits(t):
    return t.contiguous().view(torch.int32)


# ------------------------------------------------------------------------------------------------------------------ kernel

def _segments(seed):
    """Views at every alignment (offsets 0..3 floats into one buffer), odd and tiny lengths, empty ones, and separate tensors
    that span several 16 KiB chunks."""
    g = torch.Generator().manual_seed(seed)
    base = torch.randn(300000, generator=g).mul_(1e3).to(DEV)
    segs, off = [], 0
    for n in [1, 2, 3, 4, 5, 7, 0, 31, 257, 4096 + 3, 16384 + 5, 65536 - 1, 70001, 3, 0, 1000]:
        off += 1 + (n % 3)
        segs.append(base[off:off + n])
        off += n
    segs += [torch.randn(n, generator=g).to(DEV) for n in (1 << 20, 4099, 8)]
    return segs


def _run_kernel(segs, inv_scale):
    inv = torch.full((), inv_scale, dtype=torch.float32, device=DEV)
    found = torch.zeros((), dtype=torch.float32, device=DEV)
    ref = [s * inv for s in segs]
    ref_found = any(bool((~torch.isfinite(s)).any()) for s in segs)
    table = ops.grad_unscale_check(segs, inv, found)
    torch.cuda.synchronize()
    for i, (s, r) in enumerate(zip(segs, ref)):
        assert torch.equal(_bits(s), _bits(r)), ("segment", i, s.numel())
    assert float(found) == (1.0 if ref_found else 0.0)
    return table


def test_unscale_clean_segments_bit_exact():
    segs = _segments(1)
    assert any(s.data_ptr() % 16 for s in segs) and any(s.data_ptr() % 16 == 0 for s in segs)
    table = _run_kernel(segs, 2.0 ** -16)
    _run_kernel(segs, 2.0 ** -3)  # a new scale through the same table
    found = torch.zeros((), device=DEV)
    assert ops.grad_unscale_check(segs, torch.full((), 0.5, device=DEV), found, table) is table  # reused while nothing moved


@pytest.mark.parametrize("where", ["first", "last", "boundary", "every"])
@pytest.mark.parametrize("value", [float("inf"), float("-inf"), float("nan")])
def test_unscale_flags_non_finite(where, value):
    segs = _segments(2)
    live = [s for s in segs if s.numel()]
    if where == "first":
        live[0][0] = value
    elif where == "last":
        live[-1][-1] = value
    elif where == "boundary":  # both ends of a misaligned segment and the last element of a chunk
        seg = next(s for s in live if s.numel() > 16384 and s.data_ptr() % 16)
        seg[0], seg[-1] = value, value
        seg[4 * 1024 - 1 + ((16 - seg.data_ptr() % 16) % 16) // 4] = value
    else:
        for s in live:
            s[s.numel() // 2] = value
    _run_kernel(segs, 2.0 ** -16)


def test_found_inf_is_only_set():
    segs = _segments(3)
    found = torch.ones((), device=DEV)
    ops.grad_unscale_check(segs, torch.full((), 1.0, device=DEV), found)
    assert float(found) == 1.0  # a clean pass leaves an earlier flag alone: the caller zeroes it


# ------------------------------------------------------------------------------------------------------------------ underflow

def _vgg():
    os.environ["HRV_VGG_RANDOM_INIT"] = "1"
    import networks
    torch.manual_seed(11)
    return networks.Vgg19().eval()


def _vgg_loss_ref(vgg, x, y, scale, dtype):
    """CPU VGGLoss on the frozen weights: fp64 (dtype None) or fp32 under oracle.storage_rounding(dtype); d x of loss * scale / scale."""
    ft = torch.float64 if dtype is None else torch.float32
    x = x.to(ft).clone().requires_grad_(True)

    def feats(t):
        out = []
        for k in range(5):
            for layer in getattr(vgg, "slice%d" % (k + 1)):
                if isinstance(layer, torch.nn.Conv2d):
                    t = orc.conv2d_q(t, layer.weight.detach().to(ft), layer.bias.detach().to(ft), padding=1)
                elif isinstance(layer, torch.nn.ReLU):
                    t = F.relu(t)
                else:
                    t = F.max_pool2d(t, 2)
            out.append(t)
        return out

    with orc.storage_rounding(dtype) if dtype is not None else contextlib.nullcontext():
        with torch.no_grad():
            fy = feats(y.to(ft))
        fx = feats(x)
        loss = sum(w * (a - b).abs().mean() for w, a, b in zip([1 / 32, 1 / 16, 1 / 8, 1 / 4, 1.0], fx, fy)) * 10.0
        (loss * scale).backward()
    return (x.grad / scale).double()


def test_vgg_loss_fp16_underflow_and_scaled_gradient():
    n, h, w = 4, 256, 192  # relu1_1 seed 10/32/(4*64*256*192) = 2.5e-8 < 2^-25: rounds to 0 in fp16
    vgg = _vgg()
    g = torch.Generator().manual_seed(5)
    x = F.interpolate(torch.rand(n, 3, h // 8, w // 8, generator=g) * 2 - 1, size=(h, w), mode="bilinear", align_corners=False)
    y = F.interpolate(torch.rand(n, 3, h // 8, w // 8, generator=g) * 2 - 1, size=(h, w), mode="bilinear", align_corners=False)
    vd = vgg.to(DEV)
    with precision("fp16"):
        with torch.no_grad():
            fx = autograd_g.vgg_features(vd, x.to(DEV))
            fy = autograd_g.vgg_features(vd, y.to(DEV))
        seed = 10.0 / 32 / fx[0][..., :64].numel()
        assert fx[0].dtype == torch.float16 and seed < 2.0 ** -25
        d_plain = ops.l1_bwd(Act(fx[0], c=64), Act(fy[0], c=64), torch.full((1,), seed, device=DEV), relu_gate=True).buf
        d_scaled = ops.l1_bwd(Act(fx[0], c=64), Act(fy[0], c=64), torch.full((1,), seed * S16, device=DEV), relu_gate=True).buf
        assert int(torch.count_nonzero(d_plain)) == 0  # the problem: slice 1 contributes nothing
        assert int(torch.count_nonzero(d_scaled)) > d_scaled.numel() // 4
        grads = {}
        for scale in (1.0, S16):
            xd = x.to(DEV).requires_grad_(True)
            loss = autograd_g.vgg_loss(vd, [1 / 32, 1 / 16, 1 / 8, 1 / 4, 1.0], xd, y.to(DEV)) * 10.0
            (loss * scale).backward()
            grads[scale] = (xd.grad / scale).cpu().double()
    vgg = vgg.cpu()
    ref = _vgg_loss_ref(vgg, x, y, 1.0, None)
    floor = stats(_vgg_loss_ref(vgg, x, y, S16, torch.float16), ref)
    check("vgg_loss d x, fp16, S=2^16", grads[S16], ref, floor)
    unscaled = stats(grads[1.0], ref)
    print("unscaled fp16 vgg_loss d x: mean %.3e = x%.2f the scaled floor" % (unscaled["mean"], unscaled["mean"] / floor["mean"]))


def test_feature_matching_fp16_subnormal_seed():
    n, h, w, c = 2, 257, 193, 64  # seed 5 / (2*257*193*64) = 7.9e-7: a subnormal fp16 number (13 quanta of 2^-24)
    g = torch.Generator().manual_seed(9)
    buf32 = torch.randn(2 * n, h, w, c, generator=g)
    with precision("fp16"):
        buf = buf32.to(torch.float16).to(DEV).requires_grad_(True)
        got = {}
        for scale in (1.0, S16):
            buf.grad = None
            (autograd_g.FeatMatchFn.apply(buf) * 5.0 * scale).backward()
            got[scale] = (buf.grad.double() / scale).cpu()
    b64 = buf.detach().double().cpu()
    ref = torch.zeros_like(b64)
    ref[:n] = torch.sign(b64[:n] - b64[n:]) * (5.0 / (n * h * w * c))
    assert float(ref[:n].abs().max()) < 2.0 ** -14  # below fp16's normal range
    floor = stats((ref * S16).to(torch.float16).double() / S16, ref)  # one fp16 rounding of a normal number
    check("FeatMatchFn d buf, fp16, S=2^16", got[S16], ref, floor)
    plain = stats(got[1.0], ref)
    assert plain["mean"] > 10 * floor["mean"], (plain, floor)  # the unscaled gradient misses the floor by far
    print("FeatMatchFn unscaled mean error x%.1f the floor" % (plain["mean"] / floor["mean"]))


# ------------------------------------------------------------------------------------------------------------------ skip

def _filled(mod, seed):
    from hrviton_b200 import synth
    sd = mod.state_dict()
    synth.fill_state_dict(sd, seed)
    mod.load_state_dict(sd)
    return mod.cuda()


def _stage2(h, w, **kw):
    import types

    import network_generator
    import networks
    os.environ["HRV_VGG_RANDOM_INIT"] = "1"
    torch.manual_seed(0)
    topt = types.SimpleNamespace(warp_feature="T1", out_layer="relu", cuda=True)
    tocg = _filled(networks.ConditionGenerator(topt, 4, 16, 13, ngf=96, norm_layer=torch.nn.BatchNorm2d), 3).eval()
    G = _filled(network_generator.SPADEGenerator(gen_opt(h, w, True), 9), 4).train()
    D = _filled(network_generator.MultiscaleDiscriminator(gen_opt(h, w, True)), 5).train()
    tr = train_step.Stage2Trainer(tocg, G, D, networks.Vgg19().cuda().eval(), **kw)
    return tr, train_step.synthetic_batch(1, h, w, DEV, seed=7)


def _snapshot(tr):
    """{(net, parameter name, "param" | Adam state key): copy}"""
    out = {}
    for name, mod, opt in (("G", tr.G, tr.opt_g), ("D", tr.D, tr.opt_d)):
        for k, p in mod.named_parameters():
            out[(name, k, "param")] = p.detach().clone()
            for sk, sv in opt.state.get(p, {}).items():
                out[(name, k, sk)] = sv.detach().clone()
    return out


def test_overflow_step_is_skipped():
    h, w = 512, 384
    with precision("fp16"):
        tr, batch = _stage2(h, w, loss_scale="dynamic")
        tr.step(batch, h, w)  # creates the Adam state
        before = _snapshot(tr)
        for sc in tr.scalers.values():
            sc.scale.fill_(2.0 ** 60)
        tr.step(batch, h, w)
        torch.cuda.synchronize()
        after = _snapshot(tr)
        assert before.keys() == after.keys()
        moved = [k for k in before if not torch.equal(_bits(before[k].float()), _bits(after[k].float()))]
        assert not moved, moved[:10]  # parameters, exp_avg, exp_avg_sq and step untouched
        assert {k[2] for k in before} == {"param", "exp_avg", "exp_avg_sq", "step"}
        for name, sc in tr.scalers.items():
            assert float(sc.found_inf) == 1.0 and float(sc.scale) == 2.0 ** 59 and int(sc.growth_tracker) == 0, name
            sc.scale.fill_(S16)
        tr.step(batch, h, w)
        torch.cuda.synchronize()
        again = _snapshot(tr)
        for name, sc in tr.scalers.items():
            assert float(sc.found_inf) == 0.0 and float(sc.scale) == S16, name
        for net in ("G", "D"):
            assert any(not torch.equal(before[k], again[k]) for k in before if k[0] == net and k[2] == "param"), net
        assert all(int(v) == 2 for k, v in again.items() if k[2] == "step")  # the skipped step did not count


# ------------------------------------------------------------------------------------------------------------------ graphs

GRAPH_SCRIPT = textwrap.dedent(r'''
    import contextlib, io, os, sys, types
    import torch
    torch.use_deterministic_algorithms(True)
    torch.utils.deterministic.fill_uninitialized_memory = False
    sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
    import hrv_loader; hrv_loader.load()
    from hrviton_b200 import ops, synth, train_step
    assert ops.get_precision() == "fp16"
    import networks, network_generator
    from helpers import gen_opt, tocg_opt
    os.environ["HRV_VGG_RANDOM_INIT"] = "1"

    def build(stage):
        torch.manual_seed(0)
        vgg = networks.Vgg19().cuda().eval()
        if stage == "stage1":
            tocg = networks.ConditionGenerator(tocg_opt(True), 4, 16, 13, ngf=96, norm_layer=torch.nn.BatchNorm2d)
            sdt = tocg.state_dict(); synth.fill_state_dict(sdt, 3); tocg.load_state_dict(sdt)
            with contextlib.redirect_stdout(io.StringIO()):
                D = networks.define_D(input_nc=33, Ddownx2=True, Ddropout=True, n_layers_D=3, spectral=False, num_D=2)
            tr = train_step.Stage1Trainer(tocg.cuda().train(), D.cuda().train(), vgg, loss_scale="dynamic")
            return tr, {"tocg": tocg, "D": D}, (train_step.synthetic_batch_stage1(4, 256, 192, "cuda", seed=9),)
        h, w = 512, 384
        topt = types.SimpleNamespace(warp_feature="T1", out_layer="relu", cuda=True)
        tocg = networks.ConditionGenerator(topt, 4, 16, 13, ngf=96, norm_layer=torch.nn.BatchNorm2d)
        sdt = tocg.state_dict(); synth.fill_state_dict(sdt, 3); tocg.load_state_dict(sdt)
        G = network_generator.SPADEGenerator(gen_opt(h, w, True), 9)
        sdg = G.state_dict(); synth.fill_state_dict(sdg, 4); G.load_state_dict(sdg)
        D = network_generator.MultiscaleDiscriminator(gen_opt(h, w, True))
        sdd = D.state_dict(); synth.fill_state_dict(sdd, 5); D.load_state_dict(sdd)
        tr = train_step.Stage2Trainer(tocg.cuda().eval(), G.cuda().train(), D.cuda().train(), vgg, loss_scale="dynamic")
        return tr, {"G": G, "D": D}, (train_step.synthetic_batch(1, h, w, "cuda", seed=7), h, w)

    def run(stage):
        tr, mods, args = build(stage)
        for sc in tr.scalers.values():
            sc.growth_interval = 2  # let the scale move within the run
        hist = []

        def record(out):
            torch.cuda.synchronize()
            hist.append({k: (float(sc.scale), float(sc.found_inf), int(sc.growth_tracker)) for k, sc in tr.scalers.items()})
            return out

        outs = [record(tr.step(*args)) for _ in range(3)]
        tr.capture(*args)  # two warm-up steps run eagerly, then one is captured
        record(None)
        outs += [record(tr.replay(args[0])) for _ in range(3)]
        t = {}
        for mn, m in mods.items():
            for k, v in m.state_dict().items():
                t[mn + "." + k] = v.detach().clone()
        for on, o in (("opt_g", tr.opt_g), ("opt_d", tr.opt_d)):
            for i, s in enumerate(o.state.values()):
                for k, v in s.items():
                    t["%s.%d.%s" % (on, i, k)] = v.detach().clone()
        for i, out in enumerate(outs):
            for k, v in out.items():
                t["loss%d.%s" % (i, k)] = torch.as_tensor(v).detach().clone()
        for k, sc in tr.scalers.items():
            t["scale." + k] = sc.scale.clone()
        return {k: v.cpu() for k, v in t.items()}, hist

    def follows_rule(hist):
        # eager steps and graph replays move (scale, tracker) by the same rule (apex's, growth_interval 2) from the state before them;
        # hist[3] is recorded after capture(), which ran two eager warm-up steps
        for k in hist[0]:
            seq = [(2.0 ** 16, 0.0, 0)] + [h[k] for h in hist]
            for i in (0, 1, 2, 4, 5, 6):
                (s, _, trk), (s1, found, trk1) = seq[i], seq[i + 1]
                want = (s * 0.5, 0) if found else ((s * 2.0, 0) if trk + 1 == 2 else (s, trk + 1))
                assert want == (s1, trk1), (k, i, seq)
            assert len({v[0] for v in seq}) > 1, (k, seq)  # the scale did move

    stage = sys.argv[1]
    (a, ha), (b, hb) = run(stage), run(stage)
    assert ha == hb, (ha, hb)
    follows_rule(ha)
    assert a.keys() == b.keys()
    bits = lambda t: t if t.dtype == torch.bool else t.reshape(-1).view(torch.uint8)
    diff = [k for k in a if not torch.equal(bits(a[k]), bits(b[k]))]
    print("LOSS_SCALE_GRAPH %s: %d tensors compared, %d differ %s; scale history %s" % (stage, len(a), len(diff), diff[:10], ha))
    sys.exit(1 if diff else 0)
''')


@pytest.mark.parametrize("stage", ["stage1", "stage2"])
def test_scaled_training_graph_bit_identical(stage, tmp_path):
    script = tmp_path / "steps.py"
    script.write_text("ROOT = %r\n" % ROOT + GRAPH_SCRIPT)
    env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8", HRV_PRECISION="fp16")
    r = subprocess.run([sys.executable, "-s", str(script), stage], capture_output=True, text=True, env=env, timeout=1500)
    print(r.stdout[-3000:])
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-6000:]


# ------------------------------------------------------------------------------------------------------------------ reference

@pytest.mark.skipif(hrv_env.reference_dir() is None, reason="no reference copy (oracle/_ref)")
def test_reference_train_generator_fp16_uses_loss_scaling():
    import test_reference_scripts_gpu as trs
    with precision("fp16"):
        import network_generator
        import networks
        tg = hrv_env.load_reference_script("train_generator")
        from apex import amp

        from hrviton_b200.loss_scale import DynamicLossScaler
        h, w = 512, 384
        opt = trs._opt(tg, ["--name", "t", "--cuda", "True", "--gpu_ids", "0", "-b", "1", "--fine_height", str(h), "--fine_width", str(w),
                            "--keep_step", "2", "--decay_step", "0", "--display_count", "1000", "--save_count", "1000",
                            "--tensorboard_count", "1000", "--lpips_count", "1000", "--occlusion", "--fp16"])
        torch.manual_seed(0)
        tocg = networks.ConditionGenerator(opt, input1_nc=4, input2_nc=opt.semantic_nc + 3, output_nc=13, ngf=96, norm_layer=torch.nn.BatchNorm2d)
        generator = network_generator.SPADEGenerator(opt, 9)
        generator.cuda()
        generator.init_weights(opt.init_type, opt.init_variance)
        with contextlib.redirect_stdout(io.StringIO()):
            discriminator = tg.create_network(network_generator.MultiscaleDiscriminator, opt)
        g0 = generator.up_3.conv_0.weight_orig.detach().clone()
        d0 = discriminator.discriminator_0.model0[0].weight.detach().clone()
        flags = []  # (loss_id, found_inf) of every scale_loss exit
        update = DynamicLossScaler.update

        def recording_update(sc):
            flags.append((amp._SCALERS.index(sc), float(sc.found_inf)))
            update(sc)

        try:
            DynamicLossScaler.update = recording_update
            with contextlib.redirect_stdout(io.StringIO()):
                tg.train(opt, trs._Loader(1, h, w), None, None, tg.SummaryWriter(log_dir="unused"), tocg, generator, discriminator, trs._Lpips())
            torch.cuda.synchronize()
            print("apex shim, --fp16: (loss_id, found_inf) per step", flags, "scales", [float(sc.scale) for sc in amp._SCALERS])
            assert len(amp._SCALERS) == 2 and [i for i, _ in flags] == [0, 1, 0, 1]
            for i, sc in enumerate(amp._SCALERS):
                # engaged: started at 2^16, halved once per overflowing step (as apex does: the freshly initialised G may overflow at
                # first), no growth within 2 steps; at least one step of each loss was clean, so both networks move
                skips = sum(f for j, f in flags if j == i)
                assert skips <= 1 and float(sc.scale) == S16 * 0.5 ** skips, (i, flags)
        finally:
            DynamicLossScaler.update = update
            amp._SCALERS[:] = []
    gm = generator.module if hasattr(generator, "module") else generator
    dm = discriminator.module if hasattr(discriminator, "module") else discriminator
    assert float((gm.up_3.conv_0.weight_orig.detach() - g0).abs().max()) > 0
    assert float((dm.discriminator_0.model0[0].weight.detach() - d0).abs().max()) > 0
    assert all(bool(torch.isfinite(p).all()) for p in gm.parameters())
