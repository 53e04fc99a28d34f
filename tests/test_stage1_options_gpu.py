"""GPU: the stage-1 loss options of train_condition.py.

The fused flow TV (hrv_flow_tv / hrv_flow_tv_bwd through autograd_tocg.FlowTVFn):
- against train_condition.py's own TV lines (the `if opt.edgeawaretv == 'no_edge':` block, read from the reference copy under
  oracle/_ref and run as written) in float64 on the CPU: loss to 1e-5 relative, d flow and d mask to 1e-5 of their largest magnitude.
  Inputs hold exact ties (repeated flow rows and columns: D flow = 0; mask plateaus: D m = 0), so the sgn(0) = 0 convention shows.  The
  masks take values in [0, 1/8]: the fp32 interpolation then leaves errors of ~1e-8 in m, which exp(-150 |D m|) amplifies 150 times,
  well inside the bound.  d mask jumps where D m changes sign; where a smooth mask has |D m| within that fp32 error of 0 (0 < |D m| <
  1e-6 in float64) either sign is right, so the mask pixels those pairs read are left out of the d mask comparison (a few per mille);
- m_i is bit-identical to F.interpolate(mask, size, mode='bilinear') on CUDA; two runs give the same bits; forward and backward run
  under torch.use_deterministic_algorithms(True).
Stage1Trainer with each option: one eager step's losses against a torch restatement of the reference's branch; graph replays equal eager
steps bit for bit; --no_GAN_loss leaves D and its Adam state alone; --G_D_seperate moves the BatchNorm running statistics twice and
shows D the uncomposed soft-max; explicit defaults equal today's trainer; a --edgeawaretv weighted --add_lasttv run resumes bit for bit."""
import os
import sys
import textwrap

import pytest
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for _p in (ROOT, HERE):
    if _p not in sys.path:
        sys.path.insert(0, _p)
import hrv_loader  # noqa: E402

hrv_loader.load()
from hrviton_b200 import autograd_g, autograd_tocg, ops, train_loop, train_step  # noqa: E402
from test_train_loop_gpu import _assert_same, _everything, _final_state, _flags, _launch, _stage1_trainer, tree  # noqa: E402,F401

pytestmark = pytest.mark.gpu
REF_SCRIPT = os.path.join(ROOT, "oracle", "_ref", "train_condition.py")
TOCG_FLOWS = [(8, 6), (16, 12), (32, 24), (64, 48), (128, 96)]  # the tocg's five flows for a 256x192 input
ODD_FLOWS = [(7, 5), (4, 3), (9, 13), (12, 7), (25, 18)]  # of a 50x37 mask


def _reference_tv_block():
    """train_condition.py's TV lines as written: from `if opt.edgeawaretv == 'no_edge':` to the line before `N, _, iH, iW = ...`."""
    if not os.path.isfile(REF_SCRIPT):
        pytest.skip("no reference copy (oracle/_ref)")
    lines = open(REF_SCRIPT).read().splitlines()
    a = next(i for i, l in enumerate(lines) if l.strip() == "if opt.edgeawaretv == 'no_edge':")
    b = next(i for i, l in enumerate(lines) if i > a and l.strip().startswith("N, _, iH, iW"))
    return compile(textwrap.dedent("\n".join(lines[a:b])), REF_SCRIPT, "exec")


def reference_tv(flow_list, warped_clothmask_paired, edgeawaretv, add_lasttv, lasttvonly=True):
    import types
    scope = {"torch": torch, "F": F, "flow_list": flow_list, "warped_clothmask_paired": warped_clothmask_paired, "loss_tv": 0,
             "opt": types.SimpleNamespace(edgeawaretv=edgeawaretv, add_lasttv=add_lasttv, lasttvonly=lasttvonly)}
    exec(_reference_tv_block(), scope)
    return scope["loss_tv"]


def tv_inputs(n, sizes, mh, mw, seed, top=0.125):
    g = torch.Generator().manual_seed(seed)
    flows = []
    for h, w in sizes:
        f = torch.randn(n, h, w, 2, generator=g)
        rows, cols = torch.arange(h), torch.arange(w)
        rows[2::4] -= 1  # row 2 repeats row 1, ...: D_y flow = 0 exactly
        cols[1::3] -= 1
        flows.append(f[:, rows][:, :, cols].contiguous())
    lo = torch.rand(n, 1, max(2, mh // 6), max(2, mw // 6), generator=g)
    ramp = F.interpolate(lo, size=(mh, mw), mode="bilinear", align_corners=False)
    mask = ((ramp * 3 - 1).clamp(0, 1) * top).contiguous()  # plateaus at 0 and `top` (D m = 0), ramps between
    return flows, mask


def _kernel_tv(flows, mask, mode, add_lasttv):
    fl = [f.cuda().requires_grad_() for f in flows]
    m = mask.cuda().requires_grad_()
    loss = autograd_tocg.flow_tv(fl, m, mode, add_lasttv)
    loss.backward()
    return loss.detach(), [f.grad for f in fl], m.grad


@pytest.mark.parametrize("n", [1, 3])
@pytest.mark.parametrize("shape", ["tocg", "odd"])
@pytest.mark.parametrize("add_lasttv", [False, True])
@pytest.mark.parametrize("mode", ["last_only", "weighted"])
def test_flow_tv_against_reference_fp64(mode, add_lasttv, shape, n):
    sizes, (mh, mw) = (TOCG_FLOWS, (256, 192)) if shape == "tocg" else (ODD_FLOWS, (50, 37))
    flows, mask = tv_inputs(n, sizes, mh, mw, seed=len(sizes) * 10 + n)
    fl64 = [f.double().requires_grad_() for f in flows]
    m64 = mask.double().requires_grad_()
    ref = reference_tv(fl64, m64, mode, add_lasttv)
    ref.backward()
    loss, dflows, dmask = _kernel_tv(flows, mask, mode, add_lasttv)
    assert abs(float(loss) - float(ref)) <= 1e-5 * abs(float(ref)), (float(loss), float(ref))
    for i, (d, r) in enumerate(zip(dflows, fl64)):
        assert (d is None) == (r.grad is None), i
        if d is not None:
            err = float((d.cpu().double() - r.grad).abs().max())
            assert err <= 1e-5 * float(r.grad.abs().max()), (i, err, float(r.grad.abs().max()))
    keep = _away_from_sign_changes(fl64, m64.detach(), mode)
    assert float(keep.float().mean()) > 0.99
    err = float(((dmask.cpu().double() - m64.grad) * keep).abs().max())
    assert float(m64.grad.abs().max()) > 0 and err <= 1e-5 * float(m64.grad.abs().max()), (err, float(m64.grad.abs().max()))


def _away_from_sign_changes(flows, mask, mode):
    """Mask pixels read by no pair whose float64 |D m| lies in (0, 1e-6); asserts that exact ties (D m = 0) exist."""
    m = mask.clone().requires_grad_()
    near, ties = 0, 0
    for f in (flows[-1:] if mode == "last_only" else flows):
        down = F.interpolate(m, f.shape[1:3], mode="bilinear")
        dy, dx = (down[:, :, 1:] - down[:, :, :-1]).detach().abs(), (down[:, :, :, 1:] - down[:, :, :, :-1]).detach().abs()
        ties += int((dy == 0).sum() + (dx == 0).sum())
        ny, nx = ((dy > 0) & (dy < 1e-6)).double(), ((dx > 0) & (dx < 1e-6)).double()
        z = torch.zeros_like(down)
        z[:, :, 1:] += ny
        z[:, :, :-1] += ny
        z[:, :, :, 1:] += nx
        z[:, :, :, :-1] += nx
        near = near + (down * z).sum()
    assert ties > 0
    if not torch.is_tensor(near):
        return torch.ones_like(mask, dtype=torch.bool)
    g, = torch.autograd.grad(near, m, allow_unused=True)
    return torch.ones_like(mask, dtype=torch.bool) if g is None else g == 0


@pytest.mark.parametrize("n", [1, 3])
def test_flow_tv_mask_down_bit_identical_to_interpolate(n):
    flows, _ = tv_inputs(n, TOCG_FLOWS, 256, 192, seed=4)
    for sz, (mh, mw), fls in (("tocg", (256, 192), flows), ("odd", (50, 37), tv_inputs(n, ODD_FLOWS, 50, 37, seed=5)[0]),
                              ("up", (5, 4), tv_inputs(n, [(7, 5), (12, 9)], 5, 4, seed=6)[0])):
        mask = torch.rand(n, 1, mh, mw, generator=torch.Generator().manual_seed(7)).cuda()
        fc = [f.cuda() for f in fls]
        _, _, downs = ops.flow_tv(fc, [1.0] * len(fc), [0.0] * len(fc), mask, want_mask_down=True)
        for f, d in zip(fc, downs):
            want = F.interpolate(mask, size=tuple(f.shape[1:3]), mode="bilinear")
            assert torch.equal(d, want), (sz, tuple(f.shape))


def test_flow_tv_reproducible_and_deterministic_mode():
    flows, mask = tv_inputs(8, TOCG_FLOWS, 256, 192, seed=3, top=1.0)
    torch.use_deterministic_algorithms(True)
    try:
        runs = [_kernel_tv(flows, mask, "weighted", True) for _ in range(2)]
        torch.cuda.synchronize()
    finally:
        torch.use_deterministic_algorithms(False)
    (l0, d0, m0), (l1, d1, m1) = runs
    assert torch.equal(l0, l1) and torch.equal(m0, m1)
    assert all(torch.equal(a, b) for a, b in zip(d0, d1))


# ------------------------------------------------------------------------------------------------------------------------ trainer

OPTIONS = {
    "last_only": {"edgeawaretv": "last_only"},
    "last_only_add": {"edgeawaretv": "last_only", "add_lasttv": True},
    "weighted": {"edgeawaretv": "weighted"},
    "weighted_add": {"edgeawaretv": "weighted", "add_lasttv": True},
    "detach": {"clothmask_composition": "detach"},
    "no_composition": {"clothmask_composition": "no_composition"},
    "no_gan": {"no_gan_loss": True},
    "lambdas": {"tvlambda": 3.0, "ce_lambda": 5.0, "gan_lambda": 0.5},
}


def _restated_losses(tr, batch, o):
    """The losses of train_condition.py:158-282 for the options `o`, in torch (the TV from the reference's own lines), on the trainer's
    networks and the same random draws; no update."""
    o = dict(train_loop.STAGE1_OPTIONS, **o)
    c_paired, im_c, pcm = batch["cloth"], batch["parse_cloth"], batch["pcm"]
    cm_paired = (batch["cloth_mask"] > 0.5).float()
    input1 = torch.cat([c_paired, cm_paired], 1)
    input2 = torch.cat([batch["parse_agnostic"], batch["densepose"]], 1)
    with torch.no_grad():
        flow_list, fake_segmap, warped_cloth_paired, warped_clothmask_paired = autograd_tocg.tocg_forward_train(tr.tocg, input1, input2)
        warped_cm_onehot = (warped_clothmask_paired > 0.5).float()
        if o["clothmask_composition"] != "no_composition":
            cloth_mask = torch.ones_like(fake_segmap)
            cloth_mask[:, 3:4] = warped_cm_onehot if o["clothmask_composition"] == "detach" else warped_clothmask_paired
            fake_segmap = fake_segmap * cloth_mask
        warped_clothmask_paired = tr._remove_overlap(F.softmax(fake_segmap, dim=1), warped_clothmask_paired)  # --occlusion
        warped_cloth_paired = warped_cloth_paired * warped_clothmask_paired + torch.ones_like(warped_cloth_paired) * (1 - warped_clothmask_paired)
        loss_l1 = F.l1_loss(warped_clothmask_paired, pcm)
        loss_vgg = autograd_g.vgg_loss(tr.vgg, tr.vgg_weights, warped_cloth_paired, im_c)
        loss_tv = reference_tv(flow_list, warped_clothmask_paired, o["edgeawaretv"], o["add_lasttv"])
        n, _, ih, iw = c_paired.shape
        for i in range(len(flow_list) - 1):  # --interflowloss
            fh, fw = flow_list[i].shape[1], flow_list[i].shape[2]
            wc, wcm = autograd_tocg.FlowWarpNchwFn.apply(flow_list[i], c_paired, cm_paired, (ih, iw), ((fw - 1.0) / 2.0, (fh - 1.0) / 2.0))
            wcm = tr._remove_overlap(F.softmax(fake_segmap, dim=1), wcm)
            loss_l1 = loss_l1 + F.l1_loss(wcm, pcm) / (2 ** (4 - i))
            loss_vgg = loss_vgg + autograd_g.vgg_loss(tr.vgg, tr.vgg_weights, wc, im_c) / (2 ** (4 - i))
        ce = F.cross_entropy(fake_segmap, batch["parse_onehot"][:, 0].long(), ignore_index=250)
        out = {"l1": loss_l1, "vgg": loss_vgg, "ce": ce}
        if o["no_gan_loss"]:
            out["loss_g"] = (10 * loss_l1 + loss_vgg + o["tvlambda"] * loss_tv) + ce * o["ce_lambda"]
            return out
        soft = torch.softmax(fake_segmap, 1)
        loss_g_gan = tr._lsgan(autograd_tocg.tocg_discriminator_forward_train(tr.D, torch.cat((input1, input2, soft), 1)), True)
        pred_fake = autograd_tocg.tocg_discriminator_forward_train(tr.D, torch.cat((input1, input2, soft), 1))
        pred_real = autograd_tocg.tocg_discriminator_forward_train(tr.D, torch.cat((input1, input2, batch["parse"]), 1))
        out["loss_g"] = (10 * loss_l1 + loss_vgg + o["tvlambda"] * loss_tv) + (ce * o["ce_lambda"] + loss_g_gan * o["gan_lambda"])
        out["loss_d"] = tr._lsgan(pred_fake, False) + tr._lsgan(pred_real, True)
    return out


@pytest.mark.parametrize("name", list(OPTIONS))
def test_step_losses_match_restatement(name, monkeypatch):
    monkeypatch.setenv("HRV_VGG_RANDOM_INIT", "1")
    tr = _stage1_trainer(**OPTIONS[name])
    batch = train_step.synthetic_batch_stage1(2, 256, 192, "cuda", seed=2)
    with torch.random.fork_rng(devices=[torch.cuda.current_device()]):
        torch.cuda.manual_seed(11)
        ref = _restated_losses(tr, batch, OPTIONS[name])
    torch.cuda.manual_seed(11)
    out = tr.step(batch)
    torch.cuda.synchronize()
    assert sorted(out) == sorted(ref), (sorted(out), sorted(ref))
    # the same kernels on the same weights and draws: the TV's summation order (and F.cross_entropy's) are what differs
    for k in ref:
        assert abs(float(out[k]) - float(ref[k])) <= 2e-5 * abs(float(ref[k])) + 1e-7, (k, float(out[k]), float(ref[k]))


REPLAY = {
    "weighted_add_detach": ({"edgeawaretv": "weighted", "add_lasttv": True, "clothmask_composition": "detach"}, None),
    "last_only_no_composition_fp16scale": ({"edgeawaretv": "last_only", "clothmask_composition": "no_composition"}, "dynamic"),
    "no_gan": ({"no_gan_loss": True}, "dynamic"),
    "g_d_separate": ({"g_d_separate": True, "edgeawaretv": "weighted"}, None),
}


@pytest.mark.parametrize("name", list(REPLAY))
def test_graph_replays_equal_eager_steps(name, monkeypatch):
    monkeypatch.setenv("HRV_VGG_RANDOM_INIT", "1")
    opts, scale = REPLAY[name]
    batches = [train_step.synthetic_batch_stage1(2, 256, 192, "cuda", seed=s) for s in range(3)]
    tr = _stage1_trainer(loss_scale=scale, tensor_lr=True, **opts)
    d_before = {k: v.detach().clone() for k, v in tr.D.state_dict().items()}
    torch.cuda.manual_seed(7)
    tr.capture(batches[0], rollback=True)
    try:
        graph = [{k: v.clone() for k, v in tr.replay(b).items()} for b in batches[1:]]
        torch.cuda.synchronize()
        graph_state = _everything(tr)
    finally:
        tr.release_graph()
    if opts.get("no_gan_loss"):  # D, its Adam state and its loss scaler are never touched
        _assert_same(d_before, {k: v.detach() for k, v in tr.D.state_dict().items()})
        assert not any(tr.opt_d.state.get(p) for p in tr.D.parameters())
    del tr
    tr2 = _stage1_trainer(loss_scale=scale, tensor_lr=True, **opts)
    torch.cuda.manual_seed(7)
    eager = []
    for b in batches[1:]:
        ops.PARAM_GEN[0] += 1
        eager.append({k: v.clone() for k, v in tr2.step(b).items()})
    torch.cuda.synchronize()
    for i, (a, b) in enumerate(zip(graph, eager)):
        assert a.keys() == b.keys()
        assert [k for k in a if not torch.equal(a[k], b[k])] == [], i
    _assert_same(graph_state, _everything(tr2))


def test_no_gan_loss_leaves_d_alone(monkeypatch):
    monkeypatch.setenv("HRV_VGG_RANDOM_INIT", "1")
    tr = _stage1_trainer(no_gan_loss=True, loss_scale="dynamic")
    batch = train_step.synthetic_batch_stage1(2, 256, 192, "cuda", seed=4)
    d_before = {k: v.detach().clone() for k, v in tr.D.state_dict().items()}
    sc_before = {k: t.clone() for k, t in (("scale", tr.scalers["D"].scale), ("tracker", tr.scalers["D"].growth_tracker))}
    g_before = tr.tocg.flow_conv[4].weight.detach().clone()
    for _ in range(2):
        out = tr.step(batch)
    torch.cuda.synchronize()
    assert "loss_d" not in out and float((tr.tocg.flow_conv[4].weight.detach() - g_before).abs().max()) > 0
    _assert_same(d_before, {k: v.detach() for k, v in tr.D.state_dict().items()})
    assert not tr.opt_d.state and all(p.grad is None for p in tr.D.parameters())
    _assert_same(sc_before, {"scale": tr.scalers["D"].scale, "tracker": tr.scalers["D"].growth_tracker})


def test_g_d_separate_second_forward(monkeypatch):
    """The G update equals today's; the BatchNorm running statistics then equal today's step followed by one more train-mode forward
    with the updated weights; D's fake input is the soft-max of that forward's uncomposed segmentation."""
    monkeypatch.setenv("HRV_VGG_RANDOM_INIT", "1")
    batch = train_step.synthetic_batch_stage1(2, 256, 192, "cuda", seed=5)
    cm = (batch["cloth_mask"] > 0.5).float()
    input1, input2 = torch.cat([batch["cloth"], cm], 1), torch.cat([batch["parse_agnostic"], batch["densepose"]], 1)
    seen_d, seen_tocg = [], []
    fwd_d, fwd_tocg = autograd_tocg.tocg_discriminator_forward_train, autograd_tocg.tocg_forward_train

    def rec_d(D, x):
        seen_d.append(x.detach().clone())
        return fwd_d(D, x)

    def rec_tocg(m, a, b):
        out = fwd_tocg(m, a, b)
        seen_tocg.append([t.detach().clone() for t in out[1:]])
        return out
    sep = _stage1_trainer(g_d_separate=True)
    monkeypatch.setattr(autograd_tocg, "tocg_discriminator_forward_train", rec_d)
    monkeypatch.setattr(autograd_tocg, "tocg_forward_train", rec_tocg)
    torch.cuda.manual_seed(3)
    sep.step(batch)
    monkeypatch.undo()
    monkeypatch.setenv("HRV_VGG_RANDOM_INIT", "1")
    today = _stage1_trainer()
    torch.cuda.manual_seed(3)
    today.step(batch)
    params = lambda m: {k: v.detach().clone() for k, v in m.named_parameters()}
    buffers = lambda m: {k: v.detach().clone() for k, v in m.named_buffers()}
    _assert_same(params(sep.tocg), params(today.tocg))
    once = buffers(today.tocg)
    with torch.no_grad():
        autograd_tocg.tocg_forward_train(today.tocg, input1, input2)
    twice = buffers(today.tocg)
    _assert_same(buffers(sep.tocg), twice)
    assert any(not torch.equal(once[k], twice[k]) for k in once if "running_mean" in k)
    assert len(seen_tocg) == 2 and len(seen_d) == 3
    seg2, _, wcm2 = seen_tocg[1]
    fake_in = seen_d[1][:, -13:]
    assert torch.equal(fake_in, torch.softmax(seg2, 1))
    composed = seg2 * torch.cat([torch.ones_like(seg2[:, :3]), wcm2, torch.ones_like(seg2[:, 4:])], 1)
    assert not torch.equal(fake_in, torch.softmax(composed, 1))


def test_explicit_defaults_equal_todays_step(monkeypatch):
    monkeypatch.setenv("HRV_VGG_RANDOM_INIT", "1")
    batch = train_step.synthetic_batch_stage1(2, 256, 192, "cuda", seed=6)
    runs = []
    for kw in ({}, dict(train_loop.STAGE1_OPTIONS)):
        tr = _stage1_trainer(**kw)
        torch.cuda.manual_seed(5)
        outs = [{k: v.clone() for k, v in tr.step(batch).items()} for _ in range(2)]
        torch.cuda.synchronize()
        st = _everything(tr)
        st.update({"loss%d.%s" % (i, k): v for i, o in enumerate(outs) for k, v in o.items()})
        runs.append(st)
    _assert_same(*runs)


def test_weighted_run_resumes_bit_exact(tree):
    extra = ["--edgeawaretv", "weighted", "--add_lasttv"]
    full = _launch(tree, tree / "edge_full.pt", "stage1", _flags(tree, "stage1", "edge_full", False, extra))
    state = str(tree / "ckpt" / "edge_full" / "state_step_000004.pth")
    resumed = _launch(tree, tree / "edge_res.pt", "stage1", _flags(tree, "stage1", "edge_res", False, extra + ["--resume", state]))
    assert sorted(full["losses"]) == list(range(1, 7)) and sorted(resumed["losses"]) == [5, 6]
    for s in (5, 6):
        _assert_same(full["losses"][s], resumed["losses"][s])
    a, b = (_final_state(str(tree / "ckpt" / t)) for t in ("edge_full", "edge_res"))
    assert a["state_final.pth.config.edgeawaretv"] == "weighted" and a["state_final.pth.config.add_lasttv"] is True
    _assert_same(a, b)
