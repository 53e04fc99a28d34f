"""GPU: the stage-2 options of train_generator.py.

Kernels:
- hrv_parse_blur_argmax_cm (ops.parse_blur_argmax with cm) for 'warp_grad' and 'detach' is bit-identical to the torch composition
  followed by the cm-less kernel, with and without the occlusion plane, at 1024x768 and at an odd size; tryon_forward is bit-identical
  to its earlier formulation (the torch composition, restated here);
- hrv_onehot_u8_lut with the 13 -> 7 table is bit-identical to the reference's argmax -> scatter_ -> 7-group sum of the 13-plane map,
  and the loader's gen_parse equals those lines applied to the loader's own parse.
Stage2Trainer with each option: one eager step's losses against train_generator.py's own glue and loss blocks (read from the reference
copy under oracle/_ref and run as written on the trainer's networks); --no_vgg_loss never calls VGG; --no_ganFeat_loss leaves no feature
term; graph replays equal eager steps bit for bit; explicit defaults equal today's step.
Runs: a --GT --fp16 run without a tocg checkpoint resumes in a fresh process bit for bit; its LPIPS equals PerceptualLoss on
GeneratorGraph outputs; a 'detach' run evaluates through the 'detach' TryOnGraph."""
import os
import sys
import textwrap
import types

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
from hrviton_b200 import autograd_g, data, ops, pipeline, train_loop, train_step  # noqa: E402
from test_train_loop_gpu import (BATCH, N_TEST, SIZES, _assert_same, _everything, _final_state, _flags, _launch,  # noqa: E402,F401
                                 _stage2_trainer, tree)

pytestmark = pytest.mark.gpu
REF_SCRIPT = os.path.join(ROOT, "oracle", "_ref", "train_generator.py")
COMPOSITIONS = ("warp_grad", "detach")


def _regroup_reference(parse_13):
    """train_generator.py:250-273 on a 13-plane one-hot map: argmax -> scatter_ -> 7-group sum."""
    fake_parse = parse_13.argmax(dim=1)[:, None]
    n, _, h, w = parse_13.shape
    old_parse = torch.zeros(n, 13, h, w, device=parse_13.device).scatter_(1, fake_parse, 1.0)
    parse = torch.zeros(n, 7, h, w, device=parse_13.device)
    for i, grp in enumerate(train_step.LABELS7):
        for label in grp:
            parse[:, i] += old_parse[:, label]
    return parse


def _torch_composition(seg, cm, composition):
    """The composition the kernel replaces (train_generator.py:218-229)."""
    mask = torch.ones_like(seg)
    mask[:, 3:4] = (cm > 0.5).float() if composition == "detach" else cm
    return seg * mask


# ------------------------------------------------------------------------------------------------ kernels

@pytest.mark.parametrize("occlusion", [False, True], ids=["plain", "occlusion"])
@pytest.mark.parametrize("shape", [(2, 256, 192, 1024, 768), (3, 37, 29, 101, 77)], ids=["1024x768", "odd"])
@pytest.mark.parametrize("composition", COMPOSITIONS)
def test_parse_kernel_composition_bit_identical(composition, shape, occlusion):
    n, h, w, H, W = shape
    g = torch.Generator().manual_seed(h + w)
    seg = (torch.randn(n, 13, h, w, generator=g) * 3).cuda()
    cm = torch.rand(n, 1, h, w, generator=g)
    cm[:, :, ::5] = 0.5  # exactly at the threshold: not selected by 'detach'
    cm[:, :, 1::7] = 1.0
    cm = cm.cuda()
    kw = dict(group_of=train_step.GROUP_OF_13, groups=7, want_idx=True,
              overlap_classes=train_step.OCCLUSION_CLASSES if occlusion else None)
    want = ops.parse_blur_argmax(_torch_composition(seg, cm, composition), (H, W), **kw)
    got = ops.parse_blur_argmax(seg, (H, W), cm=cm, composition=composition, **kw)
    plain = ops.parse_blur_argmax(seg, (H, W), cm=cm, composition="no_composition", **kw)
    torch.cuda.synchronize()
    assert len(got) == len(want) == (3 if occlusion else 2)
    for a, b in zip(got, want):
        assert torch.equal(a, b)
    assert not torch.equal(plain[1], got[1])  # the composition changes the parse


@pytest.mark.parametrize("composition", ("warp_grad", "detach", "no_composition"))
def test_tryon_forward_equals_torch_composition(composition, monkeypatch):
    """tryon_forward against its earlier formulation: the composition in torch, then the cm-less parse kernel."""
    monkeypatch.setenv("HRV_VGG_RANDOM_INIT", "1")
    h, w = SIZES["stage2"]
    tr = _stage2_trainer(h, w)
    tocg, G = tr.tocg, tr.G.eval()
    b = train_step.synthetic_batch(2, h, w, "cuda", seed=3)

    def earlier(inputs):
        clothes, pre_cm = inputs["cloth"], (inputs["cloth_mask"] > 0.5).float()
        input1 = torch.cat([F.interpolate(clothes, size=(256, 192), mode="bilinear"), F.interpolate(pre_cm, size=(256, 192), mode="nearest")], 1)
        input2 = torch.cat([F.interpolate(inputs["parse_agnostic"], size=(256, 192), mode="nearest"),
                            F.interpolate(inputs["densepose"], size=(256, 192), mode="bilinear")], 1)
        flow_list, fake_segmap, _, warped_cm = tocg(input1, input2)
        if composition != "no_composition":
            cm = (warped_cm > 0.5).float() if composition == "detach" else warped_cm
            fake_segmap = torch.cat([fake_segmap[:, :3], fake_segmap[:, 3:4] * cm, fake_segmap[:, 4:]], 1)
        _, parse, overlap = ops.parse_blur_argmax(fake_segmap.float(), (h, w), group_of=train_step.GROUP_OF_13, groups=7, want_idx=False,
                                                  overlap_classes=train_step.OCCLUSION_CLASSES)
        div = ((96 - 1.0) / 2.0, (128 - 1.0) / 2.0)
        warped_cloth, _, _ = ops.flow_warp_nchw(flow_list[-1], clothes.float(), (h, w), div, mask=pre_cm, overlap=overlap, composite=True)
        return G(torch.cat((inputs["agnostic"], inputs["densepose"], warped_cloth), 1), parse), warped_cloth, parse
    outs = []
    for fn in (earlier, lambda i: pipeline.tryon_forward(tocg, G, i, clothmask_composition=composition)):
        torch.cuda.manual_seed(21)
        with torch.no_grad():
            outs.append([t.clone() for t in fn(b)])
    torch.cuda.synchronize()
    for a, c in zip(*outs):
        assert torch.equal(a, c)


def test_onehot_lut_equals_reference_regroup():
    g = torch.Generator().manual_seed(5)
    for n, h, w in ((2, 1024, 768), (3, 37, 29)):
        lab = torch.randint(0, 13, (n, 1, h, w), dtype=torch.uint8, generator=g).cuda()
        parse_13 = torch.zeros(n, 13, h, w, device="cuda").scatter_(1, lab.long(), 1.0)
        got = ops.onehot_u8(lab, 7, lut=train_step.GROUP_OF_13)
        assert torch.equal(got, _regroup_reference(parse_13))
        assert torch.equal(ops.onehot_u8(lab, 13), parse_13)  # no table: today's identity


def test_loader_gen_parse_equals_regrouped_parse(tree):
    h, w = SIZES["stage2"]
    loader = data.VitonHDLoader(str(tree), "train", "pairs.txt", h, w, BATCH, workers=1, keys=("parse", "gen_parse"), shuffle=False)
    try:
        for _ in range(2):
            b = loader.next_batch()
            torch.cuda.synchronize()
            assert torch.equal(b["gen_parse"], _regroup_reference(b["parse"]))
            assert int(b["gen_parse"].sum()) == BATCH * h * w
    finally:
        loader.close()
    # a CPU-fed batch takes the byte path for gen_parse too
    feeder = train_step.BatchFeeder({"gen_parse": b["gen_parse"].cpu()}, torch.device("cuda"))
    assert feeder.classes == {"gen_parse": 7}
    feeder.prefetch()
    out = feeder.consume({"gen_parse": torch.empty_like(b["gen_parse"])})
    torch.cuda.synchronize()
    assert torch.equal(out["gen_parse"], b["gen_parse"])


# ------------------------------------------------------------------------------------------------ the step

def _reference_blocks():
    """train_generator.py as written: remove_overlap, the glue (`with torch.no_grad():` before `if not opt.GT:` to `parse =
    parse.detach()`) and the generator's losses (`output_paired = generator(` to `loss_gen = sum(...)`)."""
    if not os.path.isfile(REF_SCRIPT):
        pytest.skip("no reference copy (oracle/_ref)")
    lines = open(REF_SCRIPT).read().splitlines()
    a = next(i for i, l in enumerate(lines) if l.startswith("def remove_overlap"))
    b = next(i for i, l in enumerate(lines) if i > a and l.startswith("def "))
    g0 = next(i for i, l in enumerate(lines) if l.strip() == "if not opt.GT:" and lines[i - 1].strip() == "with torch.no_grad():") - 1
    g1 = next(i for i, l in enumerate(lines) if i > g0 and l.strip() == "parse = parse.detach()")
    l0 = next(i for i, l in enumerate(lines) if i > g1 and l.strip().startswith("output_paired = generator("))
    l1 = next(i for i, l in enumerate(lines) if i > l0 and l.strip().startswith("loss_gen = sum("))
    src = lambda x, y: compile(textwrap.dedent("\n".join(lines[x:y + 1])), REF_SCRIPT, "exec")
    return src(a, b - 1), src(g0, g1), src(l0, l1)


def _reference_losses(tr, batch, o, h, w):
    """The reference's G losses for the options `o` on the trainer's networks and batch (GAN, GAN_Feat, VGG as present)."""
    import numpy
    import network_generator
    from hrviton_b200.tocg import make_grid
    fns, glue, losses = _reference_blocks()
    opt = types.SimpleNamespace(GT=o["gt"], clothmask_composition=o["clothmask_composition"], occlusion=tr.occlusion, fine_height=h,
                                fine_width=w, no_ganFeat_loss=o["no_ganFeat_loss"], no_vgg_loss=o["no_vgg_loss"],
                                lambda_feat=o["lambda_feat"], lambda_vgg=o["lambda_vgg"], gpu_ids=[0])
    scope = {"torch": torch, "F": F, "np": types.SimpleNamespace(float=numpy.float64), "opt": opt, "make_grid": make_grid,
             "gauss": train_step.gaussian_blur_15_3, "tocg": tr.tocg, "generator": tr.G,
             "discriminator": lambda x: autograd_g.discriminator_forward_train(tr.D, x, need_wgrad=False, as_float=True),
             "criterionGAN": network_generator.GANLoss("hinge"), "criterionFeat": torch.nn.L1Loss(),
             "criterionVGG": lambda x, y: autograd_g.vgg_loss(tr.vgg, tr.vgg_weights, x, y),
             "agnostic": batch["agnostic"], "pose": batch["densepose"], "im": batch["image"], "parse_GT": batch.get("parse"),
             "parse_cloth": batch.get("parse_cloth"), "parse_agnostic": batch.get("parse_agnostic"), "cm": batch.get("cloth_mask"),
             "c_paired": batch.get("cloth")}
    exec(fns, scope)
    with torch.no_grad():
        exec(glue, scope)
        exec(losses, scope)
    return scope["G_losses"], scope["loss_gen"]


OPTIONS = {
    "default": {},
    "gt": {"gt": True},
    "detach": {"clothmask_composition": "detach"},
    "no_composition": {"clothmask_composition": "no_composition"},
    "no_vgg": {"no_vgg_loss": True},
    "no_ganfeat": {"no_ganFeat_loss": True},
    "lambdas": {"lambda_feat": 5.0, "lambda_vgg": 2.0},
}


def _trainer(h, w, o, **kw):
    """_stage2_trainer with the options `o` (keys of STAGE2_OPTIONS; no_ganFeat_loss on D, as build() sets it)."""
    o = dict(o)
    no_feat = o.pop("no_ganFeat_loss", False)
    tr = _stage2_trainer(h, w, occlusion=not o.get("gt", False), **o, **kw)
    tr.D.no_ganFeat_loss = no_feat
    for d in tr.D.children():
        d.no_ganFeat_loss = no_feat
    if o.get("gt"):
        tr.tocg = None
    if o.get("no_vgg_loss"):
        tr.vgg = None
    return tr


def _batch(h, w, gt, seed):
    if not gt:
        return train_step.synthetic_batch(BATCH, h, w, "cuda", seed=seed)
    return train_step.synthetic_batch_gt(BATCH, h, w, "cuda", seed=seed)


@pytest.mark.parametrize("name", list(OPTIONS))
def test_step_losses_match_reference_blocks(name, monkeypatch):
    monkeypatch.setenv("HRV_VGG_RANDOM_INIT", "1")
    h, w = SIZES["stage2"]
    o = dict(train_loop.STAGE2_OPTIONS, **OPTIONS[name])
    tr = _trainer(h, w, OPTIONS[name])
    batch = _batch(h, w, o["gt"], seed=2)
    ref_batch = dict(batch)
    if o["gt"]:  # the reference reads the 13-plane map the loader's gen_parse is made of
        ref_batch["parse"] = train_step.synthetic_batch_stage1(BATCH, h, w, "cuda", seed=2)["parse"]
    saved = [(m, {k: v.clone() for k, v in m.state_dict().items()}) for m in (tr.G, tr.D)]
    with torch.random.fork_rng(devices=[torch.cuda.current_device()]):
        torch.cuda.manual_seed(11)
        ref, ref_gen = _reference_losses(tr, ref_batch, o, h, w)
    for m, sd in saved:  # the train-mode forwards moved the spectral-norm vectors: the step starts from the same state
        m.load_state_dict(sd)
    ops.PARAM_GEN[0] += 1
    torch.cuda.manual_seed(11)
    out = tr.step(batch, h, w)
    torch.cuda.synchronize()
    names = {"GAN": "gan", "GAN_Feat": "feat", "VGG": "vgg"}
    assert sorted(k for k in out if k not in ("loss_gen", "loss_dis")) == sorted(names[k] for k in ref)
    # the reference's glue is torch's resize / blur / argmax (a few parse pixels flip against the kernel) and its D runs without the
    # feature buffers' fused layout: the tolerances of the stage-2 oracle parity test
    gan, gan_r = float(out["gan"]), float(ref["GAN"])
    assert abs(gan - gan_r) < 0.05 + 0.05 * abs(gan_r), (gan, gan_r)
    if "GAN_Feat" in ref:
        assert abs(float(out["feat"]) - float(ref["GAN_Feat"])) < 0.05 * abs(float(ref["GAN_Feat"])) + 0.02
    if "VGG" in ref:
        assert abs(float(out["vgg"]) - float(ref["VGG"])) < 0.05 * abs(float(ref["VGG"])) + 0.01
    assert abs(float(out["loss_gen"]) - float(ref_gen)) < 0.05 * abs(float(ref_gen)) + 0.05


def test_disabled_terms_are_not_computed(monkeypatch):
    monkeypatch.setenv("HRV_VGG_RANDOM_INIT", "1")
    h, w = SIZES["stage2"]

    def no_vgg(*a, **k):
        raise AssertionError("VGG called under no_vgg_loss")
    tr = _trainer(h, w, {"no_vgg_loss": True, "no_ganFeat_loss": True})
    monkeypatch.setattr(autograd_g, "vgg_loss", no_vgg)
    feats = []
    monkeypatch.setattr(autograd_g.FeatMatchFn, "apply", lambda *a: feats.append(1))
    out = tr.step(_batch(h, w, False, seed=3), h, w)
    torch.cuda.synchronize()
    assert sorted(out) == ["gan", "loss_dis", "loss_gen"] and feats == []
    assert torch.equal(out["loss_gen"], out["gan"].mean())


REPLAY = {
    "gt_fp16scale": ({"gt": True}, "dynamic"),
    "detach": ({"clothmask_composition": "detach"}, None),
    "no_composition_no_vgg": ({"clothmask_composition": "no_composition", "no_vgg_loss": True}, None),
    "no_ganfeat_fp16scale": ({"no_ganFeat_loss": True, "lambda_vgg": 2.0}, "dynamic"),
}


@pytest.mark.parametrize("name", list(REPLAY))
def test_graph_replays_equal_eager_steps(name, monkeypatch):
    monkeypatch.setenv("HRV_VGG_RANDOM_INIT", "1")
    h, w = SIZES["stage2"]
    opts, scale = REPLAY[name]
    batches = [_batch(h, w, opts.get("gt", False), seed=s) for s in range(3)]
    tr = _trainer(h, w, opts, loss_scale=scale, tensor_lr=True)
    torch.cuda.manual_seed(7)
    tr.capture(batches[0], h, w, rollback=True)
    try:
        graph = [{k: v.clone() for k, v in tr.replay(b).items()} for b in batches[1:]]
        torch.cuda.synchronize()
        graph_state = _everything(tr)
    finally:
        tr.release_graph()
    del tr
    tr2 = _trainer(h, w, opts, loss_scale=scale, tensor_lr=True)
    torch.cuda.manual_seed(7)
    eager = []
    for b in batches[1:]:
        ops.PARAM_GEN[0] += 1
        eager.append({k: v.clone() for k, v in tr2.step(b, h, w).items()})
    torch.cuda.synchronize()
    for i, (a, b) in enumerate(zip(graph, eager)):
        assert a.keys() == b.keys()
        assert [k for k in a if not torch.equal(a[k], b[k])] == [], i
    _assert_same(graph_state, _everything(tr2))


def test_explicit_defaults_equal_todays_step(monkeypatch):
    monkeypatch.setenv("HRV_VGG_RANDOM_INIT", "1")
    h, w = SIZES["stage2"]
    batch = _batch(h, w, False, seed=6)
    runs = []
    for kw in ({}, {k: v for k, v in train_loop.STAGE2_OPTIONS.items() if k != "no_ganFeat_loss"}):
        tr = _stage2_trainer(h, w, **kw)
        torch.cuda.manual_seed(5)
        outs = []
        for _ in range(2):
            ops.PARAM_GEN[0] += 1
            outs.append({k: v.clone() for k, v in tr.step(batch, h, w).items()})
        torch.cuda.synchronize()
        assert sorted(outs[0]) == ["feat", "gan", "loss_dis", "loss_gen", "vgg"]
        st = _everything(tr)
        st.update({"loss%d.%s" % (i, k): v for i, o in enumerate(outs) for k, v in o.items()})
        runs.append(st)
    _assert_same(*runs)


# ------------------------------------------------------------------------------------------------ runs

def _gt_flags(tree, name, extra=()):
    """The stage-2 flags of test_train_loop_gpu without what a --GT run refuses (--occlusion, --tocg_checkpoint)."""
    f = _flags(tree, "stage2", name, True, ["--GT"] + list(extra))
    i = f.index("--tocg_checkpoint")
    del f[i:i + 2]
    f.remove("--occlusion")
    return f


def test_gt_fp16_run_resumes_bit_exact(tree):
    full = _launch(tree, tree / "gt_full.pt", "stage2", _gt_flags(tree, "gt_full"))
    state = str(tree / "ckpt" / "gt_full" / "state_step_000002.pth")
    resumed = _launch(tree, tree / "gt_res.pt", "stage2", _gt_flags(tree, "gt_res", ["--resume", state]))
    assert sorted(full["losses"]) == list(range(1, 7)) and sorted(resumed["losses"]) == [3, 4, 5, 6]
    for s in range(3, 7):
        _assert_same(full["losses"][s], resumed["losses"][s])
    a, b = (_final_state(str(tree / "ckpt" / t)) for t in ("gt_full", "gt_res"))
    assert a["state_final.pth.config.gt"] is True and "state_final.pth.config.tocg_sha256" not in a
    assert any(n.endswith("scalers.G.scale") for n in a)
    _assert_same(a, b)


def _lpips_run(tree, monkeypatch, opts, keys):
    import eval_models
    monkeypatch.setenv("HRV_VGG_RANDOM_INIT", "1")
    monkeypatch.setenv("HRV_ALEX_RANDOM_INIT", "1")
    monkeypatch.chdir(str(tree))
    h, w = SIZES["stage2"]
    tr = _trainer(h, w, opts, tensor_lr=True)
    loader_keys = train_step.GT_KEYS if opts.get("gt") else data.STAGE2_KEYS
    loader = data.VitonHDLoader(str(tree), "train", "pairs.txt", h, w, BATCH, workers=1, keys=loader_keys)
    test_loader = data.VitonHDLoader(str(tree), "test", "test_pairs.txt", h, w, 1, workers=1, mode="test", keys=keys, shuffle=False, shard=False)
    model = eval_models.PerceptualLoss(model="net-lin", net="alex", use_gpu=True)
    run = train_loop.TrainRun("stage2", tr, loader, str(tree / "lp2"), keep_step=1, decay_step=1, lpips_count=1,
                              evaluator=(test_loader, model), lpips_samples=N_TEST)
    return run, tr, test_loader, model


def test_gt_lpips_equals_perceptual_loss_on_generator_graph(tree, monkeypatch):
    from torchvision.transforms import transforms
    run, tr, test_loader, model = _lpips_run(tree, monkeypatch, {"gt": True}, train_loop.EVAL_GT_KEYS)
    try:
        value = run.evaluate()
        assert isinstance(run._tryon, pipeline.GeneratorGraph)
    finally:
        run._tryon.release()
    T2 = transforms.Compose([transforms.Resize((128, 128))])
    runner = pipeline.GeneratorGraph(tr.G)
    tr.G.eval()
    try:
        with torch.random.fork_rng(devices=[test_loader.device]), torch.no_grad():
            test_loader.start_at(0, 0)
            avg = 0.0
            for _ in range(N_TEST):
                b = test_loader.next_batch()
                out = runner(torch.cat((b["agnostic"], b["densepose"], b["parse_cloth"]), 1), b["gen_parse"])
                avg += model.forward(T2(b["image"]), T2(out))
            avg = avg / N_TEST
    finally:
        tr.G.train()
        runner.release()
    assert value == float(avg) and value > 0


def test_detach_run_evaluates_through_detach_tryon(tree, monkeypatch):
    from torchvision.transforms import transforms
    run, tr, test_loader, model = _lpips_run(tree, monkeypatch, {"clothmask_composition": "detach"}, train_loop.EVAL_KEYS)
    try:
        value = run.evaluate()
        assert isinstance(run._tryon, pipeline.TryOnGraph) and run._tryon.clothmask_composition == "detach"
    finally:
        run._tryon.release()
    T2 = transforms.Compose([transforms.Resize((128, 128))])
    runner = pipeline.TryOnGraph(tr.tocg, tr.G, occlusion=tr.occlusion, clothmask_composition="detach")
    tr.G.eval()
    try:
        with torch.random.fork_rng(devices=[test_loader.device]), torch.no_grad():
            test_loader.start_at(0, 0)
            avg = 0.0
            for _ in range(N_TEST):
                b = test_loader.next_batch()
                out = runner({k: b[k] for k in train_loop.EVAL_KEYS if k != "image"})[0]
                avg += model.forward(T2(b["image"]), T2(out))
            avg = avg / N_TEST
    finally:
        tr.G.train()
        runner.release()
    assert value == float(avg) and value > 0
