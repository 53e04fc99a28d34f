"""GPU: discriminator rejection (pipeline.rejection_scores / norm_constant / ConditionGraph / TryOnGraph(discriminator=)).

The fused kernel hrv_seg_softmax_cat is checked per element: copied channels are the round-to-nearest of their fp32 source bit for
bit, soft-max channels lie within u*|ref| + 64 * 2^-24 of an fp64 soft-max of the same composed scores (u = 2^-8 bf16, 2^-11 fp16,
0 with fp32 storage), and the written channel set is hrv_nchw_to_nhwc's.  The scores are held to the storage-rounding floor of the
oracle's rejection() against reject_256x192_b4.npz, and in fp32 to |dl| < 1e-3, |dscore| <= 1e-3 / ((1 - l)^2 M)."""
import contextlib
import functools
import io
import os
import sys
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import floors  # noqa: E402
import hrv_env  # noqa: E402
import rejection_oracle as rorc  # noqa: E402
from floors import orc  # noqa: E402
from helpers import gen_opt, load_golden, synth_state_dict, tocg_opt  # noqa: E402
from hrviton_b200 import ops, pipeline, synth, train_step  # noqa: E402
from hrviton_b200.ops import Act  # noqa: E402
from test_rejection_cpu import NAME, TOL_L, reject_case, score_bound  # noqa: E402

pytestmark = pytest.mark.gpu
U = {"bf16": 2.0 ** -8, "fp16": 2.0 ** -11, "fp32": 0.0}
SOFTMAX_ABS = 64 * 2.0 ** -24
SENTINEL = {torch.bfloat16: (torch.int16, 0x7FC1), torch.float16: (torch.int16, 0x7E01), torch.float32: (torch.int32, 0x7FC00123)}


@pytest.fixture(params=["bf16", "fp16"])
def precision(request):
    ops.set_precision(request.param)
    yield request.param
    ops.set_precision("bf16")


@pytest.fixture(params=["bf16", "fp16", "fp32"])
def storage(request):
    ops.set_precision(request.param)
    yield request.param
    ops.set_precision("bf16")


@pytest.fixture(autouse=True)
def _restore():
    yield
    ops.set_precision("bf16")


def _discriminator(sd):
    import networks
    with contextlib.redirect_stdout(io.StringIO()):
        D = networks.define_D(input_nc=33, Ddownx2=True, Ddropout=True, n_layers_D=3, spectral=False, num_D=2)
    D.load_state_dict(sd)
    return D.cuda().eval()


@pytest.fixture(scope="module")
def case():
    """The fixture's networks on the GPU, its batch as a cp_dataset dict at the tocg resolution, and the golden."""
    import networks
    g, sd_t, sd_d, i1, i2, label = reject_case()
    tocg = networks.ConditionGenerator(tocg_opt(True), 4, 16, 13, ngf=96, norm_layer=torch.nn.BatchNorm2d)
    tocg.load_state_dict(sd_t)
    batch = {"cloth": i1[:, :3].cuda(), "cloth_mask": i1[:, 3:4].cuda(), "parse_agnostic": i2[:, :13].cuda(), "densepose": i2[:, 13:].cuda(),
             "parse": label.cuda()}
    return types.SimpleNamespace(g=g, M=float(g["M"]), composition=str(g["composition"]), tocg=tocg.cuda().eval(), D=_discriminator(sd_d),
                                 batch=batch, sd_d=sd_d)


def _sub(batch, lo, hi):
    return {k: v[lo:hi].contiguous() for k, v in batch.items()}


# ------------------------------------------------------------------------------------------------ the kernel, per element


def _compose(seg, cm, mode, ch):
    if mode == "no_composition":
        return seg
    m = (cm > 0.5).float() if mode == "detach" else cm
    return torch.cat([seg[:, :ch], seg[:, ch:ch + 1] * m, seg[:, ch + 1:]], 1)


@pytest.mark.parametrize("softmax", [True, False])
@pytest.mark.parametrize("mode", ["no_composition", "warp_grad", "detach"])
@pytest.mark.parametrize("c1,c2,k,n,h,w", [(4, 16, 13, 2, 17, 13), (3, 2, 7, 1, 9, 11), (4, 16, 13, 1, 256, 192)])
def test_seg_softmax_cat_per_element(storage, c1, c2, k, n, h, w, mode, softmax):
    """Odd extents, K = 13 and 7, c1 + c2 = 5 (not a multiple of 8), scores over +-30 (a pixel's terms span e^-60 .. 1
    after the maximum is subtracted), cm with values on both sides of and exactly at 0.5."""
    dt = ops.STORAGE[0]
    in1 = synth.uniform((n, c1, h, w), 3, "in1", -2.0, 2.0).cuda()
    in2 = synth.uniform((n, c2, h, w), 3, "in2", -1.0, 1.0).cuda()
    seg = synth.uniform((n, k, h, w), 3, "seg", -30.0, 30.0).cuda()
    cm = synth.uniform((n, 1, h, w), 3, "cm", 0.0, 1.0)
    cm.view(-1)[::7] = 0.5
    cm = cm.cuda()
    ch = 3
    c, pitch = c1 + c2 + k, ops.round_up(c1 + c2 + k, 8) + 8
    it, bits = SENTINEL[dt]
    buf = torch.full((n, h, w, pitch), bits, dtype=it, device="cuda").view(dt)
    out, seg_out = ops.seg_softmax_cat(in1, in2, seg, cm=None if mode == "no_composition" else cm, cm_channel=ch, composition=mode,
                                       softmax=softmax, want_seg=True, out=Act(buf, c=c))
    composed = _compose(seg, cm, mode, ch)
    assert torch.equal(seg_out, composed)
    nhwc = lambda t: t.permute(0, 2, 3, 1)
    assert torch.equal(buf[..., :c1 + c2].contiguous().view(it), nhwc(torch.cat([in1, in2], 1)).to(dt).contiguous().view(it))
    third = buf[..., c1 + c2:c]
    if not softmax:
        assert torch.equal(third.contiguous().view(it), nhwc(composed).to(dt).contiguous().view(it))
    else:
        ref = torch.softmax(nhwc(composed).double().cpu(), -1)
        err = (third.double().cpu() - ref).abs()
        bound = U[storage] * ref + SOFTMAX_ABS
        worst = float((err / bound).max())
        print("FWDBOUND seg_softmax_cat %s %s k=%d %dx%d worst = %.3f of its bound" % (storage, mode, k, h, w, worst))
        assert worst <= 1.0
        assert float((third.double().sum(-1).cpu() - 1).abs().max()) <= k * (U[storage] + SOFTMAX_ABS)
    # the written set: what hrv_nchw_to_nhwc writes for a c-channel destination of this pitch — channels [0, roundup8(c)), pad zeroed
    buf2 = torch.full((n, h, w, pitch), bits, dtype=it, device="cuda").view(dt)
    ops.from_nchw(torch.cat([in1, in2, composed], 1), out=Act(buf2, c=c))
    assert torch.equal(buf.view(it) == bits, buf2.view(it) == bits)  # the same elements still hold the sentinel
    assert torch.equal(buf[..., c:].contiguous().view(it), buf2[..., c:].contiguous().view(it))  # zeroed pad of the last group


def test_seg_softmax_cat_refuses_bad_arguments():
    t = lambda c, **kw: torch.zeros(1, c, 8, 6, device="cuda", **kw)
    with pytest.raises(ValueError, match="one \\(N,H,W\\)"):
        ops.seg_softmax_cat(t(4), t(16), torch.zeros(1, 13, 8, 5, device="cuda"))
    with pytest.raises(ValueError, match="float32"):
        ops.seg_softmax_cat(t(4), t(16), t(13, dtype=torch.float16))
    with pytest.raises(ValueError, match="cm must be"):
        ops.seg_softmax_cat(t(4), t(16), t(13), cm=t(2))
    with pytest.raises(RuntimeError, match="cm_channel"):
        ops.seg_softmax_cat(t(4), t(16), t(13), cm=t(1), cm_channel=13)
    with pytest.raises(RuntimeError, match="channels"):
        ops.seg_softmax_cat(t(4), t(16), t(13), out=Act.empty(1, 8, 6, 32))


# ------------------------------------------------------------------------------------------------ the discriminator on an Act


def test_discriminator_on_fused_input_matches_nchw_path(precision):
    name = "tocgd_256x192_b1"
    g = load_golden(name)
    seed = int(g["seed"])
    D = _discriminator(synth_state_dict("tocgd", seed))
    i1, i2 = (t.cuda() for t in synth.tocg_inputs(1, 256, 192, seed))
    segs = synth.one_hot(synth.labels((1, 256, 192), 13, seed, "dseg"), 13).cuda()
    res = D.forward_act(ops.seg_softmax_cat(i1, i2, segs, softmax=False))
    with torch.no_grad():
        nchw = D(torch.cat([i1, i2, segs], 1))
    fl = floors.tocgd_floor(name, precision)
    for i, r in enumerate(res):
        floors.check("%s tocgd fused d%d" % (precision, i), r[0], g["d%d" % i], fl["d%d" % i])
        assert torch.equal(r[0], nchw[i][0])  # a copy of the same 33 channels: the same Act, the same result


# ------------------------------------------------------------------------------------------------ scores


@functools.lru_cache(maxsize=None)
def rejection_floor(name, precision):
    """What 16-bit storage costs the oracle's rejection() (tocg and discriminator chained) on the fixture, per logit map."""
    g, sd_t, sd_d, i1, i2, label = reject_case()
    with torch.no_grad(), orc.storage_rounding(floors.DT[precision]):
        _, _, maps = rorc.rejection(sd_t, sd_d, i1, i2, float(g["M"]), str(g["composition"]))
    return {"fake_d%d" % i: floors.stats(m, g["fake_d%d" % i]) for i, m in enumerate(maps)}


def _ulps(got, ref64):
    ref32 = ref64.astype(np.float32)
    return np.abs(got.astype(np.float64) - ref64) / np.spacing(np.abs(ref32)).astype(np.float64)


def _scores_and_maps(case):
    score, l, outs = pipeline.rejection_scores(case.tocg, case.D, case.batch, case.M, clothmask_composition=case.composition)
    input1 = torch.cat([case.batch["cloth"], (case.batch["cloth_mask"] > 0.5).float()], 1)
    input2 = torch.cat([case.batch["parse_agnostic"], case.batch["densepose"]], 1)
    l2, maps = pipeline.condition_logit(case.D, input1, input2, outs[1], cm=outs[3], composition=case.composition, return_maps=True)
    assert torch.equal(l, l2)
    return score.cpu().numpy(), l.cpu().numpy(), [m.cpu().numpy() for m in maps]


def _check_own_arithmetic(score, l, maps, M):
    """l is the fp32 D_logit of the call's own maps: the map values have mixed signs, so its error is measured against S = the same
    formula on |map|, at most 64 * 2^-24 * S as for every other fp32 sum of the package (measured: below 2^-24 * S, about 2 ulp of l).
    score is the fp32 l / (1 - l) / M of the call's own l: four roundings (1 - l, the quotient, the reciprocal of the scalar M that
    torch multiplies by, the product), each between half an ulp and one ulp of the result depending on where it sits in its
    binade: 4 ulp."""
    l_ref = sum(m.astype(np.float64).mean((1, 2, 3)) for m in maps) / 2
    S = sum(np.abs(m.astype(np.float64)).mean((1, 2, 3)) for m in maps) / 2
    r = np.abs(l.astype(np.float64) - l_ref) / (2.0 ** -24 * S)
    print("REJECT l error %s x 2^-24 S" % r)
    assert r.max() <= 64.0, r
    s_ref = l.astype(np.float64) / (1 - l.astype(np.float64)) / M
    assert _ulps(score, s_ref).max() <= 4.0, _ulps(score, s_ref)


def test_rejection_scores_within_storage_floor(case, precision):
    score, l, maps = _scores_and_maps(case)
    fl = rejection_floor(NAME, precision)
    assert [m.shape[0] * m.shape[2] * m.shape[3] for m in maps] == [1140, 396]
    for i, m in enumerate(maps):
        floors.check("%s reject fake_d%d" % (precision, i), m, case.g["fake_d%d" % i], fl["fake_d%d" % i])
    _check_own_arithmetic(score, l, maps, case.M)
    print("REJECT %s l %s (golden %s) score %s (golden %s)" % (precision, l, case.g["l_fake"], score, case.g["score"]))


def test_rejection_scores_fp32_meet_reference_tolerance(case):
    ops.set_precision("fp32")
    score, l, maps = _scores_and_maps(case)
    _check_own_arithmetic(score, l, maps, case.M)
    dl = np.abs(l - case.g["l_fake"])
    ds = np.abs(score - case.g["score"])
    print("REJECT fp32 |dl| %s  |dscore| / bound %s" % (dl, ds / score_bound(case.g["l_fake"], case.M)))
    assert dl.max() < TOL_L and (ds <= score_bound(case.g["l_fake"], case.M)).all()
    for i, m in enumerate(maps):
        assert float(np.abs(m - case.g["fake_d%d" % i]).max()) < TOL_L


@pytest.mark.parametrize("composition", ["no_composition", "detach"])
def test_rejection_scores_other_compositions_fp32(case, composition):
    """'detach' thresholds the warped mask on the device, 'no_composition' passes the scores through: each against the oracle."""
    ops.set_precision("fp32")
    g, sd_t, sd_d, i1, i2, label = reject_case()
    score, l, _ = pipeline.rejection_scores(case.tocg, case.D, case.batch, case.M, clothmask_composition=composition)
    with torch.no_grad():
        s_ref, l_ref, _ = rorc.rejection(sd_t, sd_d, i1, i2, case.M, composition)
    assert float((l.cpu() - l_ref).abs().max()) < TOL_L
    assert (np.abs(score.cpu().numpy() - s_ref.numpy()) <= score_bound(l_ref.numpy(), case.M)).all()


def test_norm_constant_is_the_running_maximum_without_synchronisation(case, precision):
    b = [_sub(case.batch, 0, 2), _sub(case.batch, 2, 4)]
    want = []
    for x in b:
        _, l_fake, outs = pipeline.rejection_scores(case.tocg, case.D, x, 1.0, clothmask_composition=case.composition)
        input1 = torch.cat([x["cloth"], (x["cloth_mask"] > 0.5).float()], 1)
        input2 = torch.cat([x["parse_agnostic"], x["densepose"]], 1)
        l_real = pipeline.condition_logit(case.D, input1, input2, x["parse"], softmax=False)
        want += [l_real / (1 - l_real), l_fake / (1 - l_fake)]
    want = float(torch.cat(want).max())
    assert pipeline.norm_constant(case.tocg, case.D, b, clothmask_composition=case.composition) == want

    def guarded():
        """A synchronisation while the batches are being consumed raises; the guard is lifted when the loop is done, before the
        one read of the result."""
        torch.cuda.set_sync_debug_mode("error")
        try:
            yield from b
        finally:
            torch.cuda.set_sync_debug_mode("default")

    try:
        assert pipeline.norm_constant(case.tocg, case.D, guarded(), clothmask_composition=case.composition) == want
    finally:
        torch.cuda.set_sync_debug_mode("default")
    if precision == "bf16":
        print("REJECT norm_constant %s over 2 batches of 2: %.6f (golden M, fp32 reference, one batch of 4: %.6f)" % (precision, want, case.M))


# ------------------------------------------------------------------------------------------------ graph runners


def _flat(out):
    score, l, (flows, seg, wc, wcm) = out
    return [score, l, seg, wc, wcm] + list(flows)


def _clone(out):
    return [t.clone() for t in _flat(out)]


def _assert_equal(got, ref):
    assert len(got) == len(ref)
    for i, (a, b) in enumerate(zip(got, ref)):
        assert torch.equal(a, b), "output %d: max|d| %.3e" % (i, float((a.float() - b.float()).abs().max()))


@pytest.mark.parametrize("n", [1, 4])
def test_condition_graph_equals_eager(case, precision, n):
    runner = pipeline.ConditionGraph(case.tocg, case.D, case.M, clothmask_composition=case.composition)
    try:
        for lo in (0, 4 - n):  # captured on the first call, replayed with other inputs on the second
            x = _sub(case.batch, lo, lo + n)
            ref = _clone(pipeline.rejection_scores(case.tocg, case.D, x, case.M, clothmask_composition=case.composition))
            _assert_equal(_flat(runner(x)), ref)
            d = dict(x, cloth={"paired": x["cloth"]}, cloth_mask={"paired": x["cloth_mask"]})
            _assert_equal(_flat(runner(d)), ref)
        assert len(runner._graphs) == 1
    finally:
        runner.release()


@pytest.mark.parametrize("kind", ["d_load_state_dict", "tocg_bn_stats", "precision"])
def test_condition_graph_recaptures_changed_weights(case, kind):
    runner = pipeline.ConditionGraph(case.tocg, case.D, case.M, clothmask_composition=case.composition)
    x = _sub(case.batch, 0, 1)
    undo = lambda: None
    try:
        runner(x)
        (old,) = [e.captured for e in runner._graphs.values()]
        if kind == "precision":
            ops.set_precision("fp16")
        elif kind == "d_load_state_dict":
            saved = {k: v.clone() for k, v in case.D.state_dict().items()}
            case.D.load_state_dict({k: v * 1.25 for k, v in saved.items()})
            undo = lambda: case.D.load_state_dict(saved)
        else:
            edited = [m.running_var for m in case.tocg.modules() if isinstance(m, torch.nn.BatchNorm2d)]
            saved = [t.detach().clone() for t in edited]
            with torch.no_grad():
                for t in edited:
                    t.mul_(1.5)

            def undo():
                with torch.no_grad():
                    for t, s in zip(edited, saved):
                        t.copy_(s)
        ref = _clone(pipeline.rejection_scores(case.tocg, case.D, x, case.M, clothmask_composition=case.composition))
        if kind != "d_load_state_dict":
            # what a graph that ignored the change would return.  (The discriminator's weights are packed inside the graph from
            # the live parameters, so its old graph follows a load_state_dict into the same storage; the tocg's folded BatchNorm
            # tables and the storage type are fixed at capture.)
            assert not torch.equal(_clone(old.replay())[1], ref[1])
        _assert_equal(_flat(runner(x)), ref)
    finally:
        runner.release()
        undo()


def test_condition_graph_preconditions(case):
    runner = pipeline.ConditionGraph(case.tocg, case.D, case.M)
    x = _sub(case.batch, 0, 1)
    launches = ops.LAUNCHES[0]
    case.D.train()
    try:
        with pytest.raises(RuntimeError, match="train mode"):
            runner(x)
    finally:
        case.D.eval()
    with pytest.raises(ValueError, match="'densepose'"):
        runner(dict(x, densepose=x["densepose"].cpu()))
    with pytest.raises(ValueError, match="same batch"):
        runner(dict(x, densepose=case.batch["densepose"][:2]))
    assert ops.LAUNCHES[0] == launches and not runner._graphs


@pytest.mark.parametrize("composition", ["warp_grad", "detach", "no_composition"])
def test_tryon_graph_with_discriminator(case, precision, composition):
    """The score is a fourth output; the first three are those of the runner without a discriminator (the composed scores the parse
    map is made of now come from the fused kernel), and the score is ConditionGraph's on the 256x192 inputs tryon_forward forms."""
    import network_generator
    H, W, n = 512, 384, 2
    G = network_generator.SPADEGenerator(gen_opt(H, W, True), 9)
    G.load_state_dict(synth_state_dict("gen", 24))
    G = G.cuda().eval()
    inputs = train_step.synthetic_batch(n, H, W, "cuda", seed=5)
    del inputs["image"]
    plain = pipeline.TryOnGraph(case.tocg, G, clothmask_composition=composition)
    scored = pipeline.TryOnGraph(case.tocg, G, clothmask_composition=composition, discriminator=case.D, norm_const=case.M)
    cond = pipeline.ConditionGraph(case.tocg, case.D, case.M, clothmask_composition=composition)
    try:
        for _ in range(2):  # capture, then replay
            torch.cuda.manual_seed(9)
            ref = [t.clone() for t in plain(inputs)]
            torch.cuda.manual_seed(9)
            got = [t.clone() for t in scored(inputs)]
            torch.cuda.manual_seed(9)
            eager = pipeline.tryon_forward(case.tocg, G, inputs, clothmask_composition=composition, discriminator=case.D, norm_const=case.M)
            assert len(ref) == 3 and len(got) == 4 and len(eager) == 4
            _assert_equal(got[:3], ref)
            _assert_equal(got, list(eager))
            lo = {"cloth": F.interpolate(inputs["cloth"], size=(256, 192), mode="bilinear"),
                  "cloth_mask": F.interpolate((inputs["cloth_mask"] > 0.5).float(), size=(256, 192), mode="nearest"),
                  "parse_agnostic": F.interpolate(inputs["parse_agnostic"], size=(256, 192), mode="nearest"),
                  "densepose": F.interpolate(inputs["densepose"], size=(256, 192), mode="bilinear")}
            assert torch.equal(got[3], cond(lo)[0])
    finally:
        for r in (plain, scored, cond):
            r.release()


# ------------------------------------------------------------------------------------------------ the reference's own scripts


class _Loader:
    """next_batch() and .data_loader of cp_dataset.CPDataLoader over the fixture's batch, with the entries the scripts read."""

    def __init__(self, batch):
        b = {k: v.cpu() for k, v in batch.items()}
        n, _, h, w = b["cloth"].shape
        lab = b["parse"].argmax(1, keepdim=True)
        names = ["%05d_00.jpg" % i for i in range(n)]
        self.batch = {"cloth": {"paired": b["cloth"], "unpaired": b["cloth"]}, "cloth_mask": {"paired": b["cloth_mask"], "unpaired": b["cloth_mask"]},
                      "parse_agnostic": b["parse_agnostic"], "densepose": b["densepose"], "pose": b["densepose"], "parse": b["parse"],
                      "parse_onehot": lab.float(), "pcm": (lab == 3).float(), "parse_cloth": b["cloth"], "image": b["cloth"],
                      "c_name": {"paired": names, "unpaired": names}}
        self.data_loader = [self.batch]

    def next_batch(self):
        return self.batch


@pytest.mark.skipif(hrv_env.reference_dir() is None, reason="no reference copy (oracle/_ref)")
def test_reference_scripts_agree_with_pipeline(case, tmp_path, monkeypatch):
    """get_norm_const.get_const and test_condition.test, unchanged, on the drop-in modules (torch's soft-max and D.forward(nchw)
    there, the fused kernel and the discriminator on its Act here: equal within the score bound, not bit for bit)."""
    monkeypatch.chdir(tmp_path)
    gnc = hrv_env.load_reference_script("get_norm_const")
    tcond = hrv_env.load_reference_script("test_condition")
    ops.set_precision("fp32")
    loader = _Loader(case.batch)
    opt = types.SimpleNamespace(batch_size=4, clothmask_composition=case.composition, tocg_checkpoint="ckpt/tocg.pth", datamode="test",
                                datasetting="paired", norm_const=case.M)
    with contextlib.redirect_stdout(io.StringIO()):
        M_script = gnc.get_const(opt, loader, case.tocg, case.D, 4)
    M_ours = pipeline.norm_constant(case.tocg, case.D, [case.batch], clothmask_composition=case.composition)
    l_all = np.concatenate([case.g["l_real"], case.g["l_fake"]])
    l_at_max = l_all[np.argmax(l_all / (1 - l_all))]
    assert abs(M_script - M_ours) <= TOL_L / (1 - l_at_max) ** 2, (M_script, M_ours)
    with contextlib.redirect_stdout(io.StringIO()):
        tcond.test(opt, loader, None, case.tocg, case.D)
    path = tmp_path / "output" / "ckpt" / "tocg.pth" / "test" / "paired" / "multi-task" / "rejection_prob.txt"
    written = dict((a, float(b)) for a, b in (line.split() for line in path.read_text().splitlines()))
    score, l, _ = pipeline.rejection_scores(case.tocg, case.D, case.batch, case.M, clothmask_composition=case.composition)
    score, l = score.cpu().numpy(), l.cpu().numpy()
    assert len(written) == 4
    for i in range(4):
        assert abs(written["%05d_00.png" % i] - score[i]) <= score_bound(l[i], case.M), (i, written, score)
