"""CPU: discriminator rejection on the oracle.  rejection_oracle.rejection() is pinned against reject_256x192_b4.npz (the live reference's
ConditionGenerator, define_D and D_logit), d_logit against hand-computed means, and the bound the GPU tests hold the scores to,
    |dl| < 1e-3   and   |dscore| <= 1e-3 / ((1 - l)^2 M)        (d(l / (1 - l)) / dl = 1 / (1 - l)^2),
is shown to reject input1 and input2 swapped.  The mistakes inside the third operand (the soft-max taken before the cloth-mask
composition, 'detach' composition without its > 0.5 threshold) move l too little through synthetic weights for any end-to-end
tolerance; the per-element bound on the discriminator's input rejects them.  Argument validation that needs no GPU is here too."""
import functools
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "oracle"))
import hrviton_oracle as orc  # noqa: E402
import rejection_oracle as rorc  # noqa: E402
from helpers import load_golden, synth_state_dict, tocg_opt  # noqa: E402
from hrviton_b200 import ops, pipeline, synth  # noqa: E402

NAME = "reject_256x192_b4"
TOL_L = 1e-3


def reject_case():
    """Golden, state dicts and inputs of the fixture: synthetic weights from its seed, the last-layer biases of the discriminator
    shifted as make_golden_reject.py shifted them."""
    g = load_golden(NAME)
    n, h, w = [int(v) for v in g["shape"]]
    seed = int(g["seed"])
    sd_t, sd_d = synth_state_dict("tocg", seed), synth_state_dict("tocgd", seed)
    for k in sd_d:
        if k.endswith(".bias") and sd_d[k].numel() == 1:
            sd_d[k] += float(g["d_bias_shift"])
    i1, i2 = synth.tocg_inputs(n, h, w, seed)
    label = synth.one_hot(synth.labels((n, h, w), 13, seed, "dseg"), 13)
    return g, sd_t, sd_d, i1, i2, label


@functools.lru_cache(maxsize=None)
def _tocg_out():
    g, sd_t, sd_d, i1, i2, label = reject_case()
    with torch.no_grad():
        _, seg, _, wcm = orc.tocg_forward(sd_t, i1, i2)
    return seg, wcm


def _l(sd_d, a, b, third):
    with torch.no_grad():
        return rorc.d_logit(orc.tocg_d_forward(sd_d, torch.cat([a, b, third], 1)))


def score_bound(l, M, tol_l=TOL_L):
    return tol_l / ((1.0 - np.asarray(l, np.float64)) ** 2 * M)


def test_fixture_keeps_off_the_pole():
    g = load_golden(NAME)
    l = np.concatenate([g["l_fake"], g["l_real"]])
    assert float(np.abs(1 - l).min()) >= 0.2 and abs(float(np.abs(1 - l).min()) - float(g["margin"])) < 1e-6
    assert float(g["M"]) > 0 and np.isclose(float(g["M"]), float((l / (1 - l)).max()), rtol=1e-6)
    assert np.allclose(g["score"], g["l_fake"] / (1 - g["l_fake"]) / float(g["M"]), rtol=1e-6)


def test_oracle_rejection_matches_golden():
    g, sd_t, sd_d, i1, i2, label = reject_case()
    with torch.no_grad():
        score, l, maps = rorc.rejection(sd_t, sd_d, i1, i2, float(g["M"]), str(g["composition"]))
        real = orc.tocg_d_forward(sd_d, torch.cat([i1, i2, label], 1))
    for i, m in enumerate(maps):
        assert float((m - torch.from_numpy(g["fake_d%d" % i])).abs().max()) < 1e-4
        assert float((real[i][-1] - torch.from_numpy(g["real_d%d" % i])).abs().max()) < 1e-4
    assert np.abs(l.numpy() - g["l_fake"]).max() < 1e-4
    assert np.abs(rorc.d_logit(real).numpy() - g["l_real"]).max() < 1e-4
    assert (np.abs(score.numpy() - g["score"]) <= score_bound(g["l_fake"], float(g["M"]), 1e-4)).all()


@pytest.mark.parametrize("num_d", [1, 2, 3])
@pytest.mark.parametrize("fn", [rorc.d_logit, pipeline.d_logit])
def test_d_logit_divides_by_two_for_every_num_d(fn, num_d):
    """Scale i is constant i + 1 per sample offset: the means are known exactly, and the result is their sum / 2 — the mean over
    scales only for num_D = 2."""
    per_sample = torch.tensor([0.0, 0.25, -1.5])
    preds = [[torch.full((3, 1, 2, 2), 99.0), torch.full((3, 1, 5 - i, 4), float(i + 1)) + per_sample.view(3, 1, 1, 1)] for i in range(num_d)]
    want = sum((i + 1) + per_sample for i in range(num_d)) / 2
    got = fn(preds)
    assert got.shape == (3,) and torch.allclose(got, want, atol=1e-6)


def element_bound(ref, u):
    """The per-element bound of the fused kernel's soft-max channels (tests/test_rejection_gpu.py): one rounding to the storage type
    (u = 2^-8 bf16, 2^-11 fp16, 0 fp32) plus 64 fp32 steps of the soft-max arithmetic."""
    return u * ref.abs().double() + 64 * 2.0 ** -24


@pytest.mark.parametrize("mistake", ["swapped_inputs", "softmax_before_composition", "detach_without_threshold"])
def test_bounds_reject_glue_mistakes(mistake):
    """Swapped inputs move l by 1.6e-3 .. 1.5e-2 on this fixture: outside |dl| < 1e-3 and the score bound derived from it.  The two
    mistakes inside the third operand move l by less than 3e-4 through these synthetic weights (the discriminator's response to
    one of its 33 input channels, averaged over the map), so no end-to-end tolerance on l sees them; they are caught where they
    happen, by the per-element bound on the discriminator's input, which they exceed by orders of magnitude in bf16 already."""
    g, sd_t, sd_d, i1, i2, label = reject_case()
    seg, wcm = _tocg_out()
    M = float(g["M"])
    composition = "detach" if mistake == "detach_without_threshold" else "warp_grad"
    third = F.softmax(rorc.compose_segmap(seg, wcm, composition), 1)
    if mistake == "swapped_inputs":
        right, wrong = _l(sd_d, i1, i2, third), _l(sd_d, i2, i1, third)
        dl = (wrong - right).abs().double().numpy()
        ds = (wrong / (1 - wrong) / M - right / (1 - right) / M).abs().double().numpy()
        print("REJECTBOUND %-28s |dl| %s  |dscore|/bound %s" % (mistake, dl, ds / score_bound(right.numpy(), M)))
        assert (dl > TOL_L).all() and (ds > score_bound(right.numpy(), M)).all()
        return
    if mistake == "softmax_before_composition":
        wrong_third = rorc.compose_segmap(F.softmax(seg, 1), wcm, composition)
    else:
        wrong_third = F.softmax(rorc.compose_segmap(seg, wcm, "warp_grad"), 1)
    dl = (_l(sd_d, i1, i2, wrong_third) - _l(sd_d, i1, i2, third)).abs().max()
    worst = float(((wrong_third - third).abs().double() / element_bound(third, 2.0 ** -8)).max())
    print("REJECTBOUND %-28s max|dl| %.3e  worst element %.1f x its bf16 bound" % (mistake, float(dl), worst))
    assert float(dl) < TOL_L  # what makes the per-element check necessary
    assert worst > 10.0


def test_compose_segmap_modes():
    seg = torch.arange(2 * 13 * 2 * 3, dtype=torch.float32).view(2, 13, 2, 3) - 70
    cm = torch.tensor([0.2, 0.5, 0.50001, 0.9, 1.0, 0.0]).view(1, 1, 2, 3).expand(2, 1, 2, 3)
    assert rorc.compose_segmap(seg, cm, "no_composition") is seg
    for mode, m in (("warp_grad", cm), ("detach", (cm > 0.5).float())):
        out = rorc.compose_segmap(seg, cm, mode)
        assert torch.equal(out[:, 3:4], seg[:, 3:4] * m) and torch.equal(out[:, :3], seg[:, :3]) and torch.equal(out[:, 4:], seg[:, 4:])


# ------------------------------------------------------------------------------------------------ validation (no GPU)


@pytest.mark.parametrize("bad", [None, 0, 0.0, -1.5, float("nan")])
def test_norm_const_must_be_positive(bad):
    import networks
    with pytest.raises(ValueError, match="norm_const"):
        pipeline.rejection_scores(None, None, {}, bad)
    with pytest.raises(ValueError, match="norm_const"):
        pipeline.tryon_forward(None, None, {}, discriminator=object(), norm_const=bad)
    tocg = networks.ConditionGenerator(tocg_opt(), 4, 16, 13, ngf=96, norm_layer=torch.nn.BatchNorm2d)
    with pytest.raises(ValueError, match="norm_const"):
        pipeline.ConditionGraph(tocg, torch.nn.Identity(), bad)
    with pytest.raises(ValueError, match="norm_const"):
        pipeline.TryOnGraph(tocg, torch.nn.Identity(), discriminator=torch.nn.Identity(), norm_const=bad)


def test_cpu_tensors_are_refused():
    t = lambda c: torch.zeros(1, c, 8, 6)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        pipeline.condition_logit(None, t(4), t(16), t(13))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        ops.seg_softmax_cat(t(4), t(16), t(13), cm=t(1))
    with pytest.raises(ValueError, match="composition"):
        ops.seg_softmax_cat(t(4), t(16), t(13), cm=t(1), composition="warp")


def test_norm_constant_needs_a_batch():
    with pytest.raises(ValueError, match="no batches"):
        pipeline.norm_constant(None, None, [])
