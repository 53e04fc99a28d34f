"""Dynamic loss scaling without a GPU: the scaler's state machine (growth, backoff, skip, one scaler per loss) with a torch stand-in for
the unscale kernel, the fp16 underflow of the VGG loss seeds that motivates it, and the apex shim (a no-op in bf16 storage, apex O1
semantics with a host-side skip in fp16 storage)."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import hrv_loader  # noqa: E402

hrv_loader.load()
from hrviton_b200 import loss_scale, ops  # noqa: E402


def _stub_unscale_check(grads, inv_scale, found_inf, table=None):
    """What hrv_grad_unscale_check computes, in torch (checks the input, then multiplies)."""
    for g in grads:
        if not bool(torch.isfinite(g).all()):
            found_inf.fill_(1.0)
        g.mul_(inv_scale)
    return table


@pytest.fixture
def stub_kernel(monkeypatch):
    monkeypatch.setattr(ops, "grad_unscale_check", _stub_unscale_check)


def _model(seed=0):
    g = torch.Generator().manual_seed(seed)
    p = torch.nn.Parameter(torch.randn(6, 5, generator=g))
    opt = torch.optim.Adam([p], lr=1e-2, betas=(0.0, 0.9), fused=True)
    return p, opt


def _scaled_step(sc, p, opt, poison=False):
    opt.zero_grad(set_to_none=False)
    loss = (p * p).sum() * (float("inf") if poison else 1.0)
    sc.scale_loss(loss).backward()
    sc.unscale_and_check(opt)
    opt.step()
    sc.update()


def test_defaults_are_apex_o1():
    sc = loss_scale.DynamicLossScaler("cpu")
    assert float(sc.scale) == 2.0 ** 16 and int(sc.growth_tracker) == 0 and float(sc.found_inf) == 0.0
    assert (sc.growth_factor, sc.backoff_factor, sc.growth_interval) == (2.0, 0.5, 2000)


def test_unscaled_gradient_equals_unscaled_loss_gradient(stub_kernel):
    p, opt = _model()
    sc = loss_scale.DynamicLossScaler("cpu")
    opt.zero_grad()
    sc.scale_loss((p * p).sum()).backward()
    sc.unscale_and_check(opt)
    assert torch.equal(p.grad, 2 * p.detach())  # S = 2^16: dividing by it is exact
    assert float(sc.found_inf) == 0.0


def test_growth_after_interval_clean_steps(stub_kernel):
    p, opt = _model()
    sc = loss_scale.DynamicLossScaler("cpu", init_scale=8.0, growth_interval=3)
    scales = []
    for _ in range(7):
        _scaled_step(sc, p, opt)
        scales.append(float(sc.scale))
    assert scales == [8.0, 8.0, 16.0, 16.0, 16.0, 32.0, 32.0]
    assert int(sc.growth_tracker) == 1
    assert int(opt.state[p]["step"]) == 7


def test_overflow_skips_the_step_and_backs_off(stub_kernel):
    p, opt = _model()
    sc = loss_scale.DynamicLossScaler("cpu", init_scale=1024.0, growth_interval=3)
    opt.found_inf = sc.found_inf
    _scaled_step(sc, p, opt)
    _scaled_step(sc, p, opt)
    before = (p.detach().clone(), opt.state[p]["exp_avg"].clone(), opt.state[p]["exp_avg_sq"].clone(), opt.state[p]["step"].clone())
    _scaled_step(sc, p, opt, poison=True)
    assert float(sc.found_inf) == 1.0 and float(sc.scale) == 512.0 and int(sc.growth_tracker) == 0
    after = (p.detach(), opt.state[p]["exp_avg"], opt.state[p]["exp_avg_sq"], opt.state[p]["step"])
    assert all(torch.equal(a, b) for a, b in zip(before, after))  # fused Adam left everything as it was
    _scaled_step(sc, p, opt)
    assert not torch.equal(p.detach(), before[0]) and int(opt.state[p]["step"]) == 3
    assert float(sc.found_inf) == 0.0 and float(sc.scale) == 512.0 and int(sc.growth_tracker) == 1


def test_one_scaler_per_loss(stub_kernel):
    scalers = loss_scale.make_scalers("dynamic", ["G", "D"], "cpu")
    (pg, og), (pd, od) = _model(1), _model(2)
    _scaled_step(scalers["G"], pg, og, poison=True)
    _scaled_step(scalers["D"], pd, od)
    assert float(scalers["G"].scale) == 2.0 ** 15 and float(scalers["D"].scale) == 2.0 ** 16
    assert float(scalers["G"].found_inf) == 1.0 and float(scalers["D"].found_inf) == 0.0
    assert loss_scale.make_scalers(None, ["G", "D"], "cpu") == {}
    with pytest.raises(ValueError):
        loss_scale.make_scalers("static", ["G"], "cpu")


def test_state_dict_round_trip():
    a = loss_scale.DynamicLossScaler("cpu", growth_interval=7)
    a.scale.fill_(256.0)
    a.growth_tracker.fill_(5)
    b = loss_scale.DynamicLossScaler("cpu")
    scale_tensor = b.scale
    b.load_state_dict(a.state_dict())
    assert b.scale is scale_tensor  # in place: a captured graph keeps reading the same tensor
    assert float(b.scale) == 256.0 and int(b.growth_tracker) == 5 and b.growth_interval == 7


def test_fp32_storage_refuses_loss_scaling():
    old = ops.get_precision()
    try:
        ops.set_precision("fp32")
        with pytest.raises(NotImplementedError):
            loss_scale.make_scalers("dynamic", ["G", "D"], "cpu")
    finally:
        ops.set_precision(old)


def test_gradients_prefer_reducer_buckets():
    p1, p2, p3 = (torch.nn.Parameter(torch.zeros(n)) for n in (3, 4, 5))
    opt = torch.optim.Adam([p1, p2, p3])
    flat = torch.zeros(7)
    p1.grad, p2.grad, p3.grad = flat[:3], flat[3:], torch.zeros(5)

    class _Reducer:
        _buckets = [{"flat": flat, "params": [p1, p2]}]

    got = loss_scale.DynamicLossScaler.gradients(opt, _Reducer())
    assert len(got) == 2 and got[0] is flat and got[1] is p3.grad
    assert [g is q.grad for g, q in zip(loss_scale.DynamicLossScaler.gradients(opt), (p1, p2, p3))] == [True] * 3


# ---------------------------------------------------------------------------------------------------------- the fp16 underflow

def _vgg_seeds(n, h, w):
    """Per-element gradient seed of each VGGLoss slice: lambda_vgg * weight_i / numel_i (L1 mean), relu1_1 .. relu5_1."""
    chans, scales, weights = (64, 128, 256, 512, 512), (1, 2, 4, 8, 16), (1 / 32, 1 / 16, 1 / 8, 1 / 4, 1.0)
    return [10.0 * wt / (n * c * (h // s) * (w // s)) for c, s, wt in zip(chans, scales, weights)]


def test_vgg_seeds_underflow_in_fp16_at_1024x768_b8():
    seeds = _vgg_seeds(8, 1024, 768)
    assert seeds == pytest.approx([7.76e-10, 3.10e-9, 1.24e-8, 4.97e-8, 7.95e-7], rel=2e-3)
    h16 = [float(torch.tensor(s, dtype=torch.float64).to(torch.float16)) for s in seeds]
    assert h16[:3] == [0.0, 0.0, 0.0]  # relu1_1 .. relu3_1: no gradient at all
    assert h16[3] == 2.0 ** -24  # relu4_1: one subnormal step
    assert abs(h16[4] - seeds[4]) / seeds[4] > 0.01  # relu5_1: a 13-step subnormal, 2.5 % off
    assert all(float(torch.tensor(s).to(torch.bfloat16)) > 0 for s in seeds)  # bf16 has fp32's range
    scaled = [float(torch.tensor(s * 2.0 ** 16, dtype=torch.float64).to(torch.float16)) for s in seeds]
    assert all(abs(v / 2.0 ** 16 - s) / s < 2.0 ** -10 for v, s in zip(scaled[:4], seeds[:4]))  # S = 2^16: normal fp16 numbers
    fm = 10.0 / 2 / (8 * 64 * 513 * 385)  # feature matching, D layer 0: lambda_feat / num_D / numel
    assert float(torch.tensor(fm).to(torch.float16)) == 2.0 ** -24


# ---------------------------------------------------------------------------------------------------------- the apex shim

@pytest.fixture
def amp():
    sys.path.insert(0, os.path.join(ROOT, "shims"))
    try:
        from apex import amp as mod
        yield mod
    finally:
        sys.path.remove(os.path.join(ROOT, "shims"))
        mod._SCALERS[:] = []


def test_shim_is_a_no_op_in_bf16(amp):
    old = ops.get_precision()
    try:
        ops.set_precision("bf16")
        models = [torch.nn.Linear(3, 2), torch.nn.Linear(2, 2)]
        opts = [torch.optim.Adam(m.parameters()) for m in models]
        step = opts[0].step
        got_models, got_opts = amp.initialize(models, opts, opt_level="O1", num_losses=2)
        assert got_models is models and got_opts is opts
        assert opts[0].step == step and not hasattr(opts[0], "_amp_skip_next")
        loss = models[0](torch.ones(1, 3)).sum()
        with amp.scale_loss(loss, opts[0], loss_id=0) as scaled:
            assert scaled is loss
        assert amp.initialize(models) is models
    finally:
        ops.set_precision(old)


def test_shim_scales_and_skips_in_fp16(amp, stub_kernel):
    old = ops.get_precision()
    try:
        ops.set_precision("fp16")
        model = torch.nn.Linear(3, 2)
        opt = torch.optim.Adam(model.parameters(), lr=0.1)
        amp.initialize([model], [opt], opt_level="O1", num_losses=2)
        assert len(amp._SCALERS) == 2
        x = torch.ones(1, 3)
        loss = model(x).sum()
        with amp.scale_loss(loss, opt, loss_id=0) as scaled:
            assert float(scaled.detach()) == float(loss.detach()) * 2.0 ** 16
            scaled.backward()
        torch.testing.assert_close(model.bias.grad, torch.ones(2), rtol=0, atol=0)  # unscaled on exit
        w0 = model.weight.detach().clone()
        opt.step()
        assert not torch.equal(model.weight.detach(), w0)
        w1 = model.weight.detach().clone()
        opt.zero_grad()
        with amp.scale_loss(model(x).sum() * float("inf"), opt, loss_id=0) as scaled:
            scaled.backward()
        opt.step()  # skipped
        assert torch.equal(model.weight.detach(), w1) and float(amp._SCALERS[0].scale) == 2.0 ** 15
        assert float(amp._SCALERS[1].scale) == 2.0 ** 16
        opt.zero_grad()
        with amp.scale_loss(model(x).sum(), opt, loss_id=0) as scaled:
            scaled.backward()
        opt.step()  # the skip lasts one step
        assert not torch.equal(model.weight.detach(), w1)
    finally:
        ops.set_precision(old)
