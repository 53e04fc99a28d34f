"""sync_batchnorm.SynchronizedBatchNorm2d / convert_model on the CPU: the reference's constructor defaults and state_dict, the
layer swap on a ConditionGenerator (all 34 BatchNorm layers, every value kept bit for bit), checkpoints loading both ways, and the
dispatch that keeps one process on the plain BatchNorm path."""
import os
import sys

import pytest
import torch
import torch.nn as nn

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import hrv_loader  # noqa: E402

hrv_loader.load()

import networks  # noqa: E402
import sync_batchnorm  # noqa: E402
from helpers import tocg_opt  # noqa: E402
from hrviton_b200 import ddp, synth  # noqa: E402

BN_KEYS = ["weight", "bias", "running_mean", "running_var", "num_batches_tracked"]


def _tocg(norm_layer=nn.BatchNorm2d, seed=3):
    m = networks.ConditionGenerator(tocg_opt(), 4, 16, 13, ngf=8, norm_layer=norm_layer)
    sd = m.state_dict()
    synth.fill_state_dict(sd, seed)
    m.load_state_dict(sd)
    return m


def test_public_names():
    for name in ["SynchronizedBatchNorm1d", "SynchronizedBatchNorm2d", "SynchronizedBatchNorm3d", "convert_model", "DataParallelWithCallback"]:
        assert hasattr(sync_batchnorm, name), name
    assert issubclass(sync_batchnorm.SynchronizedBatchNorm2d, nn.BatchNorm2d)


def test_constructor_defaults_and_state_dict_match_the_reference():
    # the reference: SynchronizedBatchNorm2d(num_features, eps=1e-5, momentum=0.1, affine=True) over torch's _BatchNorm
    m = sync_batchnorm.SynchronizedBatchNorm2d(24)
    assert (m.num_features, m.eps, m.momentum, m.affine, m.track_running_stats) == (24, 1e-5, 0.1, True, True)
    sd = m.state_dict()
    assert list(sd) == BN_KEYS
    ref = nn.BatchNorm2d(24).state_dict()
    for k in BN_KEYS:
        assert sd[k].shape == ref[k].shape and sd[k].dtype == ref[k].dtype and torch.equal(sd[k], ref[k]), k
    m2 = sync_batchnorm.SynchronizedBatchNorm2d(8, 1e-3, 0.2, False)
    assert (m2.eps, m2.momentum, m2.affine, m2.weight) == (1e-3, 0.2, False, None)


def test_convert_model_swaps_all_34_layers_and_keeps_every_value():
    plain = _tocg()
    before = {k: v.clone() for k, v in plain.state_dict().items()}
    n_bn = sum(isinstance(m, nn.BatchNorm2d) for m in plain.modules())
    assert n_bn == 34
    old_bn = plain.ClothEncoder[0].block[1]
    conv = sync_batchnorm.convert_model(plain)  # as the reference's: children of `plain` are replaced in place
    sync = [m for m in conv.modules() if isinstance(m, sync_batchnorm.SynchronizedBatchNorm2d)]
    assert len(sync) == 34
    assert not any(type(m) is nn.BatchNorm2d for m in conv.modules())
    after = conv.state_dict()
    assert list(after) == list(before)
    bits = lambda t: t.reshape(-1).view(torch.uint8)
    for k, v in before.items():
        assert after[k].dtype == v.dtype and torch.equal(bits(after[k]), bits(v)), k
    # affine parameters are new tensors (the converted model trains its own), the running statistics are the original buffers
    new_bn = conv.ClothEncoder[0].block[1]
    assert new_bn.weight is not old_bn.weight and new_bn.running_mean is old_bn.running_mean


def test_convert_model_keeps_mode_and_hyper_parameters():
    bn = nn.BatchNorm2d(16, eps=1e-3, momentum=0.05).eval()
    s = sync_batchnorm.convert_model(nn.Sequential(nn.Conv2d(3, 16, 3), bn))[1]
    assert isinstance(s, sync_batchnorm.SynchronizedBatchNorm2d)
    assert (s.eps, s.momentum, s.training) == (1e-3, 0.05, False)


@pytest.mark.parametrize("wrapper", [nn.DataParallel, ddp.DataParallelWithCallback])
def test_convert_model_rewraps_data_parallel(wrapper):
    net = nn.Sequential(nn.Conv2d(3, 8, 3), nn.BatchNorm2d(8))
    out = sync_batchnorm.convert_model(wrapper(net))
    assert isinstance(out, ddp.DataParallelWithCallback)
    assert isinstance(out.module[1], sync_batchnorm.SynchronizedBatchNorm2d)


def test_checkpoints_load_both_ways():
    plain = _tocg(seed=5)
    sync = _tocg(norm_layer=sync_batchnorm.SynchronizedBatchNorm2d, seed=11)
    assert sum(isinstance(m, sync_batchnorm.SynchronizedBatchNorm2d) for m in sync.modules()) == 34
    sync.load_state_dict(plain.state_dict())  # strict: same keys and shapes
    for k, v in plain.state_dict().items():
        assert torch.equal(sync.state_dict()[k], v), k
    other = _tocg(seed=7)
    sync2 = _tocg(norm_layer=sync_batchnorm.SynchronizedBatchNorm2d, seed=13)
    other.load_state_dict(sync2.state_dict())
    for k, v in sync2.state_dict().items():
        assert torch.equal(other.state_dict()[k], v), k


def test_one_process_takes_the_per_rank_path():
    assert ddp.syncbn_group() is None  # no process group: SynchronizedBatchNorm2d runs the plain BatchNorm kernels, no collectives
    m = sync_batchnorm.SynchronizedBatchNorm2d(4).train()
    x = torch.randn(2, 4, 5, 5)
    ref = nn.BatchNorm2d(4).train()
    assert torch.equal(m(x), ref(x))
    assert torch.equal(m.running_var, ref.running_var)


@pytest.mark.parametrize("cls", ["SynchronizedBatchNorm1d", "SynchronizedBatchNorm3d"])
def test_1d_and_3d_names_raise_when_used(cls):
    m = getattr(sync_batchnorm, cls)(4)
    with pytest.raises(NotImplementedError):
        m(torch.zeros(2, 4, 3) if cls.endswith("1d") else torch.zeros(2, 4, 3, 3, 3))
