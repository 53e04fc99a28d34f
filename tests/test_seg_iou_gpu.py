"""GPU: hrv_seg_iou / metrics.segmentation_iou against the restated iou_metric (seg_iou_oracle.py) bit for bit, and
pipeline.SegmentationGraph against the eager eval-mode tocg plus the oracle.

Inputs keep every probability at least 1e-5 away from 0.5 (where torch's soft-max and the kernel's could round to opposite sides),
except the exact ties the kernel must count as not predicted."""
import copy

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import seg_iou_oracle as orc
from hrviton_b200 import capi, ddp, metrics, ops, pipeline, synth

pytestmark = pytest.mark.gpu


def _bits(x):
    return np.float32(x).view(np.uint32)


def _inputs(b, h, w, seed):
    """Scores, mask and a label that agrees with the arg-max on about 70 % of the pixels, all fp32 cuda."""
    g = torch.Generator().manual_seed(seed)
    seg = torch.randn(b, 13, h, w, generator=g) * 3
    cm = torch.rand(b, 1, h, w, generator=g) * (torch.rand(b, 1, h, w, generator=g) > 0.2).float()
    seg, cm = seg.cuda(), cm.cuda()
    for _ in range(8):
        near = ((orc.probabilities(seg, cm) - 0.5).abs() < 1e-5).any(1, keepdim=True)
        if not near.any():
            break
        seg[:, :1] += near.float() * 4  # channel 0 takes the pixel
    assert not ((orc.probabilities(seg, cm) - 0.5).abs() < 1e-5).any()
    lab = orc.probabilities(seg, cm).argmax(1)
    rnd = torch.randint(0, 13, (b, h, w), generator=g).cuda()
    lab = torch.where(torch.rand(b, h, w, generator=g).cuda() < 0.7, lab, rnd)
    return seg, cm, F.one_hot(lab, 13).permute(0, 3, 1, 2).float().contiguous()


@pytest.mark.parametrize("b,h,w", [(1, 256, 192), (8, 256, 192), (3, 37, 29), (2, 1, 1), (5, 129, 255), (4, 300, 17), (7, 64, 48)])
def test_kernel_equals_oracle(b, h, w):
    seg, cm, parse = _inputs(b, h, w, b * 1000 + h)
    got = metrics.segmentation_iou(seg, cm, parse)
    assert got.shape == () and got.dtype == torch.float32 and got.is_cuda
    want = orc.segmentation_iou(seg, cm, parse)
    assert _bits(got.item()) == _bits(want), (got.item(), want)
    assert 0.0 < want < 1.0


def test_exact_ties_are_not_predicted():
    b, h, w = 2, 16, 24
    seg = torch.full((b, 13, h, w), -200.0, device="cuda")
    seg[:, 4] = 1.5
    seg[:, 7] = 1.5                                   # p = 0.5 exactly in channels 4 and 7
    seg[1, :, :, :8] = -200.0
    seg[1, 9, :, :8] = 2.0                            # sample 1, left third: channel 9 predicted (p = 1)
    cm = torch.ones(b, 1, h, w, device="cuda")
    parse = torch.zeros(b, 13, h, w, device="cuda")
    parse[:, 4] = 1
    p = orc.probabilities(seg, cm)
    assert (p[:, 4] == 0.5).all().item() is False and (p[0, 4] == 0.5).all()
    assert orc.counts(p[0], parse[0]) == (0, h * w, 0)
    got = metrics.segmentation_iou(seg, cm, parse)
    assert _bits(got.item()) == _bits(orc.segmentation_iou(seg, cm, parse))


@pytest.mark.parametrize("case", ["empty_label", "all_predicted", "mask0", "mask1"])
def test_edge_cases(case):
    b, h, w = 3, 40, 33
    seg, cm, parse = _inputs(b, h, w, 7)
    if case == "empty_label":
        parse[1] = 0                                  # L = 0 for sample 1: its term is (I + 1e-7) / (P - I + 1e-7)
    elif case == "all_predicted":
        seg[0, 5] = 50.0                              # channel 5 predicted at every pixel of sample 0
        parse[2] = 0
        parse[2, 3] = 1                               # and sample 2 labelled cloth everywhere
    elif case == "mask0":
        cm.zero_()                                    # channel 3 scores composed to zero
    else:
        cm.fill_(1.0)
    assert not ((orc.probabilities(seg, cm) - 0.5).abs() < 1e-5).any()
    got = metrics.segmentation_iou(seg, cm, parse)
    want = orc.segmentation_iou(seg, cm, parse)
    assert _bits(got.item()) == _bits(want), (got.item(), want)
    if case == "all_predicted":
        assert orc.counts(orc.probabilities(seg, cm)[0], parse[0])[0] == h * w


def test_two_calls_are_bit_identical():
    seg, cm, parse = _inputs(8, 256, 192, 99)
    a = metrics.segmentation_iou(seg, cm, parse).clone()
    b = metrics.segmentation_iou(seg, cm, parse)
    assert torch.equal(a, b)


def test_bad_inputs_are_refused_without_a_launch():
    seg, cm, parse = _inputs(2, 8, 6, 1)
    before = ops.LAUNCHES[0]
    bad = [
        ((seg.cpu(), cm, parse), RuntimeError),
        ((seg.half(), cm, parse), ValueError),
        ((seg.double(), cm, parse), ValueError),
        ((seg[:, :12], cm, parse[:, :12]), ValueError),       # 12 classes
        ((seg, torch.cat([cm, cm], 1), parse), ValueError),   # 2-channel mask
        ((seg, cm[:1], parse), ValueError),                   # batch mismatch
        ((seg, cm, parse[..., :5]), ValueError),              # size mismatch
        ((seg[0], cm, parse), ValueError),                    # 3-d
        ((seg, cm.cpu(), parse), RuntimeError),
        ((seg, cm, "parse"), TypeError),
    ]
    for args, exc in bad:
        with pytest.raises(exc):
            metrics.segmentation_iou(*args)
    with pytest.raises(ValueError, match="warp_grad"):
        metrics.segmentation_iou(seg, cm, parse, composition="no_composition")
    assert ops.LAUNCHES[0] == before
    # the C-ABI checks its own arguments too
    L, out = capi.lib(), torch.zeros((), device="cuda")
    need = int(L.hrv_seg_iou_workspace_bytes(2, 8, 6))
    assert need > 0
    ws = torch.empty(need, dtype=torch.uint8, device="cuda")
    st = ops._stream()
    for args in ((seg.data_ptr(), 13, cm.data_ptr(), parse.data_ptr(), 2, 8, 6, out.data_ptr(), ws.data_ptr(), need - 1, st),
                 (seg.data_ptr(), 3, cm.data_ptr(), parse.data_ptr(), 2, 8, 6, out.data_ptr(), ws.data_ptr(), need, st),
                 (seg.data_ptr(), 13, None, parse.data_ptr(), 2, 8, 6, out.data_ptr(), ws.data_ptr(), need, st),
                 (seg.data_ptr(), 13, cm.data_ptr(), parse.data_ptr(), 0, 8, 6, out.data_ptr(), ws.data_ptr(), need, st)):
        assert L.hrv_seg_iou(*args) != 0
    assert L.hrv_seg_iou_f16(seg.data_ptr(), 13, cm.data_ptr(), parse.data_ptr(), 2, 8, 6, out.data_ptr(), ws.data_ptr(), need, st) == 0
    assert _bits(out.item()) == _bits(orc.segmentation_iou(seg, cm, parse))


# ------------------------------------------------------------------------------------------------ the graph runner

def _tocg(seed=3):
    import networks
    from helpers import tocg_opt
    t = networks.ConditionGenerator(tocg_opt(True), 4, 16, 13, ngf=96, norm_layer=torch.nn.BatchNorm2d)
    sd = t.state_dict()
    synth.fill_state_dict(sd, seed)
    t.load_state_dict(sd)
    return t.cuda().eval()


def _batch(b, seed):
    i1, i2 = synth.tocg_inputs(b, 256, 192, seed)
    parse = synth.one_hot(synth.labels((b, 256, 192), 13, seed, "val_parse", block=16), 13)
    return {"cloth": i1[:, :3].cuda(), "cloth_mask": (i1[:, 3:4] * 0.8 + 0.1).cuda(), "parse_agnostic": i2[:, :13].cuda(),
            "densepose": i2[:, 13:].cuda(), "parse": parse.float().cuda()}


def _eager(tocg, b):
    with torch.no_grad():
        input1 = torch.cat([b["cloth"], (b["cloth_mask"] > 0.5).float()], 1)
        input2 = torch.cat([b["parse_agnostic"], b["densepose"]], 1)
        _, seg, _, wcm = tocg(input1, input2)
        return orc.segmentation_iou(seg, wcm, b["parse"]), metrics.segmentation_iou(seg, wcm, b["parse"]).item()


def test_graph_equals_eager_tocg_and_oracle_and_recaptures():
    tocg = _tocg()
    runner = pipeline.SegmentationGraph(tocg)
    batches = [_batch(4, s) for s in (1, 2)]
    try:
        for b in batches:
            got = runner(b).item()
            want, kernel = _eager(tocg, b)
            assert _bits(got) == _bits(want) == _bits(kernel), (got, want, kernel)
        entry = next(iter(runner._graphs.values()))
        runner(batches[0])
        assert next(iter(runner._graphs.values())) is entry  # same weights: replayed, not captured again
        values = [runner(batches[0]).item()]
        with torch.no_grad():
            tocg.out_layer.block[0].weight.mul_(1.5)       # a parameter edit
        values.append(runner(batches[0]).item())
        assert next(iter(runner._graphs.values())) is not entry
        assert _bits(values[-1]) == _bits(_eager(tocg, batches[0])[0])
        entry = next(iter(runner._graphs.values()))
        with torch.no_grad():
            tocg.SegDecoder[4].block[1].running_mean.add_(0.5)  # a BatchNorm running-statistics edit
        values.append(runner(batches[0]).item())
        assert next(iter(runner._graphs.values())) is not entry
        assert _bits(values[-1]) == _bits(_eager(tocg, batches[0])[0])
        assert len(set(values)) == 3, values
        tocg.train()
        with pytest.raises(RuntimeError, match="train mode"):
            runner(batches[0])
    finally:
        runner.release()


def test_syncbn_model_takes_the_folded_path(monkeypatch):
    """ddp.convert_model's tocg at one rank: its eval forward never calls a BatchNorm module (the statistics are folded into the
    convolutions) and gives the plain model's IoU bit for bit, eagerly and through the graph."""
    tocg = _tocg()
    sync = ddp.convert_model(copy.deepcopy(tocg)).eval()
    assert any(isinstance(m, ddp.SynchronizedBatchNorm2d) for m in sync.modules())
    called = []
    monkeypatch.setattr(ddp.SynchronizedBatchNorm2d, "forward", lambda self, x: called.append(self) or x)
    monkeypatch.setattr(torch.nn.BatchNorm2d, "forward", lambda self, x: called.append(self) or x)
    b = _batch(2, 5)
    want = _eager(tocg, b)[0]
    assert _bits(_eager(sync, b)[0]) == _bits(want)
    runner = pipeline.SegmentationGraph(sync)
    try:
        assert _bits(runner(b).item()) == _bits(want)
    finally:
        runner.release()
    assert not called
