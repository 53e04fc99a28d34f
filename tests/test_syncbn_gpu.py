"""Synchronised train-mode BatchNorm (sync_batchnorm.SynchronizedBatchNorm2d) on the GPU:
  (a) the combine / finalize kernels against sequential fp64 sums, an fp64 full-batch computation and torch's BatchNorm2d update;
  (b) with one process a SyncBN tocg trains bit-identically to the same tocg with nn.BatchNorm2d (eager steps and graph replays);
  (c) two processes on one GPU (gloo), 2 + 2 samples, give the loss, running statistics and gradients of one process on all 4
      samples with plain BatchNorm — and plain BatchNorm on the two ranks does not (negative control);
  (d) two GPUs (NCCL): a graph-replayed Stage1Trainer step with SyncBN equals the eager step and leaves identical running
      statistics on both ranks (skipped with fewer than 2 GPUs).
The multi-process parts run this file as a script in child processes, which are joined (or killed) before the test returns."""
import contextlib
import io
import os
import subprocess
import sys
import types

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for _p in (ROOT, HERE):
    if _p not in sys.path:
        sys.path.insert(0, _p)
import hrv_loader  # noqa: E402

hrv_loader.load()

pytestmark = pytest.mark.gpu
SEED = 17
GRAD_BOUND = 2e-3  # per-parameter relative gradient difference, as tests/test_multigpu_gpu.py
STORAGES = [torch.bfloat16, torch.float16]


def _ulp(t):
    t = t.float()
    return (torch.nextafter(t.abs(), torch.full_like(t, float("inf"))) - t.abs()).double()


# ------------------------------------------------------------------------------------------------ (a) kernels

def test_combine_is_the_sequential_fp64_sum_in_image_order():
    from hrviton_b200 import ops
    g = torch.Generator().manual_seed(SEED)
    n, c = 5, 40
    base = torch.randn(n, c, 4, generator=g, dtype=torch.float64) * 1e3 + 7.0
    for stride in (2, 4):
        sums = base[:, :, :stride].contiguous().cuda()
        wire = ops.syncbn_combine(sums, stride, 1234.0)
        ref = sums[0, :, :2].clone()
        for i in range(1, n):
            ref = ref + sums[i, :, :2]
        assert wire.shape == (2 * c + 1,) and wire.dtype == torch.float64
        assert torch.equal(wire[:2 * c].view(c, 2), ref), stride
        assert float(wire[2 * c]) == 1234.0


@pytest.mark.parametrize("storage", STORAGES, ids=["bf16", "fp16"])
def test_split_batch_forward_statistics_match_the_full_batch(storage):
    from hrviton_b200 import ops
    from hrviton_b200.ops import Act
    g = torch.Generator().manual_seed(SEED)
    n, h, w, c, c_run = 4, 12, 10, 40, 37
    x = (torch.randn(n, h, w, c, generator=g) * torch.linspace(0.5, 3.0, c) + torch.linspace(-1.0, 2.0, c)).to(storage)
    rm0 = torch.randn(c_run, generator=g) * 0.1
    rv0 = torch.rand(c_run, generator=g) + 0.5
    eps, mom = 1e-5, 0.1
    xa, xb = x[:2].contiguous().cuda(), x[2:].contiguous().cuda()
    # rank "a" contributes its wire buffer; rank "b" adds it to its own (the all-reduce of two ranks) and finalizes
    wires = []
    ops.batchnorm_stats_sync(Act(xa), eps, wires.append)
    rm, rv = rm0.clone().cuda(), rv0.clone().cuda()
    mean_nc, rstd_nc = ops.batchnorm_stats_sync(Act(xb), eps, lambda wire: wire.add_(wires[0]), rm, rv, mom)
    assert mean_nc.shape == (2, c) and torch.equal(mean_nc[0], mean_nc[1]) and torch.equal(rstd_nc[0], rstd_nc[1])
    xf = x.double().reshape(-1, c)
    mean_ref = xf.mean(0)
    var_ref = xf.var(0, unbiased=False)
    rstd_ref = 1.0 / torch.sqrt(var_ref + eps)
    mean, rstd = mean_nc[0].cpu().double(), rstd_nc[0].cpu().double()
    assert ((mean - mean_ref).abs() <= _ulp(mean_ref)).all(), (mean - mean_ref).abs().max()
    assert ((rstd - rstd_ref).abs() <= 2 * _ulp(rstd_ref)).all(), ((rstd - rstd_ref).abs() / _ulp(rstd_ref)).max()
    # running statistics: torch's BatchNorm2d update on the same (storage-rounded) full batch
    bn = nn.BatchNorm2d(c_run, eps=eps, momentum=mom).cuda().train()
    with torch.no_grad():
        bn.running_mean.copy_(rm0)
        bn.running_var.copy_(rv0)
        bn(x[..., :c_run].float().permute(0, 3, 1, 2).contiguous().cuda())
    assert torch.allclose(rm, bn.running_mean, rtol=1e-5, atol=1e-6), (rm - bn.running_mean).abs().max()
    assert torch.allclose(rv, bn.running_var, rtol=1e-5, atol=1e-6), (rv - bn.running_var).abs().max()


def test_split_batch_backward_means_match_the_full_batch():
    from hrviton_b200 import capi, ops
    g = torch.Generator().manual_seed(SEED + 1)
    n, c, hw = 4, 24, 96
    sums = torch.randn(n, c, 4, generator=g, dtype=torch.float64) * 50.0
    wa = ops.syncbn_combine(sums[:2].contiguous().cuda(), 4, 2 * hw)
    wb = ops.syncbn_combine(sums[2:].contiguous().cuda(), 4, 2 * hw)
    wb.add_(wa)
    m1 = torch.empty(2, c, device="cuda")
    m2 = torch.empty_like(m1)
    capi.check(capi.lib().hrv_syncbn_bwd_finalize(wb.data_ptr(), 2, c, m1.data_ptr(), m2.data_ptr(), ops._stream()), "bwd_finalize")
    tot = sums.sum(0) / float(n * hw)
    assert torch.equal(m1.cpu(), tot[:, 0].float().expand(2, c)) and torch.equal(m2.cpu(), tot[:, 1].float().expand(2, c))


# ------------------------------------------------------------------------------------------------ shared model set-up

def _tocg(norm_layer, ngf=96):
    import networks
    from helpers import tocg_opt
    from hrviton_b200 import synth
    m = networks.ConditionGenerator(tocg_opt(True), 4, 16, 13, ngf=ngf, norm_layer=norm_layer)
    sd = m.state_dict()
    synth.fill_state_dict(sd, SEED)
    m.load_state_dict(sd)
    return m.cuda().train()


def _tocg_batch(n, h, w):
    from hrviton_b200 import synth
    i1, i2 = synth.tocg_inputs(n, h, w, SEED)
    gen = torch.Generator().manual_seed(SEED + 2)
    target = torch.rand(n, 3, h, w, generator=gen)
    labels = torch.randint(0, 13, (n, h, w), generator=gen)
    return i1, i2, target, labels


def _fixed_loss(model, i1, i2, target, labels):
    """Train-mode forward, L1 of the warped cloth to a seeded target + cross-entropy of the segmentation, backward."""
    from hrviton_b200 import train_step
    _, seg, warped_c, _ = model(i1.cuda(), i2.cuda())
    loss = F.l1_loss(warped_c, target.cuda()) + train_step.cross_entropy_ignore(seg, labels.cuda())
    loss.backward()
    torch.cuda.synchronize()
    return float(loss)


def _bn_stats(m):
    return {k: v.detach().cpu().clone() for k, v in m.state_dict().items() if "running_" in k}


def _run_children(mode, world, tmp_path, extra=(), timeout=900):
    env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8")
    init = tmp_path / "_".join(["init", mode] + list(extra))  # a fresh rendezvous file per run
    procs = [subprocess.Popen([sys.executable, "-s", os.path.abspath(__file__), mode, str(r), str(world), str(init), str(tmp_path)] + list(extra),
                              env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True) for r in range(world)]
    outs = []
    try:
        for p in procs:
            outs.append(p.communicate(timeout=timeout)[0])
    finally:
        for p in procs:
            if p.poll() is None:
                p.kill()
                p.wait()
    for r, (p, o) in enumerate(zip(procs, outs)):
        assert p.returncode == 0, "rank %d failed:\n%s" % (r, o[-6000:])
    return [torch.load(tmp_path / ("%s_%d.pt" % (mode, r))) for r in range(world)]


# ------------------------------------------------------------------------------------------------ (b) one process

def _ws1_child(out_dir):
    import networks
    from hrviton_b200 import ddp, train_step
    os.environ["HRV_VGG_RANDOM_INIT"] = "1"
    assert ddp.syncbn_group() is None

    def run(norm_layer):
        torch.manual_seed(0)
        tocg = _tocg(norm_layer)
        with contextlib.redirect_stdout(io.StringIO()):
            D = networks.define_D(input_nc=33, Ddownx2=True, Ddropout=True, n_layers_D=3, spectral=False, num_D=2)
        D = D.cuda().train()
        tr = train_step.Stage1Trainer(tocg, D, networks.Vgg19().cuda().eval())
        batch = train_step.synthetic_batch_stage1(2, 256, 192, "cuda", seed=9)
        outs = [tr.step(batch) for _ in range(3)]
        tr.capture(batch)
        outs += [tr.replay(batch) for _ in range(3)]
        torch.cuda.synchronize()
        t = {"tocg." + k: v for k, v in tocg.state_dict().items()}
        t.update({"D." + k: v for k, v in D.state_dict().items()})
        for on, o in (("opt_g", tr.opt_g), ("opt_d", tr.opt_d)):
            for i, s in enumerate(o.state.values()):
                t.update({"%s.%d.%s" % (on, i, k): v for k, v in s.items() if torch.is_tensor(v)})
        for i, out in enumerate(outs):
            t.update({"loss%d.%s" % (i, k): v for k, v in out.items()})
        tr.release_graph()
        return {k: v.detach().cpu().clone() for k, v in t.items()}

    torch.save({"plain": run(nn.BatchNorm2d), "sync": run(ddp.SynchronizedBatchNorm2d)}, os.path.join(out_dir, "ws1_0.pt"))


def test_world_size_one_is_bit_identical_to_batchnorm(tmp_path):
    (res,) = _run_children("ws1", 1, tmp_path, timeout=1500)
    a, b = res["plain"], res["sync"]
    assert a.keys() == b.keys() and any("running_var" in k for k in a) and any(k.startswith("opt_g") for k in a)
    bits = lambda t: t.reshape(-1).view(torch.uint8) if t.dtype != torch.bool else t
    diff = [k for k in a if not torch.equal(bits(a[k]), bits(b[k]))]
    assert not diff, diff[:10]


# ------------------------------------------------------------------------------------------------ (c) two processes, one GPU, gloo

def _gloo_child(rank, world, init, out_dir, kind):
    import torch.distributed as dist
    import sync_batchnorm
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", init_method="file://" + init, rank=rank, world_size=world)
    try:
        tocg = _tocg(nn.BatchNorm2d)
        if kind == "sync":
            tocg = sync_batchnorm.convert_model(tocg)
            assert sum(isinstance(m, sync_batchnorm.SynchronizedBatchNorm2d) for m in tocg.modules()) == 34
        wrapped = sync_batchnorm.DataParallelWithCallback(tocg, device_ids=[0])
        i1, i2, target, labels = _tocg_batch(2 * world, 128, 96)
        sl = slice(2 * rank, 2 * rank + 2)
        loss = _fixed_loss(wrapped, i1[sl], i2[sl], target[sl], labels[sl])
        grads = {k: p.grad.detach().cpu().clone() for k, p in tocg.named_parameters() if p.grad is not None}
        torch.save({"loss": loss, "grads": grads, "stats": _bn_stats(tocg)}, os.path.join(out_dir, "gloo_%d.pt" % rank))
    finally:
        dist.destroy_process_group()


def _grad_rel(g, ref):
    return {k: float((g[k] - r).norm() / (r.norm() + 1e-20)) for k, r in ref.items() if float(r.norm()) >= 1e-6}


def test_two_ranks_on_gloo_equal_one_process_on_the_whole_batch(tmp_path):
    torch.cuda.set_device(0)
    ref_model = _tocg(nn.BatchNorm2d)
    i1, i2, target, labels = _tocg_batch(4, 128, 96)
    ref_loss = _fixed_loss(ref_model, i1, i2, target, labels)
    ref_grads = {k: p.grad.detach().cpu() for k, p in ref_model.named_parameters() if p.grad is not None}
    ref_stats = _bn_stats(ref_model)

    r0, r1 = _run_children("gloo", 2, tmp_path, extra=["sync"])
    # negative control: per-rank BatchNorm statistics on the same two shards
    p0, p1 = _run_children("gloo", 2, tmp_path, extra=["plain"])
    loss = 0.5 * (r0["loss"] + r1["loss"])
    rel = _grad_rel(r0["grads"], ref_grads)
    worst = max(rel.items(), key=lambda kv: kv[1])
    rel_plain = _grad_rel(p0["grads"], ref_grads)
    bn_params = [k for k in rel_plain if ".block.1." in k or ".block.4." in k]
    miss = max(rel_plain[k] for k in bn_params)
    print("SYNCBN gloo 2x2 vs 1x4: loss %.7f vs %.7f (plain BatchNorm on 2 ranks: %.7f), worst gradient rel diff %.3e (%s); plain "
          "BatchNorm on 2 ranks: %.3e" % (loss, ref_loss, 0.5 * (p0["loss"] + p1["loss"]), worst[1], worst[0], miss))
    assert abs(loss - ref_loss) <= 1e-5 * abs(ref_loss), (r0["loss"], r1["loss"], ref_loss)
    assert r0["stats"].keys() == ref_stats.keys() and len(ref_stats) == 68
    for k, v in ref_stats.items():
        assert torch.equal(r0["stats"][k], r1["stats"][k]), k
        assert torch.allclose(r0["stats"][k], v, rtol=1e-6, atol=1e-6), (k, float((r0["stats"][k] - v).abs().max()))
    for k in r0["grads"]:
        assert torch.equal(r0["grads"][k], r1["grads"][k]), k  # both ranks hold the same averaged gradient
    assert r0["grads"].keys() == ref_grads.keys()
    assert worst[1] < GRAD_BOUND, worst
    assert len(bn_params) == 68
    assert miss >= 10 * GRAD_BOUND, miss


# ------------------------------------------------------------------------------------------------ (d) two GPUs, NCCL

def _nccl_child(rank, world, init, out_dir):
    import networks
    import torch.distributed as dist
    from hrviton_b200 import ddp, train_step
    os.environ["HRV_VGG_RANDOM_INIT"] = "1"
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", init_method="file://" + init, rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        vgg = networks.Vgg19().cuda().eval()
        batch = train_step.synthetic_batch_stage1(2, 256, 192, "cuda", seed=40 + rank)

        def trainer():
            torch.manual_seed(0)
            tocg = _tocg(ddp.SynchronizedBatchNorm2d)
            with contextlib.redirect_stdout(io.StringIO()):
                D = networks.define_D(input_nc=33, Ddownx2=True, Ddropout=False, n_layers_D=3, spectral=False, num_D=2)
            D = D.cuda().train()
            ddp.broadcast_module_state(tocg)
            ddp.broadcast_module_state(D)
            reducers = {"G": ddp.GradBucketReducer(list(tocg.parameters())), "D": ddp.GradBucketReducer(list(D.parameters()))}
            return tocg, train_step.Stage1Trainer(tocg, D, vgg, reducers=reducers)

        tocg_e, tr_e = trainer()
        eager = [tr_e.step(batch) for _ in range(3)]
        torch.cuda.synchronize()
        tocg_g, tr_g = trainer()
        tr_g.capture(batch)  # two eager warm-up steps, then the captured one
        replay = tr_g.replay(batch)
        torch.cuda.synchronize()
        res = {"eager_loss": {k: v.cpu() for k, v in eager[-1].items()}, "replay_loss": {k: v.cpu() for k, v in replay.items()},
               "eager": {k: v.detach().cpu().clone() for k, v in tocg_e.state_dict().items()},
               "replay": {k: v.detach().cpu().clone() for k, v in tocg_g.state_dict().items()}}
        tr_g.release_graph()
        torch.save(res, os.path.join(out_dir, "nccl_%d.pt" % rank))
    finally:
        dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpus_graph_replay_equals_eager_step(tmp_path):
    r0, r1 = _run_children("nccl", 2, tmp_path, timeout=1500)
    for r in (r0, r1):
        for k in r["eager_loss"]:
            assert torch.equal(r["eager_loss"][k], r["replay_loss"][k]), k
        for k in r["eager"]:
            assert torch.equal(r["eager"][k], r["replay"][k]), k
    for k in r0["replay"]:
        if "running_" in k:
            assert torch.equal(r0["replay"][k], r1["replay"][k]), k


if __name__ == "__main__":
    mode, rank, world, init, out = sys.argv[1], int(sys.argv[2]), int(sys.argv[3]), sys.argv[4], sys.argv[5]
    if mode == "ws1":
        _ws1_child(out)
    elif mode == "gloo":
        _gloo_child(rank, world, init, out, sys.argv[6])
    else:
        _nccl_child(rank, world, init, out)
