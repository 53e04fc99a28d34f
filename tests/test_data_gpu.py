"""GPU: the VITON-HD loader (hrviton_b200.data) — its resize kernels against PIL, every key of its batches against the reference's
collated cp_dataset / cp_dataset_test batches bit for bit, consume() against iteration, stage-2 graph training fed by the loader
against the same batches fed by hand, and TryOnGraph on a loader batch against the reference batch."""
import numpy as np
import pytest
import torch
from PIL import Image

import hrv_env
from helpers import gen_opt, tocg_opt
from hrviton_b200 import data, synth, train_step

pytestmark = pytest.mark.gpu

N_SAMPLES, BATCH = 8, 4


@pytest.fixture(scope="module")
def tree(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("vitonhd"))
    synth.write_vitonhd(root, N_SAMPLES, seed=21, datamode="train")
    synth.write_vitonhd(root, N_SAMPLES, seed=22, datamode="test", pairs="test_pairs.txt")
    return root


def test_resize_kernels_match_pil():
    rng = np.random.default_rng(3)
    for _ in range(40):
        h, w = (int(v) for v in rng.integers(2, 300, 2))
        oh, ow = (int(v) for v in rng.integers(1, 300, 2))
        if (h, w) == (oh, ow):
            continue
        for c in (1, 3):
            a = rng.integers(0, 256, (3, h, w, c) if c == 3 else (3, h, w), dtype=np.uint8)
            got = data.resize_u8(torch.from_numpy(a).cuda(), oh, ow).cpu().numpy()
            want = np.stack([np.asarray(Image.fromarray(x).resize((ow, oh), Image.BILINEAR)) for x in a])
            assert np.array_equal(got, want), ("bilinear", h, w, oh, ow, c)
            if c == 1:
                got = data.resize_u8(torch.from_numpy(a).cuda(), oh, ow, mode="nearest").cpu().numpy()
                want = np.stack([np.asarray(Image.fromarray(x).resize((ow, oh), Image.NEAREST)) for x in a])
                assert np.array_equal(got, want), ("nearest", h, w, oh, ow)


def _reference_batches(tree, datamode, data_list, fh, fw, mode):
    if hrv_env.reference_dir() is None:
        pytest.skip("no reference copy (oracle/_ref)")
    import types
    mod = hrv_env.load_reference_script("cp_dataset" if mode == "train" else "cp_dataset_test")
    opt = types.SimpleNamespace(dataroot=tree, datamode=datamode, data_list=data_list, fine_height=fh, fine_width=fw, semantic_nc=13)
    ds = mod.CPDataset(opt) if mode == "train" else mod.CPDatasetTest(opt)
    collate = torch.utils.data.default_collate
    return [collate([ds[i] for i in range(b * BATCH, (b + 1) * BATCH)]) for b in range(N_SAMPLES // BATCH)]


def _assert_batch_equal(got, want, keys):
    assert got["im_name"] == want["im_name"] and got["c_name"] == want["c_name"]
    for k in keys:
        g, w = got[k], want[k]
        for s in (w if isinstance(w, dict) else [None]):
            gs, ws = (g[s], w[s]) if s is not None else (g, w)
            assert gs.is_cuda and gs.dtype == ws.dtype and gs.shape == ws.shape, (k, s, gs.shape, ws.shape)
            assert torch.equal(gs.cpu(), ws), (k, s, float((gs.cpu() - ws).abs().max()))


@pytest.mark.parametrize("mode,fh,fw,keys", [("train", 1024, 768, None), ("train", 512, 384, None), ("train", 256, 192, None),
                                             ("test", 1024, 768, None), ("train", 512, 384, data.STAGE2_KEYS),
                                             ("test", 256, 192, data.STAGE1_KEYS)])
def test_loader_equals_reference(tree, mode, fh, fw, keys):
    datamode, data_list = ("train", "pairs.txt") if mode == "train" else ("test", "test_pairs.txt")
    want = _reference_batches(tree, datamode, data_list, fh, fw, mode)
    loader = data.VitonHDLoader(tree, datamode, data_list, fh, fw, BATCH, workers=2, mode=mode, keys=keys, shuffle=False)
    got = list(loader)
    assert len(got) == len(want) == len(loader)
    for g, w in zip(got, want):
        assert set(k for k in g if k not in ("im_name", "c_name")) == set(keys or w.keys()) - {"im_name", "c_name"}
        _assert_batch_equal(g, w, keys or [k for k in w if k not in ("im_name", "c_name")])
    assert [b["im_name"] for b in list(loader)] == [b["im_name"] for b in got]  # the next epoch, in the same order (shuffle=False)


def _flat(batch, keys):
    return {k: (batch[k]["paired"] if k in data.PAIRED_KEYS else batch[k]) for k in keys}


def test_consume_equals_iteration(tree):
    kw = dict(workers=2, keys=data.STAGE1_KEYS, seed=4)
    it = data.VitonHDLoader(tree, "train", "pairs.txt", 256, 192, 2, **kw)
    fed = data.VitonHDLoader(tree, "train", "pairs.txt", 256, 192, 2, **kw)
    out = _flat(fed.empty_batch(), data.STAGE1_KEYS)
    for _ in range(2 * len(it) + 1):  # across epoch boundaries
        want = _flat(it.next_batch(), data.STAGE1_KEYS)
        fed.consume(out)
        for k in data.STAGE1_KEYS:
            assert torch.equal(out[k], want[k]), k
    with pytest.raises(KeyError, match="not keys of a VITON-HD batch"):  # an input the loader would leave stale
        fed.consume(dict(out, warped_cloth=torch.empty_like(out["cloth"])))
    with pytest.raises(KeyError, match="built without"):
        fed.consume(dict(out, image=torch.empty_like(out["cloth"])))


def _stage2_trainer(h, w):
    import network_generator
    import networks
    torch.manual_seed(0)
    tocg = networks.ConditionGenerator(tocg_opt(True), 4, 16, 13, ngf=96, norm_layer=torch.nn.BatchNorm2d)
    sd = tocg.state_dict(); synth.fill_state_dict(sd, 3); tocg.load_state_dict(sd)
    G = network_generator.SPADEGenerator(gen_opt(h, w, True), 9)
    sd = G.state_dict(); synth.fill_state_dict(sd, 4); G.load_state_dict(sd)
    D = network_generator.MultiscaleDiscriminator(gen_opt(h, w, True))
    sd = D.state_dict(); synth.fill_state_dict(sd, 5); D.load_state_dict(sd)
    return train_step.Stage2Trainer(tocg.cuda().eval(), G.cuda().train(), D.cuda().train(), networks.Vgg19().cuda().eval())


def _save(module, path):
    """INTEGRATION.md's checkpoint save for a captured trainer: the state on the host, the module left where the graph expects it."""
    torch.save({k: v.detach().cpu() for k, v in module.state_dict().items()}, path)


def test_stage2_graph_fed_by_loader(tree, tmp_path):
    """Three loader-fed graph steps equal three steps replayed on the same batches by hand, bit for bit, also when the loader-fed run
    saves checkpoints between its steps."""
    h, w = 512, 384
    runs = []
    for feed in ("loader", "batches"):
        loader = data.VitonHDLoader(tree, "train", "pairs.txt", h, w, 2, workers=2, keys=data.STAGE2_KEYS, seed=9)
        tr = _stage2_trainer(h, w)
        tr.capture(_flat(loader.next_batch(), data.STAGE2_KEYS), h, w)
        batches = None if feed == "loader" else [_flat(loader.next_batch(), data.STAGE2_KEYS) for _ in range(3)]
        losses, saved = [], {}
        for i in range(3):
            out = tr.replay(feeder=loader) if feed == "loader" else tr.replay(batches[i])
            losses.append({k: v.detach().clone() for k, v in out.items() if torch.is_tensor(v)})
            if feed == "loader" and i < 2:  # a checkpoint between steps must not disturb the captured step
                for name, m in (("G", tr.G), ("D", tr.D)):
                    path = str(tmp_path / ("%s_%d.pth" % (name, i)))
                    _save(m, path)
                    saved[path] = {k: v.detach().clone() for k, v in m.state_dict().items()}
        torch.cuda.synchronize()
        for path, want in saved.items():
            got = torch.load(path)
            assert list(got) == list(want) and all(torch.equal(got[k], want[k].cpu()) for k in want), path
        state = {"loss%d.%s" % (i, k): v for i, l in enumerate(losses) for k, v in l.items()}
        for name, m in (("G", tr.G), ("D", tr.D)):
            state.update({name + "." + k: v.detach().clone() for k, v in m.state_dict().items()})
        tr.release_graph()
        runs.append(state)
        del tr, loader
    a, b = runs
    assert a.keys() == b.keys()
    diff = [k for k in a if not torch.equal(a[k], b[k])]
    assert not diff, diff[:10]


def test_tryon_graph_on_loader_batch(tree):
    import network_generator
    import networks
    from hrviton_b200 import pipeline
    h, w = 512, 384
    want = _reference_batches(tree, "test", "test_pairs.txt", h, w, "test")[0]
    loader = data.VitonHDLoader(tree, "test", "test_pairs.txt", h, w, BATCH, workers=2, mode="test", shuffle=False)
    got = next(iter(loader))
    tocg = networks.ConditionGenerator(tocg_opt(True), 4, 16, 13, ngf=96, norm_layer=torch.nn.BatchNorm2d)
    sd = tocg.state_dict(); synth.fill_state_dict(sd, 6); tocg.load_state_dict(sd)
    G = network_generator.SPADEGenerator(gen_opt(h, w, True), 9)
    sd = G.state_dict(); synth.fill_state_dict(sd, 7); G.load_state_dict(sd)
    runner = pipeline.TryOnGraph(tocg.cuda().eval(), G.cuda().eval())
    keys = ("cloth", "cloth_mask", "agnostic", "densepose", "parse_agnostic")

    def run(batch):
        torch.cuda.manual_seed(5)
        return [t.clone() for t in runner({k: batch[k] for k in keys})]
    try:
        run(got)  # captures
        ours = run(got)
        ref = run({k: ({s: t.cuda() for s, t in v.items()} if isinstance(v, dict) else v.cuda()) for k, v in want.items() if k in keys})
    finally:
        runner.release()
    for a, b in zip(ours, ref):
        assert torch.equal(a, b)
