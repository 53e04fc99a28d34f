"""GPU: try-on inference replayed from CUDA graphs (pipeline.TryOnGraph, pipeline.GeneratorGraph).  A replay must equal the eager
call bit for bit — tryon_forward for the pipeline, generator(x, seg) under no_grad for the generator — for fresh inputs on every
call, advance torch's CUDA generator exactly as the eager call does, and never replay a graph captured under weights or a storage
precision that have changed since."""
import pytest
import torch

from helpers import gen_opt, synth_state_dict, tocg_opt
from hrviton_b200 import ops, pipeline, synth, train_step

pytestmark = pytest.mark.gpu

H, W = 512, 384
SEED = 23


@pytest.fixture(scope="module")
def nets():
    import network_generator
    import networks
    tocg = networks.ConditionGenerator(tocg_opt(True), 4, 16, 13, ngf=96, norm_layer=torch.nn.BatchNorm2d)
    tocg.load_state_dict(synth_state_dict("tocg", SEED))
    G = network_generator.SPADEGenerator(gen_opt(H, W, True), 9)
    G.load_state_dict(synth_state_dict("gen", SEED + 1))
    return tocg.cuda().eval(), G.cuda().eval()


@pytest.fixture(autouse=True)
def _restore():
    yield
    ops.set_precision("bf16")
    ops.PROFILE = None


def _batch(n, seed, h=H, w=W):
    b = train_step.synthetic_batch(n, h, w, "cuda", seed=seed)
    del b["image"]
    return b


def _gen_inputs(n, seed, h=H, w=W):
    x, seg = synth.gen_inputs(n, h, w, seed)
    return x.cuda(), seg.cuda()


def _table_noise(G, n):
    """Installs a noise_source that serves fixed device tensors: the k-th draw at shape (n, h, w) of a forward reads table[(n, h,
    w)][k].  Nothing is copied from the host inside the call, so the source is valid during a capture too."""
    shapes = []
    G.noise_source = lambda b, hh, ww: shapes.append((b, hh, ww)) or torch.zeros(b, hh, ww, device="cuda")
    with torch.no_grad():
        G(*_gen_inputs(n, 0))
    table = {}
    for i, s in enumerate(shapes):
        table.setdefault(s, []).append(synth.spade_noise(*s, SEED, i).cuda())
    count = {s: 0 for s in table}

    def source(b, hh, ww):
        s = (b, hh, ww)
        t = table[s][count[s] % len(table[s])]
        count[s] += 1
        return t
    G.noise_source = source
    torch.cuda.synchronize()


def _eager(tocg, G, inputs, **kw):
    return tuple(t.clone() for t in pipeline.tryon_forward(tocg, G, inputs, **kw))


def _assert_equal(got, ref):
    for i, (a, b) in enumerate(zip(got, ref)):
        assert torch.equal(a, b), "output %d: max|d| %.3e" % (i, float((a.float() - b.float()).abs().max()))


@pytest.mark.parametrize("precision", ["bf16", "fp16", "fp32"])
@pytest.mark.parametrize("n", [1, 3])
@pytest.mark.parametrize("occlusion,composition", [(True, "warp_grad"), (True, "detach"), (False, "warp_grad"), (False, "detach")])
def test_tryon_graph_equals_eager(nets, precision, n, occlusion, composition):
    tocg, G = nets
    ops.set_precision(precision)
    _table_noise(G, n)
    runner = pipeline.TryOnGraph(tocg, G, occlusion=occlusion, clothmask_composition=composition)
    try:
        inputs = _batch(n, 5)
        ref = _eager(tocg, G, inputs, occlusion=occlusion, clothmask_composition=composition)
        _assert_equal(runner(inputs), ref)  # captured on this call
        _assert_equal(runner(inputs), ref)  # replayed
        # the {setting: tensor} form of cp_dataset_test's cloth / cloth_mask
        d = dict(inputs, cloth={"paired": inputs["cloth"]}, cloth_mask={"paired": inputs["cloth_mask"]})
        _assert_equal(runner(d), ref)
        assert len(runner._graphs) == 1
    finally:
        runner.release()
        G.noise_source = None


@pytest.fixture(scope="module")
def gen_1024(nets):
    import network_generator
    G = network_generator.SPADEGenerator(gen_opt(1024, 768, True), 9)
    G.load_state_dict(nets[1].state_dict())
    return G.cuda().eval()


@pytest.mark.parametrize("precision", ["bf16", "fp16", "fp32"])
@pytest.mark.parametrize("n,h,w", [(1, H, W), (3, H, W), (1, 1024, 768)])
def test_generator_graph_equals_eager(nets, gen_1024, precision, n, h, w):
    G = gen_1024 if h == 1024 else nets[1]
    ops.set_precision(precision)
    _table_noise(G, n)
    runner = pipeline.GeneratorGraph(G)
    try:
        x, seg = _gen_inputs(n, 7, h, w)
        with torch.no_grad():
            ref = G(x, seg).clone()
        for _ in range(2):
            out = runner(x, seg)
            assert torch.equal(out, ref), float((out - ref).abs().max())
    finally:
        runner.release()
        G.noise_source = None


def test_fresh_inputs_every_call(nets):
    tocg, G = nets
    _table_noise(G, 2)
    tryon, gen = pipeline.TryOnGraph(tocg, G), pipeline.GeneratorGraph(G)
    try:
        outs = []
        for seed in (1, 2, 3):
            inputs = _batch(2, seed)
            got = tuple(t.clone() for t in tryon(inputs))
            _assert_equal(got, _eager(tocg, G, inputs))
            outs.append(got[0])
            x, seg = _gen_inputs(2, seed)
            with torch.no_grad():
                ref = G(x, seg)
            assert torch.equal(gen(x, seg), ref)
        assert not torch.equal(outs[0], outs[1]) and not torch.equal(outs[1], outs[2])
        assert len(tryon._graphs) == 1 and len(gen._graphs) == 1
    finally:
        tryon.release()
        gen.release()
        G.noise_source = None


@pytest.mark.parametrize("which", ["tryon", "generator"])
def test_torch_rng_matches_eager(nets, which):
    tocg, G = nets
    assert G.noise_source is None
    inputs = _batch(1, 4)
    x, seg = _gen_inputs(1, 4)
    if which == "tryon":
        runner = pipeline.TryOnGraph(tocg, G)
        graph_call = lambda: runner(inputs)[0].clone()
        eager_call = lambda: _eager(tocg, G, inputs)[0]
    else:
        runner = pipeline.GeneratorGraph(G)
        graph_call = lambda: runner(x, seg).clone()

        def eager_call():
            with torch.no_grad():
                return G(x, seg).clone()
    try:
        for s in (11, 12):  # the first call captures (its warm-up must not consume random numbers), the second replays
            torch.cuda.manual_seed(s)
            g1, g2 = graph_call(), graph_call()
            state_g = torch.cuda.get_rng_state()
            torch.cuda.manual_seed(s)
            e1, e2 = eager_call(), eager_call()
            state_e = torch.cuda.get_rng_state()
            assert torch.equal(g1, e1) and torch.equal(g2, e2)
            assert not torch.equal(g1, g2)  # fresh noise on every replay, as on every eager call
            assert torch.equal(state_g, state_e)
    finally:
        runner.release()


def _edit(kind, tocg, G):
    """Changes the weights (or the precision) behind a captured graph; returns a function that undoes it."""
    if kind == "precision":
        ops.set_precision("fp16")
        return lambda: ops.set_precision("bf16")
    if kind == "load_state_dict":
        sd = {k: v.clone() for k, v in G.state_dict().items()}
        G.load_state_dict(synth_state_dict("gen", SEED + 7))
        return lambda: G.load_state_dict(sd)
    if kind == "inplace":  # a SPADE modulation weight (not spectrally normalised: a uniform scale of those cancels in W / sigma)
        edited = [G.up_4.norm_1.conv_gamma.weight]
    else:  # eval-mode BatchNorm of the tocg: folded into its convolution epilogues
        edited = [m.running_var for m in tocg.modules() if isinstance(m, torch.nn.BatchNorm2d)]
    saved = [t.detach().clone() for t in edited]
    with torch.no_grad():
        for t in edited:
            t.mul_(1.5)

    def undo():
        with torch.no_grad():
            for t, s in zip(edited, saved):
                t.copy_(s)
    return undo


@pytest.mark.parametrize("kind", ["load_state_dict", "inplace", "bn_stats", "precision"])
def test_changed_weights_are_recaptured(nets, kind):
    tocg, G = nets
    _table_noise(G, 1)
    runner = pipeline.TryOnGraph(tocg, G)
    undo = None
    try:
        inputs = _batch(1, 6)
        runner(inputs)
        (old,) = [e.captured for e in runner._graphs.values()]
        undo = _edit(kind, tocg, G)
        ref = _eager(tocg, G, inputs)
        stale = tuple(t.clone() for t in old.replay())  # what a graph that ignored the change would return
        assert not torch.equal(stale[0], ref[0])
        _assert_equal(runner(inputs), ref)
    finally:
        runner.release()
        if undo is not None:
            undo()
        G.noise_source = None


def test_preconditions_raise_before_capture(nets):
    tocg, G = nets
    inputs = _batch(1, 8)
    x, seg = _gen_inputs(1, 8)
    tryon, gen = pipeline.TryOnGraph(tocg, G), pipeline.GeneratorGraph(G)
    launches = ops.LAUNCHES[0]
    tocg.ClothEncoder[1].train()
    try:
        with pytest.raises(RuntimeError, match="train mode"):
            tryon(inputs)
    finally:
        tocg.eval()
    G.train()
    try:
        with pytest.raises(RuntimeError, match="train mode"):
            gen(x, seg)
    finally:
        G.eval()
    with pytest.raises(ValueError, match="parse_agnostic"):
        tryon(dict(inputs, parse_agnostic=inputs["parse_agnostic"][:, :12]))
    with pytest.raises(ValueError, match="'x'"):
        gen(x[:, :8], seg)
    with pytest.raises(ValueError, match="'cloth'"):
        tryon(dict(inputs, cloth=inputs["cloth"].cpu()))
    with pytest.raises(ValueError, match="'seg'"):
        gen(x, seg.half())
    ops.PROFILE = []
    with pytest.raises(RuntimeError, match="PROFILE"):
        tryon(inputs)
    with pytest.raises(RuntimeError, match="PROFILE"):
        gen(x, seg)
    ops.PROFILE = None
    assert ops.LAUNCHES[0] == launches and not tryon._graphs and not gen._graphs
