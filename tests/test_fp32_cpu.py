"""CPU: the fp32 reference-precision inference mode — the static shape of its convolution kernel, the rounding model that makes the
3xTF32 split necessary, and the Python-side switches (ops.set_precision("fp32"), HRV_PRECISION, the refusal to train)."""
import os
import re
import shutil
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "..", "oracle"))
import hrviton_oracle as orc  # noqa: E402
from helpers import load_golden, maxdiff, synth_state_dict  # noqa: E402
from hrviton_b200 import ops, synth, train_step  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO = os.path.join(ROOT, "hr-viton_b200", "libhrviton_sm100.so")
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
needs_lib = pytest.mark.skipif(not (os.path.exists(SO) and os.path.exists(CUOBJDUMP)), reason="needs the built library and cuobjdump")


# ------------------------------------------------------------------------------------------------ SASS of the 3xTF32 kernel

@needs_lib
def test_tf32x3_kernel_is_tf32_wgmma_tma_without_spills():
    out = subprocess.run([CUOBJDUMP, "-sass", SO], capture_output=True, text=True, check=True).stdout
    funcs, cur = {}, None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            funcs[cur] = []
        elif cur is not None:
            m = re.search(r"/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Za-z0-9_.]*)", line)  # keeps the shape (64x64x8)
            if m:
                funcs[cur].append(m.group(1))
    res = subprocess.run([CUOBJDUMP, "--dump-resource-usage", SO], capture_output=True, text=True, check=True).stdout
    stacks = {f: int(s) for f, s in re.findall(r"Function (\S+):\s*\n\s*REG:\d+ STACK:(\d+)", res)}
    for bnt in (64, 128):
        names = [n for n in funcs if "conv_tf32x3_kernelILi%d" % bnt in n]
        assert len(names) == 1, (bnt, names)
        ops_ = funcs[names[0]]
        assert any(re.match(r"HGMMA\.64x%dx8\.F32\.TF32" % bnt, o) for o in ops_), (bnt, "no TF32 wgmma")
        assert any(o.startswith("UTMALDG") for o in ops_), (bnt, "no TMA tensor load")
        assert any(o.startswith("SYNCS") for o in ops_), (bnt, "no mbarrier")
        assert not any(o.startswith("HMMA") for o in ops_), (bnt, "legacy tensor-core instructions")
        assert stacks[names[0]] == 0, (bnt, "stack frame: local-memory spills")


# ------------------------------------------------------------------------------------------------ the rounding model

def rna_tf32(t):
    """fp32 -> TF32 (10 mantissa bits), round to nearest, ties away from zero (cvt.rna.tf32.f32)."""
    b = t.float().contiguous().view(torch.int32)
    mag = (b & 0x7FFFFFFF) + 0x1000
    return ((mag & ~0x1FFF) | (b & ~0x7FFFFFFF)).view(torch.float32)


def conv_tf32x1(x, w, b=None, stride=1, padding=0):
    return F.conv2d(rna_tf32(x), rna_tf32(w), b, stride=stride, padding=padding)


def conv_tf32x3(x, w, b=None, stride=1, padding=0):
    xh, wh = rna_tf32(x), rna_tf32(w)
    xl, wl = rna_tf32(x - xh), rna_tf32(w - wh)
    c = lambda p, q: F.conv2d(p, q, None, stride=stride, padding=padding)
    y = (c(xl, wh) + c(xh, wl)) + c(xh, wh)
    return y if b is None else y + b[None, :, None, None]


def _tocg_dev(conv, monkeypatch):
    monkeypatch.setattr(orc, "conv2d_q", conv)
    g = load_golden("tocg_256x192_b1")
    n, h, w = [int(v) for v in g["shape"]]
    seed = int(g["seed"])
    i1, i2 = synth.tocg_inputs(n, h, w, seed)
    with torch.no_grad():
        flows, seg, wc, wcm = orc.tocg_forward(synth_state_dict("tocg", seed), i1, i2)
    return max([maxdiff(seg, g["seg"]), maxdiff(wc, g["warped_c"])] + [maxdiff(f, g["flow%d" % i]) for i, f in enumerate(flows)])


def _gen_dev(conv, monkeypatch):
    monkeypatch.setattr(orc, "conv2d_q", conv)
    g = load_golden("gen_256x256_b2")
    n, h, w = [int(v) for v in g["shape"]]
    seed = int(g["seed"])
    x, seg = synth.gen_inputs(n, h, w, seed)
    cnt = [0]

    def noise(b, hh, ww):
        t = synth.spade_noise(b, hh, ww, seed, cnt[0])
        cnt[0] += 1
        return t

    with torch.no_grad():
        out = orc.spade_generator_forward(synth_state_dict("gen", seed), x, seg, noise)
    return maxdiff(out, g["out"].astype("float32"))


@pytest.mark.parametrize("which", ["tocg_256x192_b1", "gen_256x256_b2"])
def test_one_tf32_pass_misses_1e3_and_three_pass_split_meets_it(which, monkeypatch):
    """The design decision behind the fp32 mode: the oracle with its convolutions in one TF32 pass (operands rounded to TF32, fp32
    sums) leaves the 1e-3 tolerance against the fp32 goldens; with the hi/lo split (hi*hi + hi*lo + lo*hi) it stays inside it."""
    dev = _tocg_dev if which.startswith("tocg") else _gen_dev
    one = dev(conv_tf32x1, monkeypatch)
    three = dev(conv_tf32x3, monkeypatch)
    print("ROUNDING %s max|d| vs golden: 1xTF32 %.3e  3xTF32 %.3e" % (which, one, three))
    assert one > 1e-3
    assert three < 1e-3


def test_rna_tf32_model():
    x = torch.tensor([1.0, 1.0 + 2.0 ** -11, 1.0 + 3 * 2.0 ** -11, -(1.0 + 2.0 ** -11), 3.0e-3, 0.0])
    r = rna_tf32(x)
    assert r[0] == 1.0 and r[1] == 1.0 + 2.0 ** -10 and r[2] == 1.0 + 2.0 ** -9 and r[3] == -(1.0 + 2.0 ** -10) and r[5] == 0.0  # ties away
    assert (r.view(torch.int32) & 0x1FFF).eq(0).all()
    y = torch.randn(10000, generator=torch.Generator().manual_seed(0))
    hi = rna_tf32(y)
    lo = rna_tf32(y - hi)
    assert float(((hi + lo - y).abs() / y.abs()).max()) < 2.0 ** -21


# ------------------------------------------------------------------------------------------------ Python switches

def test_set_precision_fp32_switches_storage_and_invalidates_caches():
    gen = ops.PARAM_GEN[0]
    try:
        ops.set_precision("fp32")
        assert ops.STORAGE[0] == torch.float32 and ops.get_precision() == "fp32"
        assert ops.PARAM_GEN[0] == gen + 1
        ops.set_precision("fp32")
        assert ops.PARAM_GEN[0] == gen + 1
    finally:
        ops.set_precision("bf16")
    assert ops.get_precision() == "bf16" and ops.STORAGE[0] == torch.bfloat16 and ops.PARAM_GEN[0] == gen + 2
    with pytest.raises(ValueError):
        ops.set_precision("fp64")


def test_precision_from_environment():
    code = "import hrv_loader; hrv_loader.load(); from hrviton_b200 import ops; print(ops.get_precision())"
    env = dict(os.environ)
    for want in ("fp32", "fp16", "bf16"):
        env["HRV_PRECISION"] = want
        r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, capture_output=True, text=True, timeout=300)
        assert r.returncode == 0, r.stderr
        assert r.stdout.strip().splitlines()[-1] == want
    env.pop("HRV_PRECISION")
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, capture_output=True, text=True, timeout=300)
    assert r.stdout.strip().splitlines()[-1] == "bf16"


def test_trainers_refuse_fp32_storage():
    ops.set_precision("fp32")
    try:
        with pytest.raises(NotImplementedError, match="fp32 storage is inference-only"):
            object.__new__(train_step.Stage2Trainer).step(None, 0, 0)
        with pytest.raises(NotImplementedError, match="fp32 storage is inference-only"):
            object.__new__(train_step.Stage1Trainer).step(None)
    finally:
        ops.set_precision("bf16")
