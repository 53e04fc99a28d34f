"""Generates tests/golden/lpips_alex.npz and tests/golden/lpips_keys.json: LPIPS (the reference's eval_models PNetLin, AlexNet, v0.1
heads) run UNMODIFIED on the CPU in fp32, eval mode, with seeded weights.  Run where the reference checkout exists:

    python tests/golden/make_golden_lpips.py

Weights: hrviton_b200.synth.fill_state_dict(sd, SEED) on every AlexNet and head tensor (deterministic, so the tests rebuild the same
state_dict from the seed instead of storing 10 MB of it; the per-tensor fp64 sums are stored and checked), the heads made non-negative
as trained LPIPS heads are, the ScalingLayer buffers left as the reference defines them.  Inputs are 8-bit images mapped to [-1, 1] as
x = u8 / 127.5 - 1 (stored as uint8): 128x128 at batch 4, 96x160 at batch 2, and one identical pair.  Stored per case: the inputs, the
per-layer distances res[0..4] (N,) as each layer produced them, and the total."""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg  # noqa: E402  (repo root on sys.path, package loaded)
from hrviton_b200 import synth  # noqa: E402

SEED = 61
CASES = {"b4_128x128": (4, 128, 128, 1), "b2_96x160": (2, 96, 160, 2), "same_128x128": (1, 128, 128, 3)}


def seeded_state_dict(sd):
    """Fill a PNetLin(alex) state_dict in place: the tests call this on the drop-in's state_dict."""
    synth.fill_state_dict({k: v for k, v in sd.items() if not k.startswith("scaling_layer.")}, SEED)
    for k in sd:
        if k.startswith("lin"):
            sd[k].abs_()
    return sd


def images(n, h, w, seed):
    """A pair of related 8-bit image batches (N,3,H,W): blocky random content and the same content with independent pixel noise."""
    rng = np.random.RandomState(seed)
    base = np.kron(rng.randint(0, 256, (n, 3, (h + 7) // 8, (w + 7) // 8)), np.ones((1, 1, 8, 8)))[:, :, :h, :w]
    a = np.clip(base + rng.randint(-12, 13, base.shape), 0, 255).astype(np.uint8)
    b = np.clip(base + rng.randint(-40, 41, base.shape), 0, 255).astype(np.uint8)
    return a, b


def to_input(u8):
    return torch.from_numpy(u8.astype(np.float32) / np.float32(127.5) - np.float32(1.0))


def main():
    torch.set_num_threads(os.cpu_count())
    import hrv_env
    hrv_env.install()  # numpy aliases and the skimage / IPython shims the reference's eval_models imports
    sys.path.insert(0, mg.REF)
    import importlib
    nb = importlib.import_module("eval_models.networks_basic")
    sys.path.remove(mg.REF)
    assert nb.__file__.startswith(mg.REF)
    net = nb.PNetLin(pnet_rand=True, pnet_type="alex", use_dropout=True, version="0.1", lpips=True).eval()
    sd = seeded_state_dict(net.state_dict())
    net.load_state_dict(sd)
    keys = [[k, list(v.shape)] for k, v in net.state_dict().items()]
    with open(os.path.join(HERE, "lpips_keys.json"), "w") as f:
        json.dump(keys, f, indent=0)
    out = {"seed": np.int64(SEED), "sd_keys": np.array([k for k, _ in keys]),
           "sd_sums": np.array([float(v.double().sum()) for v in net.state_dict().values()]),
           "sd_abs_sums": np.array([float(v.double().abs().sum()) for v in net.state_dict().values()])}
    for name, (n, h, w, seed) in CASES.items():
        a, b = images(n, h, w, seed)
        if name.startswith("same"):
            b = a.copy()
        # PNetLin.forward sums into res[0] in place (val = res[0]; val += res[l]), so the per-layer values are recorded as
        # spatial_average returns them
        res = []
        avg = nb.spatial_average
        nb.spatial_average = lambda t, keepdim=True: (lambda r: (res.append(r.clone()), r)[1])(avg(t, keepdim=keepdim))
        try:
            with torch.no_grad():
                val = net(to_input(a), to_input(b))
        finally:
            nb.spatial_average = avg
        assert len(res) == 5
        out[name + "_in0"], out[name + "_in1"] = a, b
        out[name + "_res"] = np.stack([r.reshape(-1).numpy() for r in res])  # (5, N)
        out[name + "_val"] = val.reshape(-1).numpy()
        print(name, out[name + "_val"], out[name + "_res"].min(axis=1))
    np.savez_compressed(os.path.join(HERE, "lpips_alex.npz"), **out)
    print("wrote", os.path.join(HERE, "lpips_alex.npz"))


if __name__ == "__main__":
    main()
