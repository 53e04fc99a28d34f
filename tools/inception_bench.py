"""Inception-v3 on the kernels (hrviton_b200.metrics.InceptionV3) against torchvision's Inception3 on cuDNN, and the end-to-end time of
FID and KID for two sets of synthetic 1024x768 images.

    python tools/inception_bench.py [--batches 1,50] [--iters 20] [--rounds 3] [--images 2048] [--out DIR]

- Features per second at 299x299 for each batch size: both arms on the same seeded weights and inputs, arms alternated round by round,
  CUDA events around `iters` calls after a warm-up.  The torch arm runs with torch's defaults, which let cuDNN run convolutions in TF32
  (torch.backends.cudnn.allow_tf32); the package runs 3xTF32 (fp32-class).  The weights are seeded (tests/inception_oracle.py): the
  ImageNet ones cannot be fetched offline, and the arithmetic is the same.
- FID / KID end to end: `images` + `images` synthetic 1024x768 images in [0, 1], generated on the device in batches of 50, resized on the
  way in, pool features streamed into FeatureStats and kept for KID (100 subsets of 1000).  The generation is timed with the rest.
The card's name and power limit are read in the same run and printed with the numbers; one JSON line per result."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import hrv_loader  # noqa: E402

hrv_loader.load()
import torch  # noqa: E402

import inception_oracle  # noqa: E402
from hrviton_b200 import metrics  # noqa: E402


def card():
    name = torch.cuda.get_device_name(0)
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30)
        power = r.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def timed(fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,50")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--images", type=int, default=2048)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("inception_bench needs a GPU")
    name, power = card()
    model = inception_oracle.seeded_inception(seed=3).cuda().eval()
    net = metrics.InceptionV3.from_torchvision(model)
    results = []
    g = torch.Generator(device="cuda").manual_seed(0)
    with torch.no_grad():
        for b in [int(v) for v in a.batches.split(",")]:
            x = torch.rand((b, 3, 299, 299), generator=g, device="cuda") * 2 - 1
            arms = {"hrviton_3xtf32": lambda: net(x), "torch_cudnn": lambda: model(x)}
            for f in arms.values():  # warm-up: module loads, cuDNN algorithm choice
                timed(f, 3)
            ms = {k: [] for k in arms}
            for _ in range(a.rounds):
                for k, f in arms.items():
                    ms[k].append(timed(f, a.iters))
            ref = model(x)
            d = float((net(x)[1] - ref).abs().max() / ref.abs().max())
            for k, v in ms.items():
                results.append({"bench": "inception_features", "arm": k, "batch": b, "ms_per_call": [round(t, 3) for t in v],
                                "images_per_s_best": round(b * 1000.0 / min(v), 1), "max_rel_logit_diff_vs_torch": d,
                                "torch_cudnn_allow_tf32": torch.backends.cudnn.allow_tf32, "gpu": name, "power_limit": power})
                print(json.dumps(results[-1]), flush=True)

        # FID / KID end to end on 1024x768 images
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        feats, stats = [], []
        for s in range(2):
            st = metrics.FeatureStats()
            gs = torch.Generator(device="cuda").manual_seed(100 + s)
            fs = []
            for i in range(0, a.images, 50):
                x = torch.rand((min(50, a.images - i), 3, 1024, 768), generator=gs, device="cuda")
                if s:
                    x = x * 0.8 + 0.1
                pool, _ = net(x, unit_range=True)
                st.update(pool)
                fs.append(pool.clone())
            feats.append(torch.cat(fs))
            stats.append(st)
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        f = float(metrics.fid(stats[0], stats[1]))
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        km, ks = metrics.kid(feats[0], feats[1], subsets=100, subset_size=1000)
        km, ks = float(km), float(ks)
        t3 = time.perf_counter()
        results.append({"bench": "fid_kid_end_to_end", "images_per_set": a.images, "size": "1024x768", "features_s": round(t1 - t0, 3),
                        "fid_s": round(t2 - t1, 3), "kid_s": round(t3 - t2, 3), "total_s": round(t3 - t0, 3), "fid": f, "kid": km, "kid_std": ks,
                        "gpu": name, "power_limit": power})
        print(json.dumps(results[-1]), flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "inception_bench.json"), "w") as fh:
            json.dump(results, fh, indent=1)


if __name__ == "__main__":
    main()
