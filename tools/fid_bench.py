"""pytorch-fid's FID Inception on the kernels (metrics.InceptionV3.from_fid_weights) against the same network on torch/cuDNN, and the
end-to-end time of tools/fid.py on two folders of JPEGs.

    python tools/fid_bench.py [--batches 1,50] [--iters 10] [--rounds 5] [--images 2032] [--workers N] [--out DIR]

- Images per second from uint8 1024x768 batches already on the device, arms alternated round by round, CUDA events around `iters`
  calls after a warm-up; every round is reported, so the spread is visible.  Arms:
    hrviton_fid_u8         from_fid_weights on the uint8 (N,H,W,3) batch (the input kernel divides by 255, resizes and maps to 2x - 1)
    hrviton_fid_f32        from_fid_weights on the same images as fp32 (N,3,H,W) in [0, 1]
    hrviton_torchvision    from_torchvision on the same weights and fp32 images (unit_range=True): it folds the average pools into 3x3
                           convolutions, so against hrviton_fid_f32 the stride-1 pooling passes are the only difference
    torch_cudnn_fid        the float64 oracle's architecture (tests/fid_inception_oracle.py) in fp32 on torch/cuDNN with torch's defaults,
                           from the uint8 batch: /255, F.interpolate, 2x - 1, the network
  The weights are seeded (the real ones are not fetched); the arithmetic is the same.
- tools/fid.py end to end on `images` + `images` seeded 1024x768 JPEGs (VITON-HD's test set has 2032), with --kid: weight loading,
  feature extraction (and within it the time spent waiting for decoded batches), FID and KID; and, for the decode bound, one pass of the
  tool's DataLoader alone over one folder.
The card's name and power limit are read in the same run and printed with the numbers; one JSON line per result."""
import argparse
import json
import os
import shutil
import sys
import tempfile
import time
from multiprocessing import Pool

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")]
import hrv_loader  # noqa: E402

hrv_loader.load()
import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

import fid as fid_tool  # noqa: E402
import fid_inception_oracle as fo  # noqa: E402
from hrviton_b200 import metrics  # noqa: E402
from inception_bench import card, timed  # noqa: E402

H, W = 1024, 768


def _write_jpeg(job):
    from PIL import Image
    path, seed, shift = job
    rng = np.random.RandomState(seed)
    base = np.kron(rng.randint(0, 256, (H // 32, W // 32, 3)), np.ones((32, 32, 1)))
    im = np.clip(base * (1 - shift) + 255 * shift / 2 + rng.randint(-25, 26, base.shape), 0, 255).astype(np.uint8)
    Image.fromarray(im).save(path, quality=90)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,50")
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--images", type=int, default=2032)
    ap.add_argument("--workers", type=int, default=min(8, os.cpu_count() or 1))
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("fid_bench needs a GPU")
    name, power = card()
    sd = fo.seeded_fid_state_dict(seed=4)
    net = metrics.InceptionV3.from_fid_weights(sd)
    tv = metrics.InceptionV3.from_torchvision(metrics.fid_inception_model(sd).cuda())
    model = fo.fid_network(sd, pooling="fid").cuda()

    def torch_arm(u8):
        x = u8.permute(0, 3, 1, 2).float() / 255
        return model(2 * F.interpolate(x, size=(299, 299), mode="bilinear", align_corners=False) - 1)

    results = []
    g = torch.Generator(device="cuda").manual_seed(0)
    with torch.no_grad():
        for b in [int(v) for v in a.batches.split(",")]:
            u8 = torch.randint(0, 256, (b, H, W, 3), generator=g, device="cuda", dtype=torch.uint8)
            f01 = (u8.cpu().permute(0, 3, 1, 2).float() / 255).cuda()
            arms = {"hrviton_fid_u8": lambda: net(u8), "hrviton_fid_f32": lambda: net(f01),
                    "hrviton_torchvision": lambda: tv(f01, unit_range=True), "torch_cudnn_fid": lambda: torch_arm(u8)}
            for f in arms.values():  # warm-up: module loads, cuDNN algorithm choice, weight packing
                timed(f, 3)
            ms = {k: [] for k in arms}
            for _ in range(a.rounds):
                for k, f in arms.items():
                    ms[k].append(timed(f, a.iters))
            ref = torch_arm(u8)
            d = float((net(u8)[1] - ref).abs().max() / ref.abs().max())
            for k, v in ms.items():
                results.append({"bench": "fid_inception_features", "arm": k, "batch": b, "input": "%dx%d uint8 on device" % (H, W),
                                "ms_per_call_per_round": [round(t, 3) for t in v], "images_per_s_best": round(b * 1000.0 / min(v), 1),
                                "images_per_s_worst": round(b * 1000.0 / max(v), 1), "max_rel_logit_diff_vs_torch": d,
                                "torch_cudnn_allow_tf32": torch.backends.cudnn.allow_tf32, "gpu": name, "power_limit": power})
                print(json.dumps(results[-1]), flush=True)
    del u8, f01, model
    torch.cuda.empty_cache()

    tmp = tempfile.mkdtemp(prefix="fid_bench_")
    try:
        t0 = time.perf_counter()
        jobs, dirs = [], []
        for s in range(2):
            d = os.path.join(tmp, "set%d" % s)
            os.makedirs(d)
            dirs.append(d)
            jobs += [(os.path.join(d, "%05d_00.jpg" % i), 1000 * s + i, 0.2 * s) for i in range(a.images)]
        with Pool(max(1, os.cpu_count() or 1)) as pool:
            pool.map(_write_jpeg, jobs, chunksize=16)
        gen_s = time.perf_counter() - t0
        weights = os.path.join(tmp, "pt_inception.pth")
        torch.save(sd, weights)
        loader = torch.utils.data.DataLoader(fid_tool._Images(fid_tool.image_files(dirs[0])), batch_size=50, num_workers=a.workers,
                                             collate_fn=fid_tool._collate, pin_memory=True)
        t0 = time.perf_counter()
        for _ in loader:
            pass
        decode_s = time.perf_counter() - t0
        t0 = time.perf_counter()
        res = fid_tool.main([dirs[0], dirs[1], "--weights", weights, "--kid", "--workers", str(a.workers)])
        total_s = time.perf_counter() - t0
        results.append({"bench": "fid_tool_end_to_end", "images_per_set": a.images, "size": "%dx%d JPEG q90" % (H, W), "workers": a.workers,
                        "cpus": os.cpu_count(), "total_s": round(total_s, 3), "decode_only_one_folder_s": round(decode_s, 3),
                        "jpeg_generation_s": round(gen_s, 3), **res, "gpu": name, "power_limit": power})
        print(json.dumps(results[-1]), flush=True)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "fid_bench.json"), "w") as fh:
            json.dump(results, fh, indent=1)


if __name__ == "__main__":
    main()
