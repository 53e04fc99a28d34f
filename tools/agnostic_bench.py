"""What does rasterising the agnostic shapes on the device buy?  Prints one JSON line per measurement (and writes them to
--out/agnostic_bench.json), with the card's name and power limit.

    python tools/agnostic_bench.py [--samples 128] [--seconds 15] [--workers 2 4 8] [--out DIR]

1. Kernel time of draw.agnostic_bits and draw.parse_agnostic (1024x768) per batch of 8 and 64: CUDA events, median of 50 launches
   after 10 warm-up launches.
2. VitonHDLoader samples/s for STAGE2_KEYS at 1024x768, batch 8, for each worker count, with device_agnostic on and off alternated
   in one process (two rounds each; each round iterates --seconds after a warm-up epoch), and the host-to-device bytes per sample.
3. tools/parse_agnostic.py images/s on the synthetic tree (4 workers, batches of 16), against the reference's
   get_im_parse_agnostic + PNG save per image on one core (from oracle/_ref, skipped when absent)."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import hrv_loader  # noqa: E402

hrv_loader.load()
import torch  # noqa: E402
from PIL import Image  # noqa: E402

import draw_oracle  # noqa: E402
from hrviton_b200 import data, draw, synth  # noqa: E402

sys.path.insert(0, os.path.join(ROOT, "tools"))
import loader_bench  # noqa: E402
import parse_agnostic as tool  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout
    return q.strip().splitlines()[torch.cuda.current_device()] if q.strip() else torch.cuda.get_device_name()


def kernel_ms(fn, warm=10, reps=50):
    for _ in range(warm):
        fn()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return float(np.median(times))


def loader_rate(root, workers, flag, seconds):
    ld = data.VitonHDLoader(root, "train", "pairs.txt", 1024, 768, 8, workers=workers, keys=data.STAGE2_KEYS, device_agnostic=flag)
    out = ld.empty_batch()
    for _ in range(len(ld)):  # warm-up epoch
        ld.consume(out)
    torch.cuda.synchronize()
    n, t0 = 0, time.perf_counter()
    while time.perf_counter() - t0 < seconds:
        ld.consume(out)
        n += ld.batch_size
    torch.cuda.synchronize()
    rate = n / (time.perf_counter() - t0)
    per_sample = ld.bytes_per_step / ld.batch_size
    ld.close()
    return rate, per_sample


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--samples", type=int, default=128)
    ap.add_argument("--seconds", type=float, default=15.0)
    ap.add_argument("--workers", type=int, nargs="+", default=[2, 4, 8])
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    lines = []

    def emit(d):
        d["card"] = card()
        print(json.dumps(d), flush=True)
        lines.append(d)

    rng = np.random.default_rng(0)
    for n in (8, 64):
        kp = torch.from_numpy(np.stack([draw_oracle.random_pose(rng) for _ in range(n)])).cuda()
        lab = torch.randint(0, 20, (n, 1024, 768), dtype=torch.uint8, device="cuda")
        bits = torch.empty((n, 1024, 768), dtype=torch.uint8, device="cuda")
        ws = torch.empty(draw.workspace_bytes(n, 1024), dtype=torch.uint8, device="cuda")
        emit({"what": "kernel_ms", "batch": n, "agnostic_bits": kernel_ms(lambda: draw.agnostic_bits(kp, out=bits, workspace=ws)),
              "parse_agnostic": kernel_ms(lambda: draw.parse_agnostic(lab, kp))})

    with tempfile.TemporaryDirectory() as root:
        loader_bench.write_tree(root, a.samples)
        for w in a.workers:
            res = {True: [], False: []}
            for _ in range(2):
                for flag in (False, True):
                    res[flag].append(loader_rate(root, w, flag, a.seconds))
            emit({"what": "loader_samples_per_s", "keys": "STAGE2_KEYS", "size": "1024x768", "batch": 8, "workers": w,
                  "device_agnostic": [round(r, 1) for r, _ in res[True]], "imagedraw_workers": [round(r, 1) for r, _ in res[False]],
                  "h2d_bytes_per_sample": {"device_agnostic": res[True][0][1], "imagedraw_workers": res[False][0][1]}})

        base = os.path.join(root, "train")
        out = os.path.join(root, "out")
        tool.run(base, out, 16, 4)  # warm-up (worker start, kernel load)
        t0 = time.perf_counter()
        written, _ = tool.run(base, out, 16, 4)
        torch.cuda.synchronize()
        rate = len(written) / (time.perf_counter() - t0)
        ref_ms = None
        try:
            import hrv_env
            ref = hrv_env.load_reference_script("get_parse_agnostic")
            names = sorted(os.listdir(os.path.join(base, "image")))[:32]
            t0 = time.perf_counter()
            for name in names:
                with open(os.path.join(base, "openpose_json", name.replace(".jpg", "_keypoints.json"))) as f:
                    pose = np.array(json.load(f)["people"][0]["pose_keypoints_2d"]).reshape((-1, 3))[:, :2]
                im = Image.open(os.path.join(base, "image-parse-v3", name.replace(".jpg", ".png")))
                ref.get_im_parse_agnostic(im, pose).save(os.path.join(root, "ref.png"))
            ref_ms = (time.perf_counter() - t0) / len(names) * 1e3
        except FileNotFoundError:
            pass
        emit({"what": "parse_agnostic_tool", "images": len(written), "images_per_s": round(rate, 1), "cpus": os.cpu_count(),
              "reference_ms_per_image_one_core": ref_ms, "reference_images_per_s": None if ref_ms is None else round(1e3 / ref_ms, 1)})
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "agnostic_bench.json"), "w") as f:
            json.dump(lines, f, indent=1)


if __name__ == "__main__":
    main()
