"""JPEG decoding on the device against PIL, and what it does to the pipelines that read JPEGs from disk.

    python tools/jpeg_bench.py [--seconds 20] [--samples 256] [--workers 2 4 8] [--fid-images 1024] [--skip-stage2] [--out DIR]

1. hrviton_b200.jpeg on the synthetic tree's 1024x768 q95 4:2:0 files (image / cloth / image-densepose) at batch 1, 8, 32 and 50:
   device time per batch and its split over the three kernels (CUDA events, median of 20), against PIL's single-core decode of the
   same files on this host.  A batch of 1 is one thread Huffman-decoding one whole file: its entropy time is that thread's time.
2. VitonHDLoader samples/s at each worker count, at 1024x768 and 256x192, with the host-to-device bytes per sample: the device path
   and the PIL path alternately in this process.  The PIL path is forced by replacing jpeg.device_decodable in this process.
3. Stage-2 graph steps at 1024x768, batch 8, fed by the loader with 4 workers against one synthetic batch (tools/loader_bench.py).
4. tools/fid.py end to end on two folders of --fid-images 1024x768 JPEGs written as the reference's save_images writes (PIL's
   default q75 4:2:0), device path and PIL path, with the time spent waiting for decoded batches."""
import argparse
import io
import json
import os
import shutil
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")]
import hrv_loader  # noqa: E402

hrv_loader.load()
import numpy as np  # noqa: E402
import torch  # noqa: E402
from PIL import Image  # noqa: E402

import loader_bench  # noqa: E402
from hrviton_b200 import data, jpeg  # noqa: E402

_device_decodable = jpeg.device_decodable


def path_(pil):
    """Selects the decode path of loaders and fid.py built from now on (DataLoader workers fork with this module state)."""
    jpeg.device_decodable = (lambda h: False) if pil else _device_decodable


def emit(results, line):
    print(json.dumps(line), flush=True)
    results.append(line)


def decode_part(root, results):
    files = sorted(os.path.join(root, "train", d, f) for d in ("image", "cloth", "image-densepose")
                   for f in os.listdir(os.path.join(root, "train", d)))[:50]
    blobs = []
    for f in files:
        with open(f, "rb") as fh:
            blobs.append(fh.read())
    t0 = time.perf_counter()
    for b in blobs:
        np.asarray(Image.open(io.BytesIO(b)))
    pil_ms = (time.perf_counter() - t0) / len(blobs) * 1e3
    emit(results, {"pil_decode_1024x768_q95_ms_per_image_one_core": round(pil_ms, 3)})
    dev = torch.device("cuda")
    for n in (1, 8, 32, 50):
        items = [jpeg.compact(b) for b in blobs[:n]]
        out = [torch.empty(c.shape, dtype=torch.uint8, device=dev) for c in items]
        batch = jpeg.Batch(items)
        batch.set_destinations(out)
        split = []
        for rep in range(23):
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
            errors = batch.launch(dev, events=ev)
            torch.cuda.synchronize()
            assert not errors.any()
            if rep >= 3:
                split.append([ev[i].elapsed_time(ev[i + 1]) for i in range(3)])
        split = np.median(np.array(split), 0)
        total = float(split.sum())
        emit(results, {"device_decode_batch": n, "device_ms": round(total, 3), "huffman_ms": round(split[0], 3), "idct_ms": round(split[1], 3),
                       "color_ms": round(split[2], 3), "images_per_s": round(n * 1e3 / total, 1),
                       "pil_one_core_images_per_s": round(1e3 / pil_ms, 1)})
        for o, b in zip(out, blobs):
            assert np.array_equal(o.cpu().numpy(), np.asarray(Image.open(io.BytesIO(b))))


def loader_part(root, args, results):
    for fh, fw in ((1024, 768), (256, 192)):
        for workers in args.workers:
            for pil in (False, True):
                path_(pil)
                ld = data.VitonHDLoader(root, "train", "pairs.txt", fh, fw, 8, workers=workers)
                rate = loader_bench.timed(ld.next_batch, 8, args.seconds)
                emit(results, {"loader": "VitonHDLoader", "decode": "PIL" if pil else "device", "size": "%dx%d" % (fh, fw), "workers": workers,
                               "samples_per_s": round(rate, 2), "h2d_mb_per_sample": round(ld.bytes_per_step / 8 / 1e6, 2),
                               "device_decoded_files": ld.device_decoded})
                del ld
    path_(False)


def fid_part(args, results):
    import fid as fid_tool
    import fid_bench
    import fid_inception_oracle as fo
    tmp = tempfile.mkdtemp(prefix="fidjpeg_")
    try:
        dirs = []
        for s in range(2):
            d = os.path.join(tmp, "set%d" % s)
            os.makedirs(d)
            dirs.append(d)
            for i in range(args.fid_images):
                fid_bench._write_jpeg((os.path.join(d, "%05d_00.png" % i), 1000 * s + i, 0.2 * s))
                Image.open(os.path.join(d, "%05d_00.png" % i)).save(os.path.join(d, "%05d_00.jpg" % i))  # PIL's default: q75, 4:2:0
                os.remove(os.path.join(d, "%05d_00.png" % i))
        weights = os.path.join(tmp, "pt_inception.pth")
        torch.save(fo.seeded_fid_state_dict(seed=4), weights)
        for pil in (False, True, False, True):
            path_(pil)
            t0 = time.perf_counter()
            res = fid_tool.main([dirs[0], dirs[1], "--weights", weights, "--workers", str(min(8, os.cpu_count() or 1))])
            emit(results, {"fid_tool": "PIL" if pil else "device", "images_per_set": args.fid_images, "total_s": round(time.perf_counter() - t0, 3),
                           **res})
        path_(False)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=20.0)
    ap.add_argument("--samples", type=int, default=256)
    ap.add_argument("--workers", type=int, nargs="+", default=[2, 4, 8])
    ap.add_argument("--fid-images", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--skip-stage2", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "jpeg_bench needs a GPU"
    os.environ.setdefault("HRV_VGG_RANDOM_INIT", "1")
    results = []
    emit(results, loader_bench.device_line())
    root = tempfile.mkdtemp(prefix="vitonhd_")
    try:
        loader_bench.write_tree(root, args.samples)
        decode_part(root, results)
        loader_part(root, args, results)
        if not args.skip_stage2:
            loader_bench.stage2(root, 8, 2, args.steps, results)
    finally:
        shutil.rmtree(root, ignore_errors=True)
    if args.fid_images:
        fid_part(args, results)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "jpeg_bench.json"), "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
