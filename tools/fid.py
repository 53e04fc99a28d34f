"""FID (and KID) between two image folders, or a folder and saved statistics, with pytorch-fid's FID Inception on the package's kernels.

    python tools/fid.py A B --weights pt_inception-2015-12-05-6726825d.pth [--kid] [--batch-size 50] [--workers N]
                            [--save-stats OUT.npz] [--device cuda:0]

A and B are image folders or .npz statistics in pytorch-fid's format (mu, sigma).  A folder's images are the files with pytorch-fid's
extensions, in sorted order, decoded to RGB as PIL's .convert('RGB') does: JPEGs the device decodes (hrviton_b200.jpeg; the
reference's try-on outputs are PIL's default baseline JPEG) go to the GPU as their entropy-coded bytes and are decoded there, bit for
bit as PIL decodes them, every other file is decoded by PIL in the DataLoader workers; all images of one batch must share a size.  They go to the GPU as uint8 and are resized and normalised there (hrv_resize_bilinear_fid), as pytorch-fid's
TF.to_tensor + F.interpolate + 2x - 1 does.  --save-stats writes A's statistics (A must be a folder).  --kid (two folders only) also
prints KID's mean and std over metrics.kid's default 100 subsets of 1000 images.  The weights are never downloaded."""
import argparse
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

IMAGE_EXTENSIONS = {"bmp", "jpg", "jpeg", "pgm", "png", "ppm", "tif", "tiff", "webp"}  # pytorch-fid's
KID_SUBSETS, KID_SUBSET_SIZE = 100, 1000  # metrics.kid's defaults


def image_files(folder):
    """The images of `folder` as pytorch-fid lists them: its files with one of the (lower-case) extensions, sorted."""
    return sorted(os.path.join(folder, f) for f in os.listdir(folder)
                  if os.path.splitext(f)[1][1:] in IMAGE_EXTENSIONS and os.path.isfile(os.path.join(folder, f)))


class _Images:
    """torch Dataset of the images: a jpeg.Compact for a JPEG the device decodes, else the uint8 (H, W, 3) RGB array PIL decodes."""

    def __init__(self, files):
        self.files = files

    def __len__(self):
        return len(self.files)

    def __getitem__(self, i):
        import numpy as np
        from PIL import Image

        from hrviton_b200 import jpeg
        with Image.open(self.files[i]) as im:
            if im.format == "JPEG":
                with open(self.files[i], "rb") as f:
                    c = jpeg.compact(f.read(), self.files[i])
                if c is not None:
                    return c
            return np.asarray(im.convert("RGB"), dtype=np.uint8)


def _collate(items):
    """One pinned uint8 (N, H, W, 3) batch when PIL decoded every image, else (PIL arrays by index, jpeg.Compacts by index, packed
    entropy-coded bytes)."""
    import numpy as np
    import torch

    from hrviton_b200 import jpeg
    shapes = {(c.height, c.width, 3) if isinstance(c, jpeg.Compact) else c.shape for c in items}
    if len(shapes) != 1:
        raise ValueError("fid: the images of one batch must share a size, got %s; resize them first or use --batch-size 1" % sorted(shapes))
    dev = [(i, c) for i, c in enumerate(items) if isinstance(c, jpeg.Compact)]
    if not dev:
        return torch.from_numpy(np.stack(items))
    pil = [(i, torch.from_numpy(a)) for i, a in enumerate(items) if not isinstance(a, jpeg.Compact)]
    return {"shape": shapes.pop(), "pil": pil, "jpeg": dev, "jpeg_bytes": jpeg.pack_entropy([c for _, c in dev])}


def _device_batch(batch, device, errors):
    """The uint8 (N, H, W, 3) CUDA batch of a mixed host batch: the JPEGs decoded into their rows, the PIL images copied.  Appends
    the decode's device error codes and the files' names to `errors`."""
    import torch

    from hrviton_b200 import jpeg
    n = len(batch["pil"]) + len(batch["jpeg"])
    out = torch.empty((n,) + tuple(batch["shape"]), dtype=torch.uint8, device=device)
    for i, a in batch["pil"]:
        out[i].copy_(a, non_blocking=True)
    b = jpeg.Batch([c for _, c in batch["jpeg"]], batch["jpeg_bytes"])
    b.set_destinations([out[i] for i, _ in batch["jpeg"]])
    errors.append((b.launch(device), [c.name for _, c in batch["jpeg"]]))
    return out


def folder_features(files, net, batch_size=50, workers=0, timing=None):
    """(N, 2048) fp32 pool features of the image files through `net` (InceptionV3.from_fid_weights), in file order.  timing: a dict
    that receives 'wait_s', the time spent waiting for decoded batches."""
    import torch
    loader = torch.utils.data.DataLoader(_Images(files), batch_size=batch_size, shuffle=False, drop_last=False, num_workers=workers,
                                         collate_fn=_collate, pin_memory=True)
    from hrviton_b200 import jpeg
    feats, wait, errors = [], 0.0, []
    t0 = time.perf_counter()
    for batch in loader:
        wait += time.perf_counter() - t0
        x = batch.to(net.device, non_blocking=True) if torch.is_tensor(batch) else _device_batch(batch, net.device, errors)
        pool, _ = net(x)
        feats.append(pool)
        t0 = time.perf_counter()
    for codes, names in errors:  # corrupt JPEG data: raise naming the file
        jpeg.raise_errors(codes.cpu().numpy(), names)
    if timing is not None:
        timing["wait_s"] = timing.get("wait_s", 0.0) + wait
    return torch.cat(feats)


def _inputs(paths):
    """[(path, files or None for .npz)], refusing what cannot be scored before any GPU work."""
    out = []
    for p in paths:
        if p.endswith(".npz"):
            if not os.path.isfile(p):
                raise SystemExit("fid: no such statistics file: %s" % p)
            out.append((p, None))
        elif os.path.isdir(p):
            files = image_files(p)
            if not files:
                raise SystemExit("fid: %s holds no images (extensions: %s)" % (p, ", ".join(sorted(IMAGE_EXTENSIONS))))
            out.append((p, files))
        else:
            raise SystemExit("fid: %s is neither an image folder nor an .npz statistics file" % p)
    return out


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("a", help="image folder or .npz statistics")
    ap.add_argument("b", help="image folder or .npz statistics")
    ap.add_argument("--weights", required=True, help="pytorch-fid's pt_inception-2015-12-05-6726825d.pth (never downloaded)")
    ap.add_argument("--kid", action="store_true", help="also print KID (two folders only)")
    ap.add_argument("--batch-size", type=int, default=50)
    ap.add_argument("--workers", type=int, default=min(8, os.cpu_count() or 1))
    ap.add_argument("--save-stats", default=None, help="write A's statistics to this .npz")
    ap.add_argument("--device", default="cuda:0")
    a = ap.parse_args(argv)
    if not os.path.isfile(a.weights):
        raise SystemExit("fid: weights file not found: %s (pytorch-fid's pt_inception-2015-12-05-6726825d.pth; nothing is downloaded)"
                         % a.weights)
    if a.batch_size < 1 or a.workers < 0:
        raise SystemExit("fid: --batch-size must be >= 1 and --workers >= 0")
    inputs = _inputs([a.a, a.b])
    if a.save_stats and inputs[0][1] is None:
        raise SystemExit("fid: --save-stats needs A to be an image folder")
    if a.kid:
        if any(files is None for _, files in inputs):
            raise SystemExit("fid: --kid needs two image folders (statistics files hold no features)")
        for p, files in inputs:
            if len(files) < KID_SUBSET_SIZE:
                raise SystemExit("fid: --kid needs at least %d images per folder (the subset size); %s has %d" % (KID_SUBSET_SIZE, p, len(files)))

    import hrv_loader
    hrv_loader.load()
    import torch
    from hrviton_b200 import metrics
    t0 = time.perf_counter()
    net = metrics.InceptionV3.from_fid_weights(a.weights, device=a.device)
    timing = {"wait_s": 0.0}
    moments, feats = [], []
    with torch.no_grad():
        t1 = time.perf_counter()
        for p, files in inputs:
            if files is None:
                moments.append(metrics.FeatureStats.load_npz(p))
                feats.append(None)
                continue
            f = folder_features(files, net, a.batch_size, a.workers, timing)
            st = metrics.FeatureStats(device=net.device).update(f)
            moments.append((st.mean(), st.cov()))
            feats.append(f)
            if p == a.a and a.save_stats:
                st.save_npz(a.save_stats)
        torch.cuda.synchronize(net.device)
        t2 = time.perf_counter()
        value = float(metrics.fid_of_moments(moments[0], moments[1], device=net.device))
        t3 = time.perf_counter()
        result = {"fid": value, "images": [None if f is None else f.shape[0] for f in feats], "load_s": round(t1 - t0, 3),
                  "features_s": round(t2 - t1, 3), "decode_wait_s": round(timing["wait_s"], 3), "fid_s": round(t3 - t2, 3)}
        print("FID: %.6f" % value)
        if a.kid:
            km, ks = metrics.kid(feats[0], feats[1], subsets=KID_SUBSETS, subset_size=KID_SUBSET_SIZE)
            result["kid"], result["kid_std"] = float(km), float(ks)
            result["kid_s"] = round(time.perf_counter() - t3, 3)
            print("KID: %.6e +- %.6e" % (result["kid"], result["kid_std"]))
    return result


if __name__ == "__main__":
    main()
