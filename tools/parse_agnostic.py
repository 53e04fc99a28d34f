"""get_parse_agnostic.py on the GPU: writes image-parse-agnostic-v3.2 from a VITON-HD tree, the same files as the reference script.

    python tools/parse_agnostic.py --data_path DATA/train --output_path DATA/train/image-parse-agnostic-v3.2 [--batch_size 16] [--workers 4]

As the reference does, it walks data_path/image in os.listdir order, reads openpose_json/<name>_keypoints.json and
image-parse-v3/<name>.png, skips (printing the JSON's name) a sample whose JSON has no people[0], and writes <name>.png into
output_path in the parse image's mode and palette.  DataLoader workers decode the PNGs with PIL; the masks are drawn and applied on
the device in batches (draw.parse_agnostic); a thread pool re-encodes the labels through PIL's own save, so the bytes are the
reference's."""
import argparse
import json
import os
import os.path as osp
import sys
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = osp.dirname(osp.dirname(osp.abspath(__file__)))
sys.path.insert(0, ROOT)
import hrv_loader  # noqa: E402

hrv_loader.load()
import torch  # noqa: E402
from PIL import Image  # noqa: E402

from hrviton_b200 import draw  # noqa: E402


class ParseSet(torch.utils.data.Dataset):
    """(name, labels (H, W) uint8, keypoints (25, 2) fp64) per image name; labels None when the JSON has no people[0]."""

    def __init__(self, data_path, names):
        self.data_path, self.names = data_path, names

    def __len__(self):
        return len(self.names)

    def __getitem__(self, i):
        name = self.names[i]
        pose_name = name.replace(".jpg", "_keypoints.json")
        with open(osp.join(self.data_path, "openpose_json", pose_name)) as f:
            people = json.load(f)["people"]
        if not people:
            return name, None, None
        pose = np.array(people[0]["pose_keypoints_2d"]).reshape((-1, 3))[:, :2]
        path = osp.join(self.data_path, "image-parse-v3", name.replace(".jpg", ".png"))
        im = Image.open(path)
        if im.mode not in ("P", "L"):
            raise ValueError("%s: mode %s, the parse images are P or L" % (path, im.mode))
        return name, np.asarray(im), draw.keypoints_array(pose, pose_name)


def write_png(src, labels, dst):
    """Saves `labels` (H, W) uint8 as src's pixels: src's mode, palette and info, through the same PIL save as the reference."""
    im = Image.open(src)
    im.load()
    im.frombytes(np.ascontiguousarray(labels).tobytes())
    im.save(dst)


def run(data_path, output_path, batch_size=16, workers=4, device=None):
    """Processes the tree; returns (written, skipped) name lists."""
    os.makedirs(output_path, exist_ok=True)
    names = os.listdir(osp.join(data_path, "image"))
    loader = torch.utils.data.DataLoader(ParseSet(data_path, names), batch_size=batch_size, num_workers=workers, collate_fn=list)
    dev = torch.device("cuda") if device is None else device
    written, skipped = [], []
    with ThreadPoolExecutor(max_workers=max(1, os.cpu_count() or 1)) as pool:
        jobs = []
        for batch in loader:
            for name, lab, _ in batch:
                if lab is None:
                    print(name.replace(".jpg", "_keypoints.json"))
                    skipped.append(name)
            groups = {}  # samples of one image size run as one batch
            for item in batch:
                if item[1] is not None:
                    groups.setdefault(item[1].shape, []).append(item)
            for items in groups.values():
                lab = torch.from_numpy(np.stack([t[1] for t in items])).pin_memory().to(dev, non_blocking=True)
                kp = torch.from_numpy(np.stack([t[2] for t in items])).pin_memory().to(dev, non_blocking=True)
                out = draw.parse_agnostic(lab, kp).cpu().numpy()
                for (name, _, _), o in zip(items, out):
                    png = name.replace(".jpg", ".png")
                    jobs.append(pool.submit(write_png, osp.join(data_path, "image-parse-v3", png), o, osp.join(output_path, png)))
                    written.append(name)
        for j in jobs:
            j.result()
    return written, skipped


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--data_path", type=str, help="dataset dir")
    ap.add_argument("--output_path", type=str, help="output dir")
    ap.add_argument("--batch_size", type=int, default=16)
    ap.add_argument("--workers", type=int, default=4)
    a = ap.parse_args(argv)
    run(a.data_path, a.output_path, a.batch_size, a.workers)


if __name__ == "__main__":
    main()
