"""Generates tests/golden/parse_agnostic_512x384_b6.npz: get_parse_agnostic.get_im_parse_agnostic of the UNMODIFIED reference
(ImageDraw, Pillow 12.2) on six seeded samples, for GPU tests that cannot read the reference.  Run where oracle/_ref exists:

    python tests/golden/make_golden_parse_agnostic.py

Labels are blocks of all 20 labels with label-14 / 15 bands along the arms; poses are draw_oracle.random_pose's on a 384 x 512
image (missing joints, coincident shoulders, joints off the image), drawn on a 384 x 512 canvas (get_im_parse_agnostic's w, h).
Stored: labels (6, 512, 384) uint8, keypoints (6, 25, 2) fp64, result (6, 512, 384) uint8, pillow version."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
import hrv_env  # noqa: E402
import draw_oracle  # noqa: E402


def labels(rng, h, w, pose):
    from PIL import Image, ImageDraw
    lab = np.kron(rng.integers(0, 20, (h // 32 + 1, w // 32 + 1)), np.ones((32, 32), np.int64))[:h, :w].astype(np.uint8)
    im = Image.fromarray(lab, "L")
    d = ImageDraw.Draw(im)
    for label, joints in ((14, (5, 6, 7)), (15, (2, 3, 4))):
        d.line([tuple(pose[j]) for j in joints], label, width=40)
    return np.asarray(im)


def main():
    import PIL
    from PIL import Image
    ref = hrv_env.load_reference_script("get_parse_agnostic")
    rng = np.random.default_rng(44)
    n, h, w = 6, 512, 384
    kp = np.stack([draw_oracle.random_pose(rng, w, h) for _ in range(n)])
    lab = np.stack([labels(rng, h, w, p) for p in kp])
    out = np.stack([np.asarray(ref.get_im_parse_agnostic(Image.fromarray(l, "L"), p.copy(), w=w, h=h)) for l, p in zip(lab, kp)])
    path = os.path.join(HERE, "parse_agnostic_512x384_b6.npz")
    np.savez_compressed(path, labels=lab, keypoints=kp, result=out, pillow=np.array(PIL.__version__))
    print(path, (out != lab).mean())


if __name__ == "__main__":
    main()
