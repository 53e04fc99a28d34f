"""Run the test set and write the try-on images, as the reference's test_generator.py does, on the graph runner with JPEG encoding
on the GPU:

    python tools/test.py --dataroot ./data --tocg_checkpoint tocg.pth --gen_checkpoint gen.pth --occlusion -b 4 --output_dir out

Flags are test_generator.py's plus --seed; hrviton_b200.tryon_run documents the run and its files."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
import hrv_loader  # noqa: E402

hrv_loader.load()
from hrviton_b200 import tryon_run  # noqa: E402

if __name__ == "__main__":
    tryon_run.main()
