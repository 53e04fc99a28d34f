"""Compute the normalising constant M of discriminator rejection over the training set, as the reference's get_norm_const.py does:

    python tools/norm_const.py --dataroot ./data --tocg_checkpoint tocg.pth --D_checkpoint D.pth -b 8

prints `M: <value>`, which tools/test_condition.py takes as --norm_const.  Flags are get_norm_const.py's; hrviton_b200.condition_run
documents the run."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
import hrv_loader  # noqa: E402

hrv_loader.load()
from hrviton_b200 import condition_run  # noqa: E402

if __name__ == "__main__":
    condition_run.main_norm_const()
