"""Run the stage-1 test set and write its multi-task grids, as the reference's test_condition.py does, with PNG encoding on the GPU;
with --D_checkpoint and --norm_const also rejection_prob.txt, the samples sorted by discriminator-rejection score:

    python tools/test_condition.py --dataroot ./data --tocg_checkpoint checkpoints/tocg/tocg.pth \\
        --D_checkpoint checkpoints/tocg/D.pth --norm_const 1.52 -b 8

Flags are test_condition.py's; hrviton_b200.condition_run documents the run and its files.  tools/norm_const.py computes M."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
import hrv_loader  # noqa: E402

hrv_loader.load()
from hrviton_b200 import condition_run  # noqa: E402

if __name__ == "__main__":
    condition_run.main()
