"""Train HR-VITON's stage 1 (train_condition.py) or stage 2 (train_generator.py) to completion on the graph step and the GPU loader:

    python tools/train.py stage1 --name tocg --dataroot ./data --occlusion
    python tools/train.py stage2 --name gen --dataroot ./data --tocg_checkpoint checkpoints/tocg/tocg_final.pth --occlusion
    torchrun --nproc-per-node 8 tools/train.py stage2 ... -b 64            # -b is the global batch
    python tools/train.py stage2 ... --resume checkpoints/gen/state_step_010000.pth

Flags are the reference's (train.py stage2 --help); hrviton_b200.train_loop documents the run, its files and its resume."""
import os
import sys

os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")  # before torch makes a cuBLAS handle: reproducible training steps
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
import hrv_loader  # noqa: E402

hrv_loader.load()
from hrviton_b200 import train_loop  # noqa: E402

if __name__ == "__main__":
    train_loop.main()
