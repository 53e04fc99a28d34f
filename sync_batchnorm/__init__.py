"""Drop-in for the reference's vendored sync_batchnorm package (train_generator.py:14,171-178).  DataParallelWithCallback is a
one-process-per-GPU data-parallel wrapper: with WORLD_SIZE>1 (torchrun) gradients are averaged with NCCL all-reduce on flat
buckets (hrviton_b200.ddp); with one process it is a transparent pass-through that keeps the `.module` attribute the callers rely
on (train_generator.py:593).  SynchronizedBatchNorm2d / convert_model make train-mode BatchNorm use the statistics of every rank's
samples (see INTEGRATION.md); the 1d/3d names exist for import parity and raise when used."""
import hrv_loader

hrv_loader.load()
from hrviton_b200.ddp import (DataParallelWithCallback, SynchronizedBatchNorm1d, SynchronizedBatchNorm2d,  # noqa: E402,F401
                              SynchronizedBatchNorm3d, convert_model)
