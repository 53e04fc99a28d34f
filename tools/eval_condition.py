"""Score a stage-1 (tocg) checkpoint offline with the segmentation IoU that stage-1 training validates with (train_condition.py:314-360):

    python tools/eval_condition.py --tocg_checkpoint checkpoints/tocg/tocg_step_010000.pth --dataroot ./data --data_list test_pairs.txt

The tocg runs in eval mode (folded BatchNorm) on the first 2000 test pairs, paired cloth, in full batches of -b, through
pipeline.SegmentationGraph; the printed value is train_loop.validation_iou, the number `train.py stage1 --val_count` logs for the same
weights and batch size.  --fp16 runs the tocg in fp16 storage (as a --fp16 training run validates), bf16 otherwise."""
import argparse
import os
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
import hrv_loader  # noqa: E402

hrv_loader.load()


def main(argv=None):
    p = argparse.ArgumentParser(prog="eval_condition.py")
    p.add_argument("--tocg_checkpoint", required=True)
    p.add_argument("--dataroot", default="./data/")
    p.add_argument("--data_list", default="test_pairs.txt")
    p.add_argument("-b", "--batch_size", "--batch-size", dest="batch_size", type=int, default=8)
    p.add_argument("-j", "--workers", type=int, default=4)
    p.add_argument("--fp16", action="store_true", help="fp16 storage (bf16 otherwise)")
    opt = p.parse_args(argv)
    if opt.batch_size < 1 or opt.workers < 0:
        p.error("-b must be positive and -j non-negative")
    for k in ("tocg_checkpoint", "dataroot"):
        if not os.path.exists(getattr(opt, k)):
            p.error("--%s %s does not exist" % (k, getattr(opt, k)))
    import torch

    import networks
    from hrviton_b200 import data, ops, pipeline, train_loop
    ops.set_precision("fp16" if opt.fp16 else "bf16")
    topt = types.SimpleNamespace(warp_feature="T1", out_layer="relu", cuda=True)
    tocg = networks.ConditionGenerator(topt, 4, 16, 13, ngf=96, norm_layer=torch.nn.BatchNorm2d)
    networks.load_checkpoint(tocg, opt.tocg_checkpoint, topt)
    tocg = tocg.cuda().eval()
    loader = data.VitonHDLoader(opt.dataroot, "test", opt.data_list, 256, 192, opt.batch_size, workers=opt.workers, mode="test",
                                keys=train_loop.VAL_KEYS, shuffle=False, shard=False)
    runner = pipeline.SegmentationGraph(tocg)
    try:
        value = train_loop.validation_iou(runner, loader)
    finally:
        runner.release()
        loader.close()
    n = min(train_loop.VAL_SAMPLES, len(loader.dataset)) // opt.batch_size * opt.batch_size
    print("IoU: %.6f  (%d samples, batch %d, %s storage)" % (value, n, opt.batch_size, ops.get_precision()))
    return value


if __name__ == "__main__":
    main()
