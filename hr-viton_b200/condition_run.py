"""The reference's stage-1 test and normalising-constant scripts on the loader and the device.

test_condition.py (run): every full batch of the test set goes through the tocg (with --D_checkpoint and --norm_const, through
pipeline.ConditionGraph, which also scores the condition for discriminator rejection); png.condition_grid makes each sample's 12-panel
multi-task grid, png.encode writes it as a PNG on the device, and tryon_run's writer thread puts each file at
./output/<tocg_checkpoint parent dir>/<tocg_checkpoint file>/<datamode>/<datasetting>/multi-task/{paired cloth stem}_{unpaired cloth
stem}.png.  The grids decode to exactly the pixels the reference's save_image writes for the same tocg outputs; the compressed bytes
are png.encode's own.  With a discriminator, rejection_prob.txt is appended to in that directory after the last batch, as
test_condition.py:146-153 writes it.

    python tools/test_condition.py --dataroot ./data --tocg_checkpoint checkpoints/tocg/tocg.pth \\
        --D_checkpoint checkpoints/tocg/D.pth --norm_const 1.52 -b 8

get_norm_const.py (norm_const): pipeline.norm_constant over one epoch of full batches of the training tree, in list order; prints
`M: <value>`, the constant --norm_const takes.

    python tools/norm_const.py --dataroot ./data --tocg_checkpoint tocg.pth --D_checkpoint D.pth -b 8"""
import argparse
import os
import sys
import time
import types

import torch

from . import data, ops, png

GRID_KEYS = ("cloth", "cloth_mask", "parse_agnostic", "densepose", "parse", "pcm", "parse_cloth", "image")  # what the grid and tocg read
NORM_KEYS = ("cloth", "cloth_mask", "parse_agnostic", "densepose", "parse")
FIXED = {"warp_feature": "T1", "out_layer": "relu", "upsample": "bilinear", "semantic_nc": 13, "output_nc": 13}


def _common(p):
    """The flags test_condition.py and get_norm_const.py share."""
    p.add_argument("--gpu_ids", default="")
    p.add_argument("-j", "--workers", type=int, default=4)
    p.add_argument("-b", "--batch-size", "--batch_size", dest="batch_size", type=int, default=8)
    p.add_argument("--fp16", action="store_true", help="fp16 activation storage (default: HRV_PRECISION, bf16)")
    p.add_argument("--fine_width", type=int, default=192)
    p.add_argument("--fine_height", type=int, default=256)
    p.add_argument("--tensorboard_dir", default="tensorboard", help="accepted for the reference's command lines; nothing is written to it")
    p.add_argument("--checkpoint_dir", default="checkpoints")
    p.add_argument("--tocg_checkpoint", default="")
    p.add_argument("--D_checkpoint", default="")
    p.add_argument("--tensorboard_count", type=int, default=100)
    p.add_argument("--shuffle", action="store_true", help="accepted; the pairs are always read in list order")
    p.add_argument("--semantic_nc", type=int, default=13)
    p.add_argument("--output_nc", type=int, default=13)
    p.add_argument("--warp_feature", choices=["encoder", "T1"], default="T1")
    p.add_argument("--out_layer", choices=["relu", "conv"], default="relu")
    p.add_argument("--clothmask_composition", choices=["no_composition", "detach", "warp_grad"], default="warp_grad")
    p.add_argument("--Ddownx2", action="store_true")
    p.add_argument("--Ddropout", action="store_true")
    p.add_argument("--num_D", type=int, default=2)
    p.add_argument("--spectral", action="store_true")


def _check(p, opt, required):
    for k, v in FIXED.items():
        if getattr(opt, k, v) != v:
            p.error("--%s %s: the kernels run the reference's configuration, --%s %s" % (k, getattr(opt, k), k, v))
    if opt.batch_size < 1 or opt.workers < 0 or opt.num_D < 1:
        p.error("-b and --num_D must be positive and -j non-negative")
    if opt.fine_height < 1 or opt.fine_width < 1 or opt.fine_height % 32 or opt.fine_width % 32:
        p.error("--fine_height / --fine_width: the tocg's five stride-2 levels need multiples of 32, got %dx%d" % (opt.fine_height, opt.fine_width))
    for k in ("dataroot",) + required:
        if not os.path.exists(getattr(opt, k)):
            p.error("--%s %r does not exist" % (k, getattr(opt, k)))


def parse_args(argv=None):
    """test_condition.py's flags (get_opt, test_condition.py:17-62).  Refuses unknown flags, values the kernels do not run, and
    --D_checkpoint without --norm_const (the reference raises NotImplementedError there)."""
    p = argparse.ArgumentParser(prog="test_condition.py")
    _common(p)
    p.add_argument("--dataroot", default="./data/zalando-hd-resize")
    p.add_argument("--datamode", default="test")
    p.add_argument("--data_list", default="test_pairs.txt")
    p.add_argument("--datasetting", default="paired", choices=["paired", "unpaired"])
    p.add_argument("--upsample", choices=["nearest", "bilinear"], default="bilinear")
    p.add_argument("--occlusion", action="store_true", help="accepted; the stage-1 test does not read it")
    p.add_argument("--norm_const", type=float, help="the normalising constant M of discriminator rejection (tools/norm_const.py)")
    opt = p.parse_args(argv)
    if opt.D_checkpoint and opt.norm_const is None:
        p.error("--D_checkpoint needs --norm_const (tools/norm_const.py computes it)")
    if opt.norm_const is not None and not opt.norm_const > 0:
        p.error("--norm_const must be positive, got %r" % opt.norm_const)
    _check(p, opt, ("tocg_checkpoint",) + (("D_checkpoint",) if opt.D_checkpoint else ()))
    return opt


def parse_norm_args(argv=None):
    """get_norm_const.py's flags (get_opt, get_norm_const.py:14-58)."""
    p = argparse.ArgumentParser(prog="norm_const.py")
    _common(p)
    p.add_argument("--name", default="test")
    p.add_argument("--dataroot", default="./data")
    p.add_argument("--datamode", default="train")
    p.add_argument("--data_list", default="train_pairs_zalando.txt")
    for k, v in (("display_count", 100), ("save_count", 10000), ("load_step", 0), ("keep_step", 300000)):
        p.add_argument("--" + k, type=int, default=v)
    p.add_argument("--test_datasetting", default="unpaired")
    p.add_argument("--test_dataroot", default="./data/zalando-hd-resize")
    p.add_argument("--test_data_list", default="test_pairs.txt")
    opt = p.parse_args(argv)
    _check(p, opt, ("tocg_checkpoint", "D_checkpoint"))
    return opt


def output_dir(opt):
    """test_condition.py:73-74: ./output/<tocg_checkpoint parent dir>/<tocg_checkpoint file>/<datamode>/<datasetting>/multi-task."""
    parts = opt.tocg_checkpoint.split("/")
    if len(parts) < 2:
        raise ValueError("--tocg_checkpoint %r: the output directory is named after its parent directory and file, as the reference's "
                         "test_condition.py names it; give a path with a directory" % opt.tocg_checkpoint)
    return os.path.join("./output", parts[-2], parts[-1], opt.datamode, opt.datasetting, "multi-task")


def grid_name(c_name, i):
    """test_condition.py:142-143: '{paired cloth stem}_{unpaired cloth stem}.png', whatever --datasetting is."""
    return c_name["paired"][i].split(".")[0] + "_" + c_name["unpaired"][i].split(".")[0] + ".png"


def write_rejection(path, scored):
    """test_condition.py:146-153: (name, score) pairs sorted by score, descending (Python's stable sort), one 'name score' line each,
    appended to `path`."""
    scored = sorted(scored, key=lambda x: x[1], reverse=True)
    with open(path, "a") as f:
        for name, score in scored:
            f.write(name + " " + str(score) + "\n")


def build_models(opt, device, with_d):
    """ConditionGenerator(opt, 4, 16, 13, ngf=96, BatchNorm2d) and, with_d, define_D(33, ...) (test_condition.py:175-185), their
    checkpoints loaded, on `device` in eval mode."""
    import contextlib
    import io

    import networks
    topt = types.SimpleNamespace(warp_feature=opt.warp_feature, out_layer=opt.out_layer, cuda=True)
    tocg = networks.ConditionGenerator(topt, 4, opt.semantic_nc + 3, opt.output_nc, ngf=96, norm_layer=torch.nn.BatchNorm2d)
    networks.load_checkpoint(tocg, opt.tocg_checkpoint, topt)
    D = None
    if with_d:
        with contextlib.redirect_stdout(io.StringIO()):  # define_D prints the network
            D = networks.define_D(input_nc=4 + opt.semantic_nc + 3 + opt.output_nc, Ddownx2=opt.Ddownx2, Ddropout=opt.Ddropout, n_layers_D=3,
                                  spectral=opt.spectral, num_D=opt.num_D)
        networks.load_checkpoint(D, opt.D_checkpoint, topt)
        D = D.to(device).eval()
    return tocg.to(device).eval(), D


def _precision(opt):
    if opt.fp16:
        ops.set_precision("fp16")


def grid_inputs(batch, outs, datasetting):
    """png.condition_grid's inputs for a batch and the tocg outputs (flow_list, seg, warped_cloth, warped_cm)."""
    t = {k: batch[k] for k in ("parse_agnostic", "densepose", "parse_cloth", "pcm", "parse", "image")}
    t["cloth"], t["cloth_mask"] = batch["cloth"][datasetting], batch["cloth_mask"][datasetting]
    t["seg"], t["warped_cloth"], t["warped_cm"] = outs[1].float(), outs[2].float(), outs[3].float()
    return t


def run(opt, log=print):
    """Writes the multi-task grid of every full batch of the test set, and with a discriminator rejection_prob.txt.  Returns the list
    of files written."""
    from . import pipeline
    from .tryon_run import _Writer
    device = torch.device("cuda", torch.cuda.current_device())
    _precision(opt)
    tocg, D = build_models(opt, device, bool(opt.D_checkpoint))
    out_dir = output_dir(opt)
    os.makedirs(out_dir, exist_ok=True)
    loader = data.VitonHDLoader(opt.dataroot, opt.datamode, opt.data_list, opt.fine_height, opt.fine_width, opt.batch_size,
                                workers=opt.workers, mode="test", keys=GRID_KEYS, shuffle=False, shard=False)
    writer, graph, written, scores, names = None, None, [], [], []
    try:
        left = len(loader.dataset) - len(loader) * opt.batch_size
        if left:
            log("%d of %d pairs are left out: the last batch is incomplete (drop_last, as in the reference)" % (left, len(loader.dataset)))
        writer = _Writer()
        if D is not None:
            graph = pipeline.ConditionGraph(tocg, D, opt.norm_const, clothmask_composition=opt.clothmask_composition)
        num = 0
        start = time.time()
        with torch.no_grad():
            for batch in loader:
                if graph is not None:
                    score, _, outs = graph(batch, datasetting=opt.datasetting)
                    scores.append(score.clone())
                    names += [n.replace(".jpg", ".png") for n in batch["c_name"]["paired"]]
                else:
                    _, _, outs = pipeline._condition(tocg, batch, None, opt.datasetting)
                # on the current stream, before the next replay overwrites `outs`
                files = png.encode(png.condition_grid(grid_inputs(batch, outs, opt.datasetting), opt.clothmask_composition))
                for i, payload in enumerate(files):
                    path = os.path.join(out_dir, grid_name(batch["c_name"], i))
                    writer.put(path, payload)
                    written.append(path)
                num += len(files)
                log(num)
        writer.close()
        writer = None
        if scores:
            path = os.path.join(out_dir, "rejection_prob.txt")
            write_rejection(path, list(zip(names, torch.cat(scores).tolist())))
            written.append(path)
        log(f"Test time {time.time() - start}")
    finally:
        if writer is not None:  # an error on the way: the files queued so far are still written, the error raised is the first one
            writer.stop()
        if graph is not None:
            graph.release()
        loader.close()
    return written


def norm_const(opt):
    """get_norm_const.get_const: the normalising constant M over one epoch of full batches of the training tree, list order."""
    from . import pipeline
    device = torch.device("cuda", torch.cuda.current_device())
    _precision(opt)
    tocg, D = build_models(opt, device, True)
    loader = data.VitonHDLoader(opt.dataroot, opt.datamode, opt.data_list, opt.fine_height, opt.fine_width, opt.batch_size,
                                workers=opt.workers, mode="train", keys=NORM_KEYS, shuffle=False, shard=False)
    try:
        return pipeline.norm_constant(tocg, D, loader, clothmask_composition=opt.clothmask_composition)
    finally:
        loader.close()


def main(argv=None):
    opt = parse_args(sys.argv[1:] if argv is None else argv)
    print(opt)
    run(opt)
    print("Finished testing!")


def main_norm_const(argv=None):
    opt = parse_norm_args(sys.argv[1:] if argv is None else argv)
    print(opt)
    M = norm_const(opt)
    print("M:", M)
    return M
