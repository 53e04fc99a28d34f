"""The reference's test_generator.py run on the graph runner: every full batch of the test set goes through pipeline.TryOnGraph, its
output is JPEG-encoded on the device (jpeg.encode, byte-identical to utils.save_images' PIL encode) and a writer thread puts each
file at output_dir/{paired cloth stem}_{datasetting cloth stem}.png, JPEG bytes under the reference's .png name.

    python tools/test.py --dataroot ./data --tocg_checkpoint tocg.pth --gen_checkpoint gen.pth --occlusion -b 4 --output_dir out

The per-sample grid PNGs of test_generator.py (make_grid + save_image) are not written: they are visualisation, and zlib's bytes are
not worth reproducing."""
import argparse
import os
import queue
import sys
import threading
import time
import types
from collections import OrderedDict

import torch

from . import data, jpeg, ops

TEST_KEYS = ("cloth", "cloth_mask", "agnostic", "densepose", "parse_agnostic")  # what the try-on reads


def parse_args(argv=None):
    """test_generator.py's flags (get_opt, test_generator.py:26-71) that bear on the output, plus --seed (the SPADE noise).  Refuses
    unknown flags and values the kernels do not run."""
    p = argparse.ArgumentParser(prog="test.py")
    p.add_argument("--gpu_ids", default="")
    p.add_argument("-j", "--workers", type=int, default=4)
    p.add_argument("-b", "--batch-size", "--batch_size", dest="batch_size", type=int, default=1)
    p.add_argument("--fp16", action="store_true", help="fp16 activation storage (default: HRV_PRECISION, bf16)")
    p.add_argument("--cuda", default=False, help="accepted for the reference's command lines; the run is always on the GPU")
    p.add_argument("--test_name", default="test")
    p.add_argument("--dataroot", default="./data/zalando-hd-resize")
    p.add_argument("--datamode", default="test")
    p.add_argument("--data_list", default="test_pairs.txt")
    p.add_argument("--output_dir", default="./Output")
    p.add_argument("--datasetting", default="unpaired", choices=["paired", "unpaired"])
    p.add_argument("--fine_width", type=int, default=768)
    p.add_argument("--fine_height", type=int, default=1024)
    p.add_argument("--tocg_checkpoint", default="./eval_models/weights/v0.1/mtviton.pth")
    p.add_argument("--gen_checkpoint", default="./eval_models/weights/v0.1/gen.pth")
    p.add_argument("--semantic_nc", type=int, default=13)
    p.add_argument("--output_nc", type=int, default=13)
    p.add_argument("--gen_semantic_nc", type=int, default=7)
    p.add_argument("--warp_feature", choices=["encoder", "T1"], default="T1")
    p.add_argument("--out_layer", choices=["relu", "conv"], default="relu")
    p.add_argument("--clothmask_composition", choices=["no_composition", "detach", "warp_grad"], default="warp_grad")
    p.add_argument("--upsample", choices=["nearest", "bilinear"], default="bilinear")
    p.add_argument("--occlusion", action="store_true")
    p.add_argument("--norm_G", default="spectralaliasinstance")
    p.add_argument("--ngf", type=int, default=64)
    p.add_argument("--num_upsampling_layers", choices=("normal", "more", "most"), default="most")
    p.add_argument("--seed", type=int, default=0, help="seed of torch's CUDA generator, which draws the SPADE noise")
    opt = p.parse_args(argv)
    fixed = {"warp_feature": "T1", "out_layer": "relu", "upsample": "bilinear", "norm_G": "spectralaliasinstance", "num_upsampling_layers": "most",
             "semantic_nc": 13, "output_nc": 13, "gen_semantic_nc": 7}
    for k, v in fixed.items():
        if getattr(opt, k) != v:
            p.error("--%s %s: the kernels run the reference's configuration, --%s %s" % (k, getattr(opt, k), k, v))
    if opt.batch_size < 1 or opt.workers < 0 or opt.ngf < 1:
        p.error("-b and --ngf must be positive and -j non-negative")
    if opt.fine_width % 16 or opt.fine_height % 16:
        p.error("--fine_width / --fine_height: the device JPEG encoder takes multiples of 16, got %dx%d" % (opt.fine_width, opt.fine_height))
    want = data.resized_size(1024, 768, opt.fine_width)
    if (opt.fine_height, opt.fine_width) != want:
        p.error("--fine_height %d: VITON-HD's 1024x768 images resize to %dx%d at --fine_width %d" % (opt.fine_height, want[0], want[1], opt.fine_width))
    for k in ("dataroot", "tocg_checkpoint", "gen_checkpoint"):
        if not os.path.exists(getattr(opt, k)):
            p.error("--%s %s does not exist" % (k, getattr(opt, k)))
    return opt


def output_name(c_name, datasetting, i):
    """test_generator.py:228: '{paired cloth stem}_{datasetting cloth stem}.png' of sample i of a batch's c_name."""
    return c_name["paired"][i].split(".")[0] + "_" + c_name[datasetting][i].split(".")[0] + ".png"


def load_generator_checkpoint(model, path):
    """test_generator.py's load_checkpoint_G: the keys (and _metadata) with 'ace' -> 'alias' and '.Spade' dropped, loaded strictly."""
    sd = torch.load(path, map_location="cpu")
    fix = lambda k: k.replace("ace", "alias").replace(".Spade", "")  # noqa: E731
    new = OrderedDict((fix(k), v) for k, v in sd.items())
    meta = getattr(sd, "_metadata", None)
    if meta is not None:
        new._metadata = OrderedDict((fix(k), v) for k, v in meta.items())
    model.load_state_dict(new, strict=True)


def build_models(opt, device):
    """ConditionGenerator(opt, 4, 16, 13, ngf=96, BatchNorm2d) and SPADEGenerator(opt, 9) with semantic_nc 7 (test_generator.py:256-269),
    their checkpoints loaded, on `device` in eval mode."""
    import networks
    import network_generator
    topt = types.SimpleNamespace(warp_feature=opt.warp_feature, out_layer=opt.out_layer, cuda=True)
    tocg = networks.ConditionGenerator(topt, 4, opt.semantic_nc + 3, opt.output_nc, ngf=96, norm_layer=torch.nn.BatchNorm2d)
    networks.load_checkpoint(tocg, opt.tocg_checkpoint, topt)
    gopt = types.SimpleNamespace(norm_G=opt.norm_G, gen_semantic_nc=opt.gen_semantic_nc, semantic_nc=7, ngf=opt.ngf,
                                 num_upsampling_layers=opt.num_upsampling_layers, fine_height=opt.fine_height, fine_width=opt.fine_width, cuda=True)
    gen = network_generator.SPADEGenerator(gopt, 9)
    load_generator_checkpoint(gen, opt.gen_checkpoint)
    return tocg.to(device).eval(), gen.to(device).eval()


class _Writer:
    """A thread that writes (path, bytes) pairs; an error it meets is raised by the next put() or close()."""

    def __init__(self):
        self.q = queue.Queue(maxsize=64)
        self.error = None
        self.thread = threading.Thread(target=self._run, name="jpeg-writer", daemon=True)
        self.thread.start()

    def _run(self):
        while True:
            item = self.q.get()
            if item is None:
                return
            if self.error is None:
                try:
                    with open(item[0], "wb") as f:
                        f.write(item[1])
                except Exception as e:  # noqa: BLE001 - handed to the main thread
                    self.error = e

    def put(self, path, payload):
        if self.error is not None:
            raise self.error
        self.q.put((path, payload))

    def close(self):
        """Waits for every queued file; raises the first error met."""
        self.stop()
        if self.error is not None:
            raise self.error

    def stop(self):
        self.q.put(None)
        self.thread.join()


def run(opt, log=print):
    """Writes the try-on of every full batch of the test set to opt.output_dir.  Returns the list of files written."""
    from . import pipeline
    device = torch.device("cuda", torch.cuda.current_device())
    if opt.fp16:
        ops.set_precision("fp16")
    torch.manual_seed(opt.seed)
    torch.cuda.manual_seed(opt.seed)
    tocg, gen = build_models(opt, device)
    os.makedirs(opt.output_dir, exist_ok=True)
    loader = data.VitonHDLoader(opt.dataroot, opt.datamode, opt.data_list, opt.fine_height, opt.fine_width, opt.batch_size,
                                workers=opt.workers, mode="test", keys=TEST_KEYS, shuffle=False, shard=False)
    writer, graph, written = None, None, []
    try:
        left = len(loader.dataset) - len(loader) * opt.batch_size
        if left:
            log("%d of %d pairs are left out: the last batch is incomplete (drop_last, as in the reference)" % (left, len(loader.dataset)))
        writer = _Writer()
        graph = pipeline.TryOnGraph(tocg, gen, occlusion=opt.occlusion, clothmask_composition=opt.clothmask_composition)
        num = 0
        start = time.time()
        with torch.no_grad():
            for batch in loader:
                output = graph(batch, datasetting=opt.datasetting)[0]
                files = jpeg.encode(output)  # on the current stream, before the next replay overwrites `output`
                for i, payload in enumerate(files):
                    path = os.path.join(opt.output_dir, output_name(batch["c_name"], opt.datasetting, i))
                    writer.put(path, payload)
                    written.append(path)
                num += len(files)
                log(num)
        writer.close()
        writer = None
        log(f"Test time {time.time() - start}")
    finally:
        if writer is not None:  # an error on the way: the files queued so far are still written, the error raised is the first one
            writer.stop()
        if graph is not None:
            graph.release()
        loader.close()
    return written


def main(argv=None):
    opt = parse_args(sys.argv[1:] if argv is None else argv)
    print(opt)
    run(opt)
    print("Finished testing!")
