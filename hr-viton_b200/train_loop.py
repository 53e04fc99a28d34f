"""Training runs of both stages to completion on the graph step (train_step) fed by the GPU loader (data.VitonHDLoader): the
reference's learning-rate schedule, checkpoints in the reference's names and format, a sidecar state file from which a fresh process
resumes bit for bit, periodic LPIPS on test try-ons (stage 2) or segmentation IoU on test conditions (stage 1), and the loss prints of train_condition.py / train_generator.py.

    run = TrainRun("stage2", trainer, loader, "checkpoints/name", keep_step=100000, decay_step=100000)
    run.resume("checkpoints/name/state_step_010000.pth")     # optional, before start()
    run.start()                                              # captures the step; the capture does not train
    run.train()

An ordinary step is one replay: the schedule factor is written only on the steps where it changes, and the host synchronises only on
display, evaluation and save steps."""
import argparse
import collections
import hashlib
import os
import sys

import torch

from . import data, ops, train_step

STAGES = ("stage1", "stage2")
# train_condition.py:461-462,510-511 and train_generator.py:601-602,680-681
MODEL_FILES = {"stage1": {"tocg": ("tocg_step_%06d.pth", "tocg_final.pth"), "D": ("D_step_%06d.pth", "D_final.pth")},
               "stage2": {"G": ("gen_step_%06d.pth", "gen_model_final.pth"), "D": ("dis_step_%06d.pth", "dis_model_final.pth")}}
STATE_FILES = ("state_step_%06d.pth", "state_final.pth")
LPIPS_SAMPLES = 500  # train_generator.py:620: Subset(test_dataset, np.arange(500))
EVAL_KEYS = ("cloth", "cloth_mask", "agnostic", "densepose", "parse_agnostic", "image")
EVAL_GT_KEYS = train_step.GT_KEYS  # --GT: the ground-truth parse and cloth (train_generator.py:570-572)
VAL_SAMPLES = 2000  # train_condition.py:485: Subset(test_dataset, np.arange(2000))
VAL_KEYS = ("cloth", "cloth_mask", "parse_agnostic", "densepose", "parse")
# the stage-1 loss options a resumed run must share, with the values a state file that does not record them was trained with
STAGE1_OPTIONS = {"edgeawaretv": "no_edge", "add_lasttv": False, "clothmask_composition": "warp_grad", "no_gan_loss": False,
                  "g_d_separate": False, "tvlambda": 2.0, "ce_lambda": 10.0, "gan_lambda": 1.0}
# the same for stage 2 (train_generator.py); no_ganFeat_loss is the discriminator's option, as in the reference
STAGE2_OPTIONS = {"gt": False, "clothmask_composition": "warp_grad", "no_vgg_loss": False, "no_ganFeat_loss": False, "lambda_feat": 10.0,
                  "lambda_vgg": 10.0}


def lr_lambda(k, load_step, keep_step, decay_step, interval=1000):
    """train_generator.py:155-159: the LambdaLR factor after k scheduler steps (one every `interval` training steps)."""
    return 1.0 - max(0, k * interval + load_step - keep_step) / float(decay_step + 1)


def lr_factor(step, load_step, keep_step, decay_step, interval=1000):
    """The factor the reference trains step `step` (0-based, counted from 0 whatever load_step is) with, for a run started at load_step:
    its scheduler has stepped once for every multiple of `interval` in (load_step, step]."""
    return lr_lambda(step // interval - load_step // interval, load_step, keep_step, decay_step, interval)


def save_model(module, path):
    """networks.save_checkpoint's file (module.cpu().state_dict(): an OrderedDict of CPU tensors with its _metadata, which
    test_generator.py's load_checkpoint_G reads) without moving the module, so a captured step keeps its addresses."""
    sd = module.state_dict()
    out = collections.OrderedDict((k, v.detach().cpu()) for k, v in sd.items())
    out._metadata = sd._metadata
    _atomic_save(out, path)


def _atomic_save(obj, path):
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    tmp = path + ".tmp"
    torch.save(obj, tmp)
    os.replace(tmp, path)


def _to_cpu(obj):
    if torch.is_tensor(obj):
        return obj.detach().cpu()
    if isinstance(obj, dict):
        return type(obj)((k, _to_cpu(v)) for k, v in obj.items())
    if isinstance(obj, (list, tuple)):
        return type(obj)(_to_cpu(v) for v in obj)
    return obj


def _dist():
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized():
        return dist, dist.get_rank(), dist.get_world_size()
    return None, 0, 1


class TrainRun:
    """One training run of `stage` ("stage1": train_condition.py, "stage2": train_generator.py) on a train_step trainer built with
    tensor_lr=True (stage 2) and a data.VitonHDLoader.

    Steps are counted as the reference counts them: the run trains steps load_step .. end - 1, end = keep_step (stage 1) or
    keep_step + decay_step (stage 2).  Stage 2 follows the reference's LambdaLR (lr_factor), whose scheduler steps every `interval`
    steps (1000 in the reference); stage 1 has no schedule, as train_condition.py has none.  Every save_count steps rank 0 writes the
    model files of MODEL_FILES and a state file (state_step_%06d.pth); display_count prints the losses; lpips_count runs evaluate() (stage
    2) and val_count validate() (stage 1).
    A process group (torchrun) makes this one rank of a data-parallel run: the trainer's reducers and the sharded loader do the
    data-parallel work, and rank 0 writes the files.

    evaluator: for stage 2, (test_loader, lpips_model) — a VitonHDLoader in mode "test" with batch 1 and shard=False, and
    eval_models.PerceptualLoss or anything called as it (pred, target) -> (N,1,1,1).
    validator: for stage 1, a VitonHDLoader in mode "test" with keys VAL_KEYS, the training's per-rank batch size, shuffle=False and
    shard=False.
    on_step(step, losses): called after every step with the step's loss tensors (overwritten by the next replay)."""

    def __init__(self, stage, trainer, loader, checkpoint_dir, keep_step, decay_step=0, load_step=0, interval=1000, save_count=10000,
                 display_count=100, lpips_count=None, evaluator=None, lpips_samples=LPIPS_SAMPLES, val_count=None, validator=None,
                 val_samples=VAL_SAMPLES, log=print, on_step=None):
        if stage not in STAGES:
            raise ValueError("stage must be one of %s, not %r" % (STAGES, stage))
        if stage == "stage2" and not trainer.tensor_lr:
            raise ValueError("stage 2 follows the reference's LR schedule: build the trainer with tensor_lr=True")
        if stage == "stage2" and lpips_count and evaluator is None and _dist()[1] == 0:  # only rank 0 evaluates
            raise ValueError("lpips_count needs an evaluator (test loader, LPIPS model) on rank 0")
        if stage == "stage1" and val_count and validator is None and _dist()[1] == 0:  # only rank 0 validates
            raise ValueError("val_count needs a validator (test loader) on rank 0")
        self.stage, self.trainer, self.loader, self.dir = stage, trainer, loader, checkpoint_dir
        self.keep_step, self.decay_step, self.load_step, self.interval = int(keep_step), int(decay_step), int(load_step), int(interval)
        self.end = self.keep_step + (self.decay_step if stage == "stage2" else 0)
        self.save_count, self.display_count, self.lpips_count = save_count, display_count, lpips_count
        self.evaluator, self.lpips_samples = evaluator, lpips_samples
        self.val_count, self.validator, self.val_samples = val_count, validator, val_samples
        self.log, self.on_step = log, on_step
        self.step = self.load_step
        self.origin = self.load_step  # the load_step of the run's first process: the schedule's origin
        self.modules = {"stage1": {"tocg": trainer.tocg, "D": trainer.D}, "stage2": {"G": getattr(trainer, "G", None), "D": trainer.D}}[stage]
        self.lpips = []  # (step, value)
        self.iou = []  # (step, value)
        self._tryon = None
        self._seg = None

    # ---------------------------------------------------------------- schedule
    def factor(self, step=None):
        if self.stage == "stage1":
            return 1.0
        return lr_factor(self.step if step is None else step, self.origin, self.keep_step, self.decay_step, self.interval)

    # ---------------------------------------------------------------- files
    def config(self):
        """What a resumed run must share with the run it continues beyond the schedule: both base learning rates, --occlusion, the loss
        options of STAGE1_OPTIONS / STAGE2_OPTIONS and, for stage 2 with a tocg, the frozen tocg (a SHA-256 of its state, so another
        --tocg_checkpoint file with the same weights is accepted)."""
        cfg = {"base_lr": dict(self.trainer.base_lr), "occlusion": getattr(self.trainer, "occlusion", None)}
        if self.stage == "stage1":
            cfg.update((k, getattr(self.trainer, k, v)) for k, v in STAGE1_OPTIONS.items())  # a trainer without them trains the defaults
        if self.stage == "stage2":
            cfg.update((k, getattr(self.trainer, k, v)) for k, v in STAGE2_OPTIONS.items())
            cfg["no_ganFeat_loss"] = bool(getattr(self.trainer.D, "no_ganFeat_loss", False))
        if self.stage == "stage2" and self.trainer.tocg is not None:
            h = hashlib.sha256()
            for k, v in self.trainer.tocg.state_dict().items():
                h.update(k.encode())
                h.update(v.detach().cpu().reshape(-1).contiguous().view(torch.uint8).numpy().tobytes())
            cfg["tocg_sha256"] = h.hexdigest()
        return cfg

    def save(self, final=False):
        """Model files and the state file for the current step (rank 0 writes; every rank takes part in gathering the generator
        states).  Returns the state file's path."""
        dist, rank, world = _dist()
        rng = (torch.get_rng_state(), torch.cuda.get_rng_state())
        rngs = [rng]
        if dist is not None:
            rngs = [None] * world
            dist.all_gather_object(rngs, rng)
        path = os.path.join(self.dir, STATE_FILES[1] if final else STATE_FILES[0] % self.step)
        if rank != 0:
            return path
        models = {}
        for name, m in self.modules.items():
            fname = MODEL_FILES[self.stage][name][1 if final else 0]
            models[name] = fname if final else fname % self.step
            save_model(m, os.path.join(self.dir, models[name]))
        epoch, index = self.loader.position()
        state = {"stage": self.stage, "step": self.step, "origin": self.origin, "keep_step": self.keep_step, "decay_step": self.decay_step,
                 "interval": self.interval, "config": self.config(), "models": models, "trainer": _to_cpu(self.trainer.state_dict()),
                 "rng": [{"cpu": c, "cuda": g} for c, g in rngs],
                 "loader": {"seed": self.loader.seed, "epoch": epoch, "index": index, "batch_size": self.loader.batch_size}}
        _atomic_save(state, path)
        return path

    def resume(self, path):
        """Restores a state file written by save() (and the model files it names, from its directory), before start()."""
        if self.trainer._captured is not None:
            raise RuntimeError("resume() before start(): the captured step would keep the old state tensors")
        dist, rank, world = _dist()
        st = torch.load(path, map_location="cpu", weights_only=False)
        if st["stage"] != self.stage:
            raise ValueError("%s is a %s state, this run is %s" % (path, st["stage"], self.stage))
        for k in ("keep_step", "decay_step", "interval"):
            if self.stage == "stage2" and st[k] != getattr(self, k):
                raise ValueError("%s was saved with %s=%r, this run has %r" % (path, k, st[k], getattr(self, k)))
        cfg = self.config()
        saved = dict(STAGE1_OPTIONS if self.stage == "stage1" else STAGE2_OPTIONS)  # a state file written before the options were recorded
        saved.update(st["config"])
        for k, v in saved.items():
            if cfg.get(k) != v:
                raise ValueError("%s was saved with %s=%r, this run has %r" % (path, k, v, cfg.get(k)))
        if len(st["rng"]) != world:
            raise ValueError("%s was saved by %d ranks, this run has %d" % (path, len(st["rng"]), world))
        ld = st["loader"]
        if (ld["seed"], ld["batch_size"]) != (self.loader.seed, self.loader.batch_size):
            raise ValueError("%s was saved with loader seed %r, batch %r; this loader has %r, %r"
                             % (path, ld["seed"], ld["batch_size"], self.loader.seed, self.loader.batch_size))
        d = os.path.dirname(os.path.abspath(path))
        for name, fname in st["models"].items():
            self.modules[name].load_state_dict(torch.load(os.path.join(d, fname), map_location="cpu"))
        ops.PARAM_GEN[0] += 1
        self.trainer.load_state_dict(st["trainer"])
        torch.set_rng_state(st["rng"][rank]["cpu"])
        torch.cuda.set_rng_state(st["rng"][rank]["cuda"])
        self.loader.start_at(ld["epoch"], ld["index"])
        self.step, self.origin = st["step"], st["origin"]
        if self.stage == "stage2" and self.trainer.lr_factor != self.factor():
            raise ValueError("%s: LR factor %r, the schedule gives %r at step %d" % (path, self.trainer.lr_factor, self.factor(), self.step))
        return st

    # ---------------------------------------------------------------- steps
    def start(self):
        """Captures the trainer's step on a synthetic batch; the capture leaves every training state as it was (rollback)."""
        ds = self.loader.dataset
        n, h, w, dev = self.loader.batch_size, ds.fine_height, ds.fine_width, self.loader.device
        if self.stage == "stage2":
            self.trainer.set_lr_factor(self.factor())
            synthetic = train_step.synthetic_batch_gt if getattr(self.trainer, "gt", False) else train_step.synthetic_batch
            self.trainer.capture(synthetic(n, h, w, dev), h, w, rollback=True)
        else:
            b = train_step.synthetic_batch_stage1(n, h, w, dev)
            self.trainer.capture({k: b[k] for k in data.STAGE1_KEYS}, rollback=True)
        return self

    def train(self, until=None):
        """Trains up to step `until` (default: the end of the run); writes the final files when the run ends."""
        until = self.end if until is None else min(int(until), self.end)
        _, rank, _ = _dist()
        factor = self.trainer.lr_factor if self.stage == "stage2" else 1.0
        while self.step < until:
            f = self.factor()
            if f != factor:
                self.trainer.set_lr_factor(f)
                factor = f
            losses = self.trainer.replay(feeder=self.loader)
            self.step += 1
            if self.on_step is not None:
                self.on_step(self.step, losses)
            if self.stage == "stage2" and self.lpips_count and self.step % self.lpips_count == 0 and rank == 0:
                value = self.evaluate()
                self.lpips.append((self.step, value))
                self.log("step: %8d, LPIPS: %.6f" % (self.step, value))
            if self.stage == "stage1" and self.val_count and self.step % self.val_count == 0 and rank == 0:
                value = self.validate()
                self.iou.append((self.step, value))
                self.log("step: %8d, IoU: %.6f" % (self.step, value))
            if self.display_count and self.step % self.display_count == 0 and rank == 0:
                self.log("step: %8d, lr factor: %.6f, %s" % (self.step, factor, ", ".join("%s: %.4f" % (k, float(v)) for k, v in losses.items())))
            if self.save_count and self.step % self.save_count == 0:
                self.save()
        if self.step == self.end:
            self.save(final=True)
        return self

    def evaluate(self):
        """train_generator.py:480-584: the try-ons of the first LPIPS_SAMPLES test samples (batch 1, paired cloth) through
        pipeline.TryOnGraph with the trainer's cloth-mask composition (under --GT: the generator alone through pipeline.GeneratorGraph,
        on the ground-truth parse and cloth of a test loader with keys EVAL_GT_KEYS), each scored by lpips(T2(image), T2(output)) with
        T2 = transforms.Resize((128, 128)), summed on the device in sample order and divided by the count.  The try-on noise is drawn
        from a fork of the CUDA generator, so evaluations leave the training's random stream (and a resumed run) unchanged; the
        reference draws it from the training stream."""
        from torchvision.transforms import transforms

        from . import pipeline
        test_loader, lpips = self.evaluator
        n = min(self.lpips_samples, len(test_loader.dataset))
        T2 = transforms.Compose([transforms.Resize((128, 128))])
        G, tocg = self.trainer.G, self.trainer.tocg
        gt = getattr(self.trainer, "gt", False)
        G.eval()
        try:
            with torch.random.fork_rng(devices=[test_loader.device]), torch.no_grad():
                if self._tryon is None:
                    self._tryon = (pipeline.GeneratorGraph(G) if gt else
                                   pipeline.TryOnGraph(tocg, G, occlusion=self.trainer.occlusion,
                                                       clothmask_composition=getattr(self.trainer, "clothmask_composition", "warp_grad")))
                test_loader.start_at(0, 0)
                total = 0.0
                for _ in range(n):
                    b = test_loader.next_batch()
                    if gt:  # train_generator.py:569-576
                        out = self._tryon(torch.cat((b["agnostic"], b["densepose"], b["parse_cloth"]), 1), b["gen_parse"])
                    else:
                        out = self._tryon({k: b[k] for k in EVAL_KEYS if k != "image"})[0]
                    total += lpips.forward(T2(b["image"]), T2(out))
                value = float(total / n)
        finally:
            G.train()
        return value

    def validate(self):
        """train_condition.py:314-360: validation_iou of the tocg in eval mode over the validator, through one
        pipeline.SegmentationGraph that re-captures once per validation (the weights changed since the last).  Eval mode leaves the
        BatchNorm statistics alone and validation_iou forks the random streams, so a validation does not change the training that
        follows."""
        from . import pipeline
        tocg = self.trainer.tocg
        tocg.eval()
        try:
            if self._seg is None:
                self._seg = pipeline.SegmentationGraph(tocg)
            return validation_iou(self._seg, self.validator, self.val_samples)
        finally:
            tocg.train()


def validation_iou(runner, loader, samples=VAL_SAMPLES):
    """The value train_condition.py's validation logs: the IoU of runner (a pipeline.SegmentationGraph) on the first min(samples,
    len) samples of `loader` (a VitonHDLoader in mode "test", keys VAL_KEYS, shuffle=False) in full batches of its batch size
    (drop_last), paired cloth.  Each batch's IoU stays on the device; the result is np.mean of the batch IoUs as Python floats (the
    reference's np.mean(iou_list)), read with one copy.  Every call starts at the first sample, whereas the reference reads its test
    loader from wherever the previous validation stopped (DESIGN.md)."""
    import numpy as np
    batches = min(samples, len(loader.dataset)) // loader.batch_size
    if batches < 1:
        raise ValueError("validation_iou: %d test samples make no batch of %d" % (min(samples, len(loader.dataset)), loader.batch_size))
    with torch.random.fork_rng(devices=[loader.device]), torch.no_grad():
        loader.start_at(0, 0)
        ious = torch.empty(batches, dtype=torch.float32, device=loader.device)
        for i in range(batches):
            ious[i] = runner(loader.next_batch())
        return float(np.mean(ious.tolist()))


# -------------------------------------------------------------------------------------------------------------------- command line

def parse_args(stage, argv=None):
    """The reference's flags that matter for a run on the graph step (train_condition.py:43-115, train_generator.py:33-128), plus
    --resume (a state file), --seed and --lr_interval.  Refuses values the run could not honour."""
    if stage not in STAGES:
        raise SystemExit("stage must be one of %s, not %r" % (", ".join(STAGES), stage))
    s2 = stage == "stage2"
    p = argparse.ArgumentParser(prog="train.py %s" % stage)
    p.add_argument("--name", default="test" if not s2 else None, required=s2)
    p.add_argument("-j", "--workers", type=int, default=4)
    p.add_argument("-b", "--batch_size", "--batch-size", dest="batch_size", type=int, default=8)
    p.add_argument("--fp16", action="store_true", help="fp16 storage with dynamic loss scaling")
    p.add_argument("--dataroot", default="./data/")
    p.add_argument("--datamode", default="train")
    p.add_argument("--data_list", default="train_pairs.txt")
    p.add_argument("--fine_width", type=int, default=768 if s2 else 192)
    p.add_argument("--fine_height", type=int, default=1024 if s2 else 256)
    p.add_argument("--checkpoint_dir", default="checkpoints")
    p.add_argument("--tocg_checkpoint", default=None if s2 else "")
    p.add_argument("--display_count", type=int, default=100)
    p.add_argument("--save_count", type=int, default=10000)
    p.add_argument("--load_step", type=int, default=0)
    p.add_argument("--keep_step", type=int, default=100000 if s2 else 300000)
    p.add_argument("--G_lr", type=float, default=1e-4 if s2 else 2e-4)
    p.add_argument("--D_lr", type=float, default=4e-4 if s2 else 2e-4)
    p.add_argument("--occlusion", action="store_true")
    p.add_argument("--seed", type=int, default=0, help="model initialisation, data order and noise")
    p.add_argument("--resume", default=None, help="a state file (state_step_%%06d.pth) written by an earlier run")
    p.add_argument("--test_dataroot", default="./data/")
    p.add_argument("--test_data_list", default="test_pairs.txt")
    if s2:
        p.add_argument("--decay_step", type=int, default=100000)
        p.add_argument("--lpips_count", type=int, default=1000)
        p.add_argument("--lr_interval", type=int, default=1000, help="steps between scheduler steps (the reference's 1000)")
        p.add_argument("--GT", action="store_true", help="train on the ground-truth parse and cloth: no tocg")
        p.add_argument("--clothmask_composition", choices=train_step.CLOTHMASK_COMPOSITIONS, default="warp_grad")
        p.add_argument("--no_ganFeat_loss", action="store_true", help="no discriminator feature-matching term")
        p.add_argument("--no_vgg_loss", action="store_true", help="no VGG term")
        p.add_argument("--lambda_feat", type=float, default=10.0)
        p.add_argument("--lambda_vgg", type=float, default=10.0)
    else:
        p.add_argument("--val_count", type=int, default=None, help="steps between validations (segmentation IoU); default: none")
        p.add_argument("--edgeawaretv", choices=train_step.EDGEAWARETV, default="no_edge", help="edge-aware flow TV")
        p.add_argument("--add_lasttv", action="store_true", help="with --edgeawaretv: add the plain TV of the last flow")
        p.add_argument("--clothmask_composition", choices=train_step.CLOTHMASK_COMPOSITIONS, default="warp_grad")
        p.add_argument("--no_GAN_loss", action="store_true", help="train the tocg without the discriminator")
        p.add_argument("--G_D_seperate", action="store_true", help="step G first, then D on a new tocg forward")
        p.add_argument("--tvlambda", type=float, default=2.0)
        p.add_argument("--CElamda", type=float, default=10.0)
        p.add_argument("--GANlambda", type=float, default=1.0)
        for flag in ("--lasttvonly", "--interflowloss", "--Ddownx2", "--Ddropout"):  # the README's stage-1 command line
            p.add_argument(flag, action="store_true", help="always on: accepted so that the README's command line parses")
    opt = p.parse_args(argv)
    opt.stage = stage
    positive = ["workers", "batch_size", "fine_width", "fine_height", "display_count", "save_count", "keep_step"] + (["lpips_count", "lr_interval"]
                                                                                                                     if s2 else [])
    for k in positive:
        if getattr(opt, k) < (0 if k == "workers" else 1):
            p.error("--%s must be %s, got %d" % (k, "non-negative" if k == "workers" else "positive", getattr(opt, k)))
    if not s2 and opt.val_count is not None and opt.val_count < 1:
        p.error("--val_count must be positive, got %d" % opt.val_count)
    if not s2 and opt.val_count and opt.clothmask_composition != "warp_grad":
        p.error("--val_count validates the 'warp_grad' composition only, not --clothmask_composition %s" % opt.clothmask_composition)
    if opt.load_step < 0 or (s2 and opt.decay_step < 0):
        p.error("--load_step and --decay_step must be non-negative")
    end = opt.keep_step + (opt.decay_step if s2 else 0)
    if opt.load_step >= end:
        p.error("--load_step %d leaves nothing to train (the run ends at step %d)" % (opt.load_step, end))
    if opt.G_lr <= 0 or opt.D_lr <= 0:
        p.error("--G_lr and --D_lr must be positive")
    if s2 and opt.GT:  # each of these acts on the tocg, which a --GT run does not have
        for flag, given in (("--tocg_checkpoint", opt.tocg_checkpoint is not None), ("--occlusion", opt.occlusion),
                            ("--clothmask_composition", opt.clothmask_composition != "warp_grad")):
            if given:
                p.error("%s acts on the condition generator, which a --GT run does not have" % flag)
    elif s2 and opt.tocg_checkpoint is None:
        p.error("the following arguments are required: --tocg_checkpoint (unless --GT)")
    if opt.resume is not None and opt.load_step:
        p.error("--resume takes the step from the state file; --load_step starts a new run")
    want = data.resized_size(1024, 768, opt.fine_width)
    if (opt.fine_height, opt.fine_width) != want:
        p.error("--fine_height %d: VITON-HD's 1024x768 images resize to %dx%d at --fine_width %d" % (opt.fine_height, want[0], want[1], opt.fine_width))
    for k in ("dataroot",) + (("tocg_checkpoint",) if s2 and not opt.GT else ()) + (("test_dataroot",) if not s2 and opt.val_count else ()):
        if not os.path.exists(getattr(opt, k)):
            p.error("--%s %s does not exist" % (k, getattr(opt, k)))
    if opt.resume is not None and not os.path.isfile(opt.resume):
        p.error("--resume %s is not a file" % opt.resume)
    return opt


def stage1_options(opt):
    """The Stage1Trainer keywords (the keys of STAGE1_OPTIONS) of parsed stage-1 flags."""
    return {"edgeawaretv": opt.edgeawaretv, "add_lasttv": opt.add_lasttv, "clothmask_composition": opt.clothmask_composition,
            "no_gan_loss": opt.no_GAN_loss, "g_d_separate": opt.G_D_seperate, "tvlambda": opt.tvlambda, "ce_lambda": opt.CElamda,
            "gan_lambda": opt.GANlambda}


def stage2_options(opt):
    """The keys of STAGE2_OPTIONS of parsed stage-2 flags (no_ganFeat_loss goes to the discriminator, the rest to Stage2Trainer)."""
    return {"gt": opt.GT, "clothmask_composition": opt.clothmask_composition, "no_vgg_loss": opt.no_vgg_loss,
            "no_ganFeat_loss": opt.no_ganFeat_loss, "lambda_feat": opt.lambda_feat, "lambda_vgg": opt.lambda_vgg}


def build(opt, log=print):
    """Models, trainer, loaders and the TrainRun for parsed flags (one rank of a torchrun job when WORLD_SIZE > 1)."""
    import types

    # bit-reproducible steps (INTEGRATION.md, Reproducibility): cuBLAS (the spectral norms' power iteration) needs a fixed workspace,
    # read when its first handle is made
    os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    torch.use_deterministic_algorithms(True)
    torch.utils.deterministic.fill_uninitialized_memory = False
    import networks
    from . import ddp
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if world > 1:
        import torch.distributed as dist
        local = int(os.environ.get("LOCAL_RANK", "0"))
        torch.cuda.set_device(local)
        if not dist.is_initialized():
            dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    _, rank, world = _dist()
    if opt.batch_size % world:
        raise SystemExit("-b %d is the global batch: it must be a multiple of the %d ranks" % (opt.batch_size, world))
    dev = torch.device("cuda", torch.cuda.current_device())
    ops.set_precision("fp16" if opt.fp16 else "bf16")
    loss_scale = "dynamic" if opt.fp16 else None
    torch.manual_seed(opt.seed)
    s2 = opt.stage == "stage2"
    gt = s2 and opt.GT
    s2_opts = stage2_options(opt) if s2 else {}
    topt = types.SimpleNamespace(warp_feature="T1", out_layer="relu", cuda=True)
    tocg = None if gt else networks.ConditionGenerator(topt, 4, 16, 13, ngf=96, norm_layer=torch.nn.BatchNorm2d)
    if opt.tocg_checkpoint:
        networks.load_checkpoint(tocg, opt.tocg_checkpoint, topt)
    vgg = None if s2_opts.get("no_vgg_loss") else networks.Vgg19().to(dev).eval()
    if s2:
        import network_generator
        gopt = types.SimpleNamespace(norm_G="spectralaliasinstance", gen_semantic_nc=7, ngf=64, num_upsampling_layers="most",
                                     fine_height=opt.fine_height, fine_width=opt.fine_width, cuda=True, ndf=64, norm_D="spectralinstance",
                                     n_layers_D=3, num_D=2, no_ganFeat_loss=s2_opts.pop("no_ganFeat_loss"), init_type="xavier",
                                     init_variance=0.02)
        G = network_generator.SPADEGenerator(gopt, 9).to(dev)
        G.init_weights(gopt.init_type, gopt.init_variance)
        D = network_generator.MultiscaleDiscriminator(gopt).to(dev)
        D.init_weights(gopt.init_type, gopt.init_variance)  # utils.create_network
        tocg = None if gt else tocg.to(dev).eval()
        trained = (G.train(), D.train())
    else:
        if world > 1:  # every rank normalises over the global batch and holds the same running statistics (INTEGRATION.md)
            tocg = ddp.convert_model(tocg)
        D = networks.define_D(input_nc=33, Ddownx2=True, Ddropout=True, n_layers_D=3, spectral=False, num_D=2)
        tocg, D = tocg.to(dev).train(), D.to(dev).train()
        trained = (tocg, D)
    reducers = {}
    if world > 1:
        for m in (tocg,) + trained:
            if m is not None:
                ddp.broadcast_module_state(m)
        reducers = {"G": ddp.GradBucketReducer(list(trained[0].parameters())), "D": ddp.GradBucketReducer(list(trained[1].parameters()))}
    torch.cuda.manual_seed(opt.seed * 1000 + rank)  # per-rank noise and dropout
    if s2:
        trainer = train_step.Stage2Trainer(tocg, G, D, vgg, g_lr=opt.G_lr, d_lr=opt.D_lr, reducers=reducers, occlusion=opt.occlusion,
                                           loss_scale=loss_scale, tensor_lr=True, **s2_opts)
    else:
        trainer = train_step.Stage1Trainer(tocg, D, vgg, lr=opt.G_lr, d_lr=opt.D_lr, occlusion=opt.occlusion, reducers=reducers,
                                           loss_scale=loss_scale, **stage1_options(opt))
    keys = (train_step.GT_KEYS if gt else data.STAGE2_KEYS) if s2 else data.STAGE1_KEYS
    loader = data.VitonHDLoader(opt.dataroot, opt.datamode, opt.data_list, opt.fine_height, opt.fine_width, opt.batch_size // world,
                                workers=opt.workers, keys=keys, seed=opt.seed)
    evaluator = None
    if s2 and rank == 0:
        import eval_models
        test_loader = data.VitonHDLoader(opt.test_dataroot, "test", opt.test_data_list, opt.fine_height, opt.fine_width, 1,
                                         workers=opt.workers, mode="test", keys=EVAL_GT_KEYS if gt else EVAL_KEYS, shuffle=False, shard=False)
        evaluator = (test_loader, eval_models.PerceptualLoss(model="net-lin", net="alex", use_gpu=True, gpu_ids=[dev.index]))
    validator = None
    if not s2 and opt.val_count and rank == 0:
        validator = data.VitonHDLoader(opt.test_dataroot, "test", opt.test_data_list, opt.fine_height, opt.fine_width, opt.batch_size // world,
                                       workers=opt.workers, mode="test", keys=VAL_KEYS, shuffle=False, shard=False)
    run = TrainRun(opt.stage, trainer, loader, os.path.join(opt.checkpoint_dir, opt.name), opt.keep_step,
                   decay_step=opt.decay_step if s2 else 0, load_step=opt.load_step, interval=opt.lr_interval if s2 else 1000,
                   save_count=opt.save_count, display_count=opt.display_count, lpips_count=opt.lpips_count if s2 else None,
                   evaluator=evaluator, val_count=None if s2 else opt.val_count, validator=validator, log=log)
    if opt.resume:
        run.resume(opt.resume)
    return run


def main(argv=None):
    argv = sys.argv[1:] if argv is None else argv
    if not argv or argv[0] not in STAGES:
        raise SystemExit("usage: train.py {stage1|stage2} [flags]  (train.py stage2 --help)")
    opt = parse_args(argv[0], argv[1:])
    run = build(opt)
    try:
        run.start().train()
    finally:
        run.trainer.release_graph()
        dist, _, _ = _dist()
        if dist is not None:
            dist.destroy_process_group()
    return run
