"""One stage-2 training step (frozen tocg -> warp -> SPADE G -> D; hinge + feature-matching + VGG; Adam), restating the
body of the reference loop train_generator.py:201-360 as a callable so bench.py / tests can drive it on synthetic batches.

Hot path = the three networks (kernels of this repo).  The per-step tensor glue between them (nearest/bilinear resizes,
15x15 Gaussian blur, argmax -> one-hot -> 7-class regroup, hi-res grid_sample of the cloth) is SURVEY.md §8(f) row N2
("next"): it runs as torch ops here."""
import torch
import torch.nn.functional as F

from . import loss_scale as loss_scale_mod
from . import ops

_GRID_CACHE = {}
LABELS7 = [[0], [2, 4, 7, 8, 9, 10, 11], [3], [1], [5], [6], [12]]  # train_generator.py:261-269
GROUP_OF_13 = [next(i for i, grp in enumerate(LABELS7) if k in grp) for k in range(13)]
OCCLUSION_CLASSES = [1, 2, 5, 6, 7, 8, 9, 10, 11, 12]  # remove_overlap: seg_out[:, 1:3] and seg_out[:, 5:] (train_generator.py:26-31)


def gaussian_blur_15_3(x):
    """tgm.image.GaussianBlur((15,15),(3,3)) restated: depth-wise separable 15-tap Gaussian, sigma 3, zero padding 7
    (SURVEY.md §8c: torchgeometry is absent from the image; the restatement is pinned against scipy.ndimage.gaussian_filter, an
    independent implementation of the same published filter: tests/test_host_logic.py)."""
    k = torch.arange(15, dtype=torch.float32, device=x.device) - 7
    g = torch.exp(-(k * k) / (2 * 3.0 * 3.0))
    g = g / g.sum()
    c = x.shape[1]
    x = F.conv2d(x, g.view(1, 1, 1, 15).expand(c, 1, 1, 15), padding=(0, 7), groups=c)
    return F.conv2d(x, g.view(1, 1, 15, 1).expand(c, 1, 15, 1), padding=(7, 0), groups=c)


def make_generator_inputs(tocg, batch, fine_h, fine_w, occlusion=False, unfused_parse=False):
    """train_generator.py:201-275 (opt.GT False, clothmask_composition 'warp_grad').
    unfused_parse=True keeps the parse-map post-processing as the separate torch ops of the reference (what the tests use to
    check the fused kernel, also on CPU tensors); the product path is the kernel and needs CUDA tensors."""
    from .tocg import make_grid
    cm, c_paired = batch["cloth_mask"], batch["cloth"]
    with torch.no_grad():
        pre_cm_down = F.interpolate(cm, size=(256, 192), mode="nearest")
        parse_agn_down = F.interpolate(batch["parse_agnostic"], size=(256, 192), mode="nearest")
        clothes_down = F.interpolate(c_paired, size=(256, 192), mode="bilinear")
        dense_down = F.interpolate(batch["densepose"], size=(256, 192), mode="bilinear")
        input1 = torch.cat([clothes_down, pre_cm_down], 1)
        input2 = torch.cat([parse_agn_down, dense_down], 1)
        flow_list, fake_segmap, _, warped_cm = tocg(input1, input2)
        mask = torch.ones_like(fake_segmap)
        mask[:, 3:4] = warped_cm
        fake_segmap = fake_segmap * mask
        n, _, ih, iw = c_paired.shape
        if unfused_parse or not c_paired.is_cuda:
            key = (n, ih, iw, str(c_paired.device))
            if key not in _GRID_CACHE:  # the reference rebuilds this on the CPU and copies it every step (networks.py:162-165)
                _GRID_CACHE[key] = make_grid(n, ih, iw).to(c_paired.device)
            grid = _GRID_CACHE[key]
            flow = F.interpolate(flow_list[-1].permute(0, 3, 1, 2), size=(ih, iw), mode="bilinear").permute(0, 2, 3, 1)
            flow_norm = torch.cat([flow[..., 0:1] / ((96 - 1.0) / 2.0), flow[..., 1:2] / ((128 - 1.0) / 2.0)], 3)
            warped_grid = grid + flow_norm
            warped_cloth = F.grid_sample(c_paired, warped_grid, padding_mode="border", align_corners=False)
            warped_clothmask = F.grid_sample(cm, warped_grid, padding_mode="border", align_corners=False)
        else:
            # product path: parse post-processing in one kernel (bilinear resize -> 15x15 Gaussian -> argmax -> one-hot -> 13->7 regroup,
            # plus, under --occlusion, the softmax-overlap plane), then the hi-res warp of cloth + mask (flow x8 up-sampling, normalise,
            # base grid, grid_sample, remove_overlap, white composite) in one kernel: no (N,H,W,2) grid, no 13 blurred planes in HBM
            from . import ops
            div = ((96 - 1.0) / 2.0, (128 - 1.0) / 2.0)
            if occlusion:
                _, parse, overlap = ops.parse_blur_argmax(fake_segmap.float(), (ih, iw), group_of=GROUP_OF_13, groups=7, want_idx=False,
                                                          overlap_classes=OCCLUSION_CLASSES)
                warped_cloth, _, warped_clothmask = ops.flow_warp_nchw(flow_list[-1], c_paired.float(), (ih, iw), div, mask=cm, overlap=overlap,
                                                                       composite=True)
            else:
                _, parse = ops.parse_blur_argmax(fake_segmap.float(), (ih, iw), group_of=GROUP_OF_13, groups=7, want_idx=False)
                warped_cloth, _ = ops.flow_warp_nchw(flow_list[-1], c_paired.float(), (ih, iw), div)
            g_in = torch.cat((batch["agnostic"], batch["densepose"], warped_cloth), 1)
            return g_in.detach(), parse.detach()
        # ---- reference formulation with separate torch ops (CPU oracle pipeline of the tests; unfused_parse=True)
        fake_parse_gauss = gaussian_blur_15_3(F.interpolate(fake_segmap, size=(ih, iw), mode="bilinear"))
        fake_parse = fake_parse_gauss.argmax(dim=1)[:, None]
        if occlusion:
            so = F.softmax(fake_parse_gauss, dim=1)
            warped_clothmask = warped_clothmask - torch.cat([so[:, 1:3], so[:, 5:]], 1).sum(1, keepdim=True) * warped_clothmask
            warped_cloth = warped_cloth * warped_clothmask + (1 - warped_clothmask)
        old_parse = torch.zeros(n, 13, fine_h, fine_w, device=cm.device).scatter_(1, fake_parse, 1.0)
        mkey = ("regroup", str(cm.device))
        if mkey not in _GRID_CACHE:  # 13 -> 7 class regrouping as a constant 7x13 0/1 matrix (train_generator.py:261-273)
            m = torch.zeros(7, 13)
            for i, idx in enumerate(LABELS7):
                m[i, idx] = 1.0
            _GRID_CACHE[mkey] = m.to(cm.device)
        parse = torch.einsum("ij,njhw->nihw", _GRID_CACHE[mkey], old_parse)
        g_in = torch.cat((batch["agnostic"], batch["densepose"], warped_cloth), 1)
    return g_in.detach(), parse.detach()


def _attach_reducers(reducers):
    """Data-parallel gradient exchange of the bundled trainers: by default the reducers' hooks launch each bucket's all-reduce as soon
    as its last gradient exists (overlapping the rest of backward()); HRV_DDP_MODE=explicit reduces after backward() instead.
    Returns True when the step has to call reduce() itself."""
    import os
    if os.environ.get("HRV_DDP_MODE", "hooks") == "explicit":
        return True
    for r in reducers.values():
        r.attach()
    return False


class BatchFeeder:
    """Input feeding (SURVEY.md 8f N4; cp_dataset.py:404-426 hands the loop one CPU batch per step): pinned host tensors travel on a
    COPY stream into one of two device staging slots while the previous step still computes; one-hot maps (13-channel parse maps, half
    of the batch's bytes as fp32) travel as ONE byte per pixel and are expanded on the device (hrv_onehot_u8).  consume() hands the
    staged batch to the step as fp32 tensors (the graph's static inputs, or a per-step dict)."""
    ONEHOT = ("parse_agnostic", "parse")

    def __init__(self, batch_cpu, device):
        self.device = device
        self.host, self.classes = {}, {}
        for k, v in batch_cpu.items():
            if k in self.ONEHOT and v.dim() == 4 and v.shape[1] > 1:
                self.classes[k] = v.shape[1]
                self.host[k] = v.argmax(1, keepdim=True).to(torch.uint8).contiguous().pin_memory()
            else:
                self.host[k] = v.contiguous().pin_memory()
        self.slots = [{k: torch.empty(v.shape, dtype=v.dtype, device=device) for k, v in self.host.items()} for _ in range(2)]
        self.copy_stream = torch.cuda.Stream(device)
        self.ready = [torch.cuda.Event(), torch.cuda.Event()]
        self.free = [torch.cuda.Event(), torch.cuda.Event()]
        self.bytes_per_step = int(sum(v.numel() * v.element_size() for v in self.host.values()))
        self.slot = 0

    def prefetch(self, slot=None):
        slot = self.slot if slot is None else slot
        with torch.cuda.stream(self.copy_stream):
            self.copy_stream.wait_event(self.free[slot])  # the step that consumed this slot last has read it
            for k, v in self.host.items():
                self.slots[slot][k].copy_(v, non_blocking=True)
            self.ready[slot].record(self.copy_stream)

    def consume(self, out):
        """Makes the staged batch of the current slot available in `out` (dict of fp32 device tensors), then starts the copy of the
        next batch into the other slot.  Stream-ordered: no host synchronisation."""
        from . import ops
        slot = self.slot
        cur = torch.cuda.current_stream()
        cur.wait_event(self.ready[slot])
        for k, v in self.slots[slot].items():
            if k in self.classes:
                ops.onehot_u8(v, self.classes[k], out=out[k])
            else:
                out[k].copy_(v, non_blocking=True)
        self.free[slot].record(cur)
        self.slot ^= 1
        self.prefetch(self.slot)
        return out


class _GraphMixin:
    """Capture one whole step (all optimiser updates) into a CUDA graph over static copies of the batch: removes the thousands of
    Python-driven launches per step from the critical path.  capture(batch, *step_args) once, then replay(new_batch)."""

    _captured = None

    def capture(self, batch, *step_args, warm=2):
        from .graphs import CapturedCall
        self._static = {k: v.clone() for k, v in batch.items()}
        import torch.distributed as dist
        multi = dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1
        # with NCCL inside the graph the process group's watchdog thread keeps polling CUDA events: thread-local capture mode keeps
        # those calls from invalidating the capture
        self._captured = CapturedCall(lambda: self.step(self._static, *step_args), warm=warm,
                                      capture_error_mode="thread_local" if multi else "global")
        return self

    def replay(self, batch=None, feeder=None):
        if feeder is not None:
            feeder.consume(self._static)  # staged on the copy stream while the previous replay ran
        elif batch is not None:
            for k, v in batch.items():
                self._static[k].copy_(v, non_blocking=True)
        out = self._captured.replay()
        ops.PARAM_GEN[0] += 1  # the replayed optimiser step changed parameters without touching tensor._version: derived caches are stale
        return out

    def release_graph(self):
        """Destroy the captured graph (graphs.CapturedCall.release)."""
        if self._captured is not None:
            self._captured.release()
            self._captured = None


class _LossScaling:
    """loss_scale="dynamic": one loss_scale.DynamicLossScaler per loss ("G", "D"), as apex O1 with num_losses=2.  The scaled step keeps
    every gradient tensor allocated across steps (zero_grad(set_to_none=False)), so the device table of the unscale kernel is built once
    and a captured graph can run it; with loss_scale=None (the default) the step is exactly the unscaled one."""

    def _init_loss_scale(self, loss_scale, optimizers):
        device = optimizers["G"].param_groups[0]["params"][0].device
        self.scalers = loss_scale_mod.make_scalers(loss_scale, list(optimizers), device)
        for name, sc in self.scalers.items():
            optimizers[name].found_inf = sc.found_inf  # torch's fused Adam skips the update (and undoes its step count) where it is 1

    def _backward(self, loss, name):
        sc = self.scalers.get(name)
        (loss if sc is None else sc.scale_loss(loss)).backward()

    def _opt_step(self, opt, name):
        sc = self.scalers.get(name)
        if sc is not None:
            sc.unscale_and_check(opt, self.reducers.get(name))
        opt.step()
        if sc is not None:
            sc.update()


class Stage2Trainer(_GraphMixin, _LossScaling):
    """Holds the optimisers / criteria of train_generator.py:145-159 and runs one step.  loss_scale: None or "dynamic" (fp16 storage:
    apex O1's dynamic loss scaling, see loss_scale.py and _LossScaling)."""

    def __init__(self, tocg, generator, discriminator, vgg, lambda_feat=10.0, lambda_vgg=10.0, g_lr=1e-4, d_lr=4e-4,
                 reducers=None, occlusion=True, loss_scale=None):
        from .spade import GANLoss
        self.tocg, self.G, self.D, self.vgg = tocg, generator, discriminator, vgg
        self.crit_gan = GANLoss("hinge")
        self.vgg_weights = [1.0 / 32, 1.0 / 16, 1.0 / 8, 1.0 / 4, 1.0]
        self.lambda_feat, self.lambda_vgg = lambda_feat, lambda_vgg
        self.occlusion = occlusion  # opt.occlusion: the README trains stage 2 with --occlusion
        self.opt_g = torch.optim.Adam(generator.parameters(), lr=g_lr, betas=(0.0, 0.9), fused=True, capturable=True)
        self.opt_d = torch.optim.Adam(discriminator.parameters(), lr=d_lr, betas=(0.0, 0.9), fused=True, capturable=True)
        self.reducers = reducers or {}  # {"G": GradBucketReducer, "D": ...} for data-parallel runs
        self._explicit_reduce = _attach_reducers(self.reducers)
        self._init_loss_scale(loss_scale, {"G": self.opt_g, "D": self.opt_d})

    @staticmethod
    def _split(pred):
        fake = [[t[:t.size(0) // 2] for t in p] for p in pred]
        real = [[t[t.size(0) // 2:] for t in p] for p in pred]
        return fake, real

    def step(self, batch, fine_h, fine_w):
        from . import autograd_g
        ops.require_trainable_storage("Stage2Trainer.step")
        g_in, parse = make_generator_inputs(self.tocg, batch, fine_h, fine_w, occlusion=self.occlusion)
        im = batch["image"]
        # ---------------- generator update (train_generator.py:279-322)
        out = self.G(g_in, parse)
        d_in = torch.cat((torch.cat((parse, out), 1), torch.cat((parse, im), 1)), 0)
        pred = autograd_g.discriminator_forward_train(self.D, d_in, need_wgrad=False, as_float=False, raw=True)  # D grads are zeroed before use (:354)
        pred_fake, _ = self._split([[p[-1]] for p in pred])
        loss_gan = self.crit_gan(pred_fake, True, for_discriminator=False)
        loss_feat = 0
        num_d = len(pred)
        for i in range(num_d):
            for j in range(len(pred[i]) - 1):  # intermediate features: [fake; real] halves of one pixel-major buffer
                loss_feat = loss_feat + autograd_g.FeatMatchFn.apply(pred[i][j]) * self.lambda_feat / num_d
        loss_vgg = autograd_g.vgg_loss(self.vgg, self.vgg_weights, out, im) * self.lambda_vgg
        loss_gen = (loss_gan + loss_feat + loss_vgg).mean()
        self.opt_g.zero_grad(set_to_none=not self.scalers)
        self._backward(loss_gen, "G")  # data-parallel: bucket all-reduces are launched from gradient hooks DURING this call (ddp.py)
        if "G" in self.reducers and self._explicit_reduce:
            self.reducers["G"].reduce()
        self._opt_step(self.opt_g, "G")
        # ---------------- discriminator update (train_generator.py:327-360)
        with torch.no_grad():
            out2 = self.G(g_in, parse)
        d_in = torch.cat((torch.cat((parse, out2), 1), torch.cat((parse, im), 1)), 0)
        pred = autograd_g.discriminator_forward_train(self.D, d_in, need_wgrad=True, as_float=False)
        pred_fake, pred_real = self._split(pred)
        loss_dis = (self.crit_gan(pred_fake, False, for_discriminator=True) + self.crit_gan(pred_real, True, for_discriminator=True)).mean()
        self.opt_d.zero_grad(set_to_none=not self.scalers)
        self._backward(loss_dis, "D")
        if "D" in self.reducers and self._explicit_reduce:
            self.reducers["D"].reduce()
        self._opt_step(self.opt_d, "D")
        return {"loss_gen": loss_gen.detach(), "loss_dis": loss_dis.detach(), "gan": loss_gan.detach(),
                "feat": loss_feat.detach() if torch.is_tensor(loss_feat) else loss_feat, "vgg": loss_vgg.detach()}


def synthetic_batch(n, h, w, device, seed=0):
    """Synthetic VITON-HD-shaped batch (shapes/ranges of cp_dataset.py outputs; SURVEY.md §8d)."""
    g = torch.Generator(device="cpu").manual_seed(seed)

    def smooth(c):
        t = torch.rand((n, c, h // 16, w // 16), generator=g) * 2 - 1
        return F.interpolate(t, size=(h, w), mode="bilinear", align_corners=False)

    def onehot(c):
        lab = torch.randint(0, c, (n, h // 32, w // 32), generator=g).repeat_interleave(32, 1).repeat_interleave(32, 2)
        return torch.zeros(n, c, h, w).scatter_(1, lab[:, None], 1.0)

    b = {"cloth": smooth(3), "cloth_mask": (smooth(1) > 0).float(), "parse_agnostic": onehot(13), "densepose": smooth(3),
         "agnostic": smooth(3), "image": smooth(3)}
    return {k: v.to(device) for k, v in b.items()}


# ------------------------------------------------------------------------------------------------ stage 1 (train_condition.py)

class Stage1Trainer(_GraphMixin, _LossScaling):
    """One train_condition.py step (train_condition.py:133-286) with the README's flags (--Ddownx2 --Ddropout --lasttvonly
    --interflowloss --occlusion): tocg forward+backward on this repo's kernels (train-mode BatchNorm), L1 + VGG + TV + CE + LSGAN.
    loss_scale: None or "dynamic" (as Stage2Trainer)."""

    def __init__(self, tocg, D, vgg, lr=2e-4, lasttvonly=True, interflowloss=True, occlusion=True, tvlambda=2.0, ce_lambda=10.0,
                 gan_lambda=1.0, reducers=None, loss_scale=None):
        self.tocg, self.D, self.vgg = tocg, D, vgg
        self.lasttvonly, self.interflowloss, self.occlusion = lasttvonly, interflowloss, occlusion
        self.tvlambda, self.ce_lambda, self.gan_lambda = tvlambda, ce_lambda, gan_lambda
        self.vgg_weights = [1.0 / 32, 1.0 / 16, 1.0 / 8, 1.0 / 4, 1.0]
        self.opt_g = torch.optim.Adam(tocg.parameters(), lr=lr, betas=(0.5, 0.999), fused=True, capturable=True)
        self.opt_d = torch.optim.Adam(D.parameters(), lr=lr, betas=(0.5, 0.999), fused=True, capturable=True)
        self.reducers = reducers or {}
        self._explicit_reduce = _attach_reducers(self.reducers)
        self._init_loss_scale(loss_scale, {"G": self.opt_g, "D": self.opt_d})

    @staticmethod
    def _remove_overlap(seg_out, warped_cm):  # train_condition.py:26-31
        return warped_cm - torch.cat([seg_out[:, 1:3], seg_out[:, 5:]], 1).sum(1, keepdim=True) * warped_cm

    @staticmethod
    def _lsgan(pred, real):  # networks.GANLoss (LSGAN) on the last output of every scale (networks.py:288-299)
        return sum(F.mse_loss(p[-1].float(), torch.full_like(p[-1], 1.0 if real else 0.0, dtype=torch.float32)) for p in pred)

    def step(self, batch):
        from . import autograd_g, autograd_tocg
        ops.require_trainable_storage("Stage1Trainer.step")
        c_paired, im_c, pcm = batch["cloth"], batch["parse_cloth"], batch["pcm"]
        cm_paired = (batch["cloth_mask"] > 0.5).float()
        input1 = torch.cat([c_paired, cm_paired], 1)
        input2 = torch.cat([batch["parse_agnostic"], batch["densepose"]], 1)
        flow_list, seg, warped_c, warped_cm = autograd_tocg.tocg_forward_train(self.tocg, input1, input2)
        mask = torch.ones_like(seg.detach())
        mask = torch.cat([mask[:, :3], warped_cm, mask[:, 4:]], 1)  # clothmask_composition == 'warp_grad'
        seg = seg * mask
        if self.occlusion:
            warped_cm = self._remove_overlap(F.softmax(seg, dim=1), warped_cm)
            warped_c = warped_c * warped_cm + (1 - warped_cm)
        loss_l1 = F.l1_loss(warped_cm, pcm)
        loss_vgg = autograd_g.vgg_loss(self.vgg, self.vgg_weights, warped_c, im_c)
        loss_tv = 0
        for flow in (flow_list[-1:] if self.lasttvonly else flow_list):
            loss_tv = loss_tv + (flow[:, 1:] - flow[:, :-1]).abs().mean() + (flow[:, :, 1:] - flow[:, :, :-1]).abs().mean()
        n, _, ih, iw = c_paired.shape
        if self.interflowloss:
            # F.interpolate(size, bilinear) + normalise + base grid + grid_sample(border) of cloth and mask: hrv_flow_warp_nchw and its
            # fixed-order backward (torch's grid_sample / interpolate backward accumulate with atomics)
            for i in range(len(flow_list) - 1):
                fh, fw = flow_list[i].shape[1], flow_list[i].shape[2]
                wc, wcm = autograd_tocg.FlowWarpNchwFn.apply(flow_list[i], c_paired, cm_paired, (ih, iw), ((fw - 1.0) / 2.0, (fh - 1.0) / 2.0))
                wcm = self._remove_overlap(F.softmax(seg, dim=1), wcm)
                loss_l1 = loss_l1 + F.l1_loss(wcm, pcm) / (2 ** (4 - i))
                loss_vgg = loss_vgg + autograd_g.vgg_loss(self.vgg, self.vgg_weights, wc, im_c) / (2 ** (4 - i))
        ce = cross_entropy_ignore(seg, batch["parse_onehot"][:, 0].long(), ignore_index=250)  # utils.cross_entropy2d
        soft = torch.softmax(seg, 1)
        d_in = torch.cat((input1.detach(), input2.detach(), soft), 1)
        loss_g_gan = self._lsgan(autograd_tocg.tocg_discriminator_forward_train(self.D, d_in), True)
        pred_fake = autograd_tocg.tocg_discriminator_forward_train(self.D, d_in.detach())
        pred_real = autograd_tocg.tocg_discriminator_forward_train(self.D, torch.cat((input1.detach(), input2.detach(), batch["parse"]), 1))
        loss_d = self._lsgan(pred_fake, False) + self._lsgan(pred_real, True)
        loss_g = (10 * loss_l1 + loss_vgg + self.tvlambda * loss_tv) + (ce * self.ce_lambda + loss_g_gan * self.gan_lambda)
        self.opt_g.zero_grad(set_to_none=not self.scalers)
        self.opt_d.zero_grad(set_to_none=not self.scalers)
        self._backward(loss_g, "G")
        d_stale = [p.grad for p in self.D.parameters()]  # the G loss also back-propagates into D: the reference zeroes it (optimizer_D.zero_grad)
        if "G" in self.reducers and self._explicit_reduce:
            self.reducers["G"].reduce()
        self._opt_step(self.opt_g, "G")
        del d_stale
        self.opt_d.zero_grad(set_to_none=not self.scalers)
        self._backward(loss_d, "D")
        if "D" in self.reducers and self._explicit_reduce:
            self.reducers["D"].reduce()
        self._opt_step(self.opt_d, "D")
        return {"loss_g": loss_g.detach(), "loss_d": loss_d.detach(), "l1": loss_l1.detach(), "vgg": loss_vgg.detach(), "ce": ce.detach()}


def cross_entropy_ignore(logits, target, ignore_index=250):
    """F.cross_entropy(logits (N,C,H,W), target (N,H,W), ignore_index) (mean over the non-ignored pixels) from elementwise ops and
    fixed-tree sums: log_softmax, a one-hot comparison and a valid-pixel mask.  Unlike the NLL loss kernel it has a deterministic CUDA
    forward and backward, so it runs under torch.use_deterministic_algorithms(True)."""
    logp = F.log_softmax(logits, dim=1)
    classes = torch.arange(logits.shape[1], device=logits.device).view(1, -1, 1, 1)
    picked = (logp * (target[:, None] == classes)).sum(1)
    valid = target != ignore_index
    return -(picked * valid).sum() / valid.sum()


def synthetic_batch_stage1(n, h, w, device, seed=0):
    b = synthetic_batch(n, h, w, "cpu", seed)
    g = torch.Generator(device="cpu").manual_seed(seed + 1)
    lab = torch.randint(0, 13, (n, h // 32, w // 32), generator=g).repeat_interleave(32, 1).repeat_interleave(32, 2)
    b["parse_onehot"] = lab[:, None].float()
    b["parse"] = torch.zeros(n, 13, h, w).scatter_(1, lab[:, None], 1.0)
    b["pcm"] = (lab[:, None] == 3).float()
    b["parse_cloth"] = b["image"] * b["pcm"] + (1 - b["pcm"])
    return {k: v.to(device) for k, v in b.items()}
