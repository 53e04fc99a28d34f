"""End-to-end try-on inference: the body of the reference's test_generator.py loop (test_generator.py:117-219) as a callable.

    tocg (256x192) -> cloth-mask composition -> parse map (up-sample, 15x15 Gaussian, arg-max, 13->7 regroup) -> hi-res cloth warp
    (+ occlusion handling) -> SPADEGenerator -> image

Both networks run on this repo's kernels; the glue between them is two kernels (hrv_parse_blur_argmax, hrv_flow_warp_nchw) instead of
the reference's ~25 torch ops and three numpy round trips (the `> 0.5` thresholds at test_generator.py:128,163 run on the device).
BASELINE.json configs[4]."""
import torch
import torch.nn.functional as F

from . import ops
from .graphs import CapturedCall
from .spade import _param_key
from .train_step import GROUP_OF_13, OCCLUSION_CLASSES


def d_logit(preds):
    """The reference's D_logit (get_norm_const.py:60-64) on a MultiscaleDiscriminator result: the sum over scales of the last
    output's mean over (1,2,3), each divided by 2.  The 2 is hard-coded there: the result is the mean over scales only for
    num_D=2 (the reference's configuration); the reference's arithmetic is kept for every num_D.  (N,) fp32, no synchronisation."""
    score = 0
    for p in preds:
        score = score + p[-1].mean((1, 2, 3)) / 2
    return score


def _check_norm_const(norm_const):
    if norm_const is None or not norm_const > 0:
        raise ValueError("norm_const must be the positive normalising constant M of discriminator rejection "
                         "(pipeline.norm_constant / the reference's get_norm_const.py), got %r" % (norm_const,))


def condition_logit(D, input1, input2, third, cm=None, composition="warp_grad", softmax=True, return_maps=False):
    """l = d_logit(D([input1 | input2 | third'])) for a try-on condition, (N,) fp32 on the device (get_norm_const.py:99-120).
    third' is `third` with its cloth channel (3) multiplied by cm (composition 'warp_grad') or by (cm > 0.5) ('detach'), then
    soft-maxed over channels (softmax=True: the generated segmentation scores) or taken as is (softmax=False: the one-hot `parse`
    label of the real branch).  One kernel builds the discriminator's NHWC input; D runs its eval forward on it.
    return_maps=True also returns the per-scale logit maps the means are taken of."""
    for t in (input1, input2, third) + (() if cm is None else (cm,)):
        if not t.is_cuda:
            raise RuntimeError("condition_logit: hrviton_b200 runs on sm_90a only — got a CPU tensor (there is no CPU fallback)")
    with torch.no_grad():
        a = ops.seg_softmax_cat(input1.float(), input2.float(), third.float(), cm=None if cm is None else cm.float(),
                                composition=composition, softmax=softmax)
        preds = D.forward_act(a)
        l = d_logit(preds)
    return (l, [p[-1] for p in preds]) if return_maps else l


def _condition(tocg, inputs, opt, datasetting):
    """input1, input2 and the tocg outputs for a cp_dataset batch at the tocg resolution (test_condition.py:81-103)."""
    pick = lambda v: v[datasetting] if isinstance(v, dict) else v
    cm = (pick(inputs["cloth_mask"]) > 0.5).float()                                            # test_condition.py:84 (numpy round trip there)
    input1 = torch.cat([pick(inputs["cloth"]), cm], 1)
    input2 = torch.cat([inputs["parse_agnostic"], inputs["densepose"]], 1)
    return input1, input2, (tocg(input1, input2) if opt is None else tocg(opt, input1, input2))


def rejection_scores(tocg, D, inputs, norm_const, opt=None, clothmask_composition="warp_grad", datasetting="paired"):
    """Discriminator rejection (test_condition.py:99-127): inputs is the cp_dataset batch dict at the tocg resolution (cloth /
    cloth_mask as tensors or {setting: tensor} dicts, parse_agnostic, densepose; CUDA fp32 NCHW).  Returns (score (N,), l (N,),
    (flow_list, fake_segmap, warped_cloth, warped_clothmask)) with score = l / (1 - l) / norm_const, on the device."""
    _check_norm_const(norm_const)
    with torch.no_grad():
        input1, input2, outs = _condition(tocg, inputs, opt, datasetting)
        cm = None if clothmask_composition == "no_composition" else outs[3]
        l = condition_logit(D, input1, input2, outs[1], cm=cm, composition=clothmask_composition)
        score = l / (1 - l) / norm_const
    return score, l, outs


def norm_constant(tocg, D, batches, opt=None, clothmask_composition="warp_grad", datasetting="paired"):
    """The normalising constant M of discriminator rejection (get_norm_const.get_const, :65-132): the maximum of l / (1 - l) over
    the real (third = batch["parse"], the one-hot label, no soft-max) and the generated condition of every sample of `batches`
    (an iterable of cp_dataset batch dicts with "parse").  The maximum is kept on the device; the one synchronisation is the
    read of the result."""
    m = None
    with torch.no_grad():
        for inputs in batches:
            input1, input2, outs = _condition(tocg, inputs, opt, datasetting)
            cm = None if clothmask_composition == "no_composition" else outs[3]
            l = torch.cat([condition_logit(D, input1, input2, inputs["parse"], softmax=False),
                           condition_logit(D, input1, input2, outs[1], cm=cm, composition=clothmask_composition)])
            v = (l / (1 - l)).max()
            m = v if m is None else torch.maximum(m, v)
    if m is None:
        raise ValueError("norm_constant: no batches")
    return float(m)


def tryon_forward(tocg, generator, inputs, opt=None, occlusion=True, clothmask_composition="warp_grad", datasetting="paired",
                  discriminator=None, norm_const=None):
    """inputs: the dict a cp_dataset_test.CPDataLoader batch provides (cloth / cloth_mask may be {setting: tensor} dicts or tensors);
    CUDA fp32 NCHW tensors at the fine resolution.  Returns (output image (N,3,H,W), warped_cloth, parse (N,7,H,W)).
    With discriminator= (the stage-1 condition discriminator) and norm_const= the 256x192 condition is also scored as
    rejection_scores does, and a fourth value, score (N,), is returned; the generator still runs for every sample — the caller
    filters on score."""
    if discriminator is not None:
        _check_norm_const(norm_const)
    pick = lambda v: v[datasetting] if isinstance(v, dict) else v
    clothes, pre_cm = pick(inputs["cloth"]), pick(inputs["cloth_mask"])
    agnostic, densepose, parse_agnostic = inputs["agnostic"], inputs["densepose"], inputs["parse_agnostic"]
    with torch.no_grad():
        pre_cm = (pre_cm > 0.5).float()                                                        # test_generator.py:128 (numpy round trip there)
        input1 = torch.cat([F.interpolate(clothes, size=(256, 192), mode="bilinear"), F.interpolate(pre_cm, size=(256, 192), mode="nearest")], 1)
        input2 = torch.cat([F.interpolate(parse_agnostic, size=(256, 192), mode="nearest"), F.interpolate(densepose, size=(256, 192), mode="bilinear")], 1)
        flow_list, fake_segmap, _, warped_cm = tocg(input1, input2) if opt is None else tocg(opt, input1, input2)
        # test_generator.py:163-176: the cloth-mask composition of the scores, inside the kernel that makes the parse map
        comp = dict(cm=None if clothmask_composition == "no_composition" else warped_cm.float(), composition=clothmask_composition)
        if discriminator is not None:
            # the kernel that builds the discriminator's input also writes the composed scores the parse map is made of
            composed = comp["cm"] is not None
            a = ops.seg_softmax_cat(input1, input2, fake_segmap.float(), cm=comp["cm"], composition=clothmask_composition, want_seg=composed)
            if composed:
                a, fake_segmap = a
                comp["cm"] = None
            l = d_logit(discriminator.forward_act(a))
            score = l / (1 - l) / norm_const
        n, _, ih, iw = clothes.shape
        div = ((96 - 1.0) / 2.0, (128 - 1.0) / 2.0)
        if occlusion:
            _, parse, overlap = ops.parse_blur_argmax(fake_segmap.float(), (ih, iw), group_of=GROUP_OF_13, groups=7, want_idx=False,
                                                      overlap_classes=OCCLUSION_CLASSES, **comp)
            warped_cloth, _, _ = ops.flow_warp_nchw(flow_list[-1], clothes.float(), (ih, iw), div, mask=pre_cm, overlap=overlap, composite=True)
        else:
            _, parse = ops.parse_blur_argmax(fake_segmap.float(), (ih, iw), group_of=GROUP_OF_13, groups=7, want_idx=False, **comp)
            warped_cloth, _ = ops.flow_warp_nchw(flow_list[-1], clothes.float(), (ih, iw), div)
        output = generator(torch.cat((agnostic, densepose, warped_cloth), 1), parse)
    return (output, warped_cloth, parse) if discriminator is None else (output, warped_cloth, parse, score)


class _GraphRunner:
    """One captured CUDA graph per (input shapes, storage precision) over static copies of the inputs.  Before every replay the
    state key of the modules (ops.STORAGE and spade._param_key of each: ops.PARAM_GEN and (data_ptr, _version) of every parameter
    and buffer, the key of the derived-weight caches) is compared with the one the graph was captured under; a graph captured
    before a load_state_dict, an optimiser step, a parameter or running-statistics edit or a set_precision is released and
    captured again.  Subclasses define _body(static) -> outputs."""

    def __init__(self, modules):
        self._modules = modules
        self._graphs = {}  # (shapes, storage) -> _Entry

    class _Entry:
        def __init__(self, static, state):
            self.static, self.state = static, state
            self.captured = None
            self.keep = []

    def _state_key(self):
        return (ops.STORAGE[0],) + tuple(_param_key(m) for m in self._modules)

    def _check_ready(self, inputs, channels):
        if ops.PROFILE is not None:
            raise RuntimeError("%s: ops.PROFILE is on — profiling records CUDA events around every call, which cannot run inside a "
                               "CUDA-graph capture; set ops.PROFILE = None" % type(self).__name__)
        for m in self._modules:
            if any(s.training for s in m.modules()):
                raise RuntimeError("%s: %s is in train mode; the captured forward is the eval-mode one: call .eval()"
                                   % (type(self).__name__, type(m).__name__))
        for name, c in channels.items():
            t = inputs[name]
            if not (torch.is_tensor(t) and t.is_cuda and t.dtype == torch.float32 and t.dim() == 4 and t.shape[1] == c):
                raise ValueError("%s: input %r must be a CUDA float32 (N,%d,H,W) tensor, got %s" % (
                    type(self).__name__, name, c, "%s %s %s" % (t.device, t.dtype, tuple(t.shape)) if torch.is_tensor(t) else type(t)))

    def _run(self, inputs):
        key = tuple(tuple(t.shape) for t in inputs.values()) + (ops.STORAGE[0],)
        state = self._state_key()
        e = self._graphs.get(key)
        if e is not None and e.state != state:
            self._graphs.pop(key).captured.release()
            e = None
        if e is None:
            e = self._Entry({k: v.detach().clone() for k, v in inputs.items()}, state)
            # thread-local capture: a DataLoader's pin-memory thread in this process (data.VitonHDLoader feeding a training run that
            # evaluates through this runner) allocates pinned memory while the graph is captured, which global mode refuses
            e.captured = CapturedCall(lambda: self._body(e.static), warm=1, keep_rng=True, capture_error_mode="thread_local")
            # the graph reads the packed weights / folded BatchNorm tables of the modules' caches: keeping them alive means an
            # eager call that rebuilds a cache never frees memory a captured graph still reads
            e.keep = [getattr(s, a) for m in self._modules for s in m.modules() for a in ("_cache", "_pyr") if getattr(s, a, None) is not None]
            self._graphs[key] = e
        else:
            for k, v in inputs.items():
                e.static[k].copy_(v)
        return e.captured.replay()

    def _run_batch(self, inputs, datasetting):
        """_run on the self._channels entries of a cp_dataset batch dict ({setting: tensor} entries picked by `datasetting`)."""
        pick = lambda v: v[datasetting] if isinstance(v, dict) else v
        inputs = {k: pick(inputs[k]) for k in self._channels}
        self._check_ready(inputs, self._channels)
        if len({(t.shape[0],) + tuple(t.shape[2:]) for t in inputs.values()}) != 1:
            raise ValueError("%s: every input must have the same batch, height and width; got %s"
                             % (type(self).__name__, {k: tuple(t.shape) for k, t in inputs.items()}))
        return self._run(inputs)

    def release(self):
        """Destroy every captured graph (and the outputs they returned)."""
        for e in self._graphs.values():
            e.captured.release()
        self._graphs.clear()


class TryOnGraph(_GraphRunner):
    """tryon_forward(tocg, generator, inputs, occlusion=..., clothmask_composition=...) replayed from a CUDA graph: no Python-driven
    launches, C-ABI calls, TMA descriptor encodes or cache-key checks per network on the critical path — what matters when requests
    arrive one or a few images at a time.

    runner(inputs) takes the dict tryon_forward takes (cloth / cloth_mask as tensors or {setting: tensor} dicts, picked by
    `datasetting`); every input is a CUDA float32 NCHW tensor at the fine resolution.  The first call with a new (batch, H, W,
    storage precision) captures that shape (one eager warm-up call on a side stream, then the capture); every call copies the
    inputs into the graph's static buffers and replays.  Returns (output, warped_cloth, parse), equal to what tryon_forward
    returns for the same inputs, weights and noise.  The returned tensors belong to the runner: they stay valid until its next
    call, which overwrites them — clone() what must outlive it.

    Both modules must be in eval mode.  SPADE noise is drawn inside the graph from torch's CUDA generator (graph-safe Philox): every
    replay draws fresh noise and advances the generator exactly as one eager call does.  A generator's noise_source is called during
    the capture and what it returns there is what every replay reads; it must produce device tensors without host synchronisation.

    discriminator= (the stage-1 condition discriminator, eval mode) with norm_const= scores the 256x192 condition inside the same
    graph and returns (output, warped_cloth, parse, score), score as ConditionGraph's.  A graph cannot skip the generator for a
    rejected sample: every sample is generated and the caller filters on score."""

    def __init__(self, tocg, generator, occlusion=True, clothmask_composition="warp_grad", discriminator=None, norm_const=None):
        super().__init__([tocg, generator] + ([] if discriminator is None else [discriminator]))
        if discriminator is not None:
            _check_norm_const(norm_const)
        self.tocg, self.generator, self.discriminator, self.norm_const = tocg, generator, discriminator, norm_const
        self.occlusion, self.clothmask_composition = occlusion, clothmask_composition
        self._channels = {"cloth": 3, "cloth_mask": 1, "agnostic": 3, "densepose": 3, "parse_agnostic": tocg.io[1] - 3}

    def _body(self, static):
        return tryon_forward(self.tocg, self.generator, static, occlusion=self.occlusion, clothmask_composition=self.clothmask_composition,
                             discriminator=self.discriminator, norm_const=self.norm_const)

    def __call__(self, inputs, datasetting="paired"):
        return self._run_batch(inputs, datasetting)


class ConditionGraph(_GraphRunner):
    """rejection_scores(tocg, D, inputs, norm_const, clothmask_composition=...) replayed from a CUDA graph, with the contract of
    TryOnGraph: one graph per (input shapes, storage precision), both modules in eval mode, CUDA float32 inputs at the tocg
    resolution (cloth, cloth_mask, parse_agnostic, densepose; cloth / cloth_mask as tensors or {setting: tensor} dicts), recapture
    when the weights of either module or the precision changed.  Returns (score, l, (flow_list, fake_segmap, warped_cloth,
    warped_clothmask)), bit-identical to the eager call and owned by the runner until its next call."""

    def __init__(self, tocg, D, norm_const, clothmask_composition="warp_grad"):
        super().__init__([tocg, D])
        _check_norm_const(norm_const)
        self.tocg, self.D, self.norm_const, self.clothmask_composition = tocg, D, norm_const, clothmask_composition
        self._channels = {"cloth": 3, "cloth_mask": 1, "parse_agnostic": tocg.io[1] - 3, "densepose": 3}

    def _body(self, static):
        return rejection_scores(self.tocg, self.D, static, self.norm_const, clothmask_composition=self.clothmask_composition)

    def __call__(self, inputs, datasetting="paired"):
        return self._run_batch(inputs, datasetting)


class SegmentationGraph(_GraphRunner):
    """The stage-1 validation of train_condition.py:314-356 on one batch, replayed from a CUDA graph: the eval-mode tocg on the paired
    cloth (its mask thresholded at 0.5, test_condition.py:84) and metrics.segmentation_iou of its segmentation ('warp_grad'
    composition) against the batch's one-hot `parse`.  The contract of TryOnGraph: one graph per (input shapes, storage precision),
    the tocg in eval mode, CUDA float32 inputs at the tocg resolution (cloth, cloth_mask, parse_agnostic, densepose, parse; cloth /
    cloth_mask as tensors or {setting: tensor} dicts), recapture when its weights or BatchNorm running statistics changed.  Returns
    the batch IoU as a 0-dim fp32 cuda tensor, owned by the runner until its next call."""

    def __init__(self, tocg):
        super().__init__([tocg])
        self.tocg = tocg
        self._channels = {"cloth": 3, "cloth_mask": 1, "parse_agnostic": tocg.io[1] - 3, "densepose": 3, "parse": tocg.io[2]}

    def _body(self, static):
        from . import metrics
        with torch.no_grad():
            _, _, outs = _condition(self.tocg, static, None, "paired")
            return metrics.segmentation_iou(outs[1], outs[3], static["parse"])

    def __call__(self, inputs, datasetting="paired"):
        return self._run_batch(inputs, datasetting)


class GeneratorGraph(_GraphRunner):
    """generator(x, seg) under torch.no_grad() replayed from a CUDA graph, with the contract of TryOnGraph: one graph per (x shape,
    seg shape, storage precision), eval mode, CUDA float32 inputs, recapture when the weights or the precision changed, fresh SPADE
    noise per replay from torch's CUDA generator.  Returns the (N,3,H,W) image, owned by the runner and valid until its next call."""

    def __init__(self, generator):
        super().__init__([generator])
        self.generator = generator
        self._channels = {"x": generator.conv_0.in_channels, "seg": generator.head_0.norm_0.conv_shared[0].in_channels}

    def _body(self, static):
        with torch.no_grad():
            return self.generator(static["x"], static["seg"])

    def __call__(self, x, seg):
        inputs = {"x": x, "seg": seg}
        self._check_ready(inputs, self._channels)
        if x.shape[0] != seg.shape[0]:
            raise ValueError("GeneratorGraph: x and seg must have the same batch size; got %d and %d" % (x.shape[0], seg.shape[0]))
        return self._run(inputs)


def psnr(a, b, peak=2.0):
    """PSNR in dB for images in [-1, 1] (peak-to-peak 2)."""
    mse = float(((a.float() - b.float()) ** 2).mean())
    return float("inf") if mse == 0 else 10.0 * torch.log10(torch.tensor(peak * peak / mse)).item()
