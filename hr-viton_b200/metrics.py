"""The reference's evaluation metrics on the sm_90a kernels: LPIPS (eval_models, AlexNet with the v0.1 linear heads), skimage's
Gaussian SSIM as evaluate.py:67 calls it, and the Inception-v3 metrics: evaluate.py's Inception Score, FID and KID.

    from hrviton_b200 import metrics
    d = metrics.lpips(pred, target)        # (N,1,1,1) fp32, pred / target (N,3,H,W) fp32 cuda in [-1, 1]
    s = metrics.ssim(gt_gray, pred_gray)   # fp64 per image, (H,W) or (N,H,W) uint8 / fp32, cuda tensors or numpy arrays
    inc = torchvision.models.inception_v3(weights="IMAGENET1K_V1", transform_input=False)  # as evaluate.py:43 builds it
    net = metrics.InceptionV3.from_torchvision(inc.cuda().eval())
    pool, logits = net(images)             # (N,2048), (N,1000) fp32; images (N,3,H,W) fp32 cuda in [-1, 1] (unit_range=True: [0, 1])
    is_mean, is_std = metrics.inception_score(torch.softmax(logits, 1))
    a, b = metrics.FeatureStats(), metrics.FeatureStats()
    a.update(pool_a); b.update(pool_b)     # streamed over batches
    f = metrics.fid(a, b)
    kid_mean, kid_std = metrics.kid(pool_a, pool_b)

LPIPS and Inception always run in fp32 storage with 3xTF32 convolutions, whatever ops.get_precision() says: they are the numbers people
report, and they must not move with the training precision.  They are inference-only (no gradient).

FID and KID here are computed from torchvision's ImageNet Inception-v3.  Published FID / KID numbers use the TensorFlow-ported "FID
Inception" (pytorch-fid, clean-fid: other pool blocks, 1008 classes), so values from this module are comparable with each other, not
with those."""
import os
import warnings

import numpy as np
import torch
import torch.nn as nn

from . import ops
from .spade import _param_key

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ALEX_CHANNELS = [64, 192, 384, 256, 256]
ALEX_WEIGHTS = os.path.join("eval_models", "weights", "v0.1", "alex.pth")
# AlexNet features index of each convolution of the five slices (torchvision's alexnet().features, pretrained_networks.py:57-95)
_ALEX_SLICES = ((0, 2), (2, 5), (5, 8), (8, 10), (10, 12))
_CONVS = ((1, 0), (2, 3), (3, 6), (4, 8), (5, 10))  # (slice, features index)


def alex_weights_path():
    """Where the LPIPS v0.1 heads are looked for: ./eval_models/weights/v0.1/alex.pth under the working directory (where the reference
    keeps them next to its scripts), then the same path next to this repository's eval_models package.  None if neither exists."""
    for p in (os.path.join(os.getcwd(), ALEX_WEIGHTS), os.path.join(ROOT, ALEX_WEIGHTS)):
        if os.path.isfile(p):
            return p
    return None


def _alexnet_features(pretrained):
    """torchvision's AlexNet features with ImageNet weights, as tv.alexnet(pretrained=True) gives them; HRV_ALEX_RANDOM_INIT=1 builds them
    without weights (offline machines: hrv_env.install() sets it when the hub cache holds no AlexNet file), for weights loaded afterwards."""
    from torchvision import models
    if not pretrained or os.environ.get("HRV_ALEX_RANDOM_INIT") == "1":
        return models.alexnet(weights=None).features
    return models.alexnet(weights=models.AlexNet_Weights.IMAGENET1K_V1).features


class ScalingLayer(nn.Module):
    """networks_basic.py:94-101 (the buffers only: the kernel applies them)."""

    def __init__(self):
        super().__init__()
        self.register_buffer("shift", torch.Tensor([-.030, -.088, -.188])[None, :, None, None])
        self.register_buffer("scale", torch.Tensor([.458, .448, .450])[None, :, None, None])


class NetLinLayer(nn.Module):
    """networks_basic.py:104-111: Dropout (inert in eval mode) + 1x1 convolution without bias."""

    def __init__(self, chn_in, chn_out=1, use_dropout=True):
        super().__init__()
        layers = [nn.Dropout()] if use_dropout else []
        layers += [nn.Conv2d(chn_in, chn_out, 1, stride=1, padding=0, bias=False)]
        self.model = nn.Sequential(*layers)


class AlexFeatures(nn.Module):
    """pretrained_networks.alexnet: slice1..slice5 of torchvision's AlexNet features, frozen."""

    def __init__(self, pretrained=True):
        super().__init__()
        feats = _alexnet_features(pretrained)
        for k, (a, b) in enumerate(_ALEX_SLICES):
            seq = nn.Sequential()
            for i in range(a, b):
                seq.add_module(str(i), feats[i])
            setattr(self, "slice%d" % (k + 1), seq)
        for p in self.parameters():
            p.requires_grad = False


class PNetLin(nn.Module):
    """The LPIPS network of the reference, PNetLin(pnet_type='alex', version='0.1', lpips=True, spatial=False) (networks_basic.py:27-92),
    with its state_dict keys and shapes: scaling_layer.{shift,scale}, net.slice{1..5}.{i}.{weight,bias}, lin{0..4}.model.1.weight.
    forward(in0, in1) runs on the kernels: ScalingLayer + conv1 operand (hrv_lpips_input), the five convolutions with ReLU fused
    (hrv_conv2d_fwd, fp32 storage, 3xTF32), MaxPool2d(3, 2) (hrv_maxpool3s2) and one hrv_lpips_dist per layer."""

    def __init__(self, pretrained=True, use_dropout=True):
        super().__init__()
        self.chns = list(ALEX_CHANNELS)
        self.L = len(self.chns)
        self.scaling_layer = ScalingLayer()
        self.net = AlexFeatures(pretrained=pretrained)
        for k, c in enumerate(self.chns):
            setattr(self, "lin%d" % k, NetLinLayer(c, use_dropout=use_dropout))
        self.lins = [getattr(self, "lin%d" % k) for k in range(self.L)]
        self._packed = None

    def _pack(self):
        """fp32 3xTF32 operands of the five convolutions, rebuilt when a parameter or buffer changed (data_ptr, _version)."""
        tensors = list(self.parameters()) + list(self.buffers())
        key = tuple((t.data_ptr(), t._version, t.device) for t in tensors)
        if self._packed is not None and self._packed[0] == key:
            return self._packed[1]
        f32 = torch.float32
        packs = []
        for k, idx in _CONVS:
            conv = getattr(getattr(self.net, "slice%d" % k), str(idx))
            w = conv.weight.detach().float()
            cout, cin, kh, kw = w.shape
            if idx == 0:  # 11x11 stride 4: a 1x1 GEMM over the (ky, kx, ci) im2col operand of hrv_lpips_input
                pw = ops.pack_weight(w.permute(0, 2, 3, 1).reshape(cout, kh * kw * cin, 1, 1).contiguous(), (0, 0),
                                     flops_per_pixel=2.0 * cin * cout * kh * kw, storage=f32)
            else:
                pw = ops.pack_weight(w.contiguous(), (kh // 2, kw // 2), storage=f32)
            packs.append((pw, conv.bias.detach().float().contiguous()))
        lins = [lin.model[-1].weight.detach().float().reshape(-1).contiguous() for lin in self.lins]
        shift = self.scaling_layer.shift.detach().float().reshape(3).contiguous()
        scale = self.scaling_layer.scale.detach().float().reshape(3).contiguous()
        self._packed = (key, (packs, lins, shift, scale))
        return self._packed[1]

    def features(self, x):
        """The five ReLU outputs of AlexNet for the scaled fp32 NCHW batch x, as fp32 NHWC Acts."""
        packs, _, shift, scale = self._pack()
        h = ops.lpips_input(x, shift, scale)
        outs = []
        for k, (pw, bias) in enumerate(packs):
            if k in (1, 2):
                h = ops.maxpool3s2(h)
            out = ops.Act.empty(h.n, h.h, h.w, pw.n_gemm, dtype=torch.float32)
            h = ops.conv2d(h, pw, out, act=ops.ACT_RELU, shift=bias)
            outs.append(h)
        return outs

    def forward(self, in0, in1, retPerLayer=False):
        for t in (in0, in1):
            if not t.is_cuda:
                raise RuntimeError("LPIPS runs on the GPU only (no CPU fallback): got a %s tensor" % t.device)
        if in0.shape != in1.shape or in0.dim() != 4 or in0.shape[1] != 3:
            raise ValueError("LPIPS: in0 and in1 must both be (N,3,H,W); got %s and %s" % (tuple(in0.shape), tuple(in1.shape)))
        dev = self.scaling_layer.shift.device
        if dev.type != "cuda":
            raise RuntimeError("LPIPS: the network's weights are on the CPU; move it to the GPU with .cuda() (no CPU fallback)")
        if in0.device != dev or in1.device != dev:
            raise RuntimeError("LPIPS: the inputs (%s, %s) must be on the device of the network's weights (%s)" % (in0.device, in1.device, dev))
        n = in0.shape[0]
        with torch.cuda.device(dev):  # the kernels launch on the current device's stream
            x = torch.cat([in0.detach().float(), in1.detach().float()]).contiguous()
            _, lins, _, _ = self._pack()
            res = [ops.lpips_dist(f, lins[k]).view(n, 1, 1, 1) for k, f in enumerate(self.features(x))]
        val = res[0].clone()  # the reference sums into res[0] itself; here res keeps every layer's own distance
        for l in range(1, self.L):  # the reference's order: res[0], then += res[1..4]
            val += res[l]
        return (val, res) if retPerLayer else val


def load_lpips(path=None, pretrained=True, device="cuda"):
    """PNetLin with the v0.1 heads loaded from `path` (default: alex_weights_path()) with strict=False, as dist_model.py:62-73 does.
    A missing file raises FileNotFoundError: there is no fallback to untrained heads."""
    path = alex_weights_path() if path is None else path
    if path is None or not os.path.isfile(path):
        raise FileNotFoundError("LPIPS v0.1 weights not found: looked for %s under the working directory and next to the package (%s)"
                                % (ALEX_WEIGHTS, os.path.join(ROOT, ALEX_WEIGHTS)) if path is None else "No such file: %r" % path)
    net = PNetLin(pretrained=pretrained)
    print("Loading model from: %s" % path)
    sd = torch.load(path, map_location="cpu")
    net.load_state_dict(sd, strict=False)
    if (not pretrained or os.environ.get("HRV_ALEX_RANDOM_INIT") == "1") and not any(k.startswith("net.") for k in sd):
        warnings.warn("LPIPS: the AlexNet backbone is randomly initialised (no ImageNet weights: HRV_ALEX_RANDOM_INIT=1) and %s holds no "
                      "net.* tensors, so the distances it gives are not LPIPS; cache torchvision's alexnet-owt-7be5be79.pth or load a "
                      "file that carries the backbone" % path)
    return net.to(device).eval()


_default = [None]


def lpips(pred, target, normalize=False, net=None):
    """LPIPS distance (N,1,1,1) fp32 of two (N,3,H,W) cuda batches in [-1, 1] (normalize=True: in [0, 1]), as
    eval_models.PerceptualLoss().forward(pred, target) computes it.  net: a PNetLin (default: one loaded once by load_lpips())."""
    if torch.is_grad_enabled() and (pred.requires_grad or target.requires_grad):
        raise NotImplementedError("LPIPS has no backward pass here: call it under torch.no_grad() or on detached tensors")
    if net is None:
        if _default[0] is None:
            _default[0] = load_lpips()
        net = _default[0]
    if normalize:
        pred, target = 2 * pred - 1, 2 * target - 1
    with torch.no_grad():
        return net(target, pred)


def ssim(im1, im2, data_range=255):
    """Mean SSIM of two grayscale images or stacks, as skimage.metrics.structural_similarity(im1, im2, data_range=data_range,
    gaussian_weights=True, use_sample_covariance=False) computes it (evaluate.py:67), in fp64 on the GPU (hrv_ssim).
    im1, im2: (H,W) or (N,H,W), uint8 or float32 (pixel values), cuda tensors or numpy arrays.  Returns fp64 per image: a cuda tensor
    ((N,) or 0-d) for tensors, a numpy array ((N,) or 0-d) for arrays."""
    as_numpy = isinstance(im1, np.ndarray)
    if as_numpy:
        if not isinstance(im2, np.ndarray):
            raise TypeError("ssim: im1 and im2 must both be numpy arrays or both cuda tensors")
        im1 = torch.from_numpy(np.array(im1)).cuda()  # a copy: PIL's arrays are read-only
        im2 = torch.from_numpy(np.array(im2)).cuda()
    for t in (im1, im2):
        if not t.is_cuda:
            raise RuntimeError("ssim runs on the GPU only (no CPU fallback): got a %s tensor" % t.device)
    single = im1.dim() == 2
    if single:
        im1, im2 = im1[None], im2[None]
    out = ops.ssim(im1, im2, data_range)
    if single:
        out = out[0]
    return out.cpu().numpy() if as_numpy else out


# ----------------------------------------------------------------------------------------------- Inception-v3

INCEPTION_SIZE = 299
_F32 = torch.float32
# torchvision Inception3._transform_input: x'_c = x_c * a_c + b_c (ImageNet normalisation -> the network's [-1, 1] input)
_TRANSFORM = ((0.229 / 0.5, 0.224 / 0.5, 0.225 / 0.5), ((0.485 - 0.5) / 0.5, (0.456 - 0.5) / 0.5, (0.406 - 0.5) / 0.5))
_STEM = ["Conv2d_1a_3x3", "Conv2d_2a_3x3", "Conv2d_2b_3x3", "maxpool", "Conv2d_3b_1x1", "Conv2d_4a_3x3", "maxpool"]
_MIXED = ["Mixed_5b", "Mixed_5c", "Mixed_5d", "Mixed_6a", "Mixed_6b", "Mixed_6c", "Mixed_6d", "Mixed_6e", "Mixed_7a", "Mixed_7b", "Mixed_7c"]
# The branches of each block type in torch.cat order.  A branch is a chain of stages from the block input; a tuple stage runs its
# convolutions side by side on the previous stage's output, concatenated (InceptionE).  "maxpool" is F.max_pool2d(3, stride=2).
_BLOCKS = {
    "InceptionA": [["branch1x1"], ["branch5x5_1", "branch5x5_2"], ["branch3x3dbl_1", "branch3x3dbl_2", "branch3x3dbl_3"], ["branch_pool"]],
    "InceptionB": [["branch3x3"], ["branch3x3dbl_1", "branch3x3dbl_2", "branch3x3dbl_3"], ["maxpool"]],
    "InceptionC": [["branch1x1"], ["branch7x7_1", "branch7x7_2", "branch7x7_3"],
                   ["branch7x7dbl_1", "branch7x7dbl_2", "branch7x7dbl_3", "branch7x7dbl_4", "branch7x7dbl_5"], ["branch_pool"]],
    "InceptionD": [["branch3x3_1", "branch3x3_2"], ["branch7x7x3_1", "branch7x7x3_2", "branch7x7x3_3", "branch7x7x3_4"], ["maxpool"]],
    "InceptionE": [["branch1x1"], ["branch3x3_1", ("branch3x3_2a", "branch3x3_2b")],
                   ["branch3x3dbl_1", "branch3x3dbl_2", ("branch3x3dbl_3a", "branch3x3dbl_3b")], ["branch_pool"]],
}
_POOLED = ("InceptionA", "InceptionC", "InceptionE")  # their branch_pool is F.avg_pool2d(3, 1, 1) and a 1x1 BasicConv2d


def fold_basic_conv(bc, pool=False, affine=None):
    """A torchvision BasicConv2d (bias-free conv, eval-mode BatchNorm, ReLU) as (weight, scale, shift) in fp64, on its device:
    relu(conv(x, weight) * scale + shift) is the module's output in real arithmetic.
    pool=True: bc follows F.avg_pool2d(3, stride=1, padding=1) (count_include_pad): the pair is one 3x3 convolution, padding 1, with
    every tap w/9.  affine=(a, b): the input is a_c x_c + b_c per channel first (transform_input); the convolution must have no padding,
    so every tap sees the affine value and b folds into the shift exactly."""
    w = bc.conv.weight.detach().double()
    bn = bc.bn
    s = bn.weight.detach().double() / torch.sqrt(bn.running_var.detach().double() + bn.eps)
    t = bn.bias.detach().double() - bn.running_mean.detach().double() * s
    if affine is not None:
        assert tuple(bc.conv.padding) == (0, 0), "the input affine folds only into an unpadded convolution"
        a = torch.tensor(affine[0], dtype=torch.float64, device=w.device).view(1, -1, 1, 1)
        b = torch.tensor(affine[1], dtype=torch.float64, device=w.device).view(1, -1, 1, 1)
        t = t + s * (w * b).sum((1, 2, 3))
        w = w * a
    if pool:
        assert w.shape[2:] == (1, 1) and tuple(bc.conv.stride) == (1, 1)
        w = w.expand(-1, -1, 3, 3) / 9.0
    return w.contiguous(), s, t


class _Conv:
    """One packed BasicConv2d: 3xTF32 operand, the BatchNorm scale / shift of the epilogue, its geometry."""

    def __init__(self, bc, pool=False, affine=None):
        w, s, t = fold_basic_conv(bc, pool, affine)
        cout, cin, kh, kw = w.shape
        self.cout = cout
        self.s2d = tuple(bc.conv.stride) != (1, 1)
        if self.s2d:  # every stride-2 convolution of Inception-v3 is 3x3 without padding: a 2x2 one on the space-to-depth input
            if tuple(bc.conv.stride) != (2, 2) or (kh, kw) != (3, 3) or tuple(bc.conv.padding) != (0, 0):
                raise NotImplementedError("stride-%s %dx%d convolution with padding %s" % (bc.conv.stride, kh, kw, bc.conv.padding))
            self.pad = (0, 0)
            self.pw = ops.pack_weight(ops.s2d_weight(w.float(), 0), (0, 0), flops_per_pixel=2.0 * cin * cout * 9, storage=_F32)
        else:
            self.pad = (1, 1) if pool else tuple(bc.conv.padding)
            self.pw = ops.pack_weight(w.float(), self.pad, storage=_F32)
        self.kh, self.kw = kh, kw
        self.scale, self.shift = s.float().contiguous(), t.float().contiguous()

    def extent(self, h, w):
        if self.s2d:
            return (h - 3) // 2 + 1, (w - 3) // 2 + 1
        return h + 2 * self.pad[0] - self.kh + 1, w + 2 * self.pad[1] - self.kw + 1

    def __call__(self, x, out=None):
        src = ops.space_to_depth(x, dtype=_F32) if self.s2d else x
        if out is None:
            h, w = self.extent(x.h, x.w)
            out = ops.Act.empty(x.n, h, w, self.cout, dtype=_F32, device=x.buf.device)
        return ops.conv2d(src, self.pw, out, act=ops.ACT_RELU, scale=self.scale, shift=self.shift)


def _check_images(x, what):
    if not torch.is_tensor(x):
        raise TypeError("%s: expected a torch tensor, got %s" % (what, type(x).__name__))
    if not x.is_cuda:
        raise RuntimeError("%s runs on the GPU only (no CPU fallback): got a %s tensor" % (what, x.device))
    if torch.is_grad_enabled() and x.requires_grad:
        raise NotImplementedError("%s has no backward pass: call it under torch.no_grad() or on detached tensors" % what)


class InceptionV3:
    """torchvision's Inception3 (eval mode, transform_input honoured) up to its 2048-wide pool features and 1000-way logits, on the
    kernels: every BasicConv2d is one hrv_conv2d_fwd in fp32 storage (3xTF32) with its BatchNorm (eps 0.001) and ReLU in the epilogue,
    the stride-2 ones over hrv_space_to_depth, the average-pool branches as 3x3 convolutions with weights w/9, the max pools on
    hrv_maxpool3s2, the branches of a block written into channel slices of one buffer (the torch.cat), then hrv_global_avgpool and fc as
    a 1x1 convolution.  The aux head is never run.  Build it with from_torchvision(model); weights are re-packed whenever a parameter or
    buffer of the model changes (spade._param_key), and always kept in fp32 whatever ops.get_precision() says."""

    def __init__(self, model):
        self.model = model
        self._key = None
        self._packs = None

    @classmethod
    def from_torchvision(cls, model):
        from torchvision.models.inception import Inception3
        if not isinstance(model, Inception3):
            raise TypeError("InceptionV3.from_torchvision expects a torchvision Inception3, got %s" % type(model).__name__)
        if model.training:
            raise ValueError("InceptionV3.from_torchvision: the model must be in eval mode (BatchNorm running statistics); call .eval()")
        dev = model.fc.weight.device
        if dev.type != "cuda":
            raise RuntimeError("InceptionV3: the model's weights are on the CPU; move it to the GPU with .cuda() (no CPU fallback)")
        return cls(model)

    @property
    def device(self):
        return self.model.fc.weight.device

    def _pack(self):
        m = self.model
        key = (_param_key(m), bool(m.transform_input))
        if self._key == key:
            return self._packs
        with torch.no_grad():
            packs = {}
            for name in _STEM:
                if name != "maxpool":
                    packs[name] = _Conv(getattr(m, name), affine=_TRANSFORM if (m.transform_input and name == "Conv2d_1a_3x3") else None)
            # [0, 1] images (unit_range) reach the network as 2x - 1, which is what ImageNet normalisation followed by transform_input
            # gives: without the fold
            packs["Conv2d_1a_3x3 unit"] = _Conv(m.Conv2d_1a_3x3) if m.transform_input else packs["Conv2d_1a_3x3"]
            for blk in _MIXED:
                mod = getattr(m, blk)
                kind = type(mod).__name__
                if kind not in _BLOCKS:
                    raise NotImplementedError("%s is a %s, not a torchvision Inception block" % (blk, kind))
                for branch in _BLOCKS[kind]:
                    for stage in branch:
                        for name in (stage if isinstance(stage, tuple) else (stage,)):
                            if name != "maxpool":
                                packs[blk + "." + name] = _Conv(getattr(mod, name), pool=(name == "branch_pool" and kind in _POOLED))
            fc_w = m.fc.weight.detach().float()
            packs["fc"] = (ops.pack_weight(fc_w.reshape(fc_w.shape[0], fc_w.shape[1], 1, 1).contiguous(), (0, 0), storage=_F32),
                           m.fc.bias.detach().float().contiguous())
        self._packs, self._key = packs, key
        return packs

    def _block(self, packs, blk, x):
        kind = type(getattr(self.model, blk)).__name__
        plans = []  # per branch: (last stage names, extent, widths)
        for branch in _BLOCKS[kind]:
            h, w = x.h, x.w
            for stage in branch:
                name = stage[0] if isinstance(stage, tuple) else stage
                h, w = ((h - 3) // 2 + 1, (w - 3) // 2 + 1) if name == "maxpool" else packs[blk + "." + name].extent(h, w)
            last = branch[-1] if isinstance(branch[-1], tuple) else (branch[-1],)
            plans.append((last, (h, w), [x.c if n == "maxpool" else packs[blk + "." + n].cout for n in last]))
        (h, w) = plans[0][1]
        out = ops.Act.empty(x.n, h, w, sum(sum(p[2]) for p in plans), dtype=_F32, device=x.buf.device)
        c0 = 0
        for branch, (last, _, widths) in zip(_BLOCKS[kind], plans):
            y = x
            for stage in branch[:-1]:
                y = packs[blk + "." + stage](y)
            for name, width in zip(last, widths):
                dst = out.slice(c0, width)
                if name == "maxpool":
                    ops.maxpool3s2(y, out=dst)
                else:
                    packs[blk + "." + name](y, out=dst)
                c0 += width
        return out

    def _input(self, x, unit_range):
        n, _, h, w = x.shape
        if (h, w) != (INCEPTION_SIZE, INCEPTION_SIZE) or unit_range:
            return ops.resize_bilinear_nhwc(x, (INCEPTION_SIZE, INCEPTION_SIZE), unit_range=unit_range)
        return ops.from_nchw(x, out=ops.Act.empty(n, h, w, 3, dtype=_F32, device=x.device))

    def run(self, x, unit_range=False, keep=()):
        """(pool [N,2048], logits [N,1000], {name: Act} of the blocks named in `keep`) for fp32 NCHW x (checked by forward)."""
        packs = self._pack()
        a = self._input(x.detach().contiguous(), unit_range)
        kept = {}
        for name in _STEM:
            if name == "maxpool":
                a = ops.maxpool3s2(a)
            else:
                a = packs[name + " unit" if (unit_range and name == "Conv2d_1a_3x3") else name](a)
        for blk in _MIXED:
            a = self._block(packs, blk, a)
            if blk in keep:
                kept[blk] = a
        pool = ops.global_avgpool(a)
        pw, bias = packs["fc"]
        logits = ops.conv2d(pool, pw, ops.Act.empty(x.shape[0], 1, 1, pw.n_gemm, dtype=_F32, device=x.device), shift=bias)
        return pool.buf.view(x.shape[0], -1), logits.buf.view(x.shape[0], -1), kept

    def __call__(self, x, unit_range=False):
        return self.forward(x, unit_range)

    def forward(self, x, unit_range=False):
        """(pool_features [N,2048], logits [N,1000]), fp32 on the device, of images x: fp32 (N,3,H,W) cuda, in the range the model
        expects: [-1, 1] without transform_input (evaluate.py's T3 output), ImageNet-normalised with it.  unit_range=True takes images
        in [0, 1] whatever transform_input says: the network then sees 2x - 1, which for a transform_input model is what ImageNet
        normalisation followed by its transform gives (the transform is not applied a second time).
        Other sizes than 299x299 are resized bilinearly (F.interpolate, align_corners=False) on the way in, bit for bit as torch does."""
        _check_images(x, "InceptionV3")
        if x.dim() != 4 or x.shape[1] != 3 or x.shape[0] < 1 or x.dtype != torch.float32:
            raise ValueError("InceptionV3: expected float32 images (N,3,H,W), got %s %s" % (x.dtype, tuple(x.shape)))
        if x.device != self.device:
            raise RuntimeError("InceptionV3: the images (%s) must be on the device of the model's weights (%s)" % (x.device, self.device))
        with torch.no_grad(), torch.cuda.device(x.device):
            pool, logits, _ = self.run(x, unit_range)
        return pool, logits


def inception_score(probs_or_images, splits=1, model=None, batch_size=50):
    """evaluate.py:96-106's Inception Score in fp64 on the device: for each of `splits` equal parts of the N rows (N // splits each),
    exp(mean_i KL(p_i || mean_i p_i)) with scipy.stats.entropy's normalisation of both distributions; returns (mean, std) over the
    parts as 0-d fp64 cuda tensors (std: np.std, ddof 0).  probs_or_images: class probabilities (N,C) cuda (evaluate.py's softmax of the
    logits), or images (N,3,H,W) run through `model` (an InceptionV3) in batches of batch_size, then softmax in fp32 as evaluate.py."""
    x = probs_or_images
    _check_images(x, "inception_score")
    if x.dim() == 4:
        if model is None:
            raise ValueError("inception_score: images need model=InceptionV3.from_torchvision(...)")
        x = torch.cat([torch.softmax(model(x[i:i + batch_size])[1], 1) for i in range(0, x.shape[0], batch_size)])
    elif x.dim() != 2:
        raise ValueError("inception_score: expected probabilities (N,C) or images (N,3,H,W), got %s" % (tuple(x.shape),))
    part_n = x.shape[0] // splits if splits >= 1 else 0
    if part_n < 1:
        raise ValueError("inception_score: %d rows cannot make %d splits" % (x.shape[0], splits))
    p = x.detach().double()
    scores = []
    for k in range(splits):
        part = p[k * part_n:(k + 1) * part_n]
        pk = part / part.sum(1, keepdim=True)
        py = part.mean(0)
        qk = py / py.sum()
        kl = torch.where(pk > 0, pk * torch.log(pk / qk), torch.zeros_like(pk)).sum(1)  # scipy.special.rel_entr, summed
        scores.append(torch.exp(kl.mean()))
    s = torch.stack(scores)
    return s.mean(), s.std(unbiased=False)


def _check_features(f, what):
    _check_images(f, what)
    if f.dim() != 2 or f.shape[0] < 1 or f.dtype not in (torch.float32, torch.float64):
        raise ValueError("%s: expected fp32 / fp64 features (N,D), got %s %s" % (what, f.dtype, tuple(f.shape)))


class FeatureStats:
    """Running fp64 sums of the features of one image set, streamed over batches: sum_x and sum_x x^T (hrv_gram_f64, every sum in a
    fixed order, so the statistics do not depend on timing).  mean() and cov() give mu and the covariance with np.cov's unbiased N - 1
    normalisation."""

    def __init__(self, dim=2048, device="cuda"):
        device = torch.device(device)
        if device.type != "cuda":
            raise RuntimeError("FeatureStats runs on the GPU only (no CPU fallback): got %s" % device)
        self.dim, self.n = dim, 0
        self.sum = torch.zeros(dim, dtype=torch.float64, device=device)
        self.sum_sq = torch.zeros((dim, dim), dtype=torch.float64, device=device)

    def update(self, feats):
        """Add the rows of feats (N, dim) fp32 / fp64 cuda, on this object's device."""
        _check_features(feats, "FeatureStats.update")
        if feats.shape[1] != self.dim or feats.device != self.sum.device:
            raise ValueError("FeatureStats.update: expected (N, %d) features on %s, got %s on %s" % (self.dim, self.sum.device, tuple(feats.shape), feats.device))
        f = feats.detach()
        with torch.cuda.device(f.device):
            ops.gram_f64(f, f, out=self.sum_sq, k_major=True, accumulate=True)
            ones = torch.ones((f.shape[0], 1), dtype=f.dtype, device=f.device)
            ops.gram_f64(f, ones, out=self.sum.view(self.dim, 1), k_major=True, accumulate=True)
        self.n += f.shape[0]
        return self

    def mean(self):
        if self.n < 1:
            raise ValueError("FeatureStats: no features")
        return self.sum / self.n

    def cov(self):
        if self.n < 2:
            raise ValueError("FeatureStats: the covariance needs at least 2 features, have %d" % self.n)
        mu = self.mean()
        return (self.sum_sq - self.n * torch.outer(mu, mu)) / (self.n - 1)


def fid_from_moments(mu_a, sig_a, mu_b, sig_b, mm):
    """||mu_a - mu_b||^2 + Tr sig_a + Tr sig_b - 2 Tr sqrt(sig_a sig_b) in fp64.  The trace term is the sum of the square roots of the
    eigenvalues of the symmetric sqrt(sig_a) sig_b sqrt(sig_a), which has the eigenvalues of sig_a sig_b; sqrt(sig_a) comes from the
    eigendecomposition of sig_a.  Negative eigenvalues (rounding of a singular covariance) count as 0.  mm(a, b) = a @ b.T in fp64."""
    d = mu_a - mu_b
    ea, va = torch.linalg.eigh(sig_a)
    root_a = mm(va * ea.clamp_min(0).sqrt(), va)
    m = mm(mm(root_a, sig_b), root_a)
    em = torch.linalg.eigvalsh((m + m.mT) * 0.5).clamp_min(0)
    return (d * d).sum() + torch.diagonal(sig_a).sum() + torch.diagonal(sig_b).sum() - 2.0 * em.sqrt().sum()


def fid(stats_a, stats_b):
    """Frechet Inception Distance of two FeatureStats, a 0-d fp64 cuda tensor (fid_from_moments, products on hrv_gram_f64, the
    eigendecompositions through torch.linalg.eigh in fp64)."""
    for st in (stats_a, stats_b):
        if not isinstance(st, FeatureStats):
            raise TypeError("fid: expected FeatureStats, got %s" % type(st).__name__)
    if stats_a.sum.device != stats_b.sum.device or stats_a.dim != stats_b.dim:
        raise ValueError("fid: the two statistics must have one dimension and one device")
    with torch.cuda.device(stats_a.sum.device):
        return fid_from_moments(stats_a.mean(), stats_a.cov(), stats_b.mean(), stats_b.cov(), ops.gram_f64)


def kid_subsets(n_a, n_b, subsets, subset_size, seed=0):
    """The feature indices of KID's subsets: int32 (subsets, subset_size) for each set, each row drawn without replacement by
    np.random.RandomState(seed).choice, alternating between the two sets."""
    rng = np.random.RandomState(seed)
    ix = np.empty((subsets, subset_size), dtype=np.int32)
    iy = np.empty((subsets, subset_size), dtype=np.int32)
    for s in range(subsets):
        ix[s] = rng.choice(n_a, subset_size, replace=False)
        iy[s] = rng.choice(n_b, subset_size, replace=False)
    return ix, iy


def mmd2_from_sums(sums, m):
    """Unbiased MMD^2 per subset from the [S,3] sums (off-diagonal X-X, off-diagonal Y-Y, all X-Y) of subsets of size m."""
    return (sums[:, 0] + sums[:, 1]) / (m * (m - 1)) - 2.0 * sums[:, 2] / (m * m)


def kid(feats_a, feats_b, subsets=100, subset_size=1000, seed=0):
    """Kernel Inception Distance: the unbiased MMD^2 with the cubic polynomial kernel k(x, y) = (x.y / d + 1)^3 over `subsets` pairs of
    subsets of `subset_size` features each (kid_subsets(seed)); returns (mean, std) over the subsets as 0-d fp64 cuda tensors (std:
    ddof 0).  feats_a (Na, d), feats_b (Nb, d): fp32 / fp64 cuda.  The full Gram matrices X X^T, Y Y^T, X Y^T are computed once
    (hrv_gram_f64) and every subset sum is drawn from them (hrv_kid_sums).  They take 8 (Na^2 + Nb^2 + Na Nb) bytes of device memory:
    96 MB at 2048 + 2048 features, but 60 GB at 50k + 50k; for sets that large pass a random subset of each."""
    _check_features(feats_a, "kid")
    _check_features(feats_b, "kid")
    if feats_a.shape[1] != feats_b.shape[1] or feats_a.dtype != feats_b.dtype or feats_a.device != feats_b.device:
        raise ValueError("kid: the two feature sets must share dimension, dtype and device; got %s %s %s and %s %s %s"
                         % (tuple(feats_a.shape), feats_a.dtype, feats_a.device, tuple(feats_b.shape), feats_b.dtype, feats_b.device))
    na, nb, d = feats_a.shape[0], feats_b.shape[0], feats_a.shape[1]
    if subsets < 1 or subset_size < 2 or subset_size > min(na, nb):
        raise ValueError("kid: subset_size must be in [2, min(Na, Nb)] = [2, %d] and subsets >= 1; got %d, %d" % (min(na, nb), subset_size, subsets))
    ix, iy = kid_subsets(na, nb, subsets, subset_size, seed)
    fa, fb = feats_a.detach(), feats_b.detach()
    with torch.cuda.device(fa.device):
        ix_d = torch.from_numpy(ix).to(fa.device)
        iy_d = torch.from_numpy(iy).to(fa.device)
        sums = ops.kid_sums(ops.gram_f64(fa, fa), ops.gram_f64(fb, fb), ops.gram_f64(fa, fb), ix_d, iy_d, 1.0 / d)
        mmd = mmd2_from_sums(sums, subset_size)
        return mmd.mean(), mmd.std(unbiased=False)
