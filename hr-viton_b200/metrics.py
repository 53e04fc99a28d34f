"""The reference's evaluation metrics on the sm_90a kernels: LPIPS (eval_models, AlexNet with the v0.1 linear heads) and skimage's
Gaussian SSIM as evaluate.py:67 calls it.

    from hrviton_b200 import metrics
    d = metrics.lpips(pred, target)        # (N,1,1,1) fp32, pred / target (N,3,H,W) fp32 cuda in [-1, 1]
    s = metrics.ssim(gt_gray, pred_gray)   # fp64 per image, (H,W) or (N,H,W) uint8 / fp32, cuda tensors or numpy arrays

LPIPS always runs in fp32 storage with 3xTF32 convolutions, whatever ops.get_precision() says: it is the number people report, and it
must not move with the training precision.  It is inference-only (no gradient)."""
import os
import warnings

import numpy as np
import torch
import torch.nn as nn

from . import ops

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
