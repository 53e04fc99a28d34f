"""Drop-in for the reference's networks.py (same public names, constructor / forward signatures and state_dict
keys — networks.py:13-453) backed by the sm_90a kernels of hrviton_b200.  Put this repository first on
sys.path (or run the reference scripts from here) and `from networks import ConditionGenerator, ...` binds to it.
"""
import os

import torch
import torch.nn as nn
from torch.autograd import Variable

import hrv_loader

hrv_loader.load()
from hrviton_b200.tocg import (ConditionGenerator, MultiscaleDiscriminator, NLayerDiscriminator, ResBlock,  # noqa: E402,F401
                               define_D, get_norm_layer, load_checkpoint, make_grid, save_checkpoint, weights_init)


class Vgg19(nn.Module):
    """networks.py:201-231 — the perceptual-loss feature net.  SURVEY.md §8(f) N1: a "next" row; it stays on
    torch/cuDNN for now.  Offline boxes: HRV_VGG_RANDOM_INIT=1 builds it without downloading weights."""

    def __init__(self, requires_grad=False):
        super().__init__()
        from torchvision import models
        if os.environ.get("HRV_VGG_RANDOM_INIT") == "1":
            feats = models.vgg19(weights=None).features
        else:
            feats = models.vgg19(weights=models.VGG19_Weights.IMAGENET1K_V1).features
        cuts = [0, 2, 7, 12, 21, 30]
        for k in range(5):
            seq = nn.Sequential()
            for i in range(cuts[k], cuts[k + 1]):
                seq.add_module(str(i), feats[i])
            setattr(self, "slice%d" % (k + 1), seq)
        if not requires_grad:
            for p in self.parameters():
                p.requires_grad = False

    def forward(self, X):
        out = []
        h = X
        for k in range(5):
            h = getattr(self, "slice%d" % (k + 1))(h)
            out.append(h)
        return out


class VGGLoss(nn.Module):
    """networks.py:234-251."""

    def __init__(self, opt, layids=None):
        super().__init__()
        self.vgg = Vgg19()
        if opt.cuda:
            self.vgg.cuda()
        self.criterion = nn.L1Loss()
        self.weights = [1.0 / 32, 1.0 / 16, 1.0 / 8, 1.0 / 4, 1.0]
        self.layids = layids

    def forward(self, x, y):
        if x.is_cuda and self.layids is None:  # sm_90a conv kernels (forward + dgrad); frozen weights need no wgrad
            from hrviton_b200 import autograd_g
            return autograd_g.vgg_loss(self.vgg, self.weights, x, y)
        fx, fy = self.vgg(x), self.vgg(y)
        if self.layids is None:
            self.layids = list(range(len(fx)))
        loss = 0
        for i in self.layids:
            loss += self.weights[i] * self.criterion(fx[i], fy[i].detach())
        return loss


class GANLoss(nn.Module):
    """networks.py:258-299 (LSGAN on the last output of every scale; tiny reductions, plain torch)."""

    def __init__(self, use_lsgan=True, target_real_label=1.0, target_fake_label=0.0, tensor=torch.FloatTensor):
        super().__init__()
        self.real_label, self.fake_label = target_real_label, target_fake_label
        self.real_label_var = None
        self.fake_label_var = None
        self.Tensor = tensor
        self.loss = nn.MSELoss() if use_lsgan else nn.BCELoss()

    def get_target_tensor(self, input, target_is_real):
        attr = "real_label_var" if target_is_real else "fake_label_var"
        cur = getattr(self, attr)
        if cur is None or cur.numel() != input.numel():
            val = self.real_label if target_is_real else self.fake_label
            cur = Variable(self.Tensor(input.size()).fill_(val), requires_grad=False)
            setattr(self, attr, cur)
        return cur

    def __call__(self, input, target_is_real):
        if isinstance(input[0], list):
            loss = 0
            for scale in input:
                pred = scale[-1]
                loss += self.loss(pred, self.get_target_tensor(pred, target_is_real))
            return loss
        return self.loss(input[-1], self.get_target_tensor(input[-1], target_is_real))
