"""A float64 CPU restatement of pytorch-fid's FID Inception (fid_inception_v3) with seeded weights, for tests/test_fid_inception_*.py
and tools/fid_bench.py.

The network is torchvision's Inception3(num_classes=1008, aux_logits=False) whose InceptionA / C / E blocks pool their branch_pool
input as pytorch-fid does: F.avg_pool2d(x, 3, 1, 1, count_include_pad=False) in Mixed_5b-5d, Mixed_6b-6e and Mixed_7b, and
F.max_pool2d(x, 3, 1, 1) in Mixed_7c.  Its input is pytorch-fid's: images in [0, 1], F.interpolate to 299x299 (bilinear,
align_corners=False), then 2x - 1.  The real weights (pt_inception-2015-12-05-6726825d.pth) cannot be fetched offline, so the weights
are seeded as tests/inception_oracle.seeded_inception seeds them: BatchNorm statistics calibrated on seeded images and then perturbed,
so the activations stay O(1) through every block."""
import torch
import torch.nn as nn
import torch.nn.functional as F
from torchvision.models.inception import Inception3, InceptionA, InceptionC, InceptionE

import inception_oracle

TAPS = inception_oracle.TAPS
FID_MAX_POOL = "Mixed_7c"


def _fid_pool(x, use_max):
    return F.max_pool2d(x, 3, stride=1, padding=1) if use_max else F.avg_pool2d(x, 3, stride=1, padding=1, count_include_pad=False)


class FIDInceptionA(InceptionA):
    def forward(self, x):
        b1 = self.branch1x1(x)
        b5 = self.branch5x5_2(self.branch5x5_1(x))
        b3 = self.branch3x3dbl_3(self.branch3x3dbl_2(self.branch3x3dbl_1(x)))
        bp = self.branch_pool(_fid_pool(x, False))
        return torch.cat([b1, b5, b3, bp], 1)


class FIDInceptionC(InceptionC):
    def forward(self, x):
        b1 = self.branch1x1(x)
        b7 = self.branch7x7_3(self.branch7x7_2(self.branch7x7_1(x)))
        bd = x
        for name in ("branch7x7dbl_1", "branch7x7dbl_2", "branch7x7dbl_3", "branch7x7dbl_4", "branch7x7dbl_5"):
            bd = getattr(self, name)(bd)
        bp = self.branch_pool(_fid_pool(x, False))
        return torch.cat([b1, b7, bd, bp], 1)


class FIDInceptionE(InceptionE):
    use_max = False

    def forward(self, x):
        b1 = self.branch1x1(x)
        b3 = self.branch3x3_1(x)
        b3 = torch.cat([self.branch3x3_2a(b3), self.branch3x3_2b(b3)], 1)
        bd = self.branch3x3dbl_2(self.branch3x3dbl_1(x))
        bd = torch.cat([self.branch3x3dbl_3a(bd), self.branch3x3dbl_3b(bd)], 1)
        bp = self.branch_pool(_fid_pool(x, self.use_max))
        return torch.cat([b1, b3, bd, bp], 1)


class FIDInceptionEMax(FIDInceptionE):
    use_max = True


def _swap_blocks(m):
    """Give the blocks of a torchvision Inception3 pytorch-fid's pooling, in place (same modules, same state dict keys)."""
    for name, blk in m.named_children():
        if isinstance(blk, InceptionA):
            blk.__class__ = FIDInceptionA
        elif isinstance(blk, InceptionC):
            blk.__class__ = FIDInceptionC
        elif isinstance(blk, InceptionE):
            blk.__class__ = FIDInceptionEMax if name == FID_MAX_POOL else FIDInceptionE
    return m


def fid_network(state_dict=None, pooling="fid"):
    """An eval-mode fp32 CPU Inception3(num_classes=1008, aux_logits=False) with pooling 'fid' (pytorch-fid's) or 'torchvision'
    (count_include_pad=True averages everywhere), loaded from state_dict if given (strict, num_batches_tracked may be absent)."""
    m = Inception3(num_classes=1008, aux_logits=False, init_weights=False)
    if pooling == "fid":
        _swap_blocks(m)
    if state_dict is not None:
        missing, unexpected = m.load_state_dict(state_dict, strict=False)
        assert not unexpected and all(k.endswith("num_batches_tracked") for k in missing), (missing, unexpected)
    return m.eval()


def fid_input(x):
    """pytorch-fid's input in float64 from images in [0, 1]: fp32 (N,3,H,W) or uint8 (N,H,W,3) (as TF.to_tensor, /255)."""
    x = x.detach().cpu()
    x = x.permute(0, 3, 1, 2).double() / 255 if x.dtype == torch.uint8 else x.double()
    return 2 * F.interpolate(x, size=(299, 299), mode="bilinear", align_corners=False) - 1


def seeded_fid_state_dict(seed=0, calib_images=4):
    """The seeded weights as pytorch-fid's state dict: torchvision key names, no num_batches_tracked, fp32 CPU tensors."""
    torch.manual_seed(seed)
    m = fid_network(pooling="fid")
    g = torch.Generator().manual_seed(seed + 1)
    bns = [mod for mod in m.modules() if isinstance(mod, nn.BatchNorm2d)]
    with torch.no_grad():
        for bn in bns:
            bn.weight.copy_(torch.rand(bn.num_features, generator=g) * 0.4 + 0.3)
            bn.bias.copy_(torch.rand(bn.num_features, generator=g) * 0.5 + 0.3)
            bn.momentum = None  # cumulative average: after one batch, the running statistics are that batch's
        m.fc.weight.mul_(4.0)
        m.train()
        m(torch.rand((calib_images, 3, 299, 299), generator=g) * 2 - 1)
        m.eval()
        for bn in bns:
            sd = bn.running_var.sqrt()
            bn.running_mean.add_(0.05 * sd * torch.randn(bn.num_features, generator=g))
            bn.running_var.mul_(torch.rand(bn.num_features, generator=g) * 0.2 + 0.9)
    return {k: v.clone() for k, v in m.state_dict().items() if not k.endswith("num_batches_tracked")}


def fp64_forward(model, images):
    """({tap: fp64 NCHW}, pool fp64 (N,2048), logits fp64 (N,1008)) of `model` in float64 on pytorch-fid's input of `images`."""
    return inception_oracle.fp64_forward(model, fid_input(images))
