"""Drop-in for the reference's eval_models package (eval_models/__init__.py:13-40): `PerceptualLoss`, the LPIPS metric with AlexNet and
the v0.1 linear heads, backed by the sm_90a kernels of hrviton_b200.metrics.  Put this repository first on sys.path (hrv_env.install())
and `import eval_models as models` in train_generator.py / evaluate.py binds to it.

Supported: the configuration HR-VITON uses, PerceptualLoss(model='net-lin', net='alex', colorspace='rgb', spatial=False), under
no_grad.  Other models, backbones, colour spaces, spatial maps and gradients raise NotImplementedError.  The heads are read from
./eval_models/weights/v0.1/alex.pth under the working directory, then from weights/v0.1/alex.pth next to this package; a missing file
raises FileNotFoundError, as the reference's torch.load does.  The AlexNet backbone loads torchvision's ImageNet weights
(HRV_ALEX_RANDOM_INIT=1: none, for offline machines)."""
import torch

import hrv_loader

hrv_loader.load()
from hrviton_b200.metrics import NetLinLayer, PNetLin, ScalingLayer, alex_weights_path, load_lpips  # noqa: E402,F401


def normalize_tensor(in_feat, eps=1e-10):
    """eval_models/__init__.py:42-44 (torch; the kernels fuse it into hrv_lpips_dist)."""
    norm_factor = torch.sqrt(torch.sum(in_feat ** 2, dim=1, keepdim=True))
    return in_feat / (norm_factor + eps)


class PerceptualLoss(torch.nn.Module):
    def __init__(self, model='net-lin', net='alex', colorspace='rgb', spatial=False, use_gpu=True, gpu_ids=[0]):  # noqa: B006 (reference signature)
        super().__init__()
        print('Setting up Perceptual loss...')
        if model != 'net-lin' or net != 'alex':
            raise NotImplementedError("eval_models drop-in: only model='net-lin', net='alex' (LPIPS v0.1) runs here, got model=%r net=%r"
                                      % (model, net))
        if str(colorspace).lower() != 'rgb':
            raise NotImplementedError("eval_models drop-in: colorspace=%r is used by the L2 / SSIM models only; LPIPS takes rgb" % (colorspace,))
        if spatial:
            raise NotImplementedError("eval_models drop-in: spatial=True (per-pixel LPIPS maps) is not implemented")
        self.use_gpu = use_gpu
        self.spatial = spatial
        self.gpu_ids = gpu_ids
        self.net = load_lpips(device=("cuda:%d" % gpu_ids[0]) if use_gpu else "cpu")
        print('...[%s] initialized' % ('%s [%s]' % (model, net)))
        print('...Done')

    def forward(self, pred, target, normalize=False):
        """pred, target: (N,3,H,W) fp32 cuda in [-1, 1] (normalize=True: in [0, 1]).  Returns (N,1,1,1) fp32."""
        if torch.is_grad_enabled() and (pred.requires_grad or target.requires_grad):
            raise NotImplementedError("eval_models drop-in: LPIPS has no backward pass; call it under torch.no_grad()")
        if normalize:
            target = 2 * target - 1
            pred = 2 * pred - 1
        with torch.no_grad():
            return self.net(target, pred)
