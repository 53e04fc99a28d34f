"""CPU oracle for the HR-VITON hot path — TEST INFRASTRUCTURE ONLY.

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s cpu_baseline /
``--impl reference`` legs may import this file; the product path never does.

It restates, functionally (state_dict in, tensors out; fp32 on the host CPU), what
the reference modules compute.  The arithmetic primitives (conv2d, matmul) come
from torch-CPU fp32 — the same third-party substrate the reference itself runs on
(SURVEY.md §8c: PyTorch is un-vendored, unpinned; oracle version torch 2.11.0) —
while everything with index arithmetic (warp, bilinear/nearest resampling, pooling,
normalisation statistics) is ALSO restated in explicit numpy (``np_*`` below) so the
CUDA kernels can be checked against formulas rather than against another library.

Pinning: the reference holds no golden vectors or tests (SURVEY.md §4).  The oracle
is pinned against the *live reference modules* imported from /root/reference by
``tests/golden/make_golden.py`` (committed fixtures in tests/golden/*.npz, checked
by tests/test_oracle_vs_golden.py).  Beyond that live comparison: parity unpinned.

Citations are file:line in /root/reference.
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

# --------------------------------------------------------------------------------------
# numpy primitives (explicit index arithmetic)
# --------------------------------------------------------------------------------------


def np_linspace_grid(n):
    """torch.linspace(-1, 1, n) values (networks.py:162-163). Taken from torch on purpose:
    a hand-rolled symmetric formula does not bit-match (SURVEY.md §8c)."""
    return torch.linspace(-1.0, 1.0, n).numpy().astype(np.float32)


def np_bilinear_up2(x):
    """F.interpolate(x, scale_factor=2, mode='bilinear', align_corners=False) on (..., H, W)
    (networks.py:130-133,150,181).  src = max((d+0.5)/2-0.5, 0); i0=floor; i1=min(i0+1,n-1)."""
    x = np.asarray(x, np.float32)
    h, w = x.shape[-2:]

    def taps(n):
        d = np.arange(2 * n, dtype=np.float32)
        s = np.maximum((d + np.float32(0.5)) * np.float32(0.5) - np.float32(0.5), np.float32(0))
        i0 = np.floor(s).astype(np.int64)
        i1 = np.minimum(i0 + 1, n - 1)
        l1 = (s - i0.astype(np.float32)).astype(np.float32)
        return i0, i1, np.float32(1) - l1, l1

    y0, y1, wy0, wy1 = taps(h)
    x0, x1, wx0, wx1 = taps(w)
    # torch's CPU kernel lerps along x inside each source row first, then along y
    cols = (x[..., x0] * wx0 + x[..., x1] * wx1).astype(np.float32)
    return (cols[..., y0, :] * wy0[:, None] + cols[..., y1, :] * wy1[:, None]).astype(np.float32)


def np_nearest_resize(x, oh, ow):
    """F.interpolate(mode='nearest'): src = min(floor(dst * (in / out)), in - 1) with the scale and the product rounded to fp32, as
    torch computes them (network_generator.py:164,222).  The exact floor(dst * in / out) differs where the fp32 product falls just
    below an integer (200 -> 24: dst 15 reads row 124, not 125)."""
    h, w = x.shape[-2:]

    def idx(n_in, n_out):
        scale = np.float32(n_in) / np.float32(n_out)
        return np.minimum(np.floor(np.arange(n_out, dtype=np.float32) * scale).astype(np.int64), n_in - 1)

    yi, xi = idx(h, oh), idx(w, ow)
    return x[..., yi[:, None], xi[None, :]]


def np_avgpool3s2(x):
    """F.avg_pool2d(3, stride=2, padding=1, count_include_pad=False) (network_generator.py:302,
    networks.py:320)."""
    x = np.asarray(x, np.float32)
    h, w = x.shape[-2:]
    oh, ow = (h + 2 - 3) // 2 + 1, (w + 2 - 3) // 2 + 1
    out = np.zeros(x.shape[:-2] + (oh, ow), np.float32)
    for oy in range(oh):
        ys = [y for y in (2 * oy - 1, 2 * oy, 2 * oy + 1) if 0 <= y < h]
        for ox in range(ow):
            xs = [q for q in (2 * ox - 1, 2 * ox, 2 * ox + 1) if 0 <= q < w]
            out[..., oy, ox] = x[..., ys[0]:ys[-1] + 1, xs[0]:xs[-1] + 1].sum((-1, -2)) / np.float32(len(ys) * len(xs))
    return out


def np_instance_norm(x, eps=1e-5):
    """nn.InstanceNorm2d(affine=False): per-(n,c) mean, biased variance, eps inside sqrt
    (network_generator.py:86,427). Returns (normalised, mean, rstd)."""
    x = np.asarray(x, np.float64)
    m = x.mean((-1, -2), keepdims=True)
    v = ((x - m) ** 2).mean((-1, -2), keepdims=True)
    r = 1.0 / np.sqrt(v + eps)
    return ((x - m) * r).astype(np.float32), m.astype(np.float32), r.astype(np.float32)


def np_flow_warp_coords(flow_lo, out_h, out_w, in_h, in_w):
    """The whole coordinate chain of the flow warp (networks.py:133-135,147-152), fp32, returning
    the integer gather indices and the fp32 lerp weights.

    flow_lo: (N, h, w, 2) coarse flow.  Steps: bilinear x2 upsample -> divide by
    ((out_w/2-1)/2, (out_h/2-1)/2) [correctly rounded fp32 division] -> add linspace base grid
    -> grid_sample unnormalise ((g+1)*S-1)/2 (align_corners=False) -> clamp [0,S-1] (border)
    -> floor, frac.
    Returns x0,y0 (int32; +1 neighbours are x0+1,y0+1 and contribute only when in range), tx,ty."""
    f = np.asarray(flow_lo, np.float32)
    up = np_bilinear_up2(np.moveaxis(f, -1, 1))  # (N,2,H,W)
    assert up.shape[-2:] == (out_h, out_w)
    sx = np.float32((out_w / 2 - 1.0) / 2.0)
    sy = np.float32((out_h / 2 - 1.0) / 2.0)
    gx = (up[:, 0] / sx + np_linspace_grid(out_w)[None, None, :]).astype(np.float32)
    gy = (up[:, 1] / sy + np_linspace_grid(out_h)[None, :, None]).astype(np.float32)
    ix = ((gx + np.float32(1)) * np.float32(in_w) - np.float32(1)) / np.float32(2)
    iy = ((gy + np.float32(1)) * np.float32(in_h) - np.float32(1)) / np.float32(2)
    ix = np.minimum(np.maximum(ix, np.float32(0)), np.float32(in_w - 1)).astype(np.float32)
    iy = np.minimum(np.maximum(iy, np.float32(0)), np.float32(in_h - 1)).astype(np.float32)
    x0 = np.floor(ix)
    y0 = np.floor(iy)
    return x0.astype(np.int32), y0.astype(np.int32), (ix - x0).astype(np.float32), (iy - y0).astype(np.float32)


def np_gather_bilinear(src, x0, y0, tx, ty):
    """4-tap gather of grid_sample(bilinear, border): src (N,C,H,W); taps outside the image get
    zero weight (after the border clamp only the +1 tap at the far edge, whose weight is 0)."""
    src = np.asarray(src, np.float32)
    n, c, h, w = src.shape
    out = np.zeros((n, c) + x0.shape[1:], np.float32)
    for b in range(n):
        xa, ya = x0[b], y0[b]
        xb, yb = np.minimum(xa + 1, w - 1), np.minimum(ya + 1, h - 1)
        vx = (xa + 1 <= w - 1).astype(np.float32)
        vy = (ya + 1 <= h - 1).astype(np.float32)
        wx1, wy1 = tx[b] * vx, ty[b] * vy
        wx0, wy0 = np.float32(1) - tx[b], np.float32(1) - ty[b]
        s = src[b]
        out[b] = (s[:, ya, xa] * (wy0 * wx0) + s[:, ya, xb] * (wy0 * wx1)
                  + s[:, yb, xa] * (wy1 * wx0) + s[:, yb, xb] * (wy1 * wx1))
    return out


def np_spectral_sigma(w_orig, u, v):
    """Old-style torch spectral_norm in eval mode: sigma = u^T (W_mat v); weight = W/sigma
    (network_generator.py:138-143; SURVEY.md §8 B5)."""
    wm = np.asarray(w_orig, np.float64).reshape(w_orig.shape[0], -1)
    return float(np.asarray(u, np.float64) @ (wm @ np.asarray(v, np.float64)))


# --------------------------------------------------------------------------------------
# functional network restatements (torch-CPU fp32)
# --------------------------------------------------------------------------------------


# --- storage-rounding model ("what does 16-bit activation storage cost the fp32 algorithm itself?") -------------------------------
# With storage_rounding(torch.bfloat16 | torch.float16) active, every convolution of the restatement rounds its input
# activations, its weights and its output to that type (and, through autograd, the gradients flowing back through the same
# points) while all arithmetic stays fp32.  This is the *floor* any implementation that keeps activations in a 16-bit type
# must sit on; tests assert that the CUDA kernels deviate from the fp32 goldens by no more than 1.1x what this model does.
_ROUND = [None, True]  # [dtype | None, also round conv outputs]


class storage_rounding:
    def __init__(self, dtype, outputs=True):
        self.new = [dtype, outputs]

    def __enter__(self):
        self.old = list(_ROUND)
        _ROUND[:] = self.new
        return self

    def __exit__(self, *exc):
        _ROUND[:] = self.old
        return False


def _q(t):
    if _ROUND[0] is None or t is None:
        return t
    return t.to(_ROUND[0]).to(torch.float32)


def _qo(t):
    return _q(t) if _ROUND[1] else t


def conv2d_q(x, w, b=None, stride=1, padding=0):
    """F.conv2d under the storage-rounding model (identity when no rounding is active)."""
    return _qo(F.conv2d(_q(x), _q(w), b, stride=stride, padding=padding))


def _conv(sd, name, x, stride=1, padding=0):
    return conv2d_q(x, sd[name + ".weight"], sd.get(name + ".bias"), stride=stride, padding=padding)


def _bn_eval(sd, name, x, eps=1e-5):
    """BatchNorm2d, eval mode (networks.py:189,192)."""
    scale = sd[name + ".weight"] / torch.sqrt(sd[name + ".running_var"] + eps)
    shift = sd[name + ".bias"] - sd[name + ".running_mean"] * scale
    return x * scale[None, :, None, None] + shift[None, :, None, None]


def _bn_train(sd, name, x, eps=1e-5):
    """BatchNorm2d, train mode forward (batch statistics, biased var for normalisation)."""
    m = x.mean((0, 2, 3), keepdim=True)
    v = x.var((0, 2, 3), unbiased=False, keepdim=True)
    return (x - m) / torch.sqrt(v + eps) * sd[name + ".weight"][None, :, None, None] + sd[name + ".bias"][None, :, None, None]


def _up2(x):
    return F.interpolate(x, scale_factor=2, mode="bilinear", align_corners=False)


def resblock(sd, p, x, scale, bn_train=False):
    """networks.py:171-198."""
    bn = _bn_train if bn_train else _bn_eval
    if scale == "down":
        r = _conv(sd, p + ".scale", x, stride=2, padding=1)
    elif scale == "same":
        r = _conv(sd, p + ".scale", x)
    else:  # 'up': bilinear x2 then 1x1
        r = _conv(sd, p + ".scale.1", _up2(x))
    h = torch.relu(bn(sd, p + ".block.1", _conv(sd, p + ".block.0", r, padding=1)))
    h = bn(sd, p + ".block.4", _conv(sd, p + ".block.3", h, padding=1))
    return torch.relu(r + h)


def make_base_grid(n, h, w):
    """networks.py:161-168 (x then y, values from torch.linspace)."""
    gx = torch.linspace(-1.0, 1.0, w).view(1, 1, w, 1).expand(n, h, w, 1)
    gy = torch.linspace(-1.0, 1.0, h).view(1, h, 1, 1).expand(n, h, w, 1)
    return torch.cat([gx, gy], 3)


def flow_warp(src, flow_lo):
    """Upsample the coarse flow x2, normalise, add base grid, grid_sample(border)
    (networks.py:133-135 and :147-152).  src (N,C,H,W), flow_lo (N,H/2,W/2,2)."""
    n, _, h, w = src.shape
    fl = _up2(flow_lo.permute(0, 3, 1, 2)).permute(0, 2, 3, 1)
    fx = fl[..., 0:1] / ((w / 2 - 1.0) / 2.0)
    fy = fl[..., 1:2] / ((h / 2 - 1.0) / 2.0)
    grid = torch.cat([fx, fy], 3) + make_base_grid(n, h, w)
    return F.grid_sample(src, grid, mode="bilinear", padding_mode="border", align_corners=False)


def tocg_forward(sd, input1, input2, bn_train=False):
    """ConditionGenerator.forward with warp_feature='T1', out_layer='relu' (networks.py:98-159).
    Returns (flow_list[5 x (N,h,w,2)], seg, warped_c, warped_cm)."""
    e1, e2 = [], []
    a, b = input1, input2
    for i in range(5):
        a = resblock(sd, "ClothEncoder.%d" % i, a, "down", bn_train)
        b = resblock(sd, "PoseEncoder.%d" % i, b, "down", bn_train)
        e1.append(a)
        e2.append(b)
    flows = []
    t1 = e1[4]
    flow = _conv(sd, "flow_conv.0", torch.cat([t1, e2[4]], 1), padding=1).permute(0, 2, 3, 1)
    flows.append(flow)
    x = resblock(sd, "conv", e2[4], "same", bn_train)
    x = resblock(sd, "SegDecoder.0", x, "up", bn_train)
    for i in range(1, 5):
        lvl = 4 - i
        t1 = _up2(t1) + _conv(sd, "conv1.%d" % lvl, e1[lvl])
        # T2 update (networks.py:131) is dead code: its value is never read.
        warped = flow_warp(t1, flows[-1])
        bott = torch.relu(_conv(sd, "bottleneck.%d.0" % (i - 1), x, padding=1))
        fl_up = _up2(flows[-1].permute(0, 3, 1, 2)).permute(0, 2, 3, 1)
        flow = fl_up + _conv(sd, "flow_conv.%d" % i, torch.cat([warped, bott], 1), padding=1).permute(0, 2, 3, 1)
        flows.append(flow)
        x = resblock(sd, "SegDecoder.%d" % i, torch.cat([x, e2[lvl], warped], 1), "up", bn_train)
    warped_in = flow_warp(input1, flows[-1])
    seg = resblock(sd, "out_layer", torch.cat([x, input2, warped_in], 1), "same", bn_train)
    return flows, seg, warped_in[:, :-1], warped_in[:, -1:]


_SN_TRAIN = [False]


class spectral_train:
    """Train-mode spectral norm for the functional restatements below: one power iteration per forward, u/v updated IN PLACE in
    the state_dict (no grad), sigma = u.(W v) differentiable through W only — torch.nn.utils.spectral_norm (old style, dim 0,
    eps 1e-12) as the reference uses it (network_generator.py:138-143; SURVEY.md 8 B5)."""

    def __enter__(self):
        self.old = _SN_TRAIN[0]
        _SN_TRAIN[0] = True
        return self

    def __exit__(self, *exc):
        _SN_TRAIN[0] = self.old
        return False


def spectral_weight(sd, p):
    """Old-style spectral_norm: W_orig / (u . W_mat v).  Eval mode uses the stored u, v; under `spectral_train()` they are first
    refreshed by one power iteration (v <- normalize(W^T u), u <- normalize(W v)) written back into sd."""
    w = sd[p + ".weight_orig"]
    wm = w.reshape(w.shape[0], -1)
    u, v = sd[p + ".weight_u"], sd[p + ".weight_v"]
    if _SN_TRAIN[0]:
        with torch.no_grad():
            v.copy_(F.normalize(torch.mv(wm.detach().t(), u), dim=0, eps=1e-12))
            u.copy_(F.normalize(torch.mv(wm.detach(), v), dim=0, eps=1e-12))
        u, v = u.clone(), v.clone()
    sigma = torch.dot(u, torch.mv(wm, v))
    return w / sigma


def _inorm(x, eps=1e-5):
    m = x.mean((2, 3), keepdim=True)
    v = x.var((2, 3), unbiased=False, keepdim=True)
    return (x - m) / torch.sqrt(v + eps)


def spade_norm(sd, p, x, seg, noise_hw):
    """SPADENorm.forward (network_generator.py:101-122). noise_hw: (N,H,W) standard-normal draw,
    already transposed to image layout."""
    noise = noise_hw[:, None] * sd[p + ".noise_scale"][None, :, None, None]
    normalized = _inorm(x + noise)
    actv = torch.relu(_conv(sd, p + ".conv_shared.0", seg, padding=1))
    gamma = _conv(sd, p + ".conv_gamma", actv, padding=1)
    beta = _conv(sd, p + ".conv_beta", actv, padding=1)
    return normalized * (1 + gamma) + beta


def spade_resblock(sd, p, x, seg_full, noise_fn):
    """SPADEResBlock.forward (network_generator.py:157-173); noise draw order norm_s, norm_0, norm_1."""
    n, _, h, w = x.shape
    seg = F.interpolate(seg_full, size=(h, w), mode="nearest")
    learned = (p + ".conv_s.weight_orig") in sd
    if learned:
        hs = spade_norm(sd, p + ".norm_s", x, seg, noise_fn(n, h, w))
        x_s = conv2d_q(hs, spectral_weight(sd, p + ".conv_s"))
    else:
        x_s = x
    h0 = F.leaky_relu(spade_norm(sd, p + ".norm_0", x, seg, noise_fn(n, h, w)), 0.2)
    dx = conv2d_q(h0, spectral_weight(sd, p + ".conv_0"), sd[p + ".conv_0.bias"], padding=1)
    h1 = F.leaky_relu(spade_norm(sd, p + ".norm_1", dx, seg, noise_fn(n, h, w)), 0.2)
    dx = conv2d_q(h1, spectral_weight(sd, p + ".conv_1"), sd[p + ".conv_1.bias"], padding=1)
    return x_s + dx


def spade_generator_forward(sd, x, seg, noise_fn, num_up=7):
    """SPADEGenerator.forward, num_upsampling_layers='most' (network_generator.py:221-245)."""
    n, _, H, W = x.shape
    sh, sw = H // 2 ** num_up, W // 2 ** num_up
    feats = []
    for i in range(8):
        s = F.interpolate(x, size=(sh * 2 ** i, sw * 2 ** i), mode="nearest")
        feats.append(_conv(sd, "conv_%d" % i, s, padding=1))
    up = lambda t: F.interpolate(t, scale_factor=2, mode="nearest")
    h = spade_resblock(sd, "head_0", feats[0], seg, noise_fn)
    names = ["G_middle_0", "G_middle_1", "up_0", "up_1", "up_2", "up_3", "up_4"]
    for j, name in enumerate(names):
        h = spade_resblock(sd, name, torch.cat([up(h), feats[j + 1]], 1), seg, noise_fn)
    return torch.tanh(_conv(sd, "conv_img", F.leaky_relu(h, 0.2), padding=1))


def gen_d_forward(sd, inp, num_d=2, n_layers=3):
    """gen-D MultiscaleDiscriminator.forward with norm_D='spectralinstance'
    (network_generator.py:250-316,401-433). Returns list[num_d] of list[n_layers+1]."""
    res = []
    cur = inp
    for d in range(num_d):
        p = "discriminator_%d" % d
        feats = []
        h = F.leaky_relu(_conv(sd, p + ".model0.0", cur, stride=2, padding=2), 0.2)
        feats.append(h)
        for n in range(1, n_layers):
            q = p + ".model%d.0.0" % n
            h = conv2d_q(h, spectral_weight(sd, q), None, stride=2, padding=2)
            h = F.leaky_relu(_inorm(h), 0.2)
            feats.append(h)
        feats.append(_conv(sd, p + ".model%d.0" % n_layers, h, stride=1, padding=2))
        res.append(feats)
        cur = F.avg_pool2d(cur, 3, stride=2, padding=1, count_include_pad=False)
    return res


def tocg_d_forward(sd, inp, num_d=2, n_layers=3, ddownx2=True):
    """networks.MultiscaleDiscriminator via define_D, eval mode (Dropout = identity), no spectral,
    getIntermFeat=False (networks.py:302-408). Sequential indices: conv at 0,2,5/6..: computed from keys."""
    def run(prefix, x):
        idx = sorted({int(k.split(".")[1]) for k in sd if k.startswith(prefix + ".") and k.endswith(".weight")})
        last = idx[-1]
        for j, ci in enumerate(idx):
            w = sd["%s.%d.weight" % (prefix, ci)]
            stride = 2 if j < n_layers else 1
            x = conv2d_q(x, w, sd["%s.%d.bias" % (prefix, ci)], stride=stride, padding=2)
            if ci == last:
                break
            if j > 0:
                x = _inorm(x)
            x = F.leaky_relu(x, 0.2)
        return x

    pool = lambda t: F.avg_pool2d(t, 3, stride=2, padding=1, count_include_pad=False)
    cur = pool(inp) if ddownx2 else inp
    out = []
    for i in range(num_d):
        out.append([run("layer%d" % (num_d - 1 - i), cur)])
        if i != num_d - 1:
            cur = pool(cur)
    return out
