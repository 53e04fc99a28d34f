"""NHWC activation views + thin wrappers over the C-ABI.  torch is used here for device memory and streams only."""
import ctypes
import os
from dataclasses import dataclass

import torch

from . import capi
from .capi import ACT_LRELU, ACT_NONE, ACT_RELU, ACT_TANH, BF16, F32  # noqa: F401

LAUNCHES = [0]  # count of kernel launches issued through the C-ABI (bench.py reads this for `gpu_launches`)
PARAM_GEN = [0]  # generation of the parameter values: part of every derived-weight cache key (spade._param_key)
STORAGE = [torch.bfloat16]  # activation storage type of newly created buffers: torch.bfloat16 (default), torch.float16 or torch.float32
PROFILE = None  # bench.py sets this to a list; every C-ABI call then appends (kind, work, start_event, end_event)
PRECISIONS = {"bf16": torch.bfloat16, "fp16": torch.float16, "fp32": torch.float32}


class _Timed:
    """Brackets one C-ABI call with CUDA events on the launching stream when profiling is on (bench.py roofline)."""

    def __init__(self, kind, work, launches=1, label=""):
        self.kind, self.work, self.launches, self.label = kind, work, launches, label

    def __enter__(self):
        LAUNCHES[0] += self.launches
        if PROFILE is not None:
            self.e0 = torch.cuda.Event(enable_timing=True)
            self.e1 = torch.cuda.Event(enable_timing=True)
            self.e0.record()
        return self

    def __exit__(self, *exc):
        if PROFILE is not None:
            self.e1.record()
            PROFILE.append((self.kind, self.work, self.e0, self.e1, self.label))
        return False


def set_precision(name):
    """'bf16' (default: bf16 activations, fp32 accumulation — the training configuration), 'fp16' (IEEE half activations,
    3 more mantissa bits: the storage type of the reference's own apex-O1 --fp16 runs, train_generator.py:161-169; meets the
    1e-2 forward tolerance of BASELINE.json) or 'fp32' (fp32 activations and 3xTF32 convolutions: the reference's own fp32
    inference to the 1e-3 tolerance of BASELINE.json; inference only).  Invalidates every derived-weight cache."""
    if name not in PRECISIONS:
        raise ValueError("precision must be one of %s, got %r" % ("/".join(PRECISIONS), name))
    dt = PRECISIONS[name]
    if STORAGE[0] != dt:
        STORAGE[0] = dt
        PARAM_GEN[0] += 1


def get_precision():
    return {v: k for k, v in PRECISIONS.items()}[STORAGE[0]]


def require_trainable_storage(what):
    """Training entry points call this before any launch: fp32 storage has no backward kernels."""
    if STORAGE[0] == torch.float32:
        raise NotImplementedError("fp32 storage is inference-only (%s needs a backward pass): call ops.set_precision('bf16') or "
                                  "set_precision('fp16') to train" % what)


# The reference's inference scripts run unchanged in another precision through the environment (read once, here).
set_precision(os.environ.get("HRV_PRECISION", "bf16"))


def _L(*things):
    """The library flavour matching the storage type of the given Acts / tensors (fp16 if any of them is torch.float16)."""
    for t in things:
        if t is None:
            continue
        d = t.buf.dtype if isinstance(t, Act) else (t.dtype if torch.is_tensor(t) else t)
        if d == torch.float16:
            return capi.lib(torch.float16)
    return capi.lib()


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def round_up(v, m):
    return (v + m - 1) // m * m


class Act:
    """A pixel-major (NHWC) activation: `buf` is (N,H,W,P) bf16|fp32 on the GPU; the view covers channels
    [c0, c0+c) of every pixel.  Channel slices of one buffer replace torch.cat."""

    def __init__(self, buf, c=None, c0=0):
        assert buf.is_cuda and buf.dim() == 4 and buf.is_contiguous(), "Act needs a contiguous CUDA (N,H,W,P) buffer"
        self.buf = buf
        self.c0 = c0
        self.c = buf.shape[3] - c0 if c is None else c
        assert self.c0 + self.c <= buf.shape[3]

    @staticmethod
    def empty(n, h, w, c, dtype=None, device="cuda", pitch=None, zero=False):
        dtype = STORAGE[0] if dtype is None else dtype
        p = round_up(c, 8) if pitch is None else pitch
        f = torch.zeros if zero else torch.empty
        return Act(f((n, h, w, p), dtype=dtype, device=device), c=c)

    n = property(lambda s: s.buf.shape[0])
    h = property(lambda s: s.buf.shape[1])
    w = property(lambda s: s.buf.shape[2])
    pitch = property(lambda s: s.buf.shape[3])

    def slice(self, c0, c):
        return Act(self.buf, c=c, c0=self.c0 + c0)

    def ct(self):
        es = self.buf.element_size()
        return capi.Tensor(self.buf.data_ptr() + self.c0 * es, self.n, self.h, self.w, self.c, self.pitch,
                           F32 if self.buf.dtype == torch.float32 else BF16)

    def to_nchw(self):
        """fp32 NCHW copy (API boundary / tests)."""
        out = torch.empty((self.n, self.c, self.h, self.w), dtype=torch.float32, device=self.buf.device)
        t = self.ct()
        with _Timed("glue", 0.0, label="nhwc_to_nchw"):
            capi.check(_L(self).hrv_nhwc_to_nchw(ctypes.byref(t), out.data_ptr(), _stream()), "nhwc_to_nchw")
        return out


_NULL = capi.Tensor(None, 0, 0, 0, 0, 0, 0)


def _p(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def from_nchw(x, c_pad=None, size=None, out=None):
    """fp32 NCHW (cuda) -> NHWC Act in the storage type, optional nearest resize to `size` (F.interpolate nearest)."""
    assert x.is_cuda and x.dtype == torch.float32
    x = x.contiguous()
    n, c, h, w = x.shape
    oh, ow = (h, w) if size is None else size
    if out is None:
        out = Act.empty(n, oh, ow, c, pitch=round_up(c if c_pad is None else c_pad, 8))
    t = out.ct()
    with _Timed("glue", 0.0, label="nchw_to_nhwc"):
        capi.check(_L(out).hrv_nchw_to_nhwc(x.data_ptr(), c, h, w, ctypes.byref(t), _stream()), "nchw_to_nhwc")
    return out


SEG_CAT_MODES = {"no_composition": 0, "warp_grad": 1, "detach": 2}


def seg_softmax_cat(input1, input2, seg, cm=None, cm_channel=3, composition="warp_grad", softmax=True, want_seg=False, out=None):
    """The condition discriminator's input [input1 | input2 | third] as one NHWC Act in the storage type (hrv_seg_softmax_cat):
    third = seg with channel `cm_channel` multiplied by cm ('warp_grad') or by (cm > 0.5) ('detach'), then its channel soft-max
    (softmax=True) or itself.  All inputs fp32 NCHW (cuda) at one (N,H,W); cm (N,1,H,W), None = no composition.
    want_seg=True also returns the composed seg as fp32 NCHW; out: the destination Act (c1+c2+K channels), as for from_nchw."""
    if composition not in SEG_CAT_MODES:
        raise ValueError("composition must be one of %s, got %r" % ("/".join(SEG_CAT_MODES), composition))
    mode = 0 if cm is None else SEG_CAT_MODES[composition]
    ts = [input1, input2, seg] + ([cm] if mode else [])
    for t in ts:
        if not t.is_cuda:
            raise RuntimeError("seg_softmax_cat runs on the GPU only (no CPU fallback): got a %s tensor" % t.device)
        if t.dtype != torch.float32 or t.dim() != 4 or (t.shape[0],) + tuple(t.shape[2:]) != (seg.shape[0],) + tuple(seg.shape[2:]):
            raise ValueError("seg_softmax_cat: every input must be float32 (N,C,H,W) at one (N,H,W); got %s" % [tuple(t.shape) for t in ts])
    if mode and cm.shape[1] != 1:
        raise ValueError("seg_softmax_cat: cm must be (N,1,H,W), got %s" % (tuple(cm.shape),))
    input1, input2, seg = input1.contiguous(), input2.contiguous(), seg.contiguous()
    cm = cm.contiguous() if mode else None
    n, k, h, w = seg.shape
    if out is None:
        out = Act.empty(n, h, w, input1.shape[1] + input2.shape[1] + k)
    seg_out = torch.empty_like(seg) if want_seg else None
    t = out.ct()
    with _Timed("glue", 0.0, label="seg_softmax_cat"):
        capi.check(_L(out).hrv_seg_softmax_cat(input1.data_ptr(), input1.shape[1], input2.data_ptr(), input2.shape[1], seg.data_ptr(), k,
                                               _p(cm), cm_channel, mode, int(bool(softmax)), ctypes.byref(t), _p(seg_out), _stream()),
                   "seg_softmax_cat")
    return (out, seg_out) if want_seg else out


def seg_iou(seg, cm, parse):
    """train_condition.iou_metric(F.softmax(seg * cloth_mask, 1), parse), cloth_mask = ones with channel 3 = cm (composition
    'warp_grad'), as a 0-dim fp32 cuda tensor (hrv_seg_iou; no synchronisation).  seg, parse: fp32 (N,K,H,W) cuda; cm: (N,1,H,W).
    Shapes and dtypes are the caller's to check (metrics.segmentation_iou)."""
    seg, cm, parse = seg.contiguous(), cm.contiguous(), parse.contiguous()
    n, k, h, w = seg.shape
    out = torch.empty((), dtype=torch.float32, device=seg.device)
    L = capi.lib()
    ws = torch.empty(max(int(L.hrv_seg_iou_workspace_bytes(n, h, w)), 16), dtype=torch.uint8, device=seg.device)
    with _Timed("glue", 0.0, launches=2, label="seg_iou"):
        capi.check(L.hrv_seg_iou(seg.data_ptr(), k, cm.data_ptr(), parse.data_ptr(), n, h, w, out.data_ptr(), ws.data_ptr(), ws.numel(),
                                 _stream()), "seg_iou")
    return out


def _tv_flows(flows, edge_weights, plain_weights, mask):
    if not 1 <= len(flows) <= capi.TV_MAX_FLOWS or not len(flows) == len(edge_weights) == len(plain_weights):
        raise ValueError("flow_tv: 1..%d flows with one edge and one plain weight each, got %d / %d / %d"
                         % (capi.TV_MAX_FLOWS, len(flows), len(edge_weights), len(plain_weights)))
    n = flows[0].shape[0]
    for f in flows:
        if not f.is_cuda or f.dtype != torch.float32 or f.dim() != 4 or f.shape[0] != n or f.shape[3] != 2 or not f.is_contiguous():
            raise ValueError("flow_tv: flows must be contiguous float32 (N,h,w,2) cuda tensors, got %s %s" % (tuple(f.shape), f.dtype))
    if mask is not None and (not mask.is_cuda or mask.dtype != torch.float32 or mask.dim() != 4 or mask.shape[:2] != (n, 1)
                             or not mask.is_contiguous()):
        raise ValueError("flow_tv: mask must be a contiguous float32 (N,1,H,W) cuda tensor, got %s %s" % (tuple(mask.shape), mask.dtype))
    arr = (capi.TvFlow * len(flows))(*[capi.TvFlow(f.data_ptr(), f.shape[1], f.shape[2], float(we), float(wp))
                                       for f, we, wp in zip(flows, edge_weights, plain_weights)])
    mh, mw = (mask.shape[2], mask.shape[3]) if mask is not None else (0, 0)
    L = capi.lib()
    ws = torch.empty(int(L.hrv_flow_tv_workspace_bytes(arr, len(flows), n)), dtype=torch.uint8, device=flows[0].device)
    return L, arr, n, mh, mw, ws


def flow_tv(flows, edge_weights, plain_weights, mask=None, want_mask_down=False):
    """The stage-1 flow TV (hrv_flow_tv): sum over i of edge_weights[i] * (edge-aware TV of flows[i], weighted by exp(-150 |D m_i|),
    m_i = F.interpolate(mask, flows[i]'s size, bilinear); the plain TV without mask) + plain_weights[i] * (plain TV of flows[i]).
    flows: contiguous fp32 (N,h,w,2) cuda; mask: contiguous fp32 (N,1,H,W) or None.  Returns (loss 0-dim, per-flow terms (len,)) fp32 on
    the device, reproducible bit for bit, no synchronisation; want_mask_down=True (with mask) adds the list of m_i (N,1,h_i,w_i)."""
    L, arr, n, mh, mw, ws = _tv_flows(flows, edge_weights, plain_weights, mask)
    loss = torch.empty((), dtype=torch.float32, device=flows[0].device)
    terms = torch.empty(len(flows), dtype=torch.float32, device=flows[0].device)
    downs = [torch.empty((n, 1, f.shape[1], f.shape[2]), dtype=torch.float32, device=f.device) for f in flows] if want_mask_down else None
    dptrs = (ctypes.c_void_p * len(flows))(*[d.data_ptr() for d in downs]) if want_mask_down else None
    with _Timed("glue", 0.0, launches=3 if mask is not None else 2, label="flow_tv"):
        capi.check(L.hrv_flow_tv(arr, len(flows), n, _p(mask), mh, mw, loss.data_ptr(), terms.data_ptr(), dptrs, ws.data_ptr(), ws.numel(),
                                 _stream()), "flow_tv")
    return (loss, terms, downs) if want_mask_down else (loss, terms)


def flow_tv_bwd(flows, edge_weights, plain_weights, mask, dloss, want_dmask=True):
    """Gradients of flow_tv for the upstream scalar dloss (a 1-element fp32 cuda tensor): ([dflow_i (N,h,w,2)], dmask (N,1,H,W) or None),
    from gathers in a fixed order (hrv_flow_tv_bwd)."""
    L, arr, n, mh, mw, ws = _tv_flows(flows, edge_weights, plain_weights, mask)
    assert dloss.is_cuda and dloss.dtype == torch.float32 and dloss.numel() == 1
    dflows = [torch.empty_like(f) for f in flows]
    dmask = torch.empty_like(mask) if (mask is not None and want_dmask) else None
    dptrs = (ctypes.c_void_p * len(flows))(*[d.data_ptr() for d in dflows])
    with _Timed("glue", 0.0, launches=(1 if mask is not None else 0) + 1 + (1 if dmask is not None else 0), label="flow_tv_bwd"):
        capi.check(L.hrv_flow_tv_bwd(arr, len(flows), n, _p(mask), mh, mw, dloss.data_ptr(), dptrs, _p(dmask), ws.data_ptr(), ws.numel(),
                                     _stream()), "flow_tv_bwd")
    return dflows, dmask


# ----------------------------------------------------------------------------------------------- weights

def pick_bk(cin):
    cands = [64, 32] + ([16] if cin <= 16 else [])
    pads = {bk: round_up(cin, bk) for bk in cands}
    best = min(pads.values())
    for bk in cands:
        if pads[bk] <= 1.10 * best:
            return bk
    return cands[-1]


def pick_bn(n_gemm):
    n16 = round_up(n_gemm, 16)
    if n16 <= 256:
        return n16
    # cost model: every N tile re-streams the A operand once (+64 ~ fixed per-tile overhead in columns)
    best, best_cost = 256, None
    for bn in range(256, 15, -16):
        tiles = (n_gemm + bn - 1) // bn
        cost = (tiles * (bn + 64), tiles * bn)
        if best_cost is None or cost < best_cost:
            best, best_cost = bn, cost
    return best


def pick_bn_spade(n_gemm):
    """N tile of a gamma|beta GEMM (n_gemm = 2C interleaved columns): with several N tiles each tile's channel range ends on a
    16-channel slab (bn % 32 == 0); take the candidate with the fewest padded columns (ties: the wider tile)."""
    n16 = round_up(n_gemm, 16)
    if n16 <= 256:
        return n16
    best = None
    for bn in (256, 224, 192, 160):
        cols = round_up(n_gemm, bn)
        if best is None or cols < best[0]:
            best = (cols, bn)
    return best[1]


@dataclass
class PackedConv:
    w: torch.Tensor  # 16-bit [taps, n_pad, cin_k], or fp32 [2 (hi, lo), taps, n_pad, cin_k] on fp32 storage
    kh: int
    kw: int
    off_y: int
    off_x: int
    bk: int
    bn: int
    n_gemm: int
    cin: int
    flops_per_pixel: float = 0.0  # algorithmic 2*Cin*Cout*kh*kw of the ORIGINAL convolution (unpadded, pre-s2d)


def pack_weight(w, off, cin_total=None, interleave=None, bn=None, flops_per_pixel=None, dgrad=False, storage=None):
    """w: (Cout,Cin,kh,kw) fp32 cuda (already divided by sigma / transformed). Returns PackedConv (one kernel: hrv_pack_conv_weight).
    interleave: a second weight of identical shape whose rows are interleaved (gamma_c, beta_c pairs).
    dgrad=True packs the operand of the data-gradient convolution (flip + transpose) without materialising it.
    storage: the activation storage the convolution will run on (default: the current one, set_precision)."""
    w = w.detach()
    if w.dtype != torch.float32 or not w.is_contiguous():
        w = w.float().contiguous()
    if interleave is not None:
        interleave = interleave.detach()
        if interleave.dtype != torch.float32 or not interleave.is_contiguous():
            interleave = interleave.float().contiguous()
        assert interleave.shape == w.shape
    cout, cin, kh, kw = w.shape
    inter = 2 if interleave is not None else 1
    rows, cols = (cin, cout * inter) if dgrad else (cout * inter, cin)  # GEMM N rows, K columns
    k_eff = cols if cin_total is None else cin_total
    st = STORAGE[0] if storage is None else storage
    f32 = st == torch.float32
    if f32:
        bk = 32  # the 3xTF32 kernel's K block: 32 fp32 channels = one 128-byte swizzle row
    else:
        # Cout <= 128 with more than 32 input channels: 64-channel K blocks (zero padded), the convolution kernel's own block size
        bk = 64 if (rows <= 128 and k_eff > 32) else pick_bk(k_eff)  # K <= 32 stays on the 32-wide blocks (padding to 64 would double the MMAs)
    cin_k = round_up(k_eff, bk)
    if bn is None:
        bn = pick_bn_spade(rows) if (interleave is not None and not dgrad) else pick_bn(rows)
    n_pad = round_up(rows, bn)
    if f32:  # hi / lo planes of the 3xTF32 split
        wp = torch.empty((2, kh * kw, n_pad, cin_k), dtype=torch.float32, device=w.device)
        with _Timed("glue", 0.0, label="pack_conv_weight_tf32x2"):
            capi.check(capi.lib().hrv_pack_conv_weight_tf32x2(w.data_ptr(), _p(interleave), cout, cin, kh, kw, 1 if dgrad else 0, None,
                                                              wp.data_ptr(), n_pad, cin_k, _stream()), "pack_conv_weight_tf32x2")
    else:
        wp = torch.empty((kh * kw, n_pad, cin_k), dtype=st, device=w.device)
        with _Timed("glue", 0.0, label="pack_conv_weight"):
            capi.check(_L(wp).hrv_pack_conv_weight(w.data_ptr(), _p(interleave), cout, cin, kh, kw, 1 if dgrad else 0, None, wp.data_ptr(),
                                                       n_pad, cin_k, _stream()), "pack_conv_weight")
    fpp = 2.0 * cin * cout * inter * kh * kw if flops_per_pixel is None else flops_per_pixel
    return PackedConv(wp, kh, kw, off[0], off[1], bk, bn, rows, k_eff, fpp)


def s2d_weight(w, pad):
    """Rewrite a stride-2 conv weight (Cout,Cin,k,k) with padding `pad` as the 2x2 stride-1 weight over the space-to-depth input
    with channel order (py*2+px)*Cin8 + ci: (k=4, pad=2) and (k=3, pad=1) run with off=(1,1); (k=3, pad=0) with off=(0,0)."""
    cout, cin, k, _ = w.shape
    cin8 = round_up(cin, 8)
    out = torch.zeros((cout, 4 * cin8, 2, 2), dtype=w.dtype, device=w.device)
    shift = 1 if (k == 3 and pad == 1) else 0
    assert (k, pad) in ((4, 2), (3, 1), (3, 0)), (k, pad)
    for ky in range(k):
        ty, py = divmod(ky + shift, 2)
        for kx in range(k):
            tx, px = divmod(kx + shift, 2)
            sub = py * 2 + px
            out[:, sub * cin8:sub * cin8 + cin, ty, tx] = w[:, :, ky, kx]
    return out


def pack_s2d(w, pad):
    """PackedConv of a stride-2 convolution expressed on the space-to-depth input (algorithmic FLOPs of the original)."""
    cout, cin, k, _ = w.shape
    return pack_weight(s2d_weight(w, pad), (1, 1), flops_per_pixel=2.0 * cin * cout * k * k)


# ----------------------------------------------------------------------------------------------- ops

def conv2d(inp, pw, out, act=ACT_NONE, scale=None, shift=None, res=None, out_layout=capi.NHWC, res_mode=capi.RES_ADD):
    assert inp.c == pw.cin, (inp.c, pw.cin)
    p = capi.ConvParams()
    p.inp = inp.ct()
    p.wpack = pw.w.data_ptr()
    p.kh, p.kw, p.off_y, p.off_x = pw.kh, pw.kw, pw.off_y, pw.off_x
    p.bk, p.bn, p.n_gemm = pw.bk, pw.bn, pw.n_gemm
    if isinstance(out, Act):
        p.out = out.ct()
    else:  # raw fp32 NCHW torch tensor
        n, c, h, w = out.shape
        p.out = capi.Tensor(out.data_ptr(), n, h, w, c, c, F32)
    p.out_layout = out_layout
    p.epi = capi.EPI_LINEAR
    p.act = act
    p.scale = _p(scale)
    p.shift = _p(shift)
    p.res = res.ct() if res is not None else _NULL
    p.res_mode = res_mode if res is not None else 0
    p.x0 = _NULL
    p.x1 = _NULL
    p.gamma_out = _NULL
    with _Timed("conv", pw.flops_per_pixel * p.out.n * p.out.h * p.out.w,
                label="%d->%d k%dx%d n%d %dx%d bk%d bn%d" % (inp.c, pw.n_gemm, pw.kh, pw.kw, p.out.n, p.out.h, p.out.w, pw.bk, pw.bn)):
        capi.check(_L(inp).hrv_conv2d_fwd(ctypes.byref(p), _stream()), "conv2d_fwd")
    return out


def conv2d_spade(actv, pw, out, x0, x0_shift, x1, mean, rstd, noise, noise_scale, shift, act, gamma_out=None):
    p = capi.ConvParams()
    p.inp = actv.ct()
    p.wpack = pw.w.data_ptr()
    p.kh, p.kw, p.off_y, p.off_x = pw.kh, pw.kw, pw.off_y, pw.off_x
    p.bk, p.bn, p.n_gemm = pw.bk, pw.bn, pw.n_gemm
    p.out = out.ct()
    p.out_layout = capi.NHWC
    p.epi = capi.EPI_SPADE
    p.act = act
    p.scale = None
    p.shift = _p(shift)
    p.res = _NULL
    p.res_mode = 0
    p.x0 = x0.ct()
    p.x1 = x1.ct() if x1 is not None else _NULL
    p.x0_shift = x0_shift
    p.mean, p.rstd, p.noise, p.noise_scale = _p(mean), _p(rstd), _p(noise), _p(noise_scale)
    p.gamma_out = gamma_out.ct() if gamma_out is not None else _NULL
    with _Timed("conv_spade", pw.flops_per_pixel * out.n * out.h * out.w,
                label="%d->%d k%dx%d n%d %dx%d bk%d bn%d" % (actv.c, pw.n_gemm, pw.kh, pw.kw, out.n, out.h, out.w, pw.bk, pw.bn)):
        capi.check(_L(actv).hrv_conv2d_fwd(ctypes.byref(p), _stream()), "conv2d_fwd(spade)")
    return out


_ws = {}


def _workspace(nbytes, device):
    key = (device, "ws")
    w = _ws.get(key)
    if w is None or w.numel() < nbytes:
        w = torch.empty(max(nbytes, 1 << 20), dtype=torch.uint8, device=device)
        _ws[key] = w
    return w


def instnorm_stats(x0, x0_shift, x1, h, w, noise, noise_scale, eps=1e-5):
    n = x0.n
    c = x0.c + (x1.c if x1 is not None else 0)
    mean = torch.empty((n, c), dtype=torch.float32, device=x0.buf.device)
    rstd = torch.empty_like(mean)
    t0 = x0.ct()
    t1 = x1.ct() if x1 is not None else _NULL
    L = _L(x0)
    ws = _workspace(int(L.hrv_instnorm_stats_workspace_bytes(ctypes.byref(t0), ctypes.byref(t1), h, w)), x0.buf.device)
    nbytes = n * h * w * (2.0 * c + (4.0 if noise is not None else 0.0))  # one bf16 read of every element (+ noise)
    with _Timed("instnorm_stats", nbytes, launches=2, label="c%d n%d %dx%d shift%d" % (c, n, h, w, x0_shift)):
        capi.check(L.hrv_instnorm_stats(ctypes.byref(t0), x0_shift, ctypes.byref(t1), h, w, _p(noise), _p(noise_scale),
                                                 eps, mean.data_ptr(), rstd.data_ptr(), ws.data_ptr(), ws.numel(), _stream()),
                   "instnorm_stats")
    return mean, rstd


def instnorm_stats2(x0, x0_shift, x1, h, w, noises, noise_scales, eps=1e-5):
    """Statistics of one or two SPADE norms sharing the input cat(up2^shift(x0), x1) (hrv_instnorm_stats2): `noises` / `noise_scales`
    are lists of 1 or 2 entries (a noise entry may be None).  Returns [(mean, rstd), ...] in the same order."""
    n = x0.n
    c = x0.c + (x1.c if x1 is not None else 0)
    k = len(noises)
    assert k in (1, 2) and len(noise_scales) == k
    dev = x0.buf.device
    outs = [(torch.empty((n, c), dtype=torch.float32, device=dev), torch.empty((n, c), dtype=torch.float32, device=dev)) for _ in range(k)]
    t0 = x0.ct()
    t1 = x1.ct() if x1 is not None else _NULL
    L = _L(x0)
    ws = _workspace(int(L.hrv_instnorm_stats2_workspace_bytes(ctypes.byref(t0), ctypes.byref(t1))), dev)
    src_bytes = 2.0 * n * (x0.h * x0.w * x0.c + (h * w * x1.c if x1 is not None else 0)) + 4.0 * n * h * w * sum(z is not None for z in noises)
    nz1, ns1, m1, r1 = (noises[1], noise_scales[1], outs[1][0], outs[1][1]) if k == 2 else (None, None, None, None)
    with _Timed("instnorm_stats", src_bytes, launches=2 + (1 if x1 is not None else 0), label="c%d n%d %dx%d shift%d norms%d" % (c, n, h, w, x0_shift, k)):
        capi.check(L.hrv_instnorm_stats2(ctypes.byref(t0), x0_shift, ctypes.byref(t1), h, w, _p(noises[0]), _p(noise_scales[0]), _p(nz1), _p(ns1),
                                              eps, outs[0][0].data_ptr(), outs[0][1].data_ptr(), _p(m1), _p(r1), ws.data_ptr(), ws.numel(), _stream()),
                   "instnorm_stats2")
    return outs


def instnorm_apply(x, mean, rstd, act, out=None):
    out = x if out is None else out
    tx, ty = x.ct(), out.ct()
    with _Timed("glue", 0.0, label="instnorm_apply"):
        capi.check(_L(x).hrv_instnorm_apply(ctypes.byref(tx), mean.data_ptr(), rstd.data_ptr(), act, ctypes.byref(ty), _stream()),
                   "instnorm_apply")
    return out


def space_to_depth(x, dtype=None):
    out = Act.empty(x.n, (x.h + 1) // 2, (x.w + 1) // 2, 4 * round_up(x.c, 8), dtype=dtype)
    tx, ty = x.ct(), out.ct()
    with _Timed("glue", 0.0, label="space_to_depth"):
        capi.check(_L(x).hrv_space_to_depth(ctypes.byref(tx), ctypes.byref(ty), _stream()), "space_to_depth")
    return out


def space_to_depth_bwd(d, n, h, w, c, pitch=None):
    """dx (n,h,w,c) of space_to_depth from the gradient d of its (n,ceil(h/2),ceil(w/2),4*c8) output."""
    dx = Act.empty(n, h, w, c, pitch=pitch)
    td, tx = d.ct(), dx.ct()
    with _Timed("glue", 0.0, label="space_to_depth_bwd"):
        capi.check(_L(d).hrv_space_to_depth_bwd(ctypes.byref(td), ctypes.byref(tx), _stream()), "space_to_depth_bwd")
    return dx


def maxpool2(x):
    y = Act.empty(x.n, x.h // 2, x.w // 2, x.c, pitch=x.pitch if x.c0 == 0 else None)
    tx, ty = x.ct(), y.ct()
    with _Timed("glue", 0.0, label="maxpool2_fwd"):
        capi.check(_L(x).hrv_maxpool2_fwd(ctypes.byref(tx), ctypes.byref(ty), _stream()), "maxpool2_fwd")
    return y


def maxpool2_bwd(x, dy, relu_gate=False):
    dx = Act.empty(x.n, x.h, x.w, x.c, pitch=x.pitch if x.c0 == 0 else None)
    tx, tdy, tdx = x.ct(), dy.ct(), dx.ct()
    with _Timed("glue", 0.0, label="maxpool2_bwd"):
        capi.check(_L(x).hrv_maxpool2_bwd(ctypes.byref(tx), ctypes.byref(tdy), ctypes.byref(tdx), 1 if relu_gate else 0, _stream()), "maxpool2_bwd")
    return dx


def avgpool3s2_bwd(dy, h, w):
    dx = Act.empty(dy.n, h, w, dy.c, pitch=dy.pitch if dy.c0 == 0 else None)
    tdy, tdx = dy.ct(), dx.ct()
    with _Timed("glue", 0.0, label="avgpool3s2_bwd"):
        capi.check(_L(dy).hrv_avgpool3s2_bwd(ctypes.byref(tdy), ctypes.byref(tdx), _stream()), "avgpool3s2_bwd")
    return dx


def im2col(x, kh, kw, pad, k_pad=None):
    """(n,h,w,c) -> (n,h,w,K) with K = round_up(kh*kw*c, 64|32|16): the tap-major column form of a tiny-Cin convolution."""
    k = kh * kw * x.c
    if k_pad is None:
        k_pad = round_up(k, 64) if k > 32 else (32 if k > 16 else 16)
    out = Act.empty(x.n, x.h, x.w, k_pad)
    tx, to = x.ct(), out.ct()
    with _Timed("glue", 0.0, label="im2col"):
        capi.check(_L(x).hrv_im2col(ctypes.byref(tx), ctypes.byref(to), kh, kw, pad, _stream()), "im2col")
    return out


def l1_sum(a, b):
    """sum |a - b| as a 1-element fp64 cuda tensor (per-block partials added in a fixed order: reproducible)."""
    out = torch.empty(1, dtype=torch.float64, device=a.buf.device)
    ta, tb = a.ct(), b.ct()
    L = _L(a)
    nws = int(L.hrv_l1_sum_workspace_bytes(ctypes.byref(ta)))
    ws = torch.empty(max(nws, 8), dtype=torch.uint8, device=a.buf.device)
    with _Timed("glue", 0.0, launches=2, label="l1_sum"):
        capi.check(L.hrv_l1_sum(ctypes.byref(ta), ctypes.byref(tb), out.data_ptr(), ws.data_ptr(), ws.numel(), _stream()), "l1_sum")
    return out


def l1_bwd(a, b, gscale, relu_gate=False, out=None):
    """da = sign(a - b) * gscale (gscale: 1-element fp32 cuda tensor); relu_gate: times (a > 0).  out: Act to write into."""
    da = out if out is not None else Act.empty(a.n, a.h, a.w, a.c, pitch=a.pitch if a.c0 == 0 else None)
    ta, tb, td = a.ct(), b.ct(), da.ct()
    with _Timed("glue", 0.0, label="l1_bwd"):
        capi.check(_L(a).hrv_l1_bwd(ctypes.byref(ta), ctypes.byref(tb), gscale.data_ptr(), ctypes.byref(td), 1 if relu_gate else 0, _stream()), "l1_bwd")
    return da


def grad_unscale_check(grads, inv_scale, found_inf, table=None):
    """In place over the fp32 cuda tensors `grads`: g *= inv_scale, found_inf = 1 where any g was inf / NaN (hrv_grad_unscale_check;
    inv_scale and found_inf are 1-element fp32 cuda tensors, found_inf is only ever set, never cleared).  The kernel reads a device
    table {data_ptr, numel} of the tensors: pass the `table` returned by the previous call to reuse it while no tensor has moved.  It is
    rebuilt (a host-to-device copy) otherwise, which a CUDA-graph capture cannot record.  Returns the table."""
    key = tuple((g.data_ptr(), g.numel()) for g in grads)
    if table is None or table[0] != key:
        for g in grads:
            assert g.is_cuda and g.dtype == torch.float32 and g.is_contiguous(), "grad_unscale_check needs contiguous fp32 cuda tensors"
        if torch.cuda.is_current_stream_capturing():
            raise RuntimeError("grad_unscale_check: the gradient tensors moved during CUDA-graph capture; keep them allocated across steps "
                               "(zero_grad(set_to_none=False)) and run one step before capturing")
        table = (key, torch.tensor(key, dtype=torch.int64).reshape(len(key), 2).to(inv_scale.device))
    with _Timed("glue", 0.0, label="grad_unscale_check"):
        capi.check(capi.lib().hrv_grad_unscale_check(table[1].data_ptr(), len(key), inv_scale.data_ptr(), found_inf.data_ptr(), _stream()),
                   "grad_unscale_check")
    return table


def parse_blur_argmax(seg, size, group_of=None, groups=0, want_idx=True, overlap_classes=None, cm=None, cm_channel=3,
                      composition="warp_grad"):
    """seg (n,c,h,w) fp32 cuda -> (idx (n,1,H,W) int64 | None, onehot (n,groups,H,W) fp32 | None[, overlap (n,1,H,W)]);
    hrv_parse_blur_argmax.  overlap_classes: class ids whose softmax (over the blurred scores) is summed into `overlap`.
    cm: (n,1,h,w) fp32 cuda, the cloth-mask composition of the scores first (channel cm_channel multiplied by cm for 'warp_grad',
    by (cm > 0.5) for 'detach'; 'no_composition' or cm=None: none), as seg_softmax_cat composes."""
    assert seg.is_cuda and seg.dtype == torch.float32
    if composition not in SEG_CAT_MODES:
        raise ValueError("composition must be one of %s, got %r" % ("/".join(SEG_CAT_MODES), composition))
    mode = 0 if cm is None else SEG_CAT_MODES[composition]
    seg = seg.contiguous()
    n, c, h, w = seg.shape
    if mode:
        if not (cm.is_cuda and cm.dtype == torch.float32 and tuple(cm.shape) == (n, 1, h, w)):
            raise ValueError("parse_blur_argmax: cm must be a CUDA float32 %s tensor, got %s %s" % ((n, 1, h, w), cm.dtype, tuple(cm.shape)))
        cm = cm.contiguous()
    else:
        cm = None
    H, W = size
    idx = torch.empty((n, 1, H, W), dtype=torch.int64, device=seg.device) if want_idx else None
    onehot = torch.empty((n, groups, H, W), dtype=torch.float32, device=seg.device) if group_of is not None else None
    garr = (ctypes.c_int32 * c)(*group_of) if group_of is not None else None
    overlap = torch.empty((n, 1, H, W), dtype=torch.float32, device=seg.device) if overlap_classes else None
    mask = 0
    for k in (overlap_classes or ()):
        mask |= 1 << int(k)
    with _Timed("glue", 0.0, label="parse_blur_argmax"):
        capi.check(capi.lib().hrv_parse_blur_argmax_cm(seg.data_ptr(), n, c, h, w, H, W, garr, groups, _p(idx), _p(onehot), mask, _p(overlap),
                                                    _p(cm), cm_channel, mode, _stream()), "parse_blur_argmax")
    return (idx, onehot, overlap) if overlap_classes else (idx, onehot)


def onehot_u8(labels, classes, lut=None, out=None):
    """(N,1,H,W) or (N,H,W) uint8 label map (cuda) -> (N,classes,H,W) fp32 one-hot planes (hrv_onehot_u8): the device half of the
    input feeding — the host ships one byte per pixel instead of `classes` floats (cp_dataset.py:150-172).  lut: a sequence of
    class ids indexed by label (at most 256; labels beyond it, and ids >= classes, set no channel), e.g. train_step.GROUP_OF_13 for
    the 13 -> 7 regrouping of train_generator.py:261-273; None: class = label."""
    assert labels.is_cuda and labels.dtype == torch.uint8
    labels = labels.contiguous()
    n, h, w = labels.shape[0], labels.shape[-2], labels.shape[-1]
    if out is None:
        out = torch.empty((n, classes, h, w), dtype=torch.float32, device=labels.device)
    assert out.is_contiguous() and out.shape == (n, classes, h, w)
    table = None
    if lut is not None:
        if len(lut) > 256 or any(not 0 <= int(v) < 256 for v in lut):
            raise ValueError("onehot_u8: lut must hold at most 256 class ids in [0, 255]")
        table = (ctypes.c_uint8 * 256)(*([int(v) for v in lut] + [255] * (256 - len(lut))))
    with _Timed("glue", 0.0, label="onehot_u8"):
        capi.check(capi.lib().hrv_onehot_u8_lut(labels.data_ptr(), n, classes, h, w, table, out.data_ptr(), _stream()), "onehot_u8")
    return out


def gaussian_blur(x, ksize=15, sigma=3.0):
    """tgm.image.GaussianBlur((ksize,ksize),(sigma,sigma)) on an fp32 NCHW cuda tensor (hrv_gaussian_blur)."""
    assert x.is_cuda and x.dtype == torch.float32 and x.dim() == 4
    x = x.contiguous()
    out = torch.empty_like(x)
    n, c, h, w = x.shape
    with _Timed("glue", 0.0, label="gaussian_blur"):
        capi.check(capi.lib().hrv_gaussian_blur(x.data_ptr(), n * c, h, w, ksize, float(sigma), out.data_ptr(), _stream()), "gaussian_blur")
    return out


def flow_warp_nchw(flow_lo, src, size, div_xy, want_grid=False, mask=None, overlap=None, composite=False):
    """The hi-res cloth warp of the glue (train_generator.py:232-238): flow_lo fp32 (N,hl,wl,2) is up-sampled bilinearly to `size`,
    divided by div_xy, added to the linspace base grid and used to grid_sample (bilinear, border) src fp32 (N,C,Hs,Ws).
    mask (N,1,Hs,Ws): the cloth mask is warped with the same taps (returned third), `overlap` (N,1,H,W) applies remove_overlap to it and
    composite=True blends the cloth over white with it (train_generator.py:239-244).
    Returns (warped (N,C,H,W) fp32, grid (N,H,W,2) | None[, warped mask (N,1,H,W)])."""
    assert flow_lo.is_cuda and src.is_cuda and flow_lo.dtype == torch.float32 and src.dtype == torch.float32
    flow_lo, src = flow_lo.contiguous(), src.contiguous()
    n, hl, wl, _ = flow_lo.shape
    _, c, hs, ws = src.shape
    H, W = size
    dev = src.device
    out = torch.empty((n, c, H, W), dtype=torch.float32, device=dev)
    grid = torch.empty((n, H, W, 2), dtype=torch.float32, device=dev) if want_grid else None
    mask_out = None
    if mask is not None:
        mask = mask.float().contiguous()
        assert mask.shape == (n, 1, hs, ws)
        mask_out = torch.empty((n, 1, H, W), dtype=torch.float32, device=dev)
    if overlap is not None:
        overlap = overlap.contiguous()
        assert overlap.shape == (n, 1, H, W) and overlap.dtype == torch.float32
    with _Timed("glue", 0.0, label="flow_warp_nchw"):
        capi.check(capi.lib().hrv_flow_warp_nchw(flow_lo.data_ptr(), n, hl, wl, linspace_table(W, dev).data_ptr(), linspace_table(H, dev).data_ptr(),
                                                 src.data_ptr(), c, hs, ws, out.data_ptr(), H, W, float(div_xy[0]), float(div_xy[1]), _p(grid),
                                                 _p(mask), _p(overlap), _p(mask_out), 1 if composite else 0, _stream()), "flow_warp_nchw")
    return (out, grid, mask_out) if mask is not None else (out, grid)


def flow_warp_nchw_bwd(flow_lo, src, size, div_xy, d_dst, mask=None, d_mask=None):
    """d flow_lo (N,hl,wl,2) fp32 of flow_warp_nchw (without overlap / composite) from the gradients of the warped cloth d_dst
    (N,C,H,W) and, optionally, of the warped mask d_mask (N,1,H,W): hrv_flow_warp_nchw_bwd, fixed summation order throughout."""
    flow_lo, src = flow_lo.contiguous(), src.contiguous()
    n, hl, wl, _ = flow_lo.shape
    _, c, hs, ws_ = src.shape
    H, W = size
    dev = src.device
    d_dst = d_dst.float().contiguous() if d_dst is not None else None
    if d_mask is not None:
        mask, d_mask = mask.float().contiguous(), d_mask.float().contiguous()
    dflo = torch.empty((n, hl, wl, 2), dtype=torch.float32, device=dev)
    L = capi.lib()
    nws = int(L.hrv_flow_warp_nchw_bwd_workspace_bytes(n, H, W, wl))
    ws = torch.empty(nws, dtype=torch.uint8, device=dev)
    with _Timed("glue", 0.0, launches=3, label="flow_warp_nchw_bwd"):
        capi.check(L.hrv_flow_warp_nchw_bwd(flow_lo.data_ptr(), n, hl, wl, linspace_table(W, dev).data_ptr(), linspace_table(H, dev).data_ptr(),
                                            src.data_ptr(), c, hs, ws_, _p(d_dst), H, W, float(div_xy[0]), float(div_xy[1]),
                                            _p(mask if d_mask is not None else None), _p(d_mask), dflo.data_ptr(), ws.data_ptr(), nws, _stream()),
                   "flow_warp_nchw_bwd")
    return dflo


def avgpool3s2(x):
    out = Act.empty(x.n, (x.h - 1) // 2 + 1, (x.w - 1) // 2 + 1, x.c, pitch=x.pitch if x.c0 == 0 else None)
    tx, ty = x.ct(), out.ct()
    with _Timed("glue", 0.0, label="avgpool3s2"):
        capi.check(_L(x).hrv_avgpool3s2(ctypes.byref(tx), ctypes.byref(ty), _stream()), "avgpool3s2")
    return out


def bilinear_up2_add(a, b, out):
    ta, to = a.ct(), out.ct()
    tb = b.ct() if b is not None else _NULL
    with _Timed("glue", 0.0, label="bilinear_up2_add"):
        capi.check(_L(a).hrv_bilinear_up2_add(ctypes.byref(ta), ctypes.byref(tb), ctypes.byref(to), _stream()), "bilinear_up2_add")
    return out


_lin = {}


def linspace_table(n, device):
    """torch.linspace(-1, 1, n) — the reference's base-grid values (networks.py:162-163), built on the CPU exactly as
    the reference does, cached on the device."""
    key = (n, str(device))
    if key not in _lin:
        _lin[key] = torch.linspace(-1.0, 1.0, n).to(device)
    return _lin[key]


def flow_warp(flow_lo, src, dst, want_flow_up=True, want_idx=False):
    """flow_lo: fp32 (N,h,w,2) cuda contiguous. Returns (flow_up fp32 (N,2h,2w,2) | None, idx int32 | None)."""
    n, hl, wl, _ = flow_lo.shape
    H, W = 2 * hl, 2 * wl
    assert dst.h == H and dst.w == W
    dev = flow_lo.device
    flow_up = torch.empty((n, H, W, 2), dtype=torch.float32, device=dev) if want_flow_up else None
    idx = torch.empty((n, H, W, 2), dtype=torch.int32, device=dev) if want_idx else None
    ts, td = src.ct(), dst.ct()
    with _Timed("glue", 0.0, label="flow_warp"):
        capi.check(_L(src, dst).hrv_flow_warp(flow_lo.data_ptr(), linspace_table(W, dev).data_ptr(), linspace_table(H, dev).data_ptr(),
                                            ctypes.byref(ts), ctypes.byref(td), _p(flow_up), _p(idx), _stream()), "flow_warp")
    return flow_up, idx


def norm_bwd(dh, h, gamma, x0, x0_shift, x1, noise, noise_scale, mean, rstd, act, want_dgb, chan_scale=None, batch_stats=False,
             all_reduce=None):
    """Fused backward of the SPADE modulation + InstanceNorm (gamma given) or of InstanceNorm + activation (gamma None).
    all_reduce (with batch_stats): synchronised BatchNorm — the two means run over the pixels of every rank: the local sums go through
    one wire buffer that all_reduce sums over the ranks in place.  sum_dgamma / sum_dbeta stay local.
    Returns (dgb Act | None, dx0 Act, dx1 Act | None, d_noise_scale fp32 [C] | None, sum_dgamma fp32 [C], sum_dbeta fp32 [C])."""
    n, H, W = dh.n, dh.h, dh.w
    c0 = x0.c
    c1 = x1.c if x1 is not None else 0
    C = c0 + c1
    dev = dh.buf.device
    dxn = Act.empty(n, H, W, C)
    dgb = Act.empty(n, H, W, 2 * C) if want_dgb else None
    sums = torch.empty((n, C, 4), dtype=torch.float64, device=dev)
    tdh, tx0, tdxn = dh.ct(), x0.ct(), dxn.ct()
    th = h.ct() if h is not None else _NULL
    tg = gamma.ct() if gamma is not None else _NULL
    tx1 = x1.ct() if x1 is not None else _NULL
    tdgb = dgb.ct() if dgb is not None else _NULL
    L = _L(dh)
    nws = int(L.hrv_norm_bwd_reduce_workspace_bytes(ctypes.byref(tx0), ctypes.byref(tx1), H, W))
    if noise_scale is not None:
        nws = max(nws, int(L.hrv_norm_bwd_apply_workspace_bytes(ctypes.byref(tx0))),
                  int(L.hrv_norm_bwd_apply_workspace_bytes(ctypes.byref(tx1))) if x1 is not None else 0)
    ws = torch.empty(nws, dtype=torch.uint8, device=dev)  # per-block slabs, added in a fixed order (reproducible sums)
    with _Timed("norm_bwd", n * H * W * C * 2.0 * (4 + (1 if gamma is not None else 0) + (2 if want_dgb else 0)), launches=2):
        capi.check(L.hrv_norm_bwd_reduce(ctypes.byref(tdh), ctypes.byref(th), ctypes.byref(tg), ctypes.byref(tx0), x0_shift,
                                         ctypes.byref(tx1), H, W, _p(noise), _p(noise_scale), mean.data_ptr(), rstd.data_ptr(),
                                         _p(chan_scale), act, ctypes.byref(tdgb), ctypes.byref(tdxn), sums.data_ptr(), ws.data_ptr(), nws,
                                         _stream()), "norm_bwd_reduce")
    if batch_stats and all_reduce is not None:
        wire = syncbn_combine(sums, 4, n * H * W)
        all_reduce(wire)
        m1 = torch.empty((n, C), dtype=torch.float32, device=dev)
        m2 = torch.empty_like(m1)
        with _Timed("syncbn", C * 16.0, label="bwd_finalize c%d" % C):
            capi.check(capi.lib().hrv_syncbn_bwd_finalize(wire.data_ptr(), n, C, m1.data_ptr(), m2.data_ptr(), _stream()), "syncbn_bwd_finalize")
    elif batch_stats:  # BatchNorm: the two means run over (N,H,W)
        tot = sums.sum(0, keepdim=True) / float(n * H * W)
        m1 = tot[:, :, 0].expand(n, C).float().contiguous()
        m2 = tot[:, :, 1].expand(n, C).float().contiguous()
    else:
        inv = 1.0 / float(H * W)
        m1 = (sums[:, :, 0] * inv).float().contiguous()
        m2 = (sums[:, :, 1] * inv).float().contiguous()
    dns = torch.empty(C, dtype=torch.float64, device=dev) if noise_scale is not None else None
    dx0 = Act.empty(n, x0.h, x0.w, c0)
    tdx0 = dx0.ct()
    with _Timed("norm_bwd", n * H * W * c0 * 2.0 * 2, launches=2 if dns is not None else 1):
        capi.check(L.hrv_norm_bwd_apply(ctypes.byref(tdxn), ctypes.byref(tx0), x0_shift, 0, C, H, W, _p(noise), _p(noise_scale),
                                        mean.data_ptr(), rstd.data_ptr(), m1.data_ptr(), m2.data_ptr(), ctypes.byref(tdx0),
                                        _p(dns), ws.data_ptr(), nws, _stream()), "norm_bwd_apply(x0)")
    dx1 = None
    if x1 is not None:
        dx1 = Act.empty(n, H, W, c1)
        tdx1 = dx1.ct()
        with _Timed("norm_bwd", n * H * W * c1 * 2.0 * 3, launches=2 if dns is not None else 1):
            capi.check(L.hrv_norm_bwd_apply(ctypes.byref(tdxn), ctypes.byref(tx1), 0, c0, C, H, W, _p(noise), _p(noise_scale),
                                            mean.data_ptr(), rstd.data_ptr(), m1.data_ptr(), m2.data_ptr(), ctypes.byref(tdx1),
                                            _p(dns), ws.data_ptr(), nws, _stream()), "norm_bwd_apply(x1)")
    return dgb, dx0, dx1, (dns.float() if dns is not None else None), sums[:, :, 2].sum(0).float(), sums[:, :, 3].sum(0).float()


def act_bwd_bias(dy, y, act, want_dv=True, want_bias=True):
    """(dv Act | dy itself when act is NONE, bias_grad fp32 [c] | None) for an epilogue act(conv + b)."""
    c8 = round_up(dy.c, 8)
    dv = Act.empty(dy.n, dy.h, dy.w, dy.c, pitch=dy.pitch) if (want_dv and act != ACT_NONE) else None
    bsum = torch.empty(c8, dtype=torch.float64, device=dy.buf.device) if want_bias else None
    if dv is None and bsum is None:
        return dy, None
    tdy = dy.ct()
    ty = y.ct() if (y is not None and act != ACT_NONE) else _NULL
    tdv = dv.ct() if dv is not None else _NULL
    L = _L(dy)
    nws = int(L.hrv_act_bwd_bias_ordered_workspace_bytes(ctypes.byref(tdy))) if bsum is not None else 0
    ws = torch.empty(nws, dtype=torch.uint8, device=dy.buf.device) if nws else None  # per-block slabs, added in a fixed order
    with _Timed("act_bwd", dy.n * dy.h * dy.w * dy.c * 2.0 * (3 if dv is not None else 1), launches=2 if bsum is not None else 1):
        capi.check(L.hrv_act_bwd_bias_ordered(ctypes.byref(tdy), ctypes.byref(ty), act, ctypes.byref(tdv), _p(bsum), _p(ws), nws, _stream()),
                   "act_bwd_bias_ordered")
    return (dv if dv is not None else dy), (bsum[:dy.c].float() if bsum is not None else None)


def conv2d_wgrad(x, dy, kh, kw, pad):
    """dW (cout,cin,kh,kw) fp32 of a stride-1 convolution, on wgmma (hrv_conv2d_wgrad)."""
    dw = torch.empty((dy.c, x.c, kh, kw), dtype=torch.float32, device=x.buf.device)
    tx, tdy = x.ct(), dy.ct()
    L = _L(x)
    nws = int(L.hrv_conv2d_wgrad_workspace_bytes(ctypes.byref(tx), ctypes.byref(tdy), kh, kw))
    ws = torch.empty(nws, dtype=torch.uint8, device=x.buf.device) if nws else None  # split-K slabs, summed in a fixed order (deterministic)
    with _Timed("wgrad", 2.0 * x.c * dy.c * kh * kw * dy.n * dy.h * dy.w, launches=2 if nws else 1,
                label="%d->%d k%dx%d n%d %dx%d" % (x.c, dy.c, kh, kw, dy.n, dy.h, dy.w)):
        capi.check(L.hrv_conv2d_wgrad(ctypes.byref(tx), ctypes.byref(tdy), kh, kw, pad, dw.data_ptr(), _p(ws), nws, _stream()), "conv2d_wgrad")
    return dw


def batchnorm_stats(x, eps=1e-5):
    """Train-mode BatchNorm2d statistics over (N,H,W) from ONE pass of the statistics kernel (per-image fp64 partial sums combined
    here on [N][C] scalars) — the "single-kernel reduce" standing in for SyncBatchNorm.  Returns (mean[C], biased var[C]) fp32."""
    n, c = x.n, x.c
    mean_nc = torch.empty((n, c), dtype=torch.float32, device=x.buf.device)
    rstd_nc = torch.empty_like(mean_nc)
    t0 = x.ct()
    L = _L(x)
    ws = _workspace(int(L.hrv_instnorm_stats_workspace_bytes(ctypes.byref(t0), ctypes.byref(_NULL), x.h, x.w)), x.buf.device)
    with _Timed("instnorm_stats", n * x.h * x.w * 2.0 * c, launches=2, label="bn c%d n%d %dx%d" % (c, n, x.h, x.w)):
        capi.check(L.hrv_instnorm_stats(ctypes.byref(t0), 0, ctypes.byref(_NULL), x.h, x.w, None, None, eps, mean_nc.data_ptr(),
                                                 rstd_nc.data_ptr(), ws.data_ptr(), ws.numel(), _stream()), "batchnorm_stats")
    sums = ws[: n * c * 16].view(torch.float64).view(n, c, 2).sum(0)  # raw sum / sum of squares left in the workspace
    cnt = float(n * x.h * x.w)
    mean = sums[:, 0] / cnt
    var = (sums[:, 1] / cnt - mean * mean).clamp_min(0.0)
    return mean.float(), var.float()


def syncbn_combine(sums, stride, count):
    """The fp64 wire buffer [2C+1] of one synchronised BatchNorm layer: per-channel sums of columns 0 and 1 of `sums` ([N][C][stride]
    fp64, contiguous) over the local images, in image order, followed by the element count `count` (hrv_syncbn_combine)."""
    assert sums.dtype == torch.float64 and sums.is_contiguous() and sums.shape[2] == stride
    n, c = sums.shape[0], sums.shape[1]
    wire = torch.empty(2 * c + 1, dtype=torch.float64, device=sums.device)
    with _Timed("syncbn", n * c * 16.0, label="combine c%d n%d" % (c, n)):
        capi.check(capi.lib().hrv_syncbn_combine(sums.data_ptr(), n, c, stride, float(count), wire.data_ptr(), _stream()), "syncbn_combine")
    return wire


def batchnorm_stats_sync(x, eps, all_reduce, running_mean=None, running_var=None, momentum=0.1):
    """Train-mode BatchNorm2d statistics over the (N,H,W) of every rank: the statistics kernel on the local shard, its per-image sums
    combined into one wire buffer, all_reduce(wire) (in place, sum over the ranks), then hrv_syncbn_fwd_finalize.  Updates
    running_mean / running_var (fp32 [c_run], c_run <= x.c; optional) in place.  Returns (mean [N][C], rstd [N][C]) fp32, the tables
    of norm_apply_affine."""
    n, c = x.n, x.c
    mean_nc = torch.empty((n, c), dtype=torch.float32, device=x.buf.device)
    rstd_nc = torch.empty_like(mean_nc)
    t0 = x.ct()
    L = _L(x)
    ws = _workspace(int(L.hrv_instnorm_stats_workspace_bytes(ctypes.byref(t0), ctypes.byref(_NULL), x.h, x.w)), x.buf.device)
    with _Timed("instnorm_stats", n * x.h * x.w * 2.0 * c, launches=2, label="syncbn c%d n%d %dx%d" % (c, n, x.h, x.w)):
        capi.check(L.hrv_instnorm_stats(ctypes.byref(t0), 0, ctypes.byref(_NULL), x.h, x.w, None, None, eps, mean_nc.data_ptr(),
                                        rstd_nc.data_ptr(), ws.data_ptr(), ws.numel(), _stream()), "batchnorm_stats_sync")
    wire = syncbn_combine(ws[: n * c * 16].view(torch.float64).view(n, c, 2), 2, n * x.h * x.w)
    all_reduce(wire)
    c_run = 0
    if running_mean is not None:
        assert running_mean.dtype == torch.float32 and running_var.dtype == torch.float32 and running_mean.is_contiguous()
        c_run = running_mean.numel()
    with _Timed("syncbn", c * 16.0, label="fwd_finalize c%d" % c):
        capi.check(capi.lib().hrv_syncbn_fwd_finalize(wire.data_ptr(), n, c, c_run, eps, float(momentum), mean_nc.data_ptr(), rstd_nc.data_ptr(),
                                                      _p(running_mean), _p(running_var), _stream()), "syncbn_fwd_finalize")
    return mean_nc, rstd_nc


def norm_apply_affine(x, mean_nc, rstd_nc, gamma, beta, res, act, out=None):
    out = Act.empty(x.n, x.h, x.w, x.c) if out is None else out
    tx, ty = x.ct(), out.ct()
    tr = res.ct() if res is not None else _NULL
    with _Timed("norm_apply", x.n * x.h * x.w * x.c * 2.0 * (3 if res is not None else 2)):
        capi.check(_L(x).hrv_norm_apply_affine(ctypes.byref(tx), mean_nc.data_ptr(), rstd_nc.data_ptr(), _p(gamma), _p(beta),
                                                    ctypes.byref(tr), act, ctypes.byref(ty), _stream()), "norm_apply_affine")
    return out


def bilinear_up2_bwd(dout):
    da = Act.empty(dout.n, dout.h // 2, dout.w // 2, dout.c)
    td, ta = dout.ct(), da.ct()
    with _Timed("up2_bwd", dout.n * dout.h * dout.w * dout.c * 2.0 * 1.25):
        capi.check(_L(dout).hrv_bilinear_up2_bwd(ctypes.byref(td), ctypes.byref(ta), _stream()), "bilinear_up2_bwd")
    return da


def flow_warp_bwd(flow_lo, src, ddst, dflow_up_in, want_dsrc=True):
    """Returns (dsrc bf16 Act | None, dflow_lo fp32 (N,h,w,2)) from the ordered (bit-reproducible) backward."""
    n, hl, wl, _ = flow_lo.shape
    H, W = 2 * hl, 2 * wl
    dev = flow_lo.device
    c8 = round_up(src.c, 8)
    dsrc32 = torch.empty((n, src.h, src.w, c8), dtype=torch.float32, device=dev) if want_dsrc else None
    dfu = dflow_up_in.float().contiguous().clone() if dflow_up_in is not None else torch.zeros((n, H, W, 2), dtype=torch.float32, device=dev)
    dflo = torch.empty((n, hl, wl, 2), dtype=torch.float32, device=dev)
    ts, td = src.ct(), ddst.ct()
    L = _L(src, ddst)
    nws = int(L.hrv_flow_warp_bwd_ordered_workspace_bytes(ctypes.byref(ts), ctypes.byref(td)))
    ws = torch.empty(nws, dtype=torch.uint8, device=dev)
    with _Timed("flow_warp_bwd", n * H * W * src.c * 2.0 * 3, launches=6 if want_dsrc else 3):
        capi.check(L.hrv_flow_warp_bwd_ordered(flow_lo.data_ptr(), linspace_table(W, dev).data_ptr(), linspace_table(H, dev).data_ptr(),
                                               ctypes.byref(ts), ctypes.byref(td), _p(dsrc32), dfu.data_ptr(), dflo.data_ptr(), ws.data_ptr(), nws,
                                               _stream()), "flow_warp_bwd_ordered")
    dsrc = Act(dsrc32.to(src.buf.dtype)) if want_dsrc else None
    return dsrc, dflo


# ----------------------------------------------------------------------------------------------- evaluation metrics (fp32 / fp64)

LPIPS_K = 363  # conv1's im2col depth (11*11 taps x 3 channels)


def lpips_input(x, shift, scale):
    """LPIPS ScalingLayer + the operand of AlexNet's conv1 (11x11, stride 4, pad 2) as a 1x1 GEMM: x fp32 NCHW (n,3,h,w) cuda ->
    fp32 NHWC Act (n, (h-7)//4+1, (w-7)//4+1, 363) (hrv_lpips_input).  shift, scale: fp32 [3] cuda."""
    assert x.is_cuda and x.dtype == torch.float32 and x.dim() == 4 and x.shape[1] == 3
    x = x.contiguous()
    n, _, h, w = x.shape
    out = Act.empty(n, (h - 7) // 4 + 1, (w - 7) // 4 + 1, LPIPS_K, dtype=torch.float32)
    t = out.ct()
    with _Timed("glue", 0.0, label="lpips_input"):
        capi.check(capi.lib().hrv_lpips_input(x.data_ptr(), n, h, w, shift.data_ptr(), scale.data_ptr(), ctypes.byref(t), _stream()), "lpips_input")
    return out


def maxpool3s2(x, out=None):
    """nn.MaxPool2d(3, 2) on an fp32 NHWC Act (hrv_maxpool3s2): bit-exact.  out: the destination Act (e.g. a channel slice)."""
    y = Act.empty(x.n, (x.h - 3) // 2 + 1, (x.w - 3) // 2 + 1, x.c, dtype=torch.float32) if out is None else out
    tx, ty = x.ct(), y.ct()
    with _Timed("glue", 0.0, label="maxpool3s2"):
        capi.check(capi.lib().hrv_maxpool3s2(ctypes.byref(tx), ctypes.byref(ty), _stream()), "maxpool3s2")
    return y


def lpips_dist(feat, lin_w):
    """One LPIPS layer (hrv_lpips_dist): feat an fp32 Act of 2N images (image i against image i + N), lin_w fp32 [C] cuda.  Returns
    the per-pair spatial mean of sum_c w_c (f0_c - f1_c)^2 over unit-normalised features, fp32 [N]."""
    out = torch.empty(feat.n // 2, dtype=torch.float32, device=feat.buf.device)
    t = feat.ct()
    with _Timed("glue", 0.0, label="lpips_dist"):
        capi.check(capi.lib().hrv_lpips_dist(ctypes.byref(t), lin_w.data_ptr(), out.data_ptr(), _stream()), "lpips_dist")
    return out


def ssim(im1, im2, data_range=255.0):
    """Mean Gaussian SSIM per image (hrv_ssim; skimage's structural_similarity with gaussian_weights=True, use_sample_covariance=False)
    of two (N,H,W) cuda tensors, uint8 or fp32.  Returns fp64 [N]."""
    if im1.shape != im2.shape or im1.dtype != im2.dtype or im1.dim() != 3:
        raise ValueError("ssim: im1 and im2 must be (N,H,W) of one shape and dtype; got %s %s and %s %s"
                         % (tuple(im1.shape), im1.dtype, tuple(im2.shape), im2.dtype))
    if im1.dtype not in (torch.uint8, torch.float32):
        raise TypeError("ssim: images must be uint8 or float32, got %s" % im1.dtype)
    n, h, w = im1.shape
    if h < 11 or w < 11:
        raise ValueError("win_size exceeds image extent: the 11x11 Gaussian window needs images of at least 11x11, got %dx%d" % (h, w))
    im1, im2 = im1.contiguous(), im2.contiguous()
    out = torch.empty(n, dtype=torch.float64, device=im1.device)
    L = capi.lib()
    nws = int(L.hrv_ssim_workspace_bytes(n, h, w))
    ws = torch.empty(nws, dtype=torch.uint8, device=im1.device)
    dt = capi.SSIM_U8 if im1.dtype == torch.uint8 else capi.SSIM_F32
    with _Timed("glue", 0.0, launches=2, label="ssim"):
        capi.check(L.hrv_ssim(im1.data_ptr(), im2.data_ptr(), dt, n, h, w, float(data_range), out.data_ptr(), ws.data_ptr(), nws, _stream()), "ssim")
    return out


def resize_bilinear_nhwc(x, size, unit_range=False, pitch=None):
    """F.interpolate(x, size, mode='bilinear', align_corners=False) of fp32 NCHW x (cuda), bit-identical, as an fp32 NHWC Act
    (hrv_resize_bilinear_nhwc); unit_range=True maps x to 2x - 1 first.  The pad channels up to the next multiple of 8 are zeros."""
    assert x.is_cuda and x.dtype == torch.float32 and x.dim() == 4
    x = x.contiguous()
    n, c, h, w = x.shape
    out = Act.empty(n, size[0], size[1], c, dtype=torch.float32, device=x.device, pitch=pitch)
    t = out.ct()
    with _Timed("glue", 0.0, label="resize_bilinear_nhwc"):
        capi.check(capi.lib().hrv_resize_bilinear_nhwc(x.data_ptr(), n, c, h, w, int(bool(unit_range)), ctypes.byref(t), _stream()),
                   "resize_bilinear_nhwc")
    return out


def resize_bilinear_fid(x, size=(299, 299), pitch=None):
    """pytorch-fid's Inception input as an fp32 NHWC Act (n, size, 3) (hrv_resize_bilinear_fid): F.interpolate(v, size, 'bilinear',
    align_corners=False) and then 2v - 1, bit-identical.  x: fp32 NCHW (n,c,h,w) cuda in [0, 1], or uint8 NHWC (n,h,w,c) cuda as PIL
    decodes it (v = u8 / 255, as TF.to_tensor).  The pad channels up to the next multiple of 8 are zeros."""
    assert x.is_cuda and x.dim() == 4 and x.dtype in (torch.float32, torch.uint8)
    x = x.contiguous()
    if x.dtype == torch.uint8:
        (n, h, w, c), src = x.shape, capi.FID_SRC_U8_NHWC
    else:
        (n, c, h, w), src = x.shape, capi.FID_SRC_F32_NCHW
    out = Act.empty(n, size[0], size[1], c, dtype=torch.float32, device=x.device, pitch=pitch)
    t = out.ct()
    with _Timed("glue", 0.0, label="resize_bilinear_fid"):
        capi.check(capi.lib().hrv_resize_bilinear_fid(x.data_ptr(), src, n, c, h, w, ctypes.byref(t), _stream()), "resize_bilinear_fid")
    return out


def pool3x3s1(x, mode, out=None):
    """A 3x3, stride-1, padding-1 pool of an fp32 NHWC Act (hrv_pool3x3s1), bit-exact: mode 'avg' is F.avg_pool2d(count_include_pad=False),
    'max' is F.max_pool2d.  out: the destination Act of x's extent (e.g. a channel slice)."""
    m = {"avg": capi.POOL3X3_AVG_EXCL_PAD, "max": capi.POOL3X3_MAX}[mode]
    y = Act.empty(x.n, x.h, x.w, x.c, dtype=torch.float32, device=x.buf.device) if out is None else out
    tx, ty = x.ct(), y.ct()
    with _Timed("glue", 0.0, label="pool3x3s1 " + mode):
        capi.check(capi.lib().hrv_pool3x3s1(ctypes.byref(tx), m, ctypes.byref(ty), _stream()), "pool3x3s1")
    return y


def global_avgpool(x, out=None):
    """The mean over the pixels of an fp32 Act (hrv_global_avgpool: fp64 sum in a fixed order, one rounding) as an (n,1,1,c) fp32 Act."""
    y = Act.empty(x.n, 1, 1, x.c, dtype=torch.float32, device=x.buf.device) if out is None else out
    tx, ty = x.ct(), y.ct()
    with _Timed("glue", 0.0, label="global_avgpool"):
        capi.check(capi.lib().hrv_global_avgpool(ctypes.byref(tx), ctypes.byref(ty), _stream()), "global_avgpool")
    return y


def _gram_operand(t, k_major):
    """(strides (row, k), rows, k) of a 2-D fp32 / fp64 tensor read as a (rows, K) operand; k_major: t is (K, rows)."""
    assert t.is_cuda and t.dim() == 2 and t.dtype in (torch.float32, torch.float64)
    s0, s1 = t.stride()
    return ((s1, s0), t.shape[1], t.shape[0]) if k_major else ((s0, s1), t.shape[0], t.shape[1])


def gram_f64(a, b, out=None, k_major=False, accumulate=False):
    """a @ b.T in fp64 (hrv_gram_f64: every sum in a fixed order) of a (M,K) and b (N,K) cuda tensors, fp32 or fp64 (one dtype);
    k_major=True reads both as (K,M) / (K,N), i.e. computes a.T @ b.  out: fp64 (M,N) with unit column stride, overwritten or, with
    accumulate=True, added to."""
    assert a.dtype == b.dtype
    (sam, sak), m, k = _gram_operand(a, k_major)
    (sbn, sbk), n, kb = _gram_operand(b, k_major)
    assert k == kb, (tuple(a.shape), tuple(b.shape), k_major)
    if out is None:
        assert not accumulate
        out = torch.empty((m, n), dtype=torch.float64, device=a.device)
    assert out.dtype == torch.float64 and out.shape == (m, n) and out.stride(1) == 1
    L = capi.lib()
    nws = int(L.hrv_gram_f64_workspace_bytes(m, n, k))
    ws = torch.empty(max(nws, 8), dtype=torch.uint8, device=a.device)  # split-K slabs, added in a fixed order
    dt = capi.GRAM_F32 if a.dtype == torch.float32 else capi.GRAM_F64
    with _Timed("gram", 2.0 * m * n * k, launches=2 if nws else 1, label="gram %dx%dx%d" % (m, n, k)):
        capi.check(L.hrv_gram_f64(a.data_ptr(), sam, sak, b.data_ptr(), sbn, sbk, dt, m, n, k, out.data_ptr(), out.stride(0), int(bool(accumulate)),
                                  ws.data_ptr(), nws, _stream()), "gram_f64")
    return out


def kid_sums(gxx, gyy, gxy, ix, iy, gamma):
    """fp64 [S,3] per-subset sums of KID's polynomial kernel (g*gamma + 1)^3 over the Gram matrices (hrv_kid_sums): off-diagonal
    X-X, off-diagonal Y-Y and all X-Y pairs of subset s, whose feature indices are the rows ix[s], iy[s] (int32 (S, m) cuda)."""
    na, nb = gxx.shape[0], gyy.shape[0]
    assert gxx.shape == (na, na) and gyy.shape == (nb, nb) and gxy.shape == (na, nb)
    assert all(t.is_contiguous() and t.dtype == torch.float64 for t in (gxx, gyy, gxy))
    assert ix.dtype == torch.int32 and iy.dtype == torch.int32 and ix.shape == iy.shape and ix.is_contiguous() and iy.is_contiguous()
    s, m = ix.shape
    out = torch.empty((s, 3), dtype=torch.float64, device=gxx.device)
    with _Timed("glue", 0.0, label="kid_sums"):
        capi.check(capi.lib().hrv_kid_sums(gxx.data_ptr(), gyy.data_ptr(), gxy.data_ptr(), na, nb, ix.data_ptr(), iy.data_ptr(), s, m, float(gamma),
                                           out.data_ptr(), _stream()), "kid_sums")
    return out
