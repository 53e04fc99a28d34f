"""Written set and values of the staged convolution epilogue.  Every output lives inside a larger buffer filled with a NaN sentinel:
the kernel must write exactly the elements of its view (plus the pad channels up to the next multiple of 8 where a storage-type pitch
has room) and leave every other element bit-for-bit untouched.  Covers SPADE out / gamma_out in channel slices, bf16 pad channels with a
residual, partial pixel tiles, tiles spanning several images, fp32 NHWC at pitch 1 and 2, and fp32 NCHW, on bf16 and fp32 storage."""
import pytest
import torch
import torch.nn.functional as F

from hrviton_b200 import capi, ops, synth
from hrviton_b200.ops import Act

pytestmark = pytest.mark.gpu
DEV = "cuda"
SENTINEL = {torch.bfloat16: (torch.int16, 0x7FC1), torch.float16: (torch.int16, 0x7E01), torch.float32: (torch.int32, 0x7FC00123)}

# (n, h, w): the tile is TN x TH x TW = 128 pixels.  33 x 63 -> 2 x 64 tiles, the last row and column of tiles partial; 20 x 12 ->
# 4 x 4 x 8-image tiles, so one tile spans the image and seven past the batch; 4 x 4 with 3 images -> one tile over all of them.
SHAPES = [(1, 33, 63), (1, 20, 12), (3, 4, 4)]


@pytest.fixture(params=["bf16", "fp32"])
def storage(request):
    prev = ops.get_precision()
    ops.set_precision(request.param)
    yield ops.STORAGE[0]
    ops.set_precision(prev)


def sentinel_buf(shape, dtype):
    idt, bits = SENTINEL[dtype]
    b = torch.empty(shape, dtype=dtype, device=DEV)
    b.view(idt).fill_(bits)
    return b


def untouched(buf):
    idt, bits = SENTINEL[buf.dtype]
    return (buf.view(idt) == bits).cpu()


def rounded(t, dtype):
    return t.to(dtype).double()


def rel_err(got, ref):
    got, ref = got.double().cpu(), ref.double().cpu()
    return float((got - ref).abs().max() / (ref.abs().max() + 1e-6))


def tol(dtype):
    return 2e-3 if dtype == torch.float32 else 1.5e-2


@pytest.mark.parametrize("n,h,w", SHAPES)
@pytest.mark.parametrize("with_x1", [False, True])
def test_spade_out_and_gamma_in_slices(storage, n, h, w, with_x1):
    """SPADE out and gamma_out as channel slices of wider buffers; C = 80 leaves the second 128-column N tile 32 columns wide."""
    seed = 11
    cx0, cx1 = (64, 16) if with_x1 else (80, 0)
    C, cin = cx0 + cx1, 48
    shift = 1 if (h % 2 == 0 and w % 2 == 0) else 0
    actv = rounded(synth.normalish((n, cin, h, w), seed, "a"), storage)
    wg = rounded(synth.normalish((C, cin, 3, 3), seed, "wg", 0.05), storage)
    wb = rounded(synth.normalish((C, cin, 3, 3), seed, "wb", 0.05), storage)
    bg, bb = synth.normalish((C,), seed, "bg", 0.1), synth.normalish((C,), seed, "bb", 0.1)
    x0 = rounded(synth.normalish((n, cx0, h >> shift, w >> shift), seed, "x0"), storage)
    x1 = rounded(synth.normalish((n, cx1, h, w), seed, "x1"), storage) if cx1 else None
    noise = synth.spade_noise(n, h, w, seed, 0)
    ns = synth.normalish((C,), seed, "ns", 0.1)
    mean = synth.normalish((n, C), seed, "m", 0.2)
    rstd = synth.uniform((n, C), seed, "r", 0.5, 1.5)

    out_big = sentinel_buf((n + 1, h, w, C + 24), storage)
    gam_big = sentinel_buf((n + 1, h, w, C + 16), torch.bfloat16) if storage != torch.float32 else None
    out = Act(out_big[:n], c=C, c0=16)
    gam = Act(gam_big[:n], c=C, c0=8) if gam_big is not None else None
    pw = ops.pack_weight(wg.float().to(DEV), (1, 1), interleave=wb.float().to(DEV))
    sh = torch.stack([bg, bb], 1).reshape(-1).to(DEV)
    ops.conv2d_spade(ops.from_nchw(actv.float().to(DEV)), pw, out, ops.from_nchw(x0.float().to(DEV)), shift,
                     ops.from_nchw(x1.float().to(DEV)) if x1 is not None else None, mean.to(DEV), rstd.to(DEV), noise.to(DEV),
                     ns.to(DEV), sh, ops.ACT_LRELU, gamma_out=gam)
    torch.cuda.synchronize()

    xs = F.interpolate(x0, scale_factor=2, mode="nearest") if shift else x0
    if x1 is not None:
        xs = torch.cat([xs, x1], 1)
    xn = (xs + noise.double()[:, None] * ns.double()[None, :, None, None] - mean.double()[:, :, None, None]) * rstd.double()[:, :, None, None]
    gamma = F.conv2d(actv, wg, bg.double(), padding=1)
    beta = F.conv2d(actv, wb, bb.double(), padding=1)
    ref = F.leaky_relu(xn * (1 + gamma) + beta, 0.2)

    keep = torch.ones(out_big.shape, dtype=torch.bool)
    keep[:n, :, :, 16:16 + C] = False
    assert torch.equal(untouched(out_big), keep)
    assert rel_err(out_big[:n, :, :, 16:16 + C].permute(0, 3, 1, 2), ref) < tol(storage)
    if gam_big is not None:
        keep = torch.ones(gam_big.shape, dtype=torch.bool)
        keep[:n, :, :, 8:8 + C] = False
        assert torch.equal(untouched(gam_big), keep)
        assert rel_err(gam_big[:n, :, :, 8:8 + C].permute(0, 3, 1, 2), gamma) < 1e-2


@pytest.mark.parametrize("n,h,w", SHAPES)
def test_storage_output_pad_channels_with_residual(storage, n, h, w):
    """20 output channels in a slice of a 40-channel buffer: channels 20..23 are pad channels, written as act(0 + res)."""
    seed = 12
    cin, cout, c0, P = 24, 20, 8, 40
    x = rounded(synth.normalish((n, cin, h, w), seed, "x"), storage)
    wt = rounded(synth.normalish((cout, cin, 3, 3), seed, "w", 0.1), storage)
    b = synth.normalish((cout,), seed, "b", 0.1)
    res_buf = synth.normalish((n, h, w, 24), seed, "r").to(storage).to(DEV)  # pad channels of the residual hold data too
    out_big = sentinel_buf((n + 1, h, w, P), storage)
    out = Act(out_big[:n], c=cout, c0=c0)
    ops.conv2d(ops.from_nchw(x.float().to(DEV)), ops.pack_weight(wt.float().to(DEV), (1, 1)), out, act=ops.ACT_RELU,
               shift=b.to(DEV), res=Act(res_buf, c=cout))
    torch.cuda.synchronize()

    r = res_buf.double().cpu()
    ref = torch.relu(F.conv2d(x, wt, b.double(), padding=1) + r[..., :cout].permute(0, 3, 1, 2))
    keep = torch.ones(out_big.shape, dtype=torch.bool)
    keep[:n, :, :, c0:c0 + 24] = False
    assert torch.equal(untouched(out_big), keep)
    assert rel_err(out_big[:n, :, :, c0:c0 + cout].permute(0, 3, 1, 2), ref) < tol(storage)
    pad_ref = torch.relu(r[..., cout:24]).to(storage).double()
    assert torch.equal(out_big[:n, :, :, c0 + cout:c0 + 24].double().cpu(), pad_ref)


@pytest.mark.parametrize("n,h,w", SHAPES)
@pytest.mark.parametrize("pitch", [1, 2])
def test_fp32_nhwc_narrow_output(n, h, w, pitch):
    """fp32 NHWC outputs of 1 / 2 channels from bf16 storage (flow heads, discriminator logits), and 2 channels of a 4-wide pitch."""
    seed = 13
    cin = 32
    x = rounded(synth.normalish((n, cin, h, w), seed, "x"), torch.bfloat16)
    wt = rounded(synth.normalish((pitch, cin, 3, 3), seed, "w", 0.06), torch.bfloat16)
    b = synth.normalish((pitch,), seed, "b", 0.1)
    ref = torch.tanh(F.conv2d(x, wt, b.double(), padding=1))
    for P, c0 in ((pitch, 0), (4, 1)):
        big = sentinel_buf((n + 1, h, w, P), torch.float32)
        ops.conv2d(ops.from_nchw(x.float().to(DEV)), ops.pack_weight(wt.float().to(DEV), (1, 1)), Act(big[:n], c=pitch, c0=c0),
                   act=ops.ACT_TANH, shift=b.to(DEV))
        torch.cuda.synchronize()
        keep = torch.ones(big.shape, dtype=torch.bool)
        keep[:n, :, :, c0:c0 + pitch] = False
        assert torch.equal(untouched(big), keep), (P, c0)
        assert rel_err(big[:n, :, :, c0:c0 + pitch].permute(0, 3, 1, 2), ref) < 1e-2


@pytest.mark.parametrize("n,h,w", SHAPES)
@pytest.mark.parametrize("cout", [3, 13])
def test_fp32_nchw_output(storage, n, h, w, cout):
    """fp32 NCHW outputs (the image head, the condition generator's heads) inside a buffer with one extra image."""
    seed = 14
    cin = 40
    x = rounded(synth.normalish((n, cin, h, w), seed, "x"), storage)
    wt = rounded(synth.normalish((cout, cin, 3, 3), seed, "w", 0.05), storage)
    b = synth.normalish((cout,), seed, "b", 0.1)
    big = sentinel_buf((n + 1, cout, h, w), torch.float32)
    ops.conv2d(ops.from_nchw(x.float().to(DEV)), ops.pack_weight(wt.float().to(DEV), (1, 1)), big[:n], shift=b.to(DEV),
               out_layout=capi.NCHW)
    torch.cuda.synchronize()
    keep = torch.ones(big.shape, dtype=torch.bool)
    keep[:n] = False
    assert torch.equal(untouched(big), keep)
    assert rel_err(big[:n], F.conv2d(x, wt, b.double(), padding=1)) < tol(storage)
