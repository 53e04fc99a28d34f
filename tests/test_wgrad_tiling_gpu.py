"""hrv_conv2d_wgrad across the tilings its host plan chooses, per element against fp64 torch.nn.grad.conv2d_weight with the bound of
test_backward_kernels_gpu (bf16 and fp16 storage).

The plan (conv_wgrad.cu, wgrad_plan) puts either the output channels (dY) or the input channels (X, the box that moves with the tap)
on the 128-row M side and cuts the other side into 128-, 64- or 32-column tiles, the last one optionally narrower (128 + 64,
128 + 32).  32-column tiles read a SWIZZLE_64B box, the others SWIZZLE_128B boxes.  Each case below notes the plan it takes."""
import ctypes

import pytest
import torch

from hrviton_b200 import ops
from hrviton_b200.ops import Act
from test_backward_kernels_gpu import check, precision, upload, wgrad_case  # noqa: F401

pytestmark = pytest.mark.gpu
DEV = "cuda"

CASES = [  # n, cin, cout, H, W, k, pad, cropped dy extent or None  — plan (M side, N tiling)
    (2, 5, 128, 20, 18, 3, 1, None),          # M = cout, N = 5 in one 32-column tile (remainder 1-8)
    (2, 128, 20, 16, 20, 3, 1, None),         # M = cin, N = 20 in one 32-column tile (remainder 9-32)
    (1, 48, 128, 18, 14, 3, 1, None),         # M = cout, N = 48 in one 64-column tile (remainder 33-64)
    (1, 200, 128, 12, 10, 3, 1, None),        # M = cout, N = 200 = 128 + 72 in 128-column tiles (remainder 65-128)
    (1, 128, 180, 12, 10, 3, 1, None),        # M = cin, N = 180 = 128 + a 64-column last tile
    (1, 128, 160, 24, 20, 3, 1, None),        # gamma|beta: M = cin, N = 160 = 128 + a 32-column last tile
    (1, 128, 288, 16, 14, 3, 1, None),        # M = cin, N = 288 = 2 x 128 + 32
    (2, 96, 384, 16, 12, 1, 0, None),         # KW = 1: M = cout (3 tiles), N = 96 in one 128-column tile
    (2, 64, 96, 9, 7, 2, 1, None),            # KW = 2
    (2, 40, 72, 11, 9, 4, 2, (10, 8)),        # KW = 4, cropped dy
    (1, 128, 64, 10, 6, 2, 1, (10, 6)),       # cropped dy, M = cin, N = 64
    (1, 512, 1, 17, 13, 4, 2, None),          # D's output layer: M = cin (4 tiles), N = 1 in a 32-column tile
    (1, 32, 3, 128, 96, 3, 1, None),          # conv_img: M = cout (3 rows), N = 32, many pixels: split-K
    (2, 32, 24, 70, 58, 2, 1, None),          # few tiles, many pixels: split-K
    (1, 128, 64, 3, 40, 2, 1, (1, 40)),       # one 64-pixel chunk: one CTA per tile, no split
]


def _ids(c):
    return "n%d_%dto%d_%dx%d_k%dp%d" % c[:7] + ("_crop%dx%d" % c[7] if c[7] else "")


def workspace_bytes(xa, dya, k):
    tx, tdy = xa.ct(), dya.ct()
    return int(ops._L(xa).hrv_conv2d_wgrad_workspace_bytes(ctypes.byref(tx), ctypes.byref(tdy), k, k))


@pytest.mark.parametrize("case", CASES, ids=_ids)
def test_wgrad_tiling_per_element(case, precision):
    n, cin, cout, H, W, k, pad, crop = case
    x, dy, ref, S = wgrad_case(n, cin, cout, H, W, k, pad, crop)
    xa, dya = upload(x), upload(dy)
    got = ops.conv2d_wgrad(xa, dya, k, k, pad)
    torch.cuda.synchronize()
    check("conv wgrad", got, ref, S)
    again = ops.conv2d_wgrad(xa, dya, k, k, pad)
    torch.cuda.synchronize()
    assert torch.equal(got, again), "two identical calls must give bit-identical dW"


def test_wgrad_workspace_is_whole_slabs():
    """Split-K runs write one fp32 slab of dW per split: the workspace the library asks for is a whole number (> 1) of dW sizes,
    and zero when the grid does not split.  Both occur among the cases above."""
    seen = set()
    for n, cin, cout, H, W, k, pad, crop in CASES:
        oh, ow = crop or (H + 2 * pad - k + 1, W + 2 * pad - k + 1)
        x = torch.zeros((n, H, W, ops.round_up(cin, 8)), dtype=torch.bfloat16, device=DEV)
        dy = torch.zeros((n, oh, ow, ops.round_up(cout, 8)), dtype=torch.bfloat16, device=DEV)
        nws = workspace_bytes(Act(x, c=cin), Act(dy, c=cout), k)
        slab = cout * cin * k * k * 4
        assert nws % slab == 0 and nws != slab, (_ids((n, cin, cout, H, W, k, pad, crop)), nws, slab)
        seen.add(nws > 0)
    assert seen == {True, False}


def test_wgrad_small_workspace_is_refused():
    """A workspace one float short of what the library asks for is an error, not a short write."""
    n, cin, cout, H, W, k, pad = 2, 32, 24, 70, 58, 2, 1
    x = torch.zeros((n, H, W, ops.round_up(cin, 8)), dtype=torch.bfloat16, device=DEV)
    dy = torch.zeros((n, H + 2 * pad - k + 1, W + 2 * pad - k + 1, ops.round_up(cout, 8)), dtype=torch.bfloat16, device=DEV)
    xa, dya = Act(x, c=cin), Act(dy, c=cout)
    nws = workspace_bytes(xa, dya, k)
    assert nws > 0
    ws = torch.empty(nws, dtype=torch.uint8, device=DEV)
    dw = torch.empty((cout, cin, k, k), dtype=torch.float32, device=DEV)
    tx, tdy = xa.ct(), dya.ct()
    L = ops._L(xa)
    rc = L.hrv_conv2d_wgrad(ctypes.byref(tx), ctypes.byref(tdy), k, k, pad, ops._p(dw), ops._p(ws), nws - 4, ops._stream())
    assert rc != 0
