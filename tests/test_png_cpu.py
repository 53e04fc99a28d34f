"""CPU: png.encode_np, the numpy statement of the device PNG encoder, and png.condition_grid_np, the statement of the multi-task grid.

encode_np's files must decode (PIL, and zlib over the joined IDAT data) to the input exactly, carry a correct CRC-32 in every chunk,
fall back to stored blocks on noise, and stay within 1.25x of PIL's size on smooth content and on a grid.  condition_grid_np must
equal torchvision's make_grid + save_image's arithmetic + the reference's utils.visualize_segmap, run on the same tensors."""
import io
import os
import struct
import sys
import zlib

import numpy as np
import pytest
import torch
from PIL import Image
from scipy.ndimage import gaussian_filter

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import hrv_env  # noqa: E402
import hrv_loader  # noqa: E402

hrv_loader.load()
from hrviton_b200 import png  # noqa: E402


def chunks(b):
    assert b[:8] == png.SIGNATURE
    out, i = [], 8
    while i < len(b):
        n = struct.unpack(">I", b[i:i + 4])[0]
        kind, data, crc = b[i + 4:i + 8], b[i + 8:i + 8 + n], struct.unpack(">I", b[i + 8 + n:i + 12 + n])[0]
        out.append((kind, data, crc))
        i += 12 + n
    assert i == len(b)
    return out


def smooth(h, w, seed=0, sigma=6.0, noise=2.0):
    g = np.random.default_rng(seed)
    x = gaussian_filter(g.normal(0, 1, (h, w, 3)), (sigma, sigma, 0))
    x = (x - x.min()) / (np.ptp(x) + 1e-9) * 255 + g.normal(0, noise, (h, w, 3))
    return np.clip(x, 0, 255).astype(np.uint8)


def pil_size(a):
    f = io.BytesIO()
    Image.fromarray(a).save(f, format="PNG")
    return len(f.getvalue())


def check_file(a, b):
    assert np.array_equal(np.asarray(Image.open(io.BytesIO(b))), a)
    cs = chunks(b)
    assert [k for k, _, _ in cs][0] == b"IHDR" and cs[-1][0] == b"IEND"
    for kind, data, crc in cs:
        assert crc == zlib.crc32(kind + data)
    idat = b"".join(d for k, d, _ in cs if k == b"IDAT")
    assert zlib.decompress(idat) == png.paeth_np(a).tobytes()
    return cs


def _rand(h, w, seed=1):
    return np.random.default_rng(seed).integers(0, 256, (h, w, 3), dtype=np.uint8)


@pytest.mark.parametrize("h,w", [(1, 1), (1, 40), (37, 1), (5, 33), (31, 7), (64, 63)])
def test_round_trip_small_and_odd(h, w):
    for a in (_rand(h, w), smooth(h, w), np.full((h, w, 3), 200, np.uint8)):
        check_file(a, png.encode_np(a)[0])


def test_round_trip_flat_and_smooth():
    for a in (np.zeros((300, 257, 3), np.uint8), np.full((129, 511, 3), 77, np.uint8), smooth(400, 301)):
        cs = check_file(a, png.encode_np(a[None])[0])
        assert len([c for c in cs if c[0] == b"IDAT"]) == -(-len(png.paeth_np(a)) // png.CHUNK_BYTES)


def test_noise_takes_stored_blocks():
    a = _rand(300, 301, seed=3)
    b = png.encode_np(a)[0]
    cs = check_file(a, b)
    raw = len(png.paeth_np(a))
    idats = [d for k, d, _ in cs if k == b"IDAT"]
    assert len(idats) > 1
    # every chunk a stored block: its bytes plus a 5-byte header, the zlib header and the Adler-32 around them
    assert sum(len(d) for d in idats) == raw + 5 * len(idats) + 2 + 4
    assert len(b) <= raw + 17 * len(idats) + 6 + 33 + 12


def test_large_image_round_trip():
    a = np.kron(smooth(386, 386, seed=5), np.ones((8, 8, 1), np.uint8))[:3082, :3080]
    check_file(a, png.encode_np(a)[0])


def test_deterministic():
    a = smooth(100, 100, seed=9)
    assert png.encode_np(a) == png.encode_np(a.copy())


def test_size_within_a_quarter_of_pil():
    a = smooth(512, 384, seed=4)
    g = grid_fixture()
    for x in (a, g):
        ours, pil = len(png.encode_np(x)[0]), pil_size(x)
        print("PNG size %s: %d bytes, PIL %d (%.3fx)" % (x.shape, ours, pil, ours / pil))
        assert ours <= 1.25 * pil


def test_huffman_lengths_are_limited_and_complete():
    fib = [1, 1]
    while len(fib) < 30:
        fib.append(fib[-1] + fib[-2])
    for freq, limit in ((fib + [0] * 256, 15), (fib[:19], 7), ([0, 5] + [0] * 17, 7)):
        L = png.huffman_lengths(freq, limit)
        assert max(L) <= limit
        assert sum(2.0 ** -n for n in L if n) == 1.0  # complete: inflate refuses incomplete literal / code-length codes
        assert all(L[s] for s in range(len(freq)) if freq[s])


def test_code_length_items_expand_back():
    seq = [0] * 140 + [8] * 9 + [0, 0] + [7] * 3 + [0] * 12 + [5] * 2 + [0] * 4 + [1]
    out = []
    for s, x in png.code_length_items(seq):
        if s == 16:
            out += [out[-1]] * (3 + x)
        elif s == 17:
            out += [0] * (3 + x)
        elif s == 18:
            out += [0] * (11 + x)
        else:
            out.append(s)
    assert out == seq


def test_refuses_bad_batches():
    for bad in (np.zeros((1, 4, 4, 4), np.uint8), np.zeros((1, 4, 4, 3), np.float32), np.zeros((0, 4, 4, 3), np.uint8), np.zeros((4, 4), np.uint8)):
        with pytest.raises(ValueError):
            png.encode_np(bad)


# ------------------------------------------------------------------------------------------------ the grid

def grid_tensors(n=2, h=16, w=12, classes=13, seed=0):
    """Seeded grid inputs with values outside [-1, 1], arg-max ties, and exactly 0.5 in both thresholded masks."""
    g = torch.Generator().manual_seed(seed)
    r = lambda c, lo=-1.3, hi=1.3: torch.rand(n, c, h, w, generator=g) * (hi - lo) + lo  # noqa: E731
    t = dict(cloth=r(3), cloth_mask=r(1, 0, 1), parse_agnostic=r(classes), densepose=r(3), parse_cloth=r(3), pcm=r(1, 0, 1), warped_cloth=r(3),
             warped_cm=r(1, 0, 1), parse=r(classes), seg=r(classes), image=r(3))
    # slices: the cases that do not fit a small batch or panel are left out
    t["cloth_mask"][:1, 0, :1, :3] = 0.5
    t["warped_cm"][:1, 0, 1:2, :3] = 0.5
    t["warped_cm"][:1, 0, 2:3, :2] = 1.0
    t["seg"][:1, 3, 2:3, :4] = t["seg"][:1, 5, 2:3, :4] = 5.0     # ties at the cloth channel, composed or not
    t["seg"][1:2, 0, 3:4, :4] = t["seg"][1:2, 3, 3:4, :4] = 4.0
    t["parse"][-1:, :, :1, :1] = 1.0                              # every class tied: the first wins
    t["parse_agnostic"][:1, 7:9, 1:2, 1:2] = 9.0
    return t


def grid_fixture():
    """A 776x778 grid of smooth 256x192 panels with one-hot segmentations, as the tool writes them."""
    n, h, w = 1, 256, 192
    sm = lambda c, s: torch.from_numpy(smooth(h, w, seed=s).transpose(2, 0, 1)[None, :c].astype(np.float32) / 127.5 - 1)  # noqa: E731
    lab = lambda s: torch.nn.functional.one_hot(torch.from_numpy(np.kron(np.random.default_rng(s).integers(0, 13, (5, 4)), np.ones((64, 64), np.int64))[:h, :w]), 13).permute(2, 0, 1)[None].float()  # noqa: E731
    t = dict(cloth=sm(3, 1), cloth_mask=(sm(1, 2) > 0).float(), parse_agnostic=lab(3), densepose=sm(3, 4), parse_cloth=sm(3, 5), pcm=(sm(1, 6) > 0).float(),
             warped_cloth=sm(3, 7), warped_cm=sm(1, 8) / 2 + 0.5, parse=lab(9), seg=lab(10) * 3 + sm(1, 11), image=sm(3, 12))
    return png.condition_grid_np({k: v.numpy() for k, v in t.items()})[0]


def reference_grid(utils, t, composition):
    """test_condition.py:108-143 on CPU tensors: the uint8 arrays save_image hands to PIL."""
    from torchvision.utils import make_grid
    seg, wcm = t["seg"].clone(), t["warped_cm"]
    onehot = torch.FloatTensor((wcm.numpy() > 0.5).astype(np.float32))
    if composition != "no_composition":
        cloth_mask = torch.ones_like(seg)
        cloth_mask[:, 3:4] = onehot if composition == "detach" else wcm
        seg = seg * cloth_mask
    misalign = (torch.argmax(seg, dim=1, keepdim=True) == 3).long() - onehot
    misalign[misalign < 0.0] = 0.0
    cm = torch.FloatTensor((t["cloth_mask"].numpy() > 0.5).astype(np.float32))
    out = []
    for i in range(t["cloth"].shape[0]):
        grid = make_grid([t["cloth"][i] / 2 + 0.5, cm[i].expand(3, -1, -1), utils.visualize_segmap(t["parse_agnostic"], batch=i), (t["densepose"][i] + 1) / 2,
                          t["parse_cloth"][i] / 2 + 0.5, t["pcm"][i].expand(3, -1, -1), t["warped_cloth"][i] / 2 + 0.5, onehot[i].expand(3, -1, -1),
                          utils.visualize_segmap(t["parse"], batch=i), utils.visualize_segmap(seg, batch=i), t["image"][i] / 2 + 0.5,
                          misalign[i].expand(3, -1, -1)], nrow=4)
        out.append(grid.mul(255).add_(0.5).clamp_(0, 255).permute(1, 2, 0).to("cpu", torch.uint8).numpy())
    return np.stack(out)


@pytest.mark.skipif(hrv_env.reference_dir() is None, reason="no reference copy (oracle/_ref)")
@pytest.mark.parametrize("composition", ["warp_grad", "detach", "no_composition"])
def test_grid_restatement_equals_reference(composition):
    utils = hrv_env.load_reference_script("utils")
    t = grid_tensors()
    want = reference_grid(utils, t, composition)
    got = png.condition_grid_np({k: v.numpy() for k, v in t.items()}, composition)
    assert got.shape == want.shape == png.grid_shape(2, 16, 12)
    assert np.array_equal(got, want)
