"""Deterministic synthetic weights and inputs (SURVEY.md §8d).

Everything is derived from integer PCG64 streams and exact float arithmetic so
that the container that generates ``tests/golden`` and the GPU box that checks
them produce bit-identical tensors (no dependence on libm / SIMD width).
"""
import zlib

import numpy as np
import torch


def _rng(seed, tag):
    return np.random.Generator(np.random.PCG64([int(seed), zlib.crc32(str(tag).encode())]))


def uniform(shape, seed, tag, lo=-1.0, hi=1.0):
    g = _rng(seed, tag)
    u = g.integers(0, 1 << 24, size=tuple(shape), dtype=np.int64).astype(np.float64) / float(1 << 24)
    return torch.from_numpy((lo + (hi - lo) * u).astype(np.float32))


def normalish(shape, seed, tag, std=1.0, mean=0.0):
    """Irwin-Hall(4) pseudo-normal: exact in fp64, unit variance after scaling."""
    g = _rng(seed, tag)
    u = g.integers(0, 1 << 24, size=(4,) + tuple(shape), dtype=np.int64).astype(np.float64) / float(1 << 24)
    z = (u.sum(0) - 2.0) * np.sqrt(3.0)
    return torch.from_numpy((mean + std * z).astype(np.float32))


def labels(shape_nhw, ncls, seed, tag, block=16):
    """Piecewise-constant label map (N,H,W) int64: random labels on a coarse grid, nearest-upsampled."""
    n, h, w = shape_nhw
    g = _rng(seed, tag)
    ch, cw = max(1, (h + block - 1) // block), max(1, (w + block - 1) // block)
    coarse = g.integers(0, ncls, size=(n, ch, cw), dtype=np.int64)
    full = np.repeat(np.repeat(coarse, block, axis=1), block, axis=2)[:, :h, :w]
    return torch.from_numpy(np.ascontiguousarray(full))


def one_hot(lab, ncls):
    n, h, w = lab.shape
    out = torch.zeros(n, ncls, h, w, dtype=torch.float32)
    out.scatter_(1, lab[:, None], 1.0)
    return out


def fill_state_dict(sd, seed):
    """Overwrite every entry of a (reference-shaped) state_dict in place, keyed by name.

    conv weights ~ N(0, 1/fan_in); biases ~ N(0,0.05); BN weight ~ N(1,0.1);
    running_mean ~ N(0,0.1); running_var ~ U(0.5,1.5); noise_scale ~ N(0,0.1);
    spectral-norm u/v = 3 fp64 power iterations from a deterministic start.
    """
    keys = sorted(sd.keys())
    for k in keys:
        t = sd[k]
        leaf = k.rsplit(".", 1)[-1]
        if leaf == "num_batches_tracked":
            t.zero_()
        elif leaf == "running_mean":
            t.copy_(normalish(t.shape, seed, k, 0.1))
        elif leaf == "running_var":
            t.copy_(uniform(t.shape, seed, k, 0.5, 1.5))
        elif leaf == "noise_scale":
            t.copy_(normalish(t.shape, seed, k, 0.1))
        elif leaf in ("weight", "weight_orig") and t.dim() == 4:
            fan_in = t.shape[1] * t.shape[2] * t.shape[3]
            t.copy_(normalish(t.shape, seed, k, float(np.sqrt(1.0 / fan_in))))
        elif leaf == "weight" and t.dim() == 1:
            t.copy_(normalish(t.shape, seed, k, 0.1, 1.0))
        elif leaf == "bias":
            t.copy_(normalish(t.shape, seed, k, 0.05))
        elif leaf in ("weight_u", "weight_v"):
            pass  # below, needs weight_orig
        else:
            raise KeyError("synth.fill_state_dict: unhandled key %s" % k)
    for k in keys:
        if k.endswith(".weight_u"):
            base = k[: -len("weight_u")]
            w = sd[base + "weight_orig"].detach().double().numpy()
            w2 = w.reshape(w.shape[0], -1)
            u = normalish((w2.shape[0],), seed, k).double().numpy()
            u /= np.linalg.norm(u) + 1e-12
            for _ in range(3):
                v = w2.T @ u
                v /= np.linalg.norm(v) + 1e-12
                u = w2 @ v
                u /= np.linalg.norm(u) + 1e-12
            sd[k].copy_(torch.from_numpy(u.astype(np.float32)))
            sd[base + "weight_v"].copy_(torch.from_numpy(v.astype(np.float32)))
    return sd


def tocg_inputs(n, h, w, seed):
    """input1 = cloth(3)+mask(1); input2 = one-hot parse(13)+densepose(3)  (SURVEY §8d)."""
    # a smooth "garment": low-resolution random field, bilinearly enlarged (exact fp32 lerps), plus faint texture —
    # white-noise cloth would turn a 0.03-pixel flow difference into an O(0.1) colour difference
    import torch.nn.functional as F
    coarse = uniform((n, 3, max(2, h // 16), max(2, w // 16)), seed, "cloth")
    cloth = F.interpolate(coarse, size=(h, w), mode="bilinear", align_corners=True) * 0.9 + uniform((n, 3, h, w), seed, "cloth_tex") * 0.05
    mask = (labels((n, h, w), 2, seed, "cmask", block=32)[:, None]).float()
    parse = one_hot(labels((n, h, w), 13, seed, "parse", block=16), 13)
    dense = uniform((n, 3, h, w), seed, "dense")
    return torch.cat([cloth, mask], 1), torch.cat([parse, dense], 1)


def gen_inputs(n, h, w, seed, input_nc=9, seg_nc=7):
    x = uniform((n, input_nc, h, w), seed, "gx")
    seg = one_hot(labels((n, h, w), seg_nc, seed, "gseg", block=16), seg_nc)
    return x, seg


def spade_noise(n, h, w, seed, idx):
    """The idx-th noise draw of a forward, already in (N,H,W) layout.

    Reference: ``torch.randn(b, w, h, 1)`` then ``.transpose(1, 3)`` (network_generator.py:104-107),
    i.e. noise[b, 0, y, x] = draw[b, x, y, 0].
    """
    draw = normalish((n, w, h, 1), seed, "noise%d" % idx)
    return draw.transpose(1, 3)[:, 0].contiguous()


def write_vitonhd(root, n, h=1024, w=768, seed=0, datamode="train", pairs="pairs.txt"):
    """A seeded synthetic VITON-HD tree under root/datamode in the real layout and image modes, plus root/pairs (each person paired
    with the next sample's cloth for the unpaired setting): image / cloth / image-densepose RGB jpg, cloth-mask L jpg, image-parse-v3
    and image-parse-agnostic-v3.2 P png (all 20 labels in blobs, arm labels 14 / 15 along the arms), openpose_img RGB png, and
    openpose_json with a plausible body (every third sample misses an elbow or a wrist: the (0,0) keypoints get_agnostic skips).
    Returns the sample names."""
    import json
    import os

    from PIL import Image, ImageDraw
    g = _rng(seed, "vitonhd")
    base = os.path.join(root, datamode)
    for d in ("image", "cloth", "cloth-mask", "image-parse-v3", "image-parse-agnostic-v3.2", "openpose_img", "openpose_json", "image-densepose"):
        os.makedirs(os.path.join(base, d), exist_ok=True)
    palette = [int(v) for v in g.integers(0, 256, 256 * 3)]

    def smooth(c):
        t = g.integers(0, 256, (max(2, h // 32), max(2, w // 32), c), dtype=np.uint8)
        return Image.fromarray(t[..., 0] if c == 1 else t).resize((w, h), Image.BILINEAR)

    def labels(arms, kp):
        lab = np.kron(g.integers(0, 20, (max(1, h // 64) + 1, max(1, w // 64) + 1)), np.ones((64, 64), np.int64))[:h, :w].astype(np.uint8)
        im = Image.fromarray(lab, "P")
        im.putpalette(palette)
        if arms:
            d = ImageDraw.Draw(im)
            for label, joints in ((14, (5, 6, 7)), (15, (2, 3, 4))):
                pts = [tuple(kp[j]) for j in joints if kp[j][0] or kp[j][1]]
                if len(pts) > 1:
                    d.line(pts, label, width=max(2, w // 12))
        return im

    names = []
    for i in range(n):
        name = "%06d_00.jpg" % i
        names.append(name)
        s = np.array([w, h], np.float64)
        kp = np.zeros((25, 3))
        body = {0: (0.5, 0.12), 1: (0.5, 0.22), 2: (0.33, 0.23), 3: (0.27, 0.38), 4: (0.25, 0.52), 5: (0.67, 0.23), 6: (0.73, 0.38),
                7: (0.75, 0.52), 8: (0.5, 0.55), 9: (0.42, 0.56), 12: (0.58, 0.56), 10: (0.42, 0.75), 13: (0.58, 0.75)}
        for j, (fx, fy) in body.items():
            kp[j, :2] = (np.array([fx, fy]) + g.uniform(-0.03, 0.03, 2)) * s
            kp[j, 2] = 0.9
        if i % 3 == 1:
            kp[(4, 7)[i % 2], :2] = 0.0  # a missing wrist
        elif i % 3 == 2:
            kp[(3, 6)[i % 2], :2] = 0.0  # a missing elbow
        p = os.path.join
        smooth(3).save(p(base, "image", name), quality=95)
        smooth(3).save(p(base, "cloth", name), quality=95)
        Image.fromarray(((np.asarray(smooth(1)) > 128) * 255).astype(np.uint8), "L").save(p(base, "cloth-mask", name), quality=95)
        labels(True, kp[:, :2]).save(p(base, "image-parse-v3", name.replace(".jpg", ".png")))
        labels(False, kp[:, :2]).save(p(base, "image-parse-agnostic-v3.2", name.replace(".jpg", ".png")))
        smooth(3).save(p(base, "openpose_img", name.replace(".jpg", "_rendered.png")))
        smooth(3).save(p(base, "image-densepose", name), quality=95)
        with open(p(base, "openpose_json", name.replace(".jpg", "_keypoints.json")), "w") as f:
            json.dump({"version": 1.3, "people": [{"person_id": [-1], "pose_keypoints_2d": kp.ravel().tolist()}]}, f)
    with open(os.path.join(root, pairs), "w") as f:
        f.write("".join("%s %s\n" % (names[i], names[(i + 1) % n]) for i in range(n)))
    return names


def jpeg_corpus(seed=0):
    """Seeded JPEG files as PIL writes them, smooth and noisy: [(name, bytes)] over sizes 1x1 to 256x192, quality 1-100, subsampling
    4:4:4 / 4:2:2 / 4:2:0, optimized Huffman tables, restart intervals (blocks and rows) and mode L."""
    import io

    from PIL import Image, ImageFile
    g = _rng(seed, "jpeg")

    def content(w, h, c, noisy):
        if noisy:
            a = g.integers(0, 256, (h, w, c), dtype=np.uint8)
        else:
            t = g.integers(0, 256, (max(2, h // 16), max(2, w // 16), c), dtype=np.uint8)
            a = np.asarray(Image.fromarray(t[..., 0] if c == 1 else t).resize((w, h), Image.BILINEAR)).reshape(h, w, c)
        return Image.fromarray(a[..., 0] if c == 1 else a, "L" if c == 1 else "RGB")

    def save(im, **kw):
        buf = io.BytesIO()
        ImageFile.MAXBLOCK = max(ImageFile.MAXBLOCK, 4 * im.width * im.height * 3)  # optimize=True encodes in one buffer
        im.save(buf, "JPEG", **kw)
        return buf.getvalue()

    out = []
    sizes = [(1, 1), (8, 8), (9, 17), (17, 9), (3, 5), (45, 67), (67, 45), (256, 192)]
    for w, h in sizes:
        for q in (1, 10, 50, 75, 95, 100):
            for sub in (0, 1, 2):
                noisy = (w * 7 + q + sub) % 2 == 1
                out.append(("%dx%d_q%d_s%d" % (w, h, q, sub), save(content(w, h, 3, noisy), quality=q, subsampling=sub)))
        for name, kw in (("opt", {"optimize": True}), ("rstb", {"restart_marker_blocks": 3}), ("rstr", {"restart_marker_rows": 1})):
            for sub in (0, 1, 2):
                for noisy in (False, True):
                    out.append(("%dx%d_%s_s%d_%d" % (w, h, name, sub, noisy), save(content(w, h, 3, noisy), quality=90, subsampling=sub, **kw)))
        for q in (10, 75, 95):
            out.append(("%dx%d_L_q%d" % (w, h, q), save(content(w, h, 1, q == 75), quality=q)))
        out.append(("%dx%d_L_rst" % (w, h), save(content(w, h, 1, False), quality=90, restart_marker_blocks=1)))
    return out


def encode_corpus(seed=0, sizes=((16, 16), (32, 48), (80, 64), (256, 192), (512, 384), (1024, 768))):
    """Seeded RGB images for the JPEG encoder, as {(h, w): [(name, uint8 (h, w, 3))]}: per size uniform noise (many 0xFF bytes to
    stuff, large AC categories), a smooth gradient, a flat colour (EOB and ZRL) and saturated 0 / 255 primaries in 8x8 cells, plus at
    256x192 and up the image of a write_vitonhd tree resized to that size (a try-on-like picture)."""
    import os
    import tempfile

    from PIL import Image
    g = _rng(seed, "jpeg_encode")
    out = {}
    with tempfile.TemporaryDirectory() as d:
        write_vitonhd(d, 1, seed=seed)
        person = Image.open(os.path.join(d, "train", "image", "000000_00.jpg")).convert("RGB")
        for h, w in sizes:
            items = [("noise", g.integers(0, 256, (h, w, 3), dtype=np.uint8))]
            t = g.integers(0, 256, (max(2, h // 64), max(2, w // 64), 3), dtype=np.uint8)
            items.append(("smooth", np.asarray(Image.fromarray(t).resize((w, h), Image.BILINEAR))))
            items.append(("flat", np.broadcast_to(g.integers(0, 256, 3).astype(np.uint8), (h, w, 3)).copy()))
            cells = (g.integers(0, 2, (h // 8, w // 8, 3)) * 255).astype(np.uint8)
            items.append(("primaries", cells.repeat(8, 0).repeat(8, 1)))
            if h >= 256:
                items.append(("person", np.asarray(person.resize((w, h), Image.BILINEAR))))
            out[(h, w)] = items
    return out
