"""VITON-HD input pipeline: the tensors of cp_dataset.CPDataset / cp_dataset_test.CPDatasetTest, bit-identical, from the on-disk
VITON-HD tree (jpg / png / json), with the pixel work on the GPU.

The CPU workers (VitonHDDataset, run by a torch DataLoader) read each JPEG's header and ship the files the device decodes
(jpeg.device_decodable: baseline, grayscale or YCbCr, 4:4:4 / 4:2:2 / 4:2:0) as their entropy-coded bytes, which hrviton_b200.jpeg
decodes on the device bit for bit as PIL does, straight into the batch's staged uint8 planes; every other file (the PNGs, and JPEGs
such as progressive ones) they decode with PIL and ship as uint8 at source resolution.  For the agnostic image they ship the
OpenPose keypoints, from which the device rasterises get_agnostic's pose shapes as one bit plane (hrviton_b200.draw), bit for bit as
ImageDraw draws them in agnostic_bits.  The file's header selects the path; there is no option.  The device (include/hrviton_sm100_data.h) composites the agnostic image,
resizes with Pillow's own fixed-point arithmetic (tables built here), regroups the 20 parse labels to 13 and writes the fp32 outputs
in one assembly launch; the 13-channel maps are expanded from one byte per pixel by hrv_onehot_u8.  VitonHDLoader stages each batch
on a copy stream with two slots (train_step.BatchFeeder), so `Stage2Trainer.replay(feeder=loader)` trains from disk.

Data-parallel runs: every rank derives one permutation from (seed, epoch) and takes a disjoint 1/W share of it.  The reference's
CPDataLoader instead gives every rank its own RandomSampler over the whole set, so its ranks see overlapping samples."""
import json
import math
import os.path as osp

import numpy as np
import torch
from PIL import Image, ImageDraw

from . import capi, draw, jpeg
from .train_step import GROUP_OF_13, LABELS7, BatchFeeder

PRECISION_BITS = 22  # Pillow's fixed-point precision for 8-bit resampling
# cp_dataset.py:150-164: group g of the 13-channel parse map collects these labels of the 20-label parse
GROUPS = [[0, 10], [1, 2], [4, 13], [5, 6, 7], [9, 12], [14], [15], [16], [17], [18], [19], [8], [3, 11]]
GROUP_OF = np.zeros(256, np.uint8)
for _g, _labels in enumerate(GROUPS):
    GROUP_OF[_labels] = _g
SEMANTIC_NC = len(GROUPS)
ARM_CANVAS = (768, 1024)  # get_agnostic draws the arm masks on a fixed 768x1024 canvas, whatever the image size

TRAIN_KEYS = ("cloth", "cloth_mask", "parse_agnostic", "densepose", "pose", "agnostic", "parse_onehot", "parse", "pcm", "parse_cloth",
              "image")
STAGE2_KEYS = ("cloth", "cloth_mask", "parse_agnostic", "densepose", "agnostic", "image")
STAGE1_KEYS = ("cloth", "cloth_mask", "parse_agnostic", "densepose", "parse_onehot", "parse", "pcm", "parse_cloth")
ONEHOT_KEYS = ("parse", "parse_agnostic")
PAIRED_KEYS = ("cloth", "cloth_mask")  # {'paired': ..., 'unpaired': ...} in the reference's batches
# the source planes a key is computed from
_NEEDS = {"cloth": ("cloth",), "cloth_mask": ("cloth_mask",), "image": ("image",), "pose": ("pose",), "densepose": ("densepose",),
          "parse_agnostic": ("parse_agnostic",), "parse": ("parse",), "pcm": ("parse",), "parse_onehot": ("parse",),
          "parse_cloth": ("image", "parse"), "agnostic": ("image", "parse", "keypoints"), "gen_parse": ("parse",)}
GEN_PARSE_NC = len(LABELS7)  # gen_parse: the 13-channel parse regrouped into the generator's 7 classes (train_generator.py:250-273)
_RGB_ORDER = ("image", "cloth", "pose", "densepose")


# ------------------------------------------------------------------------------------------------ host tables (Pillow's arithmetic)

def resized_size(h, w, fine_width):
    """(height, width) that transforms.Resize(fine_width) gives an h x w image: the shorter edge becomes fine_width, the other is
    scaled and truncated."""
    if w <= h:
        return int(fine_width * h / w), fine_width
    return fine_width, int(fine_width * w / h)


def bilinear_tables(n_in, n_out):
    """Pillow's precompute_coeffs + normalize_coeffs_8bpc for the bilinear filter: int32 bounds [n_out][2] = (first tap, taps) and
    int32 coefficients [n_out][ksize] in 22-bit fixed point (rounded half away from zero)."""
    scale = n_in / n_out
    fs = max(scale, 1.0)
    ksize = int(math.ceil(fs)) * 2 + 1
    bounds = np.zeros((n_out, 2), np.int32)
    coeffs = np.zeros((n_out, ksize), np.int32)
    for x in range(n_out):
        center = (x + 0.5) * scale
        xmin = max(int(center - fs + 0.5), 0)
        xmax = min(int(center + fs + 0.5), n_in) - xmin
        w = [max(0.0, 1.0 - abs((t + xmin - center + 0.5) / fs)) for t in range(xmax)]
        ww = sum(w)
        for t, v in enumerate(w):
            v = v / ww if ww != 0.0 else v
            coeffs[x, t] = int(0.5 + v * (1 << PRECISION_BITS)) if v >= 0 else int(-0.5 + v * (1 << PRECISION_BITS))
        bounds[x] = (xmin, xmax)
    return bounds, coeffs


def nearest_index(n_in, n_out):
    """Source index of every output of Pillow's nearest resize: it steps through the source from 0.5*scale in increments of scale
    (in double) and floors, which differs from floor((x + 0.5) * scale) at non-integer ratios."""
    scale = n_in / n_out
    out = np.empty(n_out, np.int32)
    xx = 0.5 * scale
    for x in range(n_out):
        out[x] = min(int(math.floor(xx)), n_in - 1)
        xx += scale
    return out


def resize_bilinear_np(a, oh, ow):
    """numpy restatement of the two integer passes (x, then y) over the host tables: uint8 (h, w) or (h, w, c)."""
    def one_pass(a, n_out, axis):
        a = np.moveaxis(a, axis, 0).astype(np.int64)
        bounds, coeffs = bilinear_tables(a.shape[0], n_out)
        out = np.empty((n_out,) + a.shape[1:], np.int64)
        for i, ((x0, n), k) in enumerate(zip(bounds, coeffs)):
            s = np.full(a.shape[1:], 1 << (PRECISION_BITS - 1), np.int64)
            for t in range(n):
                s += a[x0 + t] * int(k[t])
            out[i] = np.clip(s >> PRECISION_BITS, 0, 255)
        return np.moveaxis(out.astype(np.uint8), 0, axis)
    if a.shape[:2] == (oh, ow):
        return a
    return one_pass(one_pass(a, ow, 1), oh, 0)


def resize_nearest_np(a, oh, ow):
    return a[nearest_index(a.shape[0], oh)][:, nearest_index(a.shape[1], ow)]


# ------------------------------------------------------------------------------------------------ get_agnostic's shapes as bits

def agnostic_bits(pose_data, size):
    """The shapes cp_dataset.get_agnostic draws, rasterised by ImageDraw in mode 'L' (no antialiasing, so the covered pixels are those
    its 'gray' / 'black' calls cover): uint8 (h, w) with bit 0 = a grey torso / neck / arm shape, bits 1 and 2 = the black shapes of the
    label-14 and label-15 arm masks.  pose_data: (25, 2) OpenPose keypoints, copied (keypoints 9 and 12 are rescaled to the shoulder
    width, as the reference does in place); size: the image's (width, height)."""
    p = np.array(pose_data, dtype=np.float64)
    shoulders = np.linalg.norm(p[5] - p[2])
    hips = np.linalg.norm(p[12] - p[9])
    mid = (p[9] + p[12]) / 2
    p[9] = mid + (p[9] - mid) / hips * shoulders
    p[12] = mid + (p[12] - mid) / hips * shoulders
    r = int(shoulders / 16) + 1

    def pt(i):
        return tuple(p[i])

    def box(i, rx, ry):
        x, y = p[i]
        return (x - r * rx, y - r * ry, x + r * rx, y + r * ry)

    def absent(i):
        return p[i, 0] == 0.0 and p[i, 1] == 0.0

    grey = Image.new("L", size, 0)
    d = ImageDraw.Draw(grey)
    for i in (9, 12):  # torso
        d.ellipse(box(i, 3, 6), 255, 255)
    d.line([pt(2), pt(9)], 255, width=r * 6)
    d.line([pt(5), pt(12)], 255, width=r * 6)
    d.line([pt(9), pt(12)], 255, width=r * 12)
    d.polygon([pt(2), pt(5), pt(12), pt(9)], 255, 255)
    x, y = p[1]  # neck
    d.rectangle((x - r * 5, y - r * 9, x + r * 5, y), 255, 255)
    d.line([pt(2), pt(5)], 255, width=r * 12)  # arms
    for i in (2, 5):
        d.ellipse(box(i, 5, 6), 255, 255)
    for i in (3, 4, 6, 7):
        if absent(i - 1) or absent(i):
            continue
        d.line([pt(i - 1), pt(i)], 255, width=r * 10)
        d.ellipse(box(i, 5, 5), 255, 255)
    bits = (np.asarray(grey) != 0).astype(np.uint8)

    for bit, joints in ((1, (5, 6, 7)), (2, (2, 3, 4))):  # arm masks of labels 14 and 15
        arm = Image.new("L", ARM_CANVAS, 0)
        d = ImageDraw.Draw(arm)
        d.ellipse(box(joints[0], 5, 6), 255, 255)
        last = joints[0]
        for i in joints[1:]:
            if absent(i - 1) or absent(i):
                continue
            d.line([pt(i - 1), pt(i)], 255, width=r * 10)
            last = i
            if i != joints[-1]:
                d.ellipse(box(i, 5, 5), 255, 255)
        d.ellipse(box(last, 4, 4), 255, 255)
        bits |= (np.asarray(arm) != 0).astype(np.uint8) << bit
    return bits


def agnostic_np(image, parse, bits):
    """numpy statement of hrv_agnostic_composite: image (h, w, 3) uint8, parse (h, w) labels, bits from agnostic_bits."""
    restore = ((bits & 2 == 0) & (parse == 14)) | ((bits & 4 == 0) & (parse == 15)) | np.isin(parse, (4, 13, 9, 12, 16, 17, 18, 19))
    out = image.copy()
    out[((bits & 1) != 0) & ~restore] = 128
    return out


# ------------------------------------------------------------------------------------------------ worker side

class VitonHDDataset(torch.utils.data.Dataset):
    """One VITON-HD sample as uint8 arrays at source resolution (what the CPU workers ship).  Reads `dataroot/datamode/...` and the
    pairs file `dataroot/data_list` as cp_dataset.CPDataset(opt) does.

    mode="train": cp_dataset.CPDataset (paired cloth, im_name = 'image/' + name).  mode="test": cp_dataset_test.CPDatasetTest (paired
    and unpaired cloth, im_name = name; with keys=STAGE... or without 'agnostic' also cp_dataset.CPDatasetTest).  keys: the outputs
    wanted (default: every key of the reference's batch); only the files they need are opened.

    Raises ValueError on input the device path does not reproduce: an image, pose or densepose file that is not RGB (ToTensor would
    keep its other channels), a cloth mask that is not mode 'L', parse labels above 19, planes of different sizes, or a fine_height
    other than torchvision's height for fine_width.

    device_agnostic=True ships each sample's (25, 2) fp64 keypoints ('keypoints') instead of the agnostic bit plane ('bits'), for
    the device to rasterise (draw.agnostic_bits); such a sample raises ValueError on keypoints draw.keypoints_array refuses."""

    def __init__(self, dataroot, datamode, data_list, fine_height, fine_width, mode="train", keys=None, device_agnostic=False):
        if mode not in ("train", "test"):
            raise ValueError("mode must be 'train' or 'test', not %r" % (mode,))
        self.mode = mode
        self.keys = tuple(TRAIN_KEYS if keys is None else keys)
        unknown = [k for k in self.keys if k not in _NEEDS]
        if unknown:
            raise ValueError("unknown keys %s (known: %s)" % (unknown, ", ".join(_NEEDS)))
        self.fine_height, self.fine_width = int(fine_height), int(fine_width)
        self.data_path = osp.join(dataroot, datamode)
        self.im_names, self.c_unpaired = [], []
        with open(osp.join(dataroot, data_list)) as f:
            for line in f.readlines():
                im_name, c_name = line.strip().split()
                self.im_names.append(im_name)
                self.c_unpaired.append(c_name)
        self.sets = ("paired", "unpaired") if mode == "test" else ("paired",)
        needs = {s for k in self.keys for s in _NEEDS[k]}
        # plane layout of a sample: RGB planes (one per cloth set), label planes, cloth-mask planes
        self.rgb_planes = [p for p in _RGB_ORDER if p in needs for _ in (self.sets if p == "cloth" else (None,))]
        self.lab_planes = [p for p in ("parse", "parse_agnostic") if p in needs]
        self.mask_sets = len(self.sets) if "cloth_mask" in needs else 0
        self.keypoints = "keypoints" in needs
        self.device_agnostic = bool(device_agnostic)
        if not self.im_names:
            raise ValueError("%s lists no samples" % osp.join(dataroot, data_list))
        first = self._open(self._paths(0)[self.rgb_planes[0] if self.rgb_planes else (self.lab_planes or ["cloth_mask"])[0]])
        self.src_h, self.src_w = first.height, first.width
        want = resized_size(self.src_h, self.src_w, self.fine_width)
        if want != (self.fine_height, self.fine_width):
            raise ValueError("fine_height %d: transforms.Resize(%d) makes %dx%d images %dx%d" % (self.fine_height, self.fine_width, self.src_h,
                                                                                                 self.src_w, want[0], want[1]))
        if self.keypoints and (self.src_w, self.src_h) != ARM_CANVAS:
            raise ValueError("the agnostic image needs 768x1024 sources (get_agnostic's arm masks are fixed at that size), not %dx%d"
                             % (self.src_w, self.src_h))
        self.__getitem__(0)  # every mode / size check on the first sample, in the constructor

    def __len__(self):
        return len(self.im_names)

    def names(self, index):
        name = self.im_names[index]
        im_name = "image/" + name if self.mode == "train" else name
        c_name = {"paired": name, "unpaired": self.c_unpaired[index]}
        return im_name, {s: c_name[s] for s in self.sets}

    def _paths(self, index):
        """File of every source plane, derived from the names as the reference derives them (string replacement included)."""
        im_name, c_name = self.names(index)
        j = lambda *a: osp.join(self.data_path, *a)  # noqa: E731
        if self.mode == "train":
            parse = im_name.replace("image", "image-parse-v3").replace(".jpg", ".png")
            paths = {"image": j(im_name), "parse": j(parse), "parse_agnostic": j(parse.replace("image-parse-v3", "image-parse-agnostic-v3.2")),
                     "pose": j(im_name.replace("image", "openpose_img").replace(".jpg", "_rendered.png")),
                     "keypoints": j(im_name.replace("image", "openpose_json").replace(".jpg", "_keypoints.json")),
                     "densepose": j(im_name.replace("image", "image-densepose"))}
        else:
            parse = im_name.replace(".jpg", ".png")
            paths = {"image": j("image", im_name), "parse": j("image-parse-v3", parse), "parse_agnostic": j("image-parse-agnostic-v3.2", parse),
                     "pose": j("openpose_img", im_name.replace(".jpg", "_rendered.png")),
                     "keypoints": j("openpose_json", im_name.replace(".jpg", "_keypoints.json")),
                     "densepose": j("image-densepose", im_name.replace("image", "image-densepose"))}
        paths["cloth"] = [j("cloth", c_name[s]) for s in self.sets]
        paths["cloth_mask"] = [j("cloth-mask", c_name[s]) for s in self.sets]
        return paths

    @staticmethod
    def _open(path):
        return Image.open(path[0] if isinstance(path, list) else path)

    def _array(self, im, path, modes):
        if modes and im.mode not in modes:
            raise ValueError("%s: mode %s, the loader reproduces %s only" % (path, im.mode, "/".join(modes)))
        a = np.asarray(im)
        if a.shape[:2] != (self.src_h, self.src_w):
            raise ValueError("%s: %dx%d, the other planes are %dx%d" % (path, a.shape[0], a.shape[1], self.src_h, self.src_w))
        return a

    def _plane(self, path, modes, to_rgb=False):
        """A JPEG plane the device decodes as its jpeg.Compact (header and entropy-coded bytes; PIL only reads the header, so the mode
        and size checks keep their messages), any other file as PIL's uint8 array (converted to RGB with to_rgb)."""
        im = Image.open(path)
        if modes and im.mode not in modes:
            raise ValueError("%s: mode %s, the loader reproduces %s only" % (path, im.mode, "/".join(modes)))
        if (im.height, im.width) != (self.src_h, self.src_w):
            raise ValueError("%s: %dx%d, the other planes are %dx%d" % (path, im.height, im.width, self.src_h, self.src_w))
        if im.format == "JPEG":
            with open(path, "rb") as f:
                c = jpeg.compact(f.read())
            if c is not None and (c.height, c.width) == (self.src_h, self.src_w):
                c.name = path
                return c
        return self._array(im.convert("RGB") if to_rgb else im, path, modes)

    def __getitem__(self, index):
        paths = self._paths(index)
        im_name, c_name = self.names(index)
        out = {"im_name": im_name, "c_name": c_name}
        rgb, cloth_i = [], 0
        for p in self.rgb_planes:
            if p == "cloth":  # the reference converts the cloth to RGB; the other images go to ToTensor as decoded
                path = paths["cloth"][cloth_i]
                cloth_i += 1
                rgb.append(self._plane(path, None, to_rgb=True))
            else:
                rgb.append(self._plane(paths[p], ("RGB",)))
        if rgb:
            out["rgb"] = rgb
        if self.lab_planes:
            lab = np.stack([self._array(Image.open(paths[p]), paths[p], ("P", "L")) for p in self.lab_planes])
            if lab.max() > 19:
                raise ValueError("%s: parse label %d, cp_dataset's one-hot has 20 classes" % (paths[self.lab_planes[0]], lab.max()))
            out["lab"] = lab
        if self.mask_sets:
            out["cm"] = [self._plane(p, ("L",)) for p in paths["cloth_mask"]]
        if self.keypoints:
            with open(paths["keypoints"]) as f:
                pose = np.array(json.load(f)["people"][0]["pose_keypoints_2d"]).reshape((-1, 3))[:, :2]
            if self.device_agnostic:
                out["keypoints"] = draw.keypoints_array(pose, paths["keypoints"])
            else:
                out["bits"] = agnostic_bits(pose, (self.src_w, self.src_h))
        return out


def collate(samples):
    """Stacks a batch plane-major ((planes, n, h, w[, 3]) uint8), so that each plane of the batch is one contiguous device image stack.
    Images the device decodes travel as their entropy-coded bytes instead: 'jpeg' lists their jpeg.Compacts and 'jpeg_to' their
    (key, plane, sample) destinations, with the bytes packed into one buffer 'jpeg_bytes'.  Where a key mixes both, its PIL images
    travel as one stack '<key>_pil' with their (plane, sample) in '<key>_to'."""
    out = {k: torch.from_numpy(np.stack([s[k] for s in samples], 1)) for k in ("lab",) if k in samples[0]}
    items, item_to = [], []
    for k in ("rgb", "cm"):
        if k not in samples[0]:
            continue
        pil, pil_to = [], []
        for p in range(len(samples[0][k])):
            for i, s in enumerate(samples):
                if isinstance(s[k][p], jpeg.Compact):
                    items.append(s[k][p])
                    item_to.append((k, p, i))
                else:
                    pil.append(s[k][p])
                    pil_to.append((p, i))
        if len(pil) == len(samples) * len(samples[0][k]):
            out[k] = torch.from_numpy(np.stack(pil)).unflatten(0, (-1, len(samples)))
        elif pil:
            out[k + "_pil"], out[k + "_to"] = torch.from_numpy(np.stack(pil)), pil_to
    if items:
        out["jpeg_bytes"] = jpeg.pack_entropy(items)
        out["jpeg"], out["jpeg_to"] = items, item_to
    for k in ("bits", "keypoints"):
        if k in samples[0]:
            out[k] = torch.from_numpy(np.stack([s[k] for s in samples]))
    out["im_name"] = [s["im_name"] for s in samples]
    out["c_name"] = {k: [s["c_name"][k] for s in samples] for k in samples[0]["c_name"]}
    return out


# ------------------------------------------------------------------------------------------------ sampling

def shard_indices(n_items, batch_size, epoch, seed=0, shuffle=True, rank=0, world=1):
    """The sample indices of rank `rank` of `world` for one epoch: one permutation of range(n_items) derived from (seed, epoch) (the
    identity with shuffle=False), cut to the largest multiple of world * batch_size, rank r taking every world-th entry from r.  Ranks
    are disjoint and get the same number of full batches; world 1 is the plain seeded shuffle."""
    order = np.random.default_rng([int(seed), int(epoch)]).permutation(n_items) if shuffle else np.arange(n_items)
    per_rank = n_items // (world * batch_size) * batch_size
    return order[:per_rank * world][rank::world]


class _EpochSampler(torch.utils.data.Sampler):
    def __init__(self, n_items, batch_size, seed, shuffle, rank, world):
        self.args = (n_items, batch_size)
        self.seed, self.shuffle, self.rank, self.world = seed, shuffle, rank, world
        self.epoch = 0
        self.start = 0  # samples of the epoch to skip (VitonHDLoader.start_at)

    def __iter__(self):
        return iter(shard_indices(*self.args, self.epoch, self.seed, self.shuffle, self.rank, self.world)[self.start:].tolist())

    def __len__(self):
        return len(shard_indices(*self.args, 0, self.seed, False, self.rank, self.world))


# ------------------------------------------------------------------------------------------------ device side

def resize_u8(x, oh, ow, mode="bilinear"):
    """Image.resize((ow, oh), BILINEAR or NEAREST) of every image of x on the device, bit-identical to Pillow: x (planes, h, w) or
    (planes, h, w, 3) uint8 CUDA -> (planes, oh, ow[, 3]).  An unchanged size returns x (torchvision's Resize does not resample)."""
    assert x.is_cuda and x.dtype == torch.uint8 and x.dim() in (3, 4) and mode in ("bilinear", "nearest")
    x = x.contiguous()
    planes, h, w = x.shape[:3]
    c = x.shape[3] if x.dim() == 4 else 1
    if (h, w) == (oh, ow):
        return x
    L, st, dev = capi.lib(), torch.cuda.current_stream().cuda_stream, x.device
    if mode == "nearest":
        assert c == 1
        ys, xs = (torch.from_numpy(nearest_index(a, b)).to(dev) for a, b in ((h, oh), (w, ow)))
        out = torch.empty((planes, oh, ow), dtype=torch.uint8, device=dev)
        capi.check(L.hrv_pil_nearest(x.data_ptr(), planes, h, w, ys.data_ptr(), oh, xs.data_ptr(), ow, None, out.data_ptr(), st), "pil_nearest")
        return out
    tmp = torch.empty((planes, h, ow) + x.shape[3:], dtype=torch.uint8, device=dev)
    out = torch.empty((planes, oh, ow) + x.shape[3:], dtype=torch.uint8, device=dev)
    for axis, (src, dst, n_in, n_out) in enumerate(((x, tmp, w, ow), (tmp, out, h, oh))):
        b, k = (torch.from_numpy(t).to(dev) for t in bilinear_tables(n_in, n_out))
        capi.check(L.hrv_pil_resample_pass(src.data_ptr(), planes, h, ow if axis else w, c, axis, b.data_ptr(), k.data_ptr(), k.shape[1], n_out,
                                           dst.data_ptr(), st), "pil_resample_pass")
    return out


class VitonHDLoader(BatchFeeder):
    """Batches of the VITON-HD tree as CUDA fp32 tensors, bit-identical to the reference's collated batches.

    Iterating yields one epoch of dicts keyed as cp_dataset's (cloth / cloth_mask as {'paired': ...[, 'unpaired': ...]}, c_name,
    im_name); next_batch() cycles through epochs forever, as CPDataLoader.next_batch does; consume(out) writes the next batch into
    given tensors (flat keys; cloth / cloth_mask take the paired cloth), stream-ordered, and starts the copy of the following batch,
    so a captured trainer replays with replay(feeder=loader).  Incomplete batches are dropped (drop_last, as in the reference).

    With an initialised process group of world size W, rank r reads a disjoint 1/W of each epoch's permutation (shard_indices);
    shard=False reads the whole set on every rank.  position() and start_at() save and restore where the batches stand.

    The agnostic image's shapes are rasterised on the device from the keypoints the workers ship (device_agnostic=True), or drawn
    by ImageDraw in the workers (False); the batches are the same bit for bit."""

    def __init__(self, dataroot, datamode, data_list, fine_height, fine_width, batch_size, workers=4, mode="train", keys=None, shuffle=True,
                 seed=0, shard=True, device_agnostic=True):
        import torch.distributed as dist
        self.dataset = VitonHDDataset(dataroot, datamode, data_list, fine_height, fine_width, mode=mode, keys=keys,
                                      device_agnostic=device_agnostic)
        ds = self.dataset
        self.keys, self.batch_size, self.seed = ds.keys, int(batch_size), seed
        rank, world = (dist.get_rank(), dist.get_world_size()) if shard and dist.is_available() and dist.is_initialized() else (0, 1)
        self.sampler = _EpochSampler(len(ds), self.batch_size, seed, shuffle, rank, world)
        if len(self.sampler) == 0:
            raise ValueError("%d samples make no full batch of %d on each of %d ranks" % (len(ds), self.batch_size, world))
        self.loader = torch.utils.data.DataLoader(ds, batch_size=self.batch_size, sampler=self.sampler, num_workers=workers, collate_fn=collate,
                                                  pin_memory=True, drop_last=True, persistent_workers=workers > 0,
                                                  generator=torch.Generator().manual_seed(int(seed)))  # leaves torch's CPU generator alone
        self._init_staging(torch.device("cuda", torch.cuda.current_device()))  # the kernels launch on the current device's stream
        self.slots, self.host, self.names, self.epochs = [None, None], [None, None], [None, None], [None, None]
        self.positions = [None, None]
        self._iter, self._epoch, self._index, self._skip = None, 0, 0, 0
        h, w, fh, fw = ds.src_h, ds.src_w, ds.fine_height, ds.fine_width
        self.resize = (h, w) != (fh, fw)  # torchvision returns an image of the requested size unchanged
        dev = self.device
        if self.resize:
            self.tables = {"x": [torch.from_numpy(t).to(dev) for t in bilinear_tables(w, fw)],
                           "y": [torch.from_numpy(t).to(dev) for t in bilinear_tables(h, fh)]}
        self.ys = torch.from_numpy(nearest_index(h, fh)).to(dev)
        self.xs = torch.from_numpy(nearest_index(w, fw)).to(dev)
        self.lut = torch.from_numpy(GROUP_OF).to(dev)
        n = self.batch_size
        n_rgb = len(ds.rgb_planes) + (1 if ds.keypoints else 0)  # + the agnostic image, composited on the device
        self.scratch = {"lab": torch.empty((len(ds.lab_planes), n, fh, fw), dtype=torch.uint8, device=dev)}
        if self.resize and n_rgb:
            self.scratch["rgb_x"] = torch.empty((n_rgb, n, h, fw, 3), dtype=torch.uint8, device=dev)
            self.scratch["rgb"] = torch.empty((n_rgb, n, fh, fw, 3), dtype=torch.uint8, device=dev)
        if self.resize and ds.mask_sets:
            self.scratch["cm"] = torch.empty((ds.mask_sets, n, fh, fw), dtype=torch.uint8, device=dev)
        self.bytes_per_step = None
        self.device_decoded = 0  # JPEG files decoded on the device so far (the others were decoded by PIL in the workers)
        self._jpeg_pending = None

    def __len__(self):
        return len(self.sampler) // self.batch_size

    # -------- host batches, cycling through epochs
    def _next_host(self):
        """(epoch, batch index in the epoch, host batch) of the next batch from the workers."""
        while True:
            if self._iter is None:
                self.sampler.epoch, self.sampler.start = self._epoch, self._skip * self.batch_size
                self._index, self._skip = self._skip, 0
                self._iter = iter(self.loader)
            try:
                b = next(self._iter)
                self._index += 1
                return self._epoch, self._index - 1, b
            except StopIteration:
                self._iter = None
                self._epoch += 1

    def position(self):
        """(epoch, batch index) of the batch that the next consume() / next_batch() delivers."""
        if self.host[self.slot] is not None:
            return self.positions[self.slot]
        if self._iter is None:
            return self._epoch, self._skip
        return self._epoch, self._index

    def start_at(self, epoch, index):
        """The next batch delivered is batch `index` of epoch `epoch` (position()), as an uninterrupted run would have delivered it:
        each epoch's order derives from (seed, epoch) alone, and the workers skip the earlier samples without reading them.  Batches
        already staged are dropped.  An index at or past the end of the epoch starts the next one."""
        if int(epoch) < 0 or int(index) < 0:
            raise ValueError("start_at(%r, %r): epoch and index must be >= 0" % (epoch, index))
        torch.cuda.current_stream().wait_stream(self.copy_stream)  # a staged copy may still be writing a slot
        self.host, self.names, self.epochs, self.positions = [None, None], [None, None], [None, None], [None, None]
        self._iter, self._epoch, self._skip = None, int(epoch), int(index)

    def prefetch(self, slot=None):
        """Takes the next host batch from the workers and starts its copy into staging slot `slot` on the copy stream."""
        slot = self.slot if slot is None else slot
        epoch, index, b = self._next_host()
        ds = self.dataset
        n = self.batch_size
        self._check_jpeg_errors()  # the previous batch's decode: the loader raises no later than the next batch
        if self.slots[slot] is None:
            h, w, dev = ds.src_h, ds.src_w, self.device
            s = {}
            if ds.rgb_planes or ds.keypoints:  # one plane more for the agnostic image
                s["rgb"] = torch.empty((len(ds.rgb_planes) + (1 if ds.keypoints else 0), n, h, w, 3), dtype=torch.uint8, device=dev)
            if ds.lab_planes:
                s["lab"] = torch.empty((len(ds.lab_planes), n, h, w), dtype=torch.uint8, device=dev)
            if ds.mask_sets:
                s["cm"] = torch.empty((ds.mask_sets, n, h, w), dtype=torch.uint8, device=dev)
            if ds.keypoints:
                s["bits"] = torch.empty((n, h, w), dtype=torch.uint8, device=dev)
            if ds.keypoints and ds.device_agnostic:
                s["keypoints"] = torch.empty((n, 25, 2), dtype=torch.float64, device=dev)
                s["draw_ws"] = torch.empty(draw.workspace_bytes(n, h), dtype=torch.uint8, device=dev)
            self.slots[slot] = s
        st = self.slots[slot]
        with torch.cuda.stream(self.copy_stream):
            self.copy_stream.wait_event(self.free[slot])  # the batch that used this slot last has been assembled
            for k, v in b.items():
                if k in ("rgb", "lab", "cm", "bits", "keypoints"):
                    st[k][:v.shape[0]].copy_(v, non_blocking=True)
                elif k in ("rgb_pil", "cm_pil"):
                    for (p, i), img in zip(b[k[:-4] + "_to"], v):
                        st[k[:-4]][p, i].copy_(img, non_blocking=True)
            if "keypoints" in b:
                draw.agnostic_bits(st["keypoints"], out=st["bits"], workspace=st["draw_ws"])
            if "jpeg" in b:
                batch = jpeg.Batch(b["jpeg"], b["jpeg_bytes"])
                batch.set_destinations([st[k][p, i] for k, p, i in b["jpeg_to"]])
                errors = batch.launch(self.device, stream=self.copy_stream)
                self._jpeg_pending = (torch.empty(errors.shape, dtype=torch.int32).pin_memory(), torch.cuda.Event(), b)
                self._jpeg_pending[0].copy_(errors, non_blocking=True)
                self._jpeg_pending[1].record(self.copy_stream)
                self.device_decoded += len(b["jpeg"])
            self.ready[slot].record(self.copy_stream)
        self.bytes_per_step = int(sum(v.numel() * v.element_size() for k, v in b.items() if torch.is_tensor(v))) + len(b.get("jpeg", ())) * jpeg.DESCRIPTOR_BYTES
        self.host[slot], self.names[slot], self.epochs[slot], self.positions[slot] = b, (b["im_name"], b["c_name"]), epoch, (epoch, index)

    def _check_jpeg_errors(self):
        """Raises OSError naming the file when the last device decode met corrupt data (waits for that decode)."""
        if self._jpeg_pending is None:
            return
        codes, done, b = self._jpeg_pending
        self._jpeg_pending = None
        done.synchronize()
        if codes.any():
            names = [c.name for c in b["jpeg"]]
            jpeg.raise_errors(codes.numpy(), names)

    def consume(self, out):
        unknown = [k for k in out if k not in _NEEDS]
        if unknown:  # a graph input the loader does not write would keep stale data
            raise KeyError("consume(): %s are not keys of a VITON-HD batch (%s)" % (unknown, ", ".join(_NEEDS)))
        missing = [k for k in out if k not in self.keys]
        if missing:
            raise KeyError("consume(): the loader was built without keys %s (keys=%s)" % (missing, self.keys))
        if self.slots[self.slot] is None or self.host[self.slot] is None:
            self.prefetch()
        return super().consume(out)

    def _expand(self, staged, out):
        """The device half on the current stream: composite, resize, regroup, assemble, one-hot expansion into `out`."""
        ds, L, st = self.dataset, capi.lib(), torch.cuda.current_stream().cuda_stream
        n, h, w, fh, fw = self.batch_size, ds.src_h, ds.src_w, ds.fine_height, ds.fine_width
        rgb = staged.get("rgb")
        if ds.keypoints:
            img = rgb[ds.rgb_planes.index("image")]
            par = staged["lab"][ds.lab_planes.index("parse")]
            capi.check(L.hrv_agnostic_composite(img.data_ptr(), par.data_ptr(), staged["bits"].data_ptr(), n, h, w, rgb[-1].data_ptr(), st),
                   "agnostic_composite")
        if rgb is not None and self.resize:
            planes = rgb.shape[0] * n
            (bx, cx), (by, cy) = self.tables["x"], self.tables["y"]
            capi.check(L.hrv_pil_resample_pass(rgb.data_ptr(), planes, h, w, 3, 0, bx.data_ptr(), cx.data_ptr(), cx.shape[1], fw,
                                           self.scratch["rgb_x"].data_ptr(), st), "pil_resample_pass")
            capi.check(L.hrv_pil_resample_pass(self.scratch["rgb_x"].data_ptr(), planes, h, fw, 3, 1, by.data_ptr(), cy.data_ptr(), cy.shape[1], fh,
                                           self.scratch["rgb"].data_ptr(), st), "pil_resample_pass")
            rgb = self.scratch["rgb"]
        lab = self.scratch["lab"]
        if ds.lab_planes:
            capi.check(L.hrv_pil_nearest(staged["lab"].data_ptr(), len(ds.lab_planes) * n, h, w, self.ys.data_ptr(), fh, self.xs.data_ptr(), fw,
                                     self.lut.data_ptr(), lab.data_ptr(), st), "pil_nearest")
        cm = staged.get("cm")
        if cm is not None and self.resize:
            capi.check(L.hrv_pil_nearest(cm.data_ptr(), ds.mask_sets * n, h, w, self.ys.data_ptr(), fh, self.xs.data_ptr(), fw, None,
                                     self.scratch["cm"].data_ptr(), st), "pil_nearest")
            cm = self.scratch["cm"]

        src, dst = capi.VitonPlanes(), capi.VitonOutputs()
        for name in ("image", "pose", "densepose"):
            if name in ds.rgb_planes:
                setattr(src, name, rgb[ds.rgb_planes.index(name)].data_ptr())
        if ds.keypoints:
            src.agnostic = rgb[-1].data_ptr()
        c0 = ds.rgb_planes.index("cloth") if "cloth" in ds.rgb_planes else None
        for s in range(len(ds.sets)):
            if c0 is not None:
                src.cloth[s] = rgb[c0 + s].data_ptr()
            if cm is not None:
                src.cloth_mask[s] = cm[s].data_ptr()
        if "parse" in ds.lab_planes:
            src.parse = lab[ds.lab_planes.index("parse")].data_ptr()
        for k, t in out.items():
            if k in PAIRED_KEYS:
                for s, name in enumerate(ds.sets):
                    tt = t.get(name) if isinstance(t, dict) else (t if name == "paired" else None)
                    if tt is not None:
                        self._check_out(k, tt, 1 if k == "cloth_mask" else 3)
                        getattr(dst, k)[s] = tt.data_ptr()
            elif k in ONEHOT_KEYS:
                self._check_out(k, t, SEMANTIC_NC)
            elif k == "gen_parse":
                self._check_out(k, t, GEN_PARSE_NC)
            elif k in ("image", "pose", "densepose", "agnostic", "parse_cloth"):
                self._check_out(k, t, 3)
                setattr(dst, k, t.data_ptr())
            elif k in ("pcm", "parse_onehot"):
                self._check_out(k, t, 1)
                setattr(dst, k, t.data_ptr())
        capi.check(L.hrv_viton_assemble(src, dst, n, fh, fw, st), "viton_assemble")
        from . import ops
        for k in ONEHOT_KEYS:
            if k in out:
                ops.onehot_u8(lab[ds.lab_planes.index(k)], SEMANTIC_NC, out=out[k])
        if "gen_parse" in out:  # argmax -> scatter_ -> 7-group sum of the one-hot 13-plane map: its label through the group table
            ops.onehot_u8(lab[ds.lab_planes.index("parse")], GEN_PARSE_NC, lut=GROUP_OF_13, out=out["gen_parse"])

    def _check_out(self, key, t, c):
        want = (self.batch_size, c, self.dataset.fine_height, self.dataset.fine_width)
        if not (t.is_cuda and t.dtype == torch.float32 and t.is_contiguous() and tuple(t.shape) == want):
            raise ValueError("%s: need a contiguous CUDA fp32 tensor of shape %s, got %s %s" % (key, want, t.dtype, tuple(t.shape)))

    # -------- batches as new tensors
    def empty_batch(self):
        """A dict of device tensors for one batch of this loader's keys (cloth / cloth_mask per cloth set)."""
        ds, n = self.dataset, self.batch_size
        chans = {"cloth_mask": 1, "pcm": 1, "parse_onehot": 1, "parse": SEMANTIC_NC, "parse_agnostic": SEMANTIC_NC, "gen_parse": GEN_PARSE_NC}

        def new(k):
            return torch.empty((n, chans.get(k, 3), ds.fine_height, ds.fine_width), dtype=torch.float32, device=self.device)
        return {k: ({s: new(k) for s in ds.sets} if k in PAIRED_KEYS else new(k)) for k in self.keys}

    def _take(self):
        if self.slots[self.slot] is None or self.host[self.slot] is None:
            self.prefetch()
        im_name, c_name = self.names[self.slot]
        out = self.consume(self.empty_batch())
        out["im_name"], out["c_name"] = im_name, c_name
        return out

    def next_batch(self):
        return self._take()

    def close(self):
        """Stops the worker processes (they persist across epochs otherwise); the loader is not used after this."""
        self._iter = None
        it = getattr(self.loader, "_iterator", None)
        if it is not None:
            it._shutdown_workers()
            self.loader._iterator = None

    def __iter__(self):
        if self.slots[self.slot] is None or self.host[self.slot] is None:
            self.prefetch()
        epoch = self.epochs[self.slot]
        while self.epochs[self.slot] == epoch:
            yield self._take()
