"""GPU: JPEG decoding on the device (hrviton_b200.jpeg) against PIL byte for byte — the seeded corpus in one batched call mixing sizes,
samplings and L / RGB, and 32 synth-tree 1024x768 files in one call; a cut entropy segment reports its error code and raises; the
VITON-HD loader on a tree with a progressive image and an L-mode cloth still equals the reference's batches, with the other JPEGs
decoded on the device; tools/fid.py's features of a JPEG folder equal those of the PIL-decoded arrays."""
import glob
import io
import os
import shutil
import sys
import types

import numpy as np
import pytest
import torch
from PIL import Image

import hrv_env
from hrviton_b200 import data, jpeg, synth

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _pil(d, rgb=False):
    im = Image.open(io.BytesIO(d))
    return np.asarray(im.convert("RGB") if rgb else im)


def test_corpus_in_one_call():
    corpus = synth.jpeg_corpus(0)
    got = jpeg.decode([d for _, d in corpus])
    assert len(got) == len(corpus)
    for (name, d), g in zip(corpus, got):
        want = _pil(d)
        assert g.is_cuda and g.shape == want.shape and np.array_equal(g.cpu().numpy(), want), name
    gray = [d for n, d in corpus if "_L_" in n]
    for d, g in zip(gray, jpeg.decode(gray, rgb=True)):  # convert('RGB') replication
        assert np.array_equal(g.cpu().numpy(), _pil(d, rgb=True))


def test_synth_tree_files_in_one_call(tmp_path):
    synth.write_vitonhd(str(tmp_path), 8, seed=31)
    files = sorted(glob.glob(str(tmp_path / "train" / "*" / "*.jpg")))
    assert len(files) == 32
    for f, g in zip(files, jpeg.decode(files)):
        assert np.array_equal(g.cpu().numpy(), np.asarray(Image.open(f))), f


def test_cut_entropy_segment_raises():
    corpus = dict(synth.jpeg_corpus(0))
    good = corpus["256x192_q95_s2"]
    h = jpeg.parse(good)
    s0, s1 = h.segment
    cut = good[:s0 + (s1 - s0) // 3] + b"\xff\xd9"  # well formed, but the scan's data stops a third of the way in
    items = [jpeg.compact(good), jpeg.compact(cut, "cut.jpg")]
    out = [torch.empty(c.shape, dtype=torch.uint8, device="cuda") for c in items]
    b = jpeg.Batch(items)
    b.set_destinations(out)
    codes = b.launch(torch.device("cuda")).cpu().numpy()
    assert codes.tolist() == [0, jpeg.ERR_TRUNCATED]
    assert np.array_equal(out[0].cpu().numpy(), _pil(good))  # the other image of the batch decodes
    with pytest.raises(OSError, match="image 1: .*truncated"):  # bytes are named by their index
        jpeg.decode([good, cut])


def _reference_batches(tree, fh, fw, n, batch):
    if hrv_env.reference_dir() is None:
        pytest.skip("no reference copy (oracle/_ref)")
    mod = hrv_env.load_reference_script("cp_dataset")
    opt = types.SimpleNamespace(dataroot=tree, datamode="train", data_list="pairs.txt", fine_height=fh, fine_width=fw, semantic_nc=13)
    ds = mod.CPDataset(opt)
    collate = torch.utils.data.default_collate
    return [collate([ds[i] for i in range(b * batch, (b + 1) * batch)]) for b in range(n // batch)]


def test_loader_mixes_device_and_pil_decoding(tmp_path):
    tree = str(tmp_path)
    n, batch = 4, 2
    synth.write_vitonhd(tree, n, seed=33)
    img = os.path.join(tree, "train", "image", "000001_00.jpg")
    Image.open(img).save(img, quality=90, progressive=True)  # stays on PIL
    cloth = os.path.join(tree, "train", "cloth", "000002_00.jpg")
    Image.open(cloth).convert("L").save(cloth, quality=90)  # decoded on the device, replicated to RGB as convert('RGB') does
    assert not jpeg.device_decodable(jpeg.parse(img)) and jpeg.device_decodable(jpeg.parse(cloth))
    want = _reference_batches(tree, 512, 384, n, batch)
    loader = data.VitonHDLoader(tree, "train", "pairs.txt", 512, 384, batch, workers=2, shuffle=False)
    got = list(loader)
    assert len(got) == len(want)
    for g, w in zip(got, want):
        assert g["im_name"] == w["im_name"]
        for k in w:
            if k in ("im_name", "c_name"):
                continue
            for s in (w[k] if isinstance(w[k], dict) else [None]):
                gs, ws = (g[k][s], w[k][s]) if s is not None else (g[k], w[k])
                assert torch.equal(gs.cpu(), ws), (k, s)
    # image, cloth, image-densepose and cloth-mask are JPEGs: all but the progressive image went through the device, over the epoch
    # and the next epoch's first batch, which the loader has staged (it holds the progressive image too)
    assert loader.device_decoded == (4 * n - 1) + (4 * batch - 1)


def test_fid_folder_features_on_jpegs(tmp_path):
    import fid_inception_oracle as fo
    from hrviton_b200 import metrics
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    try:
        import fid as fid_tool
    finally:
        sys.path.pop(0)
    net = metrics.InceptionV3.from_fid_weights(fo.seeded_fid_state_dict(seed=4))
    folder = tmp_path / "jpegs"
    folder.mkdir()
    rng = np.random.default_rng(5)
    for i in range(20):
        t = rng.integers(0, 256, (16, 12, 3), dtype=np.uint8)
        im = Image.fromarray(t).resize((192, 256), Image.BILINEAR)
        if i == 3:
            im.save(str(folder / ("%03d.jpg" % i)), progressive=True)  # PIL
        elif i == 4:
            im.convert("L").save(str(folder / ("%03d.jpg" % i)))  # device, replicated
        else:
            im.save(str(folder / ("%03d.jpg" % i)))  # PIL's default: q75, 4:2:0, as the reference's save_images writes
    files = fid_tool.image_files(str(folder))
    decoded = torch.from_numpy(np.stack([np.asarray(Image.open(f).convert("RGB")) for f in files]))
    with torch.no_grad():
        got = fid_tool.folder_features(files, net, batch_size=8, workers=2)
        direct = torch.cat([net(decoded[i:i + 8].cuda())[0] for i in range(0, len(files), 8)])
    assert torch.equal(got, direct)
    shutil.rmtree(str(folder))
