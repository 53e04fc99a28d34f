"""CPU: the numpy JPEG encoder (hrviton_b200.jpeg.encode_np) against PIL's Image.fromarray(rgb).save(format='JPEG') byte for byte on
a seeded corpus (16x16 to 1024x768: noise, smooth, flat, 0/255 primaries, a synth try-on picture); the save_images conversion of
fp32 generator output at rounding edges and outside [-1, 1] against torch; the header against PIL's; refusals of sizes and dtypes;
and tools/test.py's flag parsing, refusals and output names from a test-mode batch."""
import io

import numpy as np
import pytest
import torch
from PIL import Image

from hrviton_b200 import data, jpeg, synth, tryon_run


def _pil(rgb):
    buf = io.BytesIO()
    Image.fromarray(rgb).save(buf, format="JPEG")
    return buf.getvalue()


@pytest.fixture(scope="module")
def corpus():
    return synth.encode_corpus(0)


def test_encode_np_equals_pil(corpus):
    for (h, w), items in corpus.items():
        got = jpeg.encode_np(np.stack([a for _, a in items]))
        for (name, a), g in zip(items, got):
            assert g == _pil(a), (h, w, name)


def test_noise_stuffs_and_decodes(corpus):
    noise = dict(corpus[(256, 192)])["noise"]
    data_ = jpeg.encode_np(noise)[0]
    h = jpeg.parse(data_)
    seg = np.frombuffer(data_, np.uint8)[h.segment[0]:h.segment[1]]
    assert int(((seg[:-1] == 0xFF) & (seg[1:] == 0)).sum()) > 20  # stuffed bytes
    assert np.array_equal(jpeg.decode_np(data_), np.asarray(Image.open(io.BytesIO(_pil(noise)))))


def test_header_equals_pil():
    for h, w in ((16, 16), (16, 32), (256, 192), (1024, 768), (4096, 48)):
        head = jpeg.encode_header(h, w)
        assert _pil(np.zeros((h, w, 3), np.uint8))[:len(head)] == head, (h, w)


def _torch_save_images(x):
    """utils.save_images' arithmetic, in torch as the reference runs it."""
    t = ((torch.from_numpy(x) + 1) * 0.5 * 255).clamp(0, 255)
    return t.numpy().astype("uint8").transpose(0, 2, 3, 1)


def test_save_images_conversion_at_edges():
    k = np.arange(256, dtype=np.float64)
    edges = (k + 0.0) / 127.5 - 1  # values whose conversion lands on or next to an integer
    vals = np.concatenate([edges, (k + 0.5) / 127.5 - 1, (k + 1e-6) / 127.5 - 1, (k - 1e-6) / 127.5 - 1]).astype(np.float32)
    vals = np.concatenate([vals, np.nextafter(vals, np.float32(2)), np.nextafter(vals, np.float32(-2)),
                           np.array([-3, -1.5, -1.0000001, 1.0000001, 1.2, 7, np.inf, -np.inf, 0.0, -0.0], np.float32)])
    x = np.resize(vals, 3 * 16 * 48).reshape(1, 3, 16, 48).astype(np.float32)
    assert np.array_equal(jpeg.save_images_u8_np(x), _torch_save_images(x))
    assert jpeg.encode_np(x)[0] == _pil(_torch_save_images(x)[0])


def test_refusals():
    for bad in (np.zeros((1, 17, 16, 3), np.uint8), np.zeros((1, 16, 24, 3), np.uint8), np.zeros((1, 16, 16, 4), np.uint8),
                np.zeros((1, 16, 16, 3), np.float32), np.zeros((1, 3, 16, 16), np.float64), np.zeros((1, 16, 16, 3), np.uint16),
                np.zeros((16, 16), np.uint8), np.zeros((0, 16, 16, 3), np.uint8)):
        with pytest.raises(ValueError):
            jpeg.encode_np(bad)
    with pytest.raises(ValueError):
        jpeg.encode(torch.zeros(1, 16, 24, 3, dtype=torch.uint8))
    with pytest.raises(ValueError):  # a well-formed batch on the host: the device encoder takes CUDA tensors
        jpeg.encode(torch.zeros(1, 16, 16, 3, dtype=torch.uint8))


@pytest.fixture
def files(tmp_path):
    (tmp_path / "data").mkdir()
    for f in ("tocg.pth", "gen.pth"):
        (tmp_path / f).write_bytes(b"")
    return tmp_path


def _args(files, *extra):
    return ["--dataroot", str(files / "data"), "--tocg_checkpoint", str(files / "tocg.pth"), "--gen_checkpoint", str(files / "gen.pth")] + list(extra)


def test_driver_flags(files):
    opt = tryon_run.parse_args(_args(files, "-b", "4", "--occlusion", "--datasetting", "paired", "--fine_width", "192", "--fine_height", "256",
                                     "--seed", "3", "--cuda", "True", "--gpu_ids", "0", "--test_name", "t", "--fp16"))
    assert (opt.batch_size, opt.occlusion, opt.datasetting, opt.fine_height, opt.fine_width, opt.seed, opt.fp16) == (4, True, "paired", 256, 192, 3, True)
    opt = tryon_run.parse_args(_args(files))
    assert (opt.batch_size, opt.datasetting, opt.fine_height, opt.fine_width, opt.clothmask_composition) == (1, "unpaired", 1024, 768, "warp_grad")
    refused = [["--warp_feature", "encoder"], ["--out_layer", "conv"], ["--upsample", "nearest"], ["--num_upsampling_layers", "more"],
               ["--norm_G", "spectralinstance"], ["--semantic_nc", "20"], ["--gen_semantic_nc", "8"], ["--fine_width", "500", "--fine_height", "667"],
               ["--fine_width", "192", "--fine_height", "192"], ["-b", "0"], ["--datasetting", "both"], ["--shuffle"], ["--tensorboard_dir", "x"],
               ["--no_such_flag"]]
    for extra in refused:
        with pytest.raises(SystemExit):
            tryon_run.parse_args(_args(files, *extra))
    with pytest.raises(SystemExit):
        tryon_run.parse_args(["--dataroot", str(files / "missing"), "--tocg_checkpoint", str(files / "tocg.pth"), "--gen_checkpoint", str(files / "gen.pth")])


def test_output_names_from_a_test_batch(tmp_path):
    synth.write_vitonhd(str(tmp_path), 3, h=256, w=192, seed=4, datamode="test", pairs="test_pairs.txt")
    ds = data.VitonHDDataset(str(tmp_path), "test", "test_pairs.txt", 256, 192, mode="test", keys=("cloth", "cloth_mask"))
    batch = data.collate([ds[i] for i in range(3)])
    pairs = [line.split() for line in open(tmp_path / "test_pairs.txt").read().splitlines()]
    for setting in ("paired", "unpaired"):
        got = [tryon_run.output_name(batch["c_name"], setting, i) for i in range(3)]
        want = [p[0].split(".")[0] + "_" + (p[0] if setting == "paired" else p[1]).split(".")[0] + ".png" for p in pairs]
        assert got == want
    assert got[0] != tryon_run.output_name(batch["c_name"], "paired", 0)
