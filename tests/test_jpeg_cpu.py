"""CPU: the JPEG host side (hrviton_b200.jpeg) — the marker parser against PIL's fields, decode_np (the numpy statement of the device
decoder) against PIL byte for byte, which files device_decodable keeps on PIL, and the refusal of cut files."""
import ctypes
import io

import numpy as np
import pytest
from PIL import Image

import hrv_loader

hrv_loader.load()
from hrviton_b200 import jpeg, synth  # noqa: E402

CORPUS = synth.jpeg_corpus(0)


@pytest.fixture(scope="module")
def synth_file(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("vitonhd"))
    synth.write_vitonhd(root, 1, seed=7)
    with open(root + "/train/image/000000_00.jpg", "rb") as f:
        return f.read()


def test_corpus_covers_the_cases():
    names = [n for n, _ in CORPUS]
    for part in ("1x1_", "8x8_", "9x17_", "45x67_", "256x192_", "_q1_", "_q100_", "_s0", "_s1", "_s2", "_opt_", "_rstb_", "_rstr_", "_L_"):
        assert any(part in n for n in names), part
    samplings = {tuple((c[1], c[2]) for c in jpeg.parse(d).components) for _, d in CORPUS}
    assert {((1, 1), (1, 1), (1, 1)), ((2, 1), (1, 1), (1, 1)), ((2, 2), (1, 1), (1, 1)), ((1, 1),)} <= samplings
    assert any(jpeg.parse(d).restart_interval for _, d in CORPUS)


@pytest.mark.parametrize("i", range(len(CORPUS)), ids=[n for n, _ in CORPUS])
def test_parser_and_decode_np_match_pil(i):
    name, d = CORPUS[i]
    im = Image.open(io.BytesIO(d))
    h = jpeg.parse(d)
    assert (h.size, h.mode) == (im.size, im.mode)
    assert h.layer == [tuple(int(v) for v in t) for t in im.layer]
    assert h.quantization == {k: list(v) for k, v in im.quantization.items()}
    assert jpeg.device_decodable(h)
    got, want = jpeg.decode_np(d), np.asarray(im)
    assert got.dtype == np.uint8 and got.shape == want.shape and np.array_equal(got, want), name
    if h.mode == "L":
        assert np.array_equal(jpeg.decode_np(d, rgb=True), np.asarray(im.convert("RGB")))


def test_decode_np_synth_tree_file(synth_file):
    assert np.array_equal(jpeg.decode_np(synth_file), np.asarray(Image.open(io.BytesIO(synth_file))))


def _save(im, **kw):
    buf = io.BytesIO()
    im.save(buf, "JPEG", **kw)
    return buf.getvalue()


def test_pil_only_files_are_not_device_decodable():
    rgb = Image.fromarray(np.random.default_rng(0).integers(0, 256, (24, 40, 3), dtype=np.uint8))
    progressive = jpeg.parse(_save(rgb, progressive=True))
    assert progressive.sof == 0xC2 and not jpeg.device_decodable(progressive)
    cmyk = jpeg.parse(_save(rgb.convert("CMYK")))
    assert cmyk.mode == "CMYK" and not jpeg.device_decodable(cmyk)
    rgb_coded = jpeg.parse(_save(rgb, keep_rgb=True))  # component ids 'R', 'G', 'B' and Adobe transform 0: no colour conversion
    assert rgb_coded.color_space() == "RGB" and not jpeg.device_decodable(rgb_coded)
    with pytest.raises(ValueError, match="not a file the device decodes"):
        jpeg.decode_np(_save(rgb, progressive=True))


def test_cut_file_is_refused_like_pil():
    d = dict(CORPUS)["256x192_q95_s2"]
    for cut in (len(d) - 2, len(d) // 2, 200):
        with pytest.raises(OSError, match="(?i)truncated"):
            Image.open(io.BytesIO(d[:cut])).load()
        with pytest.raises(OSError, match="(?i)truncated"):
            jpeg.parse(d[:cut])


def test_short_entropy_segment_is_an_error():
    """A well-formed file whose entropy-coded data was cut short (the EOI moved up) parses, but decoding it raises."""
    d = dict(CORPUS)["256x192_q95_s2"]
    h = jpeg.parse(d)
    s0, s1 = h.segment
    short = d[:s0 + (s1 - s0) // 2] + b"\xff\xd9"
    assert jpeg.device_decodable(jpeg.parse(short))
    with pytest.raises(ValueError, match="truncated"):
        jpeg.decode_np(short)


def test_descriptor_layout():
    """jpeg.Image mirrors include/hrviton_sm100_jpeg.h's hrv_jpeg_image (jpeg_kernels.cu asserts the same size)."""
    assert ctypes.sizeof(jpeg.Image) == 2120
    assert jpeg.Image.quant.offset == 100 and jpeg.Image.vals.offset == 580
