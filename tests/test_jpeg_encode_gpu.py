"""GPU: the device JPEG encoder (hrviton_b200.jpeg.encode) against PIL byte for byte — every size of the seeded corpus in one batched
call, uint8 and fp32 inputs, a batch of 16 at 1024x768, two launches alike, the device decoder reading the result — and tools/test.py
end to end on a synthetic test tree with seeded weights: the file names, every file equal to PIL's encoding of save_images applied to
TryOnGraph's outputs for the same batches and seed, a second run byte-identical, and no module of the reference loaded."""
import collections
import io
import os
import sys
import types

import numpy as np
import pytest
import torch
from PIL import Image

from hrviton_b200 import data, jpeg, pipeline, synth, tryon_run

pytestmark = pytest.mark.gpu


def _pil(rgb):
    buf = io.BytesIO()
    Image.fromarray(rgb).save(buf, format="JPEG")
    return buf.getvalue()


def _save_images_u8(out):
    """utils.save_images' arithmetic as the reference runs it: on the device, then clamp and uint8 on the host."""
    t = ((out.clone() + 1) * 0.5 * 255).cpu().clamp(0, 255)
    return t.numpy().astype("uint8").transpose(0, 2, 3, 1)


def test_corpus_each_size_in_one_call():
    for (h, w), items in synth.encode_corpus(0).items():
        batch = torch.from_numpy(np.stack([a for _, a in items])).cuda()
        for (name, a), g in zip(items, jpeg.encode(batch)):
            assert g == _pil(a), (h, w, name)


def test_fp32_input_and_batch_of_16():
    g = torch.Generator().manual_seed(3)
    x = (torch.rand(16, 3, 1024, 768, generator=g) * 2.4 - 1.2)
    x[:8] = torch.nn.functional.interpolate(x[:8, :, ::64, ::64], size=(1024, 768), mode="bilinear")  # smooth half
    x = x.cuda()
    want = [_pil(a) for a in _save_images_u8(x)]
    got = jpeg.encode(x)
    assert got == want
    assert jpeg.encode(x) == got  # a second launch: the same bytes
    rgb = torch.from_numpy(_save_images_u8(x)).cuda()
    assert jpeg.encode(rgb) == want
    for d, w in zip(jpeg.decode(got[:4]), want[:4]):
        assert np.array_equal(d.cpu().numpy(), np.asarray(Image.open(io.BytesIO(w))))


def _tree_and_weights(tmp_path, n):
    import network_generator
    import networks
    root = tmp_path / "data"
    synth.write_vitonhd(str(root), n, seed=11, datamode="test", pairs="test_pairs.txt")
    topt = types.SimpleNamespace(warp_feature="T1", out_layer="relu", cuda=True)
    tocg = networks.ConditionGenerator(topt, 4, 16, 13, ngf=96, norm_layer=torch.nn.BatchNorm2d)
    sd = tocg.state_dict()
    synth.fill_state_dict(sd, 5)
    torch.save(sd, str(tmp_path / "tocg.pth"))
    gopt = types.SimpleNamespace(norm_G="spectralaliasinstance", gen_semantic_nc=7, semantic_nc=7, ngf=64, num_upsampling_layers="most",
                                 fine_height=256, fine_width=192, cuda=True)
    gen = network_generator.SPADEGenerator(gopt, 9)
    sd = gen.state_dict()
    synth.fill_state_dict(sd, 6)
    out = collections.OrderedDict(sd)
    out._metadata = sd._metadata
    torch.save(out, str(tmp_path / "gen.pth"))
    return root


def test_driver_end_to_end(tmp_path, capsys):
    n, b, seed = 5, 2, 9
    before = set(sys.modules)
    root = _tree_and_weights(tmp_path, n)
    args = ["--dataroot", str(root), "--tocg_checkpoint", str(tmp_path / "tocg.pth"), "--gen_checkpoint", str(tmp_path / "gen.pth"),
            "--fine_width", "192", "--fine_height", "256", "-b", str(b), "-j", "2", "--occlusion", "--seed", str(seed)]
    opt = tryon_run.parse_args(args + ["--output_dir", str(tmp_path / "out1")])
    written = tryon_run.run(opt)
    printed = capsys.readouterr().out
    assert "1 of 5 pairs are left out" in printed and "Test time" in printed
    pairs = [line.split() for line in open(root / "test_pairs.txt").read().splitlines()][:4]
    names = sorted(p[0].split(".")[0] + "_" + p[1].split(".")[0] + ".png" for p in pairs)
    assert sorted(os.listdir(tmp_path / "out1")) == names and len(written) == 4

    # the restatement: the same models, loader and seed through TryOnGraph, save_images' arithmetic, PIL's encoder
    torch.manual_seed(seed)
    torch.cuda.manual_seed(seed)
    tocg, gen = tryon_run.build_models(opt, torch.device("cuda"))
    loader = data.VitonHDLoader(str(root), "test", "test_pairs.txt", 256, 192, b, workers=0, mode="test", keys=tryon_run.TEST_KEYS,
                                shuffle=False, shard=False)
    graph = pipeline.TryOnGraph(tocg, gen, occlusion=True)
    with torch.no_grad():
        for batch in loader:
            for i, a in enumerate(_save_images_u8(graph(batch, datasetting="unpaired")[0])):
                name = tryon_run.output_name(batch["c_name"], "unpaired", i)
                assert (tmp_path / "out1" / name).read_bytes() == _pil(a), name
    graph.release()
    loader.close()

    tryon_run.run(tryon_run.parse_args(args + ["--output_dir", str(tmp_path / "out2")]))
    for name in names:
        assert (tmp_path / "out1" / name).read_bytes() == (tmp_path / "out2" / name).read_bytes(), name
    ref = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref")
    loaded = [k for k in set(sys.modules) - before if ref in (getattr(sys.modules[k], "__file__", None) or "")]
    assert not loaded, loaded
