"""Measures test-set inference with device JPEG encoding (hrviton_b200.tryon_run, tools/test.py) on one GPU:

  1. jpeg.encode of fp32 generator-like output at 1024x768, batches of 1, 4 and 16 (CUDA events around the call, which includes the
     two device-to-host copies, after warm-up), against PIL's encode of the same images on one host core;
  2. tools/test.py end to end on a synthetic 1024x768 test tree (-b 4, 4 workers, seeded random weights), in samples/s, against an
     arm that writes through utils.save_images' CPU path (device-to-host of the fp32 output, clamp, uint8, PIL) in a thread pool;
     the arms alternate over --rounds rounds;
  3. bytes copied device-to-host per image by each arm.

    python tools/test_bench.py [--samples 64] [--rounds 3]"""
import argparse
import concurrent.futures
import io
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def _gpu():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    except OSError:
        return "unknown"


def _images(n, seed):
    import torch
    g = torch.Generator().manual_seed(seed)
    low = torch.rand(n, 3, 16, 12, generator=g) * 2 - 1
    x = torch.nn.functional.interpolate(low, size=(1024, 768), mode="bilinear") + 0.05 * torch.randn(n, 3, 1024, 768, generator=g)
    return x.clamp(-1.05, 1.05).cuda()


def encode_times(reps=10):
    import numpy as np
    import torch
    from PIL import Image

    from hrviton_b200 import jpeg
    out = {}
    for n in (1, 4, 16):
        x = _images(n, n)
        for _ in range(3):
            jpeg.encode(x)
        times = []
        for _ in range(reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            files = jpeg.encode(x)
            b.record()
            b.synchronize()
            times.append(a.elapsed_time(b))
        stats = {}
        jpeg.encode(x, stats=stats)
        u8 = ((x + 1) * 0.5 * 255).cpu().clamp(0, 255).numpy().astype("uint8").transpose(0, 2, 3, 1)
        pil = []
        for rgb in np.concatenate([u8] * max(1, 8 // n)):
            t = time.perf_counter()
            buf = io.BytesIO()
            Image.fromarray(rgb).save(buf, format="JPEG")
            pil.append((time.perf_counter() - t) * 1e3)
        out[n] = {"device_ms_per_batch": statistics.median(times), "device_ms_min": min(times), "device_ms_max": max(times),
                  "pil_ms_per_image": statistics.median(pil), "pil_ms_min": min(pil), "pil_ms_max": max(pil),
                  "bytes_per_image": sum(map(len, files)) / n, "d2h_bytes_per_image": stats["d2h_bytes"] / n}
    return out


def _save_images_arm(opt, log=lambda *a: None):
    """tools/test.py's loop with utils.save_images' CPU path (fp32 output to the host, clamp, uint8, PIL) in a thread pool instead
    of the device encoder.  Returns (files, device-to-host bytes)."""
    import torch
    from PIL import Image

    from hrviton_b200 import data, pipeline, tryon_run
    tocg, gen = tryon_run.build_models(opt, torch.device("cuda"))
    torch.cuda.manual_seed(opt.seed)
    loader = data.VitonHDLoader(opt.dataroot, opt.datamode, opt.data_list, opt.fine_height, opt.fine_width, opt.batch_size,
                                workers=opt.workers, mode="test", keys=tryon_run.TEST_KEYS, shuffle=False, shard=False)
    graph = pipeline.TryOnGraph(tocg, gen, occlusion=opt.occlusion, clothmask_composition=opt.clothmask_composition)
    os.makedirs(opt.output_dir, exist_ok=True)

    def save(array, path):
        Image.fromarray(array).save(path, format="JPEG")

    n, d2h = 0, 0
    try:
        with concurrent.futures.ThreadPoolExecutor(opt.workers) as pool, torch.no_grad():
            pending = []
            for batch in loader:
                out = graph(batch, datasetting=opt.datasetting)[0]
                host = ((out.clone() + 1) * 0.5 * 255).cpu().clamp(0, 255)
                d2h += host.numel() * 4
                arrays = host.numpy().astype("uint8").transpose(0, 2, 3, 1)
                for i, a in enumerate(arrays):
                    pending.append(pool.submit(save, a, os.path.join(opt.output_dir, tryon_run.output_name(batch["c_name"], opt.datasetting, i))))
                n += len(arrays)
            for f in pending:
                f.result()
    finally:
        graph.release()
        loader.close()
    return n, d2h


def end_to_end(samples, rounds):
    import collections
    import types

    import torch

    import network_generator
    import networks
    from hrviton_b200 import jpeg, synth, tryon_run
    tmp = tempfile.mkdtemp(prefix="test_bench_")
    root = os.path.join(tmp, "data")
    synth.write_vitonhd(root, samples, seed=2, datamode="test", pairs="test_pairs.txt")
    topt = types.SimpleNamespace(warp_feature="T1", out_layer="relu", cuda=True)
    t = networks.ConditionGenerator(topt, 4, 16, 13, ngf=96, norm_layer=torch.nn.BatchNorm2d)
    sd = t.state_dict()
    synth.fill_state_dict(sd, 1)
    torch.save(sd, os.path.join(tmp, "tocg.pth"))
    gopt = types.SimpleNamespace(norm_G="spectralaliasinstance", gen_semantic_nc=7, semantic_nc=7, ngf=64, num_upsampling_layers="most",
                                 fine_height=1024, fine_width=768, cuda=True)
    g = network_generator.SPADEGenerator(gopt, 9)
    sd = g.state_dict()
    synth.fill_state_dict(sd, 2)
    out = collections.OrderedDict(sd)
    out._metadata = sd._metadata
    torch.save(out, os.path.join(tmp, "gen.pth"))
    res = {"device": [], "save_images": []}
    d2h = {}
    for r in range(rounds):
        for arm in ("device", "save_images") if r % 2 == 0 else ("save_images", "device"):
            opt = tryon_run.parse_args(["--dataroot", root, "--tocg_checkpoint", os.path.join(tmp, "tocg.pth"), "--gen_checkpoint",
                                        os.path.join(tmp, "gen.pth"), "-b", "4", "-j", "4", "--occlusion", "--output_dir",
                                        os.path.join(tmp, "out_" + arm)])
            t0 = time.perf_counter()
            if arm == "device":
                stats = {}
                orig = jpeg.encode
                tryon_run.jpeg.encode = lambda x, **kw: orig(x, stats=stats)
                try:
                    n = len(tryon_run.run(opt, log=lambda *a: None))
                finally:
                    tryon_run.jpeg.encode = orig
                d2h[arm] = stats["d2h_bytes"] / n
            else:
                n, b = _save_images_arm(opt)
                d2h[arm] = b / n
            res[arm].append(n / (time.perf_counter() - t0))
    return {arm: {"samples_per_s": v, "median": statistics.median(v), "d2h_bytes_per_image": d2h[arm]} for arm, v in res.items()}


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--samples", type=int, default=64)
    p.add_argument("--rounds", type=int, default=3)
    a = p.parse_args()
    import hrv_loader
    hrv_loader.load()
    os.environ.setdefault("HRV_VGG_RANDOM_INIT", "1")
    result = {"gpu": _gpu(), "host_cpus": os.cpu_count(), "encode": encode_times(), "end_to_end": end_to_end(a.samples, a.rounds)}
    print(json.dumps(result, indent=1))


if __name__ == "__main__":
    main()
