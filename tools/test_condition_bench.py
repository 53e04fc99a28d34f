"""Stage-1 test run and PNG encoding: the device against the reference's host path.

    python tools/test_condition_bench.py [--samples 64] [--batch 8] [--out results/test_condition_bench.json]

Prints one JSON line per measurement, with the card's name and power limit read in the same run:
  * tool: samples/s of tools/test_condition.py (condition_run.run: loader, ConditionGraph with the discriminator, grid kernel, device
    PNG encoder, writer thread) over a synthetic 1024x768 VITON-HD test tree at 256x192, second run (the first captures the graph);
  * loader: samples/s of the loader alone over the same tree (what bounds the tool when it is the slower of the two);
  * reference: samples/s of the reference's test_condition.test(), unchanged, on the drop-in modules over the same batches already
    moved to the CPU (its loader is not timed), fp32 storage for both, as the reference computes in fp32;
  * encode: png.encode of a batch of 8 776x778 grids (one sync included) against PIL's Image.save(format='PNG') of the same arrays,
    on one core and on a thread pool over every core.
The synthetic tree and the output files go to a temporary directory."""
import argparse
import concurrent.futures
import contextlib
import io
import json
import os
import subprocess
import sys
import tempfile
import time
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import hrv_loader  # noqa: E402

hrv_loader.load()


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        name, power = [s.strip() for s in q.stdout.splitlines()[0].split(",")]
        return {"gpu": name, "power_limit": power}
    except Exception as e:  # noqa: BLE001 - reported as is
        return {"gpu": "unknown (%s)" % e, "power_limit": "unknown"}


def main(argv=None):
    p = argparse.ArgumentParser()
    p.add_argument("--samples", type=int, default=64)
    p.add_argument("--batch", type=int, default=8)
    p.add_argument("--out", default=None)
    a = p.parse_args(argv)
    a.out = a.out and os.path.abspath(a.out)
    import numpy as np
    import torch
    from PIL import Image

    import hrv_env
    from hrviton_b200 import condition_run, data, ops, png, synth
    from test_png_cpu import grid_fixture
    from test_rejection_cpu import reject_case
    info = card()
    lines = []

    def emit(d):
        d = dict(d, **info)
        lines.append(d)
        print(json.dumps(d), flush=True)

    tmp = tempfile.mkdtemp(prefix="hrv_tc_bench_")
    root = os.path.join(tmp, "data")
    synth.write_vitonhd(root, a.samples, seed=41, datamode="test", pairs="test_pairs.txt")
    g, sd_t, sd_d, _, _, _ = reject_case()
    os.makedirs(os.path.join(tmp, "ckpt"))
    torch.save(sd_t, os.path.join(tmp, "ckpt", "tocg.pth"))
    torch.save(sd_d, os.path.join(tmp, "ckpt", "D.pth"))
    os.chdir(tmp)
    argv = ["--dataroot", root, "--tocg_checkpoint", "ckpt/tocg.pth", "--D_checkpoint", "ckpt/D.pth", "--norm_const", repr(float(g["M"])),
            "-b", str(a.batch), "-j", "4", "--Ddownx2", "--Ddropout"]
    opt = condition_run.parse_args(argv)
    n = a.samples // a.batch * a.batch
    for precision in ("bf16", "fp32"):
        ops.set_precision(precision)
        for rep in range(2):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            with contextlib.redirect_stdout(io.StringIO()):
                condition_run.run(opt, log=lambda *x: None)
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
        emit({"what": "tool", "precision": precision, "samples": n, "seconds": dt, "samples_per_s": n / dt})
    loader = data.VitonHDLoader(root, "test", "test_pairs.txt", 256, 192, a.batch, workers=4, mode="test", keys=condition_run.GRID_KEYS,
                                shuffle=False, shard=False)
    for rep in range(2):
        t0 = time.perf_counter()
        for _ in loader:
            pass
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
    loader.close()
    emit({"what": "loader", "samples": n, "seconds": dt, "samples_per_s": n / dt})

    # the reference's loop over the same batches on the CPU
    keys = condition_run.GRID_KEYS + ("pose", "parse_onehot")
    loader = data.VitonHDLoader(root, "test", "test_pairs.txt", 256, 192, a.batch, workers=4, mode="test", keys=keys, shuffle=False, shard=False)
    batches = [{k: ({s: t.cpu() for s, t in v.items()} if isinstance(v, dict) and k != "c_name" else (v.cpu() if torch.is_tensor(v) else v))
                for k, v in b.items()} for b in loader]
    loader.close()
    ops.set_precision("fp32")
    tcond = hrv_env.load_reference_script("test_condition")
    tocg, D = condition_run.build_models(opt, torch.device("cuda"), True)
    ropt = types.SimpleNamespace(tocg_checkpoint="ref/tocg.pth", datamode="test", datasetting="paired", clothmask_composition="warp_grad",
                                 norm_const=float(g["M"]))
    for rep in range(2):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        with contextlib.redirect_stdout(io.StringIO()):
            tcond.test(ropt, types.SimpleNamespace(data_loader=batches), None, tocg, D)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
    emit({"what": "reference", "precision": "fp32", "samples": n, "seconds": dt, "samples_per_s": n / dt})

    # the encoder against PIL on 8 grids
    grid = grid_fixture()
    grids = np.stack([np.roll(grid, 7 * i, axis=1) for i in range(8)])
    dev = torch.from_numpy(grids).cuda()
    for _ in range(3):
        png.encode(dev)
    reps = 20
    t0 = time.perf_counter()
    for _ in range(reps):
        files = png.encode(dev)
    enc_ms = (time.perf_counter() - t0) / reps * 1e3

    def pil(x):
        f = io.BytesIO()
        Image.fromarray(x).save(f, format="PNG")
        return len(f.getvalue())

    t0 = time.perf_counter()
    sizes = [pil(x) for x in grids]
    one_ms = (time.perf_counter() - t0) * 1e3
    cores = os.cpu_count() or 1
    with concurrent.futures.ThreadPoolExecutor(cores) as ex:
        list(ex.map(pil, grids))
        t0 = time.perf_counter()
        list(ex.map(pil, grids))
        pool_ms = (time.perf_counter() - t0) * 1e3
    emit({"what": "encode", "images": 8, "shape": list(grids.shape[1:]), "png_encode_ms": enc_ms, "pil_one_core_ms": one_ms,
          "pil_pool_ms": pool_ms, "pool_threads": cores, "bytes_vs_pil": sum(map(len, files)) / sum(sizes)})
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(lines, f, indent=1)


if __name__ == "__main__":
    main()
