"""Measures stage-1 validation (TrainRun.validate, `train.py stage1 --val_count`) on one GPU:

  1. one validation: 2000 test samples at 256x192, batch 8 (250 batches), as train_loop.validation_iou runs it through
     pipeline.SegmentationGraph (re-captured once, as after every stretch of training), against an eager loop over the same batches:
     the package's eval-mode tocg, torch's soft-max and iou_metric as train_condition.py:18-36 writes it, on the GPU, with one .item()
     per batch as the reference reads it.  Each arm is timed end to end from the loader (synthetic 1024x768 JPEG/PNG tree whose
     test list cycles over --unique samples) and on the compute alone (8 batches resident on the device, cycled).  Before every
     timed arm the parameter generation is bumped, as a training replay bumps it, so both arms rebuild the derived weights (packed
     convolutions, folded BatchNorm) they read; the graph's first call after such a change (re-capture and one replay) is also timed
     on its own;
  2. the stage-1 graph step (batch 8, bf16) from the same loader, and the step amortised over 1000 steps with one validation every
     1000 steps (--val_count 1000): step + validation / 1000, both measured in this call;
  3. the card name and power limit.

    python tools/val_bench.py [--unique 64] [--rounds 2] [--steps 30]"""
import argparse
import json
import os
import shutil
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
B, SAMPLES = 8, 2000


def _gpu():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    except OSError:
        return "unknown"


def _reference_iou_metric(y_pred_batch, y_true_batch):
    """train_condition.py:18-36 as written."""
    import torch
    B = y_pred_batch.shape[0]
    iou = 0
    for i in range(B):
        y_pred = (y_pred_batch[i] > 0.5).flatten()
        y_true = y_true_batch[i].flatten()
        intersection = torch.sum(y_pred[y_true == 1])
        union = torch.sum(y_pred) + torch.sum(y_true)
        iou += (intersection + 1e-7) / (union - intersection + 1e-7) / B
    return iou


def _eager_batch_iou(tocg, b):
    import torch
    import torch.nn.functional as F
    pick = lambda v: v["paired"] if isinstance(v, dict) else v
    input1 = torch.cat([pick(b["cloth"]), (pick(b["cloth_mask"]) > 0.5).float()], 1)
    input2 = torch.cat([b["parse_agnostic"], b["densepose"]], 1)
    _, seg, _, wcm = tocg(input1, input2)
    mask = torch.ones_like(seg)
    mask[:, 3:4] = wcm
    return _reference_iou_metric(F.softmax(seg * mask, dim=1), b["parse"]).item()


def _timed(fn):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    v = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, v


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--unique", type=int, default=64, help="distinct samples in the synthetic test tree (its list cycles over them)")
    p.add_argument("--rounds", type=int, default=2)
    p.add_argument("--steps", type=int, default=30)
    p.add_argument("--workers", type=int, default=min(8, os.cpu_count() or 1))
    a = p.parse_args()
    import hrv_loader
    hrv_loader.load()
    os.environ.setdefault("HRV_VGG_RANDOM_INIT", "1")
    import numpy as np
    import torch

    from hrviton_b200 import data, ops, pipeline, synth, train_loop
    tmp = tempfile.mkdtemp(prefix="val_bench_")
    synth.write_vitonhd(tmp, 16, seed=1, datamode="train")
    names = synth.write_vitonhd(tmp, a.unique, seed=2, datamode="test", pairs="unique_pairs.txt")
    with open(os.path.join(tmp, "test_pairs.txt"), "w") as f:
        f.write("".join("%s %s\n" % (names[i % a.unique], names[(i + 1) % a.unique]) for i in range(SAMPLES)))
    flags = ["--name", "bench", "--dataroot", tmp, "--data_list", "pairs.txt", "-b", str(B), "-j", str(a.workers), "--checkpoint_dir",
             os.path.join(tmp, "ckpt"), "--display_count", "1000000", "--save_count", "1000000", "--keep_step", "1000000", "--occlusion",
             "--val_count", "1000", "--test_dataroot", tmp, "--test_data_list", "test_pairs.txt"]
    run = train_loop.build(train_loop.parse_args("stage1", flags), log=lambda *x: None)
    loader, tocg = run.validator, run.trainer.tocg
    result = {"gpu": _gpu(), "host_cpus": os.cpu_count(), "workers": a.workers, "batch": B, "samples": SAMPLES, "size": "256x192"}
    try:
        run.start()
        run.train(until=5)  # warm-up steps
        ms, _ = _timed(lambda: run.train(until=5 + a.steps))
        step_ms = ms / a.steps
        # one validation from the loader: graph runner vs the eager loop, alternating
        val = {"graph": [], "eager": []}
        values = {}
        cached = None
        for _ in range(a.rounds):
            ops.PARAM_GEN[0] += 1  # as after training steps: the graph re-captures once
            ms, values["graph"] = _timed(run.validate)
            val["graph"].append(ms)
            ops.PARAM_GEN[0] += 1  # the eager arm rebuilds its derived weights too
            tocg.eval()
            try:
                def eager():
                    loader.start_at(0, 0)
                    with torch.no_grad():
                        return float(np.mean([_eager_batch_iou(tocg, loader.next_batch()) for _ in range(SAMPLES // B)]))
                ms, values["eager"] = _timed(eager)
                val["eager"].append(ms)
                if cached is None:
                    loader.start_at(0, 0)
                    cached = [{k: ({s: t.clone() for s, t in v.items()} if isinstance(v, dict) else v.clone()) for k, v in loader.next_batch().items()
                               if k in train_loop.VAL_KEYS} for _ in range(8)]
            finally:
                tocg.train()
        # the compute alone: 250 batches cycled from 8 resident ones
        comp = {"graph": [], "eager": []}
        first_call = []
        tocg.eval()
        try:
            runner = pipeline.SegmentationGraph(tocg)
            runner(cached[0])
            for _ in range(a.rounds):
                ops.PARAM_GEN[0] += 1
                first_call.append(_timed(lambda: runner(cached[0]).item())[0])
            for _ in range(a.rounds):
                def graph():
                    ious = torch.empty(SAMPLES // B, device="cuda")
                    for i in range(SAMPLES // B):
                        ious[i] = runner(cached[i % 8])
                    return float(np.mean(ious.tolist()))
                comp["graph"].append(_timed(graph)[0])
                with torch.no_grad():
                    comp["eager"].append(_timed(lambda: [_eager_batch_iou(tocg, cached[i % 8]) for i in range(SAMPLES // B)])[0])
            runner.release()
        finally:
            tocg.train()
        val_ms = statistics.median(val["graph"])
        result.update({
            "validation_ms": {k: {"rounds": v, "median": statistics.median(v)} for k, v in val.items()},
            "validation_compute_ms": {k: {"rounds": v, "median": statistics.median(v)} for k, v in comp.items()},
            "graph_first_call_after_weight_change_ms": {"rounds": first_call, "median": statistics.median(first_call)},
            "iou": values,
            "stage1_step_ms": step_ms,
            "stage1_step_ms_with_val_count_1000": step_ms + val_ms / 1000.0,
        })
    finally:
        run.trainer.release_graph()
        if run._seg is not None:
            run._seg.release()
        for ld in (run.loader, run.validator):
            ld.close()
        shutil.rmtree(tmp, ignore_errors=True)
    print(json.dumps(result, indent=1))


if __name__ == "__main__":
    main()
