"""What the evaluation metrics cost: hrv_ssim against the float64 CPU restatement of skimage's Gaussian SSIM on this machine's host,
and the drop-in LPIPS (eval_models.PerceptualLoss on the kernels) against the reference's PerceptualLoss on torch / cuDNN.

    python tools/metrics_bench.py [--rounds 5] [--calls 20]

SSIM: one 1024x768 uint8 pair and a batch of 8, the images already in device memory for the kernel arm and in host memory for the CPU
arm (tests/metrics_oracle.py, numpy).  LPIPS: 128x128 (the size evaluate.py and train_generator.py resize to) at batch 1 and 8, seeded
weights written to a temporary alex.pth for both arms; the reference arm needs the reference copy under oracle/_ref and is skipped
without it.  The arms agree before they are timed and are timed alternately for --rounds rounds; the columns are those of
tools/inference_graph_bench.py (device_ms over --calls back-to-back calls, host_ms to issue one, latency_ms = one call + synchronize,
median; the CPU arm has latency_ms only).  Medians over the rounds are printed as a table and one JSON line, with the card's name and
power limit."""
import argparse
import contextlib
import io
import json
import os
import statistics
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import hrv_env  # noqa: E402
import hrv_loader  # noqa: E402
from inference_graph_bench import card, measure  # noqa: E402

hrv_loader.load()
import numpy as np  # noqa: E402
import torch  # noqa: E402

import make_golden_lpips as mgl  # noqa: E402  (seeded LPIPS weights)
import metrics_oracle as mo  # noqa: E402


def cpu_latency(fn, calls):
    lat = []
    for _ in range(calls):
        t = time.perf_counter()
        fn()
        lat.append(time.perf_counter() - t)
    return {"latency_ms": 1e3 * statistics.median(lat)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--calls", type=int, default=20)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "metrics_bench measures on the GPU"
    hrv_env.install()
    from hrviton_b200 import metrics
    import eval_models
    rng = np.random.RandomState(0)
    cases = []
    # --- SSIM
    for n in (1, 8):
        a = rng.randint(0, 256, (n, 1024, 768)).astype(np.uint8)
        b = np.clip(a.astype(np.int32) + rng.randint(-20, 21, a.shape), 0, 255).astype(np.uint8)
        da, db = torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()
        got = metrics.ssim(da, db).cpu().numpy()
        ref = np.array([mo.ssim(a[i], b[i]) for i in range(n)])
        assert np.abs(got - ref).max() < 1e-10
        cases.append(("ssim 1024x768 b%d" % n, {"kernel": (lambda da=da, db=db: metrics.ssim(da, db), True),
                                                  "cpu_fp64": (lambda a=a, b=b: [mo.ssim(a[i], b[i]) for i in range(len(a))], False)}))
    # --- LPIPS
    tmp = tempfile.mkdtemp()
    net = metrics.PNetLin(pretrained=False)
    wdir = os.path.join(tmp, "eval_models", "weights", "v0.1")
    os.makedirs(wdir)
    alex = os.path.join(wdir, "alex.pth")
    torch.save(mgl.seeded_state_dict(net.state_dict()), alex)
    os.environ["HRV_ALEX_RANDOM_INIT"] = "1"
    cwd = os.getcwd()
    os.chdir(tmp)
    try:
        with contextlib.redirect_stdout(io.StringIO()):
            ours = eval_models.PerceptualLoss(model="net-lin", net="alex", use_gpu=True)
    finally:
        os.chdir(cwd)
    theirs = None
    if hrv_env.reference_dir():
        with mo.reference_eval_models(alex) as ref_models, contextlib.redirect_stdout(io.StringIO()):
            theirs = ref_models.PerceptualLoss(model="net-lin", net="alex", use_gpu=True)
    for n in (1, 8):
        g = torch.Generator(device="cuda").manual_seed(n)
        x = torch.rand((n, 3, 128, 128), generator=g, device="cuda") * 2 - 1
        y = (x + 0.1 * torch.randn((n, 3, 128, 128), generator=g, device="cuda")).clamp(-1, 1)
        arms = {"drop_in": (lambda x=x, y=y: ours.forward(x, y), True)}
        if theirs is not None:
            with torch.no_grad():
                assert float((ours.forward(x, y) - theirs.forward(x, y)).abs().max()) < 1e-4
            arms["reference_torch"] = (lambda x=x, y=y: theirs.forward(x, y), True)
        cases.append(("lpips 128x128 b%d" % n, arms))
    results = {}
    with torch.no_grad():
        for name, arms in cases:
            for arm, (fn, _) in arms.items():  # warm-up
                fn()
            torch.cuda.synchronize()
            rows = {arm: [] for arm in arms}
            for _ in range(args.rounds):
                for arm, (fn, gpu) in arms.items():
                    rows[arm].append(measure(fn, args.calls) if gpu else cpu_latency(fn, max(2, args.calls // 10)))
            results[name] = {arm: {k: statistics.median(r[k] for r in rs) for k in rs[0]} for arm, rs in rows.items()}
    c = card()
    print("card: %s" % c)
    for name, arms in results.items():
        for arm, r in arms.items():
            print("%-20s %-16s %s" % (name, arm, "  ".join("%s=%.3f" % kv for kv in r.items())))
    print(json.dumps({"card": c, "rounds": args.rounds, "calls": args.calls, "results": results}))


if __name__ == "__main__":
    main()
