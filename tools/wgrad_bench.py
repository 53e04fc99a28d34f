"""Per-layer timing of hrv_conv2d_wgrad at the shapes one training step runs (CUDA events, device-resident seeded inputs).

The shapes come from the `wgrad` rows of a `bench.py --dump-profile` CSV (label `cin->cout kKxK nN HxW`, HxW the dY extent); each
distinct shape is timed once and counted as often as the step runs it.  Per shape it prints the time per call, the useful rate
(2 cin cout K^2 N H W FLOP), the MMA work the kernel's tiling issues, issued / useful, and the bytes TMA stages into shared memory
per useful FLOP, which follow from the host plan of the kernel named by --kernel:
  parent  M = cout in 128-row tiles, N = cin in 64-column (cin <= 64) or 128-column tiles
  tiled   M = cin or cout, N in 128-, 64- or 32-column tiles with an optional narrower last tile (conv_wgrad.cu, wgrad_plan)
Usage: python tools/wgrad_bench.py --profile prof.csv [--root TREE] [--kernel tiled|parent] [--reps 20]"""
import argparse
import collections
import csv
import os
import re
import subprocess
import sys

PX = 64  # pixels per pipeline stage (kPX)
TILE_COST = 32


def plan_parent(cin, cout):
    bn = 64 if cin <= 64 else 128
    m_tiles = (cout + 127) // 128
    n_widths = [bn] * ((cin + bn - 1) // bn)
    return "M=cout", m_tiles, n_widths


def plan_tiled(cin, cout):
    best = None
    for a_is_x in (0, 1):
        cm, cn = (cin, cout) if a_is_x else (cout, cin)
        mt = (cm + 127) // 128
        for bn, bt in ((128, 0), (128, 64), (128, 32), (64, 0), (32, 0)):
            rem = cn % bn
            if bt and (rem == 0 or rem > bt):
                continue
            widths = [bn] * (cn // bn) + [bt] if bt else [bn] * ((cn + bn - 1) // bn)
            cost = mt * sum(w + TILE_COST for w in widths)
            if best is None or cost < best[0]:
                best = (cost, "M=cin" if a_is_x else "M=cout", mt, widths)
    return best[1:]


def stage_bytes(w, kernel):
    if kernel == "parent":
        return PX * 128 * (2 + w // 64)
    return 2 * PX * 128 + (PX * 64 if w == 32 else PX * 128 * (w // 64))


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--profile", required=True, help="CSV written by bench.py --dump-profile")
    ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                    help="source tree whose built library to time (default: this one)")
    ap.add_argument("--kernel", default="tiled", choices=["tiled", "parent"], help="tiling rules for the issued-work columns")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()

    shapes = collections.Counter()
    with open(args.profile) as f:
        for row in csv.DictReader(f):
            if row["kind"] != "wgrad":
                continue
            m = re.match(r"(\d+)->(\d+) k(\d+)x(\d+) n(\d+) (\d+)x(\d+)", row["label"])
            shapes[tuple(int(v) for v in m.groups())] += 1
    if not shapes:
        sys.exit("no wgrad rows in %s" % args.profile)

    sys.path.insert(0, os.path.abspath(args.root))
    import hrv_loader
    hrv_loader.load()
    import torch
    from hrviton_b200 import ops
    from hrviton_b200.ops import Act

    if not torch.cuda.is_available():
        sys.exit("wgrad_bench needs a GPU")
    plan = plan_tiled if args.kernel == "tiled" else plan_parent
    print("card: %s (name, power limit, max SM clock)" % card())
    print("library: %s  tiling: %s" % (os.path.abspath(args.root), args.kernel))
    hdr = "%-28s %3s %-6s %-14s %9s %9s %9s %9s %7s %9s" % ("layer (cin->cout kKxK nN HxW)", "x", "M", "N tiles", "ms/call", "useful TF",
                                                           "TF/s", "issued TF", "iss/use", "B/FLOP")
    print(hdr)
    tot = collections.Counter()
    g = torch.Generator(device="cuda").manual_seed(1234)
    for (cin, cout, kh, kw, n, h, w), count in sorted(shapes.items(), key=lambda kv: -kv[0][0] * kv[0][1] * kv[0][2] * kv[0][3] * kv[0][5] * kv[0][6] * kv[1]):
        pad = kh // 2
        x = Act(torch.randn((n, h, w, ops.round_up(cin, 8)), generator=g, device="cuda").to(ops.STORAGE[0]), c=cin)
        dy = Act(torch.randn((n, h, w, ops.round_up(cout, 8)), generator=g, device="cuda").to(ops.STORAGE[0]), c=cout)
        for _ in range(args.warmup):
            ops.conv2d_wgrad(x, dy, kh, kw, pad)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.reps):
            ops.conv2d_wgrad(x, dy, kh, kw, pad)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / args.reps
        del x, dy

        side, mt, widths = plan(cin, cout)
        chunks = n * h * ((w + PX - 1) // PX)
        useful = 2.0 * cin * cout * kh * kw * n * h * w
        issued = 2.0 * mt * 128 * sum(widths) * kh * kw * chunks * PX
        staged = float(mt * sum(stage_bytes(wd, args.kernel) for wd in widths) * kh * kw * chunks)
        label = "%d->%d k%dx%d n%d %dx%d" % (cin, cout, kh, kw, n, h, w)
        ntiles = "+".join("%dx%d" % (widths.count(v), v) for v in sorted(set(widths), reverse=True))
        print("%-28s %3d %-6s %-14s %9.3f %9.3f %9.1f %9.3f %7.2f %9.4f" % (label, count, side, "%dx(%s)" % (mt, ntiles), ms, useful / 1e12,
                                                                           useful / (ms * 1e-3) / 1e12, issued / 1e12, issued / useful, staged / useful))
        tot["ms"] += ms * count
        tot["useful"] += useful * count
        tot["issued"] += issued * count
        tot["staged"] += staged * count
    print("TOTAL: %.2f ms per step, useful %.3f TFLOP at %.1f TFLOP/s, issued %.3f TFLOP (issued / useful %.2f), %.4f B staged per useful FLOP"
          % (tot["ms"], tot["useful"] / 1e12, tot["useful"] / (tot["ms"] * 1e-3) / 1e12, tot["issued"] / 1e12, tot["issued"] / tot["useful"],
             tot["staged"] / tot["useful"]))


if __name__ == "__main__":
    main()
