"""Bytes the 16-bit forward / data-gradient convolution stages into shared memory, per layer of a `bench.py --dump-profile` CSV.

    python tools/conv_staging.py TAP.csv [HALO.csv]

TAP.csv is the profile of a build whose convolutions all run the tap-by-tap main loop; HALO.csv (optional) that of a build with the
halo main loop.  For each distinct conv / conv_spade label ("cin->n_gemm kKHxKW nN HxW bk bn", one layer shape) the table gives
launches, time and useful TFLOP/s, the bytes TMA stages under either loop (computed from the shape with the tiling rules of
conv_fwd in csrc/conv_fwd.cuh), the staged TB/s, and whether the halo rule takes the layer.  Staged bytes include TMA's zero fill
(padding, channels past cin, weight rows past n_gemm): it is written to shared memory like data.
"""
import argparse
import csv
import re
import sys
from collections import OrderedDict

ROW = 128                  # bytes of one K block (64 16-bit channels) of one pixel / weight row
BUDGET = 110 * 1024        # dynamic shared memory of one CTA (two CTAs per SM)
HALO_TW = 64
LABEL = re.compile(r"^(\d+)->(\d+) k(\d+)x(\d+) n(\d+) (\d+)x(\d+) bk(\d+) bn(\d+)$")


def pick_pow2(dim, cap):
    best, best_waste = 1, 1e30
    p = 1
    while p <= cap:
        waste = -(-dim // p) * p / dim
        if waste <= best_waste + 0.031:
            best_waste = min(best_waste, waste)
            best = p
        p <<= 1
    return best


def bnt(n_gemm):
    return 64 if n_gemm <= 64 else 128


def halo_slot(kh, kw):
    box = ROW * (HALO_TW + kw - 1) * (1 + kh)
    return box, (box + 1023) // 1024 * 1024


def halo_eligible(cin, n_gemm, kh, kw, w):
    """conv_fwd's rule for the halo main loop of 16-bit storage."""
    chunks = -(-cin // 64)
    return kh * kw > 1 and w % HALO_TW == 0 and chunks * halo_slot(kh, kw)[1] + 2 * bnt(n_gemm) * ROW <= BUDGET - 2048


def staged_bytes(cin, n_gemm, kh, kw, n, h, w, halo):
    """Bytes one launch stages: A and B boxes per K step (tap loop) or one halo box per chunk plus B boxes per K step (halo loop)."""
    chunks = -(-cin // 64)
    bn = bnt(n_gemm)
    kt = kh * kw * chunks
    tiles_n = -(-n_gemm // bn)
    if halo:
        tiles = tiles_n * (w // HALO_TW) * -(-h // 2) * n
        return tiles * (chunks * halo_slot(kh, kw)[0] + kt * bn * ROW)
    tw = pick_pow2(w, 128)
    th = pick_pow2(h, 128 // tw)
    tn = 128 // (tw * th)
    tiles = tiles_n * -(-w // tw) * -(-h // th) * -(-n // tn)
    return tiles * kt * (128 * ROW + bn * ROW)


def read_profile(path):
    layers = OrderedDict()
    with open(path) as f:
        for r in csv.DictReader(f):
            if r["kind"] not in ("conv", "conv_spade"):
                continue
            key = (r["kind"], r["label"])
            e = layers.setdefault(key, [0, 0.0, 0.0])
            e[0] += 1
            e[1] += float(r["ms"])
            e[2] += float(r["work"])
    return layers


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("tap", help="profile CSV of a build with the tap-by-tap loop only")
    ap.add_argument("halo", nargs="?", help="profile CSV of a build with the halo loop")
    ap.add_argument("--top", type=int, default=0, help="only the N layers with the most tap-loop time")
    args = ap.parse_args(argv)
    tap = read_profile(args.tap)
    halo = read_profile(args.halo) if args.halo else {}
    rows = []
    for (kind, label), (launches, ms, flops) in tap.items():
        m = LABEL.match(label)
        if not m:
            continue
        cin, ng, kh, kw, n, h, w = (int(v) for v in m.groups()[:7])
        el = halo_eligible(cin, ng, kh, kw, w)
        b_tap = staged_bytes(cin, ng, kh, kw, n, h, w, False) * launches
        b_halo = staged_bytes(cin, ng, kh, kw, n, h, w, True) * launches if el else b_tap
        rows.append((kind, label, launches, ms, flops, el, b_tap, b_halo, halo.get((kind, label))))
    rows.sort(key=lambda r: -r[3])
    shown = rows[:args.top] if args.top else rows

    hdr = ["layer", "launches", "tap ms", "tap TFLOP/s", "tap GB", "tap TB/s", "halo", "halo GB"]
    if halo:
        hdr += ["halo ms", "halo TFLOP/s", "halo TB/s", "speed-up"]
    print("| " + " | ".join(hdr) + " |")
    print("|" + "---|" * len(hdr))
    for kind, label, launches, ms, flops, el, b_tap, b_halo, new in shown:
        cells = ["%s%s" % (label, " (spade)" if kind == "conv_spade" else ""), "%d" % launches, "%.3f" % ms, "%.0f" % (flops / ms / 1e9),
                 "%.2f" % (b_tap / 1e9), "%.2f" % (b_tap / ms / 1e9), "yes" if el else "no", "%.2f" % (b_halo / 1e9) if el else "-"]
        if halo:
            if new:
                nms = new[1]
                cells += ["%.3f" % nms, "%.0f" % (new[2] / nms / 1e9), "%.2f" % (b_halo / nms / 1e9), "%.2fx" % (ms / nms)]
            else:
                cells += ["-"] * 4
        print("| " + " | ".join(cells) + " |")

    tot = sum(r[3] for r in rows)
    el_ms = sum(r[3] for r in rows if r[5])
    print()
    print("conv launches: %d, %.2f ms, %.0f TFLOP/s; halo-eligible: %.2f ms (%.0f %% of conv time), staged %.1f GB -> %.1f GB"
          % (sum(r[2] for r in rows), tot, sum(r[4] for r in rows) / max(tot, 1e-9) / 1e9, el_ms, 100 * el_ms / max(tot, 1e-9),
             sum(r[6] for r in rows if r[5]) / 1e9, sum(r[7] for r in rows if r[5]) / 1e9))
    if halo:
        new_tot = sum(v[1] for v in halo.values())
        new_el = sum(r[8][1] for r in rows if r[5] and r[8])
        print("halo build: conv %.2f ms (%.2f ms less); halo-eligible layers %.2f ms -> %.2f ms" % (new_tot, tot - new_tot, el_ms, new_el))
    return 0


if __name__ == "__main__":
    sys.exit(main())
