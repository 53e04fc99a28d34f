"""Lists the arrays that differ between two `bench.py --dump-outputs` directories, with the count of differing elements and the
largest |difference|.  Exit status 0 when every array is bit-identical (and both directories hold the same names), 1 otherwise.

    python tools/compare_dumps.py DIR_A DIR_B"""
import os
import sys

import numpy as np


def compare(a, b):
    """[(name, differing elements, elements, max |a - b|)] for every array that is not bit-identical; arrays present in only one
    directory are listed with a count of -1."""
    na = {f[:-4] for f in os.listdir(a) if f.endswith(".npy")}
    nb = {f[:-4] for f in os.listdir(b) if f.endswith(".npy")}
    rows = [(n, -1, 0, float("nan")) for n in sorted(na ^ nb)]
    for n in sorted(na & nb):
        x, y = np.load(os.path.join(a, n + ".npy")), np.load(os.path.join(b, n + ".npy"))
        if x.shape != y.shape:
            rows.append((n, -1, x.size, float("nan")))
            continue
        xb, yb = x.reshape(-1).view(np.uint8).reshape(x.size, -1), y.reshape(-1).view(np.uint8).reshape(y.size, -1)
        diff = (xb != yb).any(axis=1) if x.size else np.zeros(0, bool)
        if diff.any():
            d = np.abs(x.astype(np.float64) - y.astype(np.float64)).reshape(-1)
            rows.append((n, int(diff.sum()), x.size, float(np.nanmax(d))))
    return rows, len(na | nb)


def main(argv):
    if len(argv) != 3:
        sys.exit(__doc__)
    rows, total = compare(argv[1], argv[2])
    for n, cnt, size, mx in rows:
        print("%-60s %s  max|d| %.3g" % (n, "only in one directory / shape differs" if cnt < 0 else "%d of %d differ" % (cnt, size), mx))
    print("%d of %d arrays differ" % (len(rows), total))
    return 1 if rows else 0


if __name__ == "__main__":
    sys.exit(main(sys.argv))
