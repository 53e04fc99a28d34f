"""Places the UNMODIFIED reference (its .py files) under oracle/_ref/ — git-ignored, but shipped with the working tree — so that
bench.py's reference arm and the tests that run the reference's own training scripts on this repository's drop-in modules can
import them.  The reference is a directory of scripts without setup.py / pyproject.toml, so its files are copied verbatim; nothing
under oracle/_ref is tracked or edited.

The reference checkout is taken from $HRV_REFERENCE_DIR, else from a directory `reference` next to this repository, else from
/root/reference, where the original project is checked out on the build machines.
    python oracle/install_reference.py"""
import os
import shutil
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DST = os.path.join(ROOT, "oracle", "_ref")


def source_dir():
    cands = [os.environ.get("HRV_REFERENCE_DIR"), os.path.join(os.path.dirname(ROOT), "reference"), "/root/reference"]
    for d in cands:
        if d and os.path.isfile(os.path.join(d, "train_generator.py")):
            return d
    return cands[1]


def install(verbose=True):
    src = source_dir()
    if not os.path.isfile(os.path.join(src, "train_generator.py")):
        return os.path.isdir(DST)
    os.makedirs(DST, exist_ok=True)
    n = 0
    for dirpath, dirnames, filenames in os.walk(src):
        dirnames[:] = [d for d in dirnames if not d.startswith(".") and d not in ("figures", "data", "__pycache__")]
        rel = os.path.relpath(dirpath, src)
        for f in filenames:
            if not f.endswith((".py", ".txt", ".md")):
                continue
            os.makedirs(os.path.join(DST, rel), exist_ok=True)
            shutil.copy2(os.path.join(dirpath, f), os.path.join(DST, rel, f))
            n += 1
    if verbose:
        print("oracle/_ref: %d reference files copied verbatim from %s" % (n, src))
    return True


if __name__ == "__main__":
    sys.exit(0 if install() else 1)
