"""Stage the reference's Python forward path under oracle/_ref/ so that the comparisons against it run from this tree.

The reference (Atten4Vis/LW-DETR) is pure Python on this path.  This recipe (run by __graft_entry__.build() whenever a
reference checkout is found at $LWDETR_REFERENCE_SRC) copies the packages the forward imports - models/ and util/ -
byte for byte into oracle/_ref/ (git-ignored: never part of the history), where `bench.py --impl reference`, the
cpu_baseline leg and the tests that drive the reference's own code find it.  Nothing is edited: the three missing third-party imports (timm, fairscale, the compiled
MultiScaleDeformableAttention module) are shimmed at import time by tools/ref_import.py, exactly as for the
golden-vector generator.  MANIFEST.json records the source, the file list and their sha256.

    python oracle/vendor_reference.py            # copy (no-op without a reference checkout)
    python oracle/vendor_reference.py --check    # verify oracle/_ref against its manifest
"""
import hashlib
import json
import os
import shutil
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.environ.get("LWDETR_REFERENCE_SRC", "/root/reference")
DST = os.path.join(ROOT, "oracle", "_ref")
PACKAGES = ("models", "util")            # what `from models import build_model` pulls in (models/__init__.py:16-17)
EXTRA_FILES = ("demo/demo.py",)          # the caller the drop-in tests drive end to end (tests/test_dropin_demo.py)
SKIP_DIRS = {"__pycache__", "src", "build"}   # models/ops/src is the CUDA op's C++/CUDA source: not on the CPU forward


def _sha(path):
    h = hashlib.sha256()
    with open(path, "rb") as f:
        h.update(f.read())
    return h.hexdigest()


def vendor(verbose=False):
    if not os.path.isdir(os.path.join(SRC, "models")):
        return None
    files = {}
    for pkg in PACKAGES:
        for dirpath, dirnames, filenames in os.walk(os.path.join(SRC, pkg)):
            dirnames[:] = [d for d in dirnames if d not in SKIP_DIRS]
            for fn in filenames:
                if not fn.endswith(".py"):
                    continue
                src = os.path.join(dirpath, fn)
                rel = os.path.relpath(src, SRC)
                dst = os.path.join(DST, rel)
                os.makedirs(os.path.dirname(dst), exist_ok=True)
                if not os.path.exists(dst) or _sha(dst) != _sha(src):
                    shutil.copyfile(src, dst)
                files[rel] = _sha(dst)
    for rel in EXTRA_FILES:
        src, dst = os.path.join(SRC, rel), os.path.join(DST, rel)
        if os.path.isfile(src):
            os.makedirs(os.path.dirname(dst), exist_ok=True)
            if not os.path.exists(dst) or _sha(dst) != _sha(src):
                shutil.copyfile(src, dst)
            files[rel] = _sha(dst)
    with open(os.path.join(DST, "MANIFEST.json"), "w") as f:
        json.dump({"source": "Atten4Vis/LW-DETR (unmodified files, copied by oracle/vendor_reference.py)", "packages": PACKAGES,
                   "files": files}, f, indent=1, sort_keys=True)
    if verbose:
        print("vendored %d reference files into %s" % (len(files), DST))
    return DST


def check():
    man = os.path.join(DST, "MANIFEST.json")
    if not os.path.exists(man):
        return False
    with open(man) as f:
        files = json.load(f)["files"]
    return all(os.path.exists(os.path.join(DST, rel)) and _sha(os.path.join(DST, rel)) == h for rel, h in files.items())


if __name__ == "__main__":
    if "--check" in sys.argv:
        ok = check()
        print("oracle/_ref:", "ok" if ok else "missing or modified")
        sys.exit(0 if ok else 1)
    print(vendor(verbose=True) or "no reference at %s - nothing to do" % SRC)
