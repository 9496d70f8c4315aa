"""Build liblwdetr_b200.so (CUDA kernels + C-ABI) and the CPU oracle helpers.

nvcc cross-compiles for sm_90a without a GPU, so this runs on a machine without a GPU as well.  Objects are cached by source mtime under lw-detr_b200/build/.
"""
import concurrent.futures as cf
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "lw-detr_b200")
CSRC = os.path.join(PKG, "csrc")
OBJ = os.path.join(PKG, "build")
LIB = os.path.join(PKG, "lib", "liblwdetr_b200.so")

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden", "-I", os.path.join(ROOT, "include"), "-I", CSRC,
]


def _stale(out, deps):
    if not os.path.exists(out):
        return True
    t = os.path.getmtime(out)
    return any(os.path.getmtime(d) > t for d in deps)


def _compile(src, obj, headers, verbose):
    if not _stale(obj, [src] + headers):
        return obj
    cmd = [NVCC] + FLAGS + ["-c", src, "-o", obj]
    if verbose:
        print(" ".join(cmd), flush=True)
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed for %s:\n%s\n%s" % (src, r.stdout, r.stderr))
    return obj


def build(verbose=False, force=False):
    os.makedirs(OBJ, exist_ok=True)
    os.makedirs(os.path.dirname(LIB), exist_ok=True)
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".h", ".cuh"))]
    headers += [os.path.join(ROOT, "include", f) for f in os.listdir(os.path.join(ROOT, "include"))]
    srcs = sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cu", ".cpp")))
    if force:
        for f in os.listdir(OBJ):
            os.remove(os.path.join(OBJ, f))
    objs = []
    with cf.ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        futs = [ex.submit(_compile, s, os.path.join(OBJ, os.path.basename(s) + ".o"), headers, verbose) for s in srcs]
        for f in futs:
            objs.append(f.result())
    if _stale(LIB, objs):
        cmd = [NVCC, "-shared", "-o", LIB] + objs + ["-gencode", "arch=compute_90a,code=sm_90a"]
        if verbose:
            print(" ".join(cmd), flush=True)
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("link failed:\n%s\n%s" % (r.stdout, r.stderr))
    return LIB


if __name__ == "__main__":
    print(build(verbose=True, force="--force" in sys.argv))
