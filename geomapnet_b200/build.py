"""Builds geomapnet_b200/csrc/libmapnet_b200.so in-tree with nvcc for sm_90a (H100).

    python -m geomapnet_b200.build [--force]

The shared library is a plain C ABI (include/mapnet_b200.h): no torch, no
pybind -- Python binds it with ctypes (geomapnet_b200/_lib.py).  It is a build
product and git-ignored.
"""
import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(CSRC, "libmapnet_b200.so")
OBJ = os.path.join(CSRC, "_obj")
SOURCES = ["api.cu", "net.cu", "bn.cu", "conv_simt.cu", "conv_tc.cu", "layout.cu", "head.cu", "loss.cu", "adam.cu",
           "optim.cu", "preprocess.cu", "pgo.cu"]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
         "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr", "-Xptxas", "-v"]


def _digest():
    h = hashlib.sha256()
    for root in (CSRC, os.path.join(os.path.dirname(HERE), "include")):
        for f in sorted(os.listdir(root)):
            if f.endswith((".cu", ".cuh", ".h")):
                with open(os.path.join(root, f), "rb") as fh:
                    h.update(f.encode()); h.update(fh.read())
    h.update(" ".join(FLAGS).encode())
    return h.hexdigest()


def _compile(src):
    obj = os.path.join(OBJ, src.replace(".cu", ".o"))
    cmd = [NVCC] + FLAGS + ["-c", os.path.join(CSRC, src), "-o", obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    with open(obj + ".log", "w") as f:
        f.write(" ".join(cmd) + "\n" + r.stdout + r.stderr)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed for %s:\n%s" % (src, r.stderr[-6000:]))
    return obj


def build(force=False, verbose=True):
    os.makedirs(OBJ, exist_ok=True)
    stamp = os.path.join(OBJ, "digest.txt")
    dig = _digest()
    if not force and os.path.exists(OUT) and os.path.exists(stamp) and open(stamp).read() == dig:
        return OUT
    if not os.path.exists(NVCC):
        raise RuntimeError("nvcc not found at %s and no up-to-date %s present" % (NVCC, OUT))
    with ThreadPoolExecutor(max_workers=min(8, len(SOURCES))) as ex:
        objs = list(ex.map(_compile, SOURCES))
    cmd = [NVCC, "-shared", "-o", OUT] + objs + ["-lcudart"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("link failed:\n" + r.stderr[-4000:])
    with open(stamp, "w") as f:
        f.write(dig)
    if verbose:
        print("built", OUT)
    return OUT


if __name__ == "__main__":
    build(force="--force" in sys.argv)
