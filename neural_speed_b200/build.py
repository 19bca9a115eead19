"""Build libns_b200.so (hand-written sm_90a CUDA + the C-ABI) in-tree with nvcc.

The .so and the objects are git-ignored build products.  Cross-compiles without a GPU.
"""
from __future__ import annotations

import concurrent.futures as cf
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "build")
LIB = os.path.join(HERE, "libns_b200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")

NVCC_FLAGS = [
    "-std=c++17", "-O3", "-lineinfo",
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-Xcompiler", "-fPIC,-fvisibility=hidden,-fopenmp,-Wall,-Wno-unused-function",
    "-Xptxas", "-v",
]


def _sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith((".cu", ".cpp")))


def _digest(path: str) -> str:
    h = hashlib.sha1()
    for dep in [path] + [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC)) if f.endswith((".cuh", ".h"))] + [
        os.path.join(HERE, "..", "include", "ns_b200.h"), __file__]:
        with open(dep, "rb") as fh:
            h.update(fh.read())
    return h.hexdigest()


def _compile(src: str) -> str:
    path = os.path.join(CSRC, src)
    obj = os.path.join(OBJ, src + ".o")
    stamp = obj + ".sha1"
    dig = _digest(path)
    if os.path.exists(obj) and os.path.exists(stamp) and open(stamp).read() == dig:
        return obj
    cmd = [NVCC] + NVCC_FLAGS + ["-c", path, "-o", obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    with open(obj + ".log", "w") as fh:
        fh.write(" ".join(cmd) + "\n" + r.stdout + r.stderr)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError(f"nvcc failed on {src}")
    with open(stamp, "w") as fh:
        fh.write(dig)
    return obj


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(OBJ, exist_ok=True)
    if force:
        for f in os.listdir(OBJ):
            os.remove(os.path.join(OBJ, f))
    srcs = _sources()
    with cf.ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        objs = list(ex.map(_compile, srcs))
    newest = max(os.path.getmtime(o) for o in objs)
    if force or not os.path.exists(LIB) or os.path.getmtime(LIB) < newest:
        cmd = [NVCC, "-shared", "-cudart", "static", "-o", LIB] + objs + ["-Xcompiler", "-fopenmp", "-lgomp"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
            raise RuntimeError("link failed")
    if verbose:
        print("built", LIB)
    return LIB


if __name__ == "__main__":
    build(force="--force" in sys.argv, verbose=True)
