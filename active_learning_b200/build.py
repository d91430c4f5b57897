"""In-tree build of libalq.so (the C-ABI CUDA library) for sm_90a (H100).

    python -m active_learning_b200.build            # or: make

nvcc cross-compiles without a GPU.  The .so is written next to this file
(active_learning_b200/libalq.so, git-ignored), so the package is importable from the source
tree.  Nothing is JIT-compiled at import time.
"""
from __future__ import annotations

import concurrent.futures
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libalq.so")
OBJ = os.path.join(HERE, "csrc", "_obj")

GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = [
    *GENCODE,
    "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC,-O3,-Wall,-Wno-unused-function",
]


def sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        raise RuntimeError("nvcc not found: libalq.so cannot be built here")
    os.makedirs(OBJ, exist_ok=True)
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    headers.append(os.path.join(os.path.dirname(HERE), "include", "alq.h"))
    jobs = []
    for src in sources():
        s = os.path.join(CSRC, src)
        o = os.path.join(OBJ, src[:-3] + ".o")
        if force or _stale(o, [s] + headers):
            jobs.append([nvcc, *NVCC_FLAGS, "-c", s, "-o", o])

    def run(cmd):
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed:\n" + " ".join(cmd) + "\n" + r.stdout + r.stderr)
        if verbose and (r.stdout or r.stderr):
            print(r.stdout + r.stderr)

    with concurrent.futures.ThreadPoolExecutor(max_workers=min(8, max(1, len(jobs)))) as ex:
        list(ex.map(run, jobs))
    objs = [os.path.join(OBJ, s[:-3] + ".o") for s in sources()]
    if force or jobs or _stale(OUT, objs):
        run([nvcc, "-shared", *GENCODE, "-o", OUT, *objs])
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
