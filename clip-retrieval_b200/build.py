"""Build the b200clip shared library (sm_90a only: H100) in-tree with nvcc.

`python clip-retrieval_b200/build.py` or `__graft_entry__.build()`.  Objects land in
clip-retrieval_b200/build/, the library in clip-retrieval_b200/lib/libb200clip.so (both git-ignored).
"""
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "build")
LIB = os.path.join(HERE, "lib", "libb200clip.so")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC",
    "-Xcompiler", "-Wall",
    "--expt-relaxed-constexpr",
]


def _nvcc():
    exe = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(exe):
        raise RuntimeError("nvcc not found; the b200clip library needs the CUDA 12.9 toolchain")
    return exe


def _deps_mtime():
    newest = 0.0
    for root in (CSRC, os.path.join(HERE, "..", "include")):
        for name in os.listdir(root):
            if name.endswith((".cuh", ".h")):
                newest = max(newest, os.path.getmtime(os.path.join(root, name)))
    return newest


def build(verbose=False, force=False):
    """Compile every csrc/*.cu for sm_90a and link the C-ABI library.  Returns its path."""
    os.makedirs(OBJ, exist_ok=True)
    os.makedirs(os.path.dirname(LIB), exist_ok=True)
    nvcc = _nvcc()
    sources = sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))
    hdr_time = _deps_mtime()
    jobs = []
    objs = []
    for src in sources:
        s = os.path.join(CSRC, src)
        o = os.path.join(OBJ, src[:-3] + ".o")
        objs.append(o)
        if force or not os.path.exists(o) or os.path.getmtime(o) < max(os.path.getmtime(s), hdr_time):
            jobs.append((s, o))

    def compile_one(job):
        s, o = job
        cmd = [nvcc] + NVCC_FLAGS + ["-c", s, "-o", o]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed for %s:\n%s\n%s" % (s, r.stdout, r.stderr))
        return r.stderr

    if jobs:
        with ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            for log in ex.map(compile_one, jobs):
                if verbose and log:
                    print(log)
    if jobs or not os.path.exists(LIB) or any(os.path.getmtime(o) > os.path.getmtime(LIB) for o in objs):
        cmd = [nvcc, "-shared", "-o", LIB] + objs + ["-gencode", "arch=compute_90a,code=sm_90a"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("link failed:\n%s\n%s" % (r.stdout, r.stderr))
    return LIB


if __name__ == "__main__":
    path = build(verbose="-v" in sys.argv, force="-f" in sys.argv)
    print(path)
