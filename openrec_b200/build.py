"""Build liborx.so (the sm_90a CUDA kernels + C-ABI) in-tree with nvcc.

    python -m openrec_b200.build [--force] [--verbose]

The shared object lands next to the sources (openrec_b200/csrc/liborx.so, git-ignored), so the
package is importable straight from the source tree.  sm_90a (H100) only, no other arch, no fallback.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(CSRC, "liborx.so")
ROOT = os.path.dirname(HERE)

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17", "--expt-relaxed-constexpr",
    "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden",
]


def _nvcc():
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found (set NVCC=/path/to/nvcc)")


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _stale():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cu", ".cuh", ".h"))]
    deps.append(os.path.join(ROOT, "include", "orx.h"))
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    """Compile every .cu under csrc/ into liborx.so; returns the path."""
    if not force and not _stale():
        return LIB
    nvcc = _nvcc()
    objs = []
    procs = []
    for src in sources():
        obj = src[:-3] + ".o"
        cmd = [nvcc, *NVCC_FLAGS, "-c", src, "-o", obj]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            failed = True
            sys.stderr.write(f"nvcc failed on {src}:\n{out}\n")
        elif verbose or out.strip():
            sys.stderr.write(out)
    if failed:
        raise RuntimeError("liborx build failed")
    # exported symbols carry default visibility via ORX_API in the sources
    link = [nvcc, "-shared", "-o", LIB, *objs, "-gencode", "arch=compute_90a,code=sm_90a", "-cudart", "static"]
    r = subprocess.run(link, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError("liborx link failed:\n" + r.stdout)
    return LIB


if __name__ == "__main__":
    path = build(force="--force" in sys.argv, verbose="--verbose" in sys.argv)
    print(path)
