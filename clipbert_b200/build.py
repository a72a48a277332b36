"""Build libclipbert_sm90.so (hand-written sm_90a kernels + C ABI) in-tree with nvcc.

The library is compiled ahead of time into ``clipbert_b200/lib/`` so that it travels with the
repository tree to the machine that runs it; there is no JIT cache and no torch extension machinery.
"""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
OBJDIR = os.path.join(LIBDIR, "obj")
LIB = os.path.join(LIBDIR, "libclipbert_sm90.so")

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC", "--use_fast_math", "-Xptxas", "-v",
    "-I", os.path.join(HERE, "..", "include"),
]


def _sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def _deps_mtime():
    m = 0.0
    for f in os.listdir(CSRC):
        if f.endswith((".cuh", ".h")):
            m = max(m, os.path.getmtime(os.path.join(CSRC, f)))
    m = max(m, os.path.getmtime(os.path.join(HERE, "..", "include", "clipbert_b200.h")))
    return m


def _compile(src, verbose):
    obj = os.path.join(OBJDIR, src[:-3] + ".o")
    srcp = os.path.join(CSRC, src)
    if os.path.exists(obj) and os.path.getmtime(obj) >= max(os.path.getmtime(srcp), _deps_mtime()):
        return obj, ""
    cmd = [NVCC] + FLAGS + ["-c", srcp, "-o", obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed for %s:\n%s\n%s" % (src, r.stdout, r.stderr))
    return obj, r.stderr


def build(verbose=False, force=False):
    """Compile every .cu under csrc/ for sm_90a and link the shared library. Returns its path."""
    os.makedirs(OBJDIR, exist_ok=True)
    if force:
        for f in os.listdir(OBJDIR):
            os.remove(os.path.join(OBJDIR, f))
    srcs = _sources()
    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        results = list(ex.map(lambda s: _compile(s, verbose), srcs))
    objs = [o for o, _ in results]
    if verbose:
        for _, log in results:
            if log:
                sys.stderr.write(log)
    newest = max(os.path.getmtime(o) for o in objs)
    if not os.path.exists(LIB) or os.path.getmtime(LIB) < newest:
        cmd = [NVCC, "-shared", "-o", LIB] + objs + ["-lcudart"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("link failed:\n%s\n%s" % (r.stdout, r.stderr))
    return LIB


if __name__ == "__main__":
    print(build(verbose="-v" in sys.argv, force="-f" in sys.argv))
