"""The GEMM main loops keep one wgmma group in flight: every kernel that issues wgmma (HGMMA in SASS) waits on them with exactly
two WARPGROUP.DEPBAR, the wgmma_wait<1> of the stage loop and the wgmma_wait<0> after it. When ptxas serialises wgmma (its
advisory C7520, e.g. around compiler-inserted warpgroup arrives on a path it takes for divergent), it puts a DEPBAR after every
HGMMA and the pipelining is gone with no other sign. Reads the built library; skips where it or cuobjdump is absent."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "clipbert_b200", "lib", "libclipbert_sm90.so")
MAX_DEPBAR = 2      # mma_tile / mma_tile_pp: wgmma_wait<1> in the stage loop, wgmma_wait<0> after it


def _cuobjdump():
    found = shutil.which("cuobjdump")
    if found:
        return found
    for home in (os.environ.get("CUDA_HOME"), os.environ.get("CUDA_PATH"), "/usr/local/cuda"):
        if home and os.path.exists(os.path.join(home, "bin", "cuobjdump")):
            return os.path.join(home, "bin", "cuobjdump")
    return None


def _wgmma_kernels():
    """{mangled kernel name: (HGMMA count, WARPGROUP.DEPBAR count)} of every kernel in the library that issues wgmma."""
    tool = _cuobjdump()
    if tool is None or not os.path.exists(LIB):
        pytest.skip("needs the built library and cuobjdump")
    sass = subprocess.run([tool, "-sass", LIB], capture_output=True, text=True, check=True).stdout
    counts, fn = {}, None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            fn = m.group(1)
            continue
        if fn is None:
            continue
        c = counts.setdefault(fn, [0, 0])
        if "HGMMA." in line:
            c[0] += 1
        elif "WARPGROUP.DEPBAR" in line:
            c[1] += 1
    return {f: tuple(c) for f, c in counts.items() if c[0]}


def test_wgmma_kernels_are_not_serialised():
    """Both wgmma kernels are in the library (TN / NN ping-pong; every weight gradient, single or grouped), and no wgmma kernel
    waits on its wgmma more often than the pipelined main loop does."""
    kernels = _wgmma_kernels()
    names = " ".join(kernels)
    for k in ("gemm_pingpong_kernel", "wgrad_group_kernel"):
        assert k in names, "no wgmma kernel %s in the library" % k
    bad = {f: c for f, c in kernels.items() if c[1] > MAX_DEPBAR}
    assert not bad, "wgmma serialised (HGMMA, WARPGROUP.DEPBAR): %s" % bad


def test_gemm_kernels_do_not_spill():
    """No GEMM kernel (TN / NN ping-pong, weight gradients, split reduce) uses local memory or a stack: a spill in the
    consumer warpgroups' fused epilogue, beside 2 x BN / 2 fp32 accumulators, would put local-memory traffic on every tile."""
    tool = _cuobjdump()
    if tool is None or not os.path.exists(LIB):
        pytest.skip("needs the built library and cuobjdump")
    out = subprocess.run([tool, "-res-usage", LIB], capture_output=True, text=True, check=True).stdout
    usage, fn = {}, None
    for line in out.splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            fn = m.group(1)
            continue
        m = re.search(r"STACK:(\d+).*LOCAL:(\d+)", line)
        if m and fn and ("gemm" in fn or "wgrad" in fn):
            usage[fn] = (int(m.group(1)), int(m.group(2)))
    assert any("gemm_pingpong_kernel" in f for f in usage) and any("wgrad_group_kernel" in f for f in usage), sorted(usage)
    bad = {f: u for f, u in usage.items() if u != (0, 0)}
    assert not bad, "GEMM kernels with stack / local memory (spills): %s" % bad
