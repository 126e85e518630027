"""The tile kernels' MMA groups are pipelined by ptxas, not serialized.

ptxas waits for every wgmma before issuing the next one when it cannot prove an MMA group convergent and free of calls (C7510, C7517 to
C7520 in its output).  The SASS then has a `WARPGROUP.DEPBAR` after every `HGMMA`.  Every MMA group of the tile kernels contains at least
one full k-step of the split-operand scheme (three products), so no wait may cover fewer than three HGMMA.  CPU only: reads the built
library and its build log."""
import functools
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "nice_slam_b200", "libnsb.so")
BUILD_LOG = os.path.join(ROOT, "nice_slam_b200", "csrc", "build.log")
KERNELS = ("render_fwd_tile_kernel", "render_fwd_tile_h16_kernel", "render_bwd_tile_kernel", "render_bwd_wg_tile_kernel")


def _cuobjdump():
    for cand in (shutil.which("cuobjdump"), os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")):
        if cand and os.path.exists(cand):
            return cand
    return None


@functools.lru_cache(maxsize=None)
def _kernel_sass():
    tool = _cuobjdump()
    if not os.path.exists(LIB) or tool is None:
        pytest.skip("libnsb.so or cuobjdump not available")
    sass = subprocess.run([tool, "-sass", LIB], check=True, capture_output=True, text=True).stdout
    out = {}
    for m in re.finditer(r"Function : (\S+)\n(.*?)(?=\n\s*Function : |\Z)", sass, re.S):
        for k in KERNELS:
            if re.search(r"\d%s[A-Z]" % k, m.group(1)):
                out[k] = m.group(2)
    return out


def _wait_runs(body):
    """Number of HGMMA since the previous wait, at every WARPGROUP.DEPBAR of the kernel."""
    runs, n = [], 0
    for line in body.splitlines():
        if "HGMMA" in line:
            n += 1
        elif "WARPGROUP.DEPBAR" in line:
            runs.append(n)
            n = 0
    return runs


@pytest.mark.parametrize("kernel", KERNELS)
def test_tile_kernel_mma_groups_not_serialized(kernel):
    body = _kernel_sass().get(kernel)
    assert body is not None, "%s not found in %s" % (kernel, LIB)
    runs = _wait_runs(body)
    n_mma = body.count("HGMMA")
    assert n_mma > 0 and runs, kernel
    assert min(runs) >= 3, "%s: a wait after %d HGMMA (waits after %s of %d HGMMA): ptxas serialized the MMA groups" % (
        kernel, min(runs), runs, n_mma)


def test_build_log_has_no_wgmma_serialization_notes():
    if not os.path.exists(BUILD_LOG):
        pytest.skip("no build log")
    notes = [ln.strip() for ln in open(BUILD_LOG) if re.search(r"\(C75(10|17|18|19|20)\)", ln) and any(k in ln for k in KERNELS)]
    assert not notes, "\n".join(notes)
