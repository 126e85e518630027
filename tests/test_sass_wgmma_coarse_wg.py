"""The coarse decoder's tensor-core weight-gradient kernel (render_bwd_wg_coarse_tile_kernel, option wgrad_all) keeps its MMA groups
pipelined like the other tile kernels: no `WARPGROUP.DEPBAR` after fewer than three `HGMMA` in its SASS, and no wgmma serialisation note
(C7510, C7517 to C7520) for it in the build log.  CPU only: reads the built library and its build log."""
import os
import re
import subprocess

import pytest

from test_sass_wgmma import BUILD_LOG, LIB, _cuobjdump, _wait_runs

KERNEL = "render_bwd_wg_coarse_tile_kernel"


def _sass(kernel):
    tool = _cuobjdump()
    if not os.path.exists(LIB) or tool is None:
        pytest.skip("libnsb.so or cuobjdump not available")
    sass = subprocess.run([tool, "-sass", LIB], check=True, capture_output=True, text=True).stdout
    for m in re.finditer(r"Function : (\S+)\n(.*?)(?=\n\s*Function : |\Z)", sass, re.S):
        if re.search(r"\d%s[A-Z]" % kernel, m.group(1)):
            return m.group(2)
    return None


def test_coarse_weight_gradient_kernel_mma_groups_not_serialized():
    body = _sass(KERNEL)
    assert body is not None, "%s not found in %s" % (KERNEL, LIB)
    runs = _wait_runs(body)
    assert body.count("HGMMA") > 0 and runs
    assert min(runs) >= 3, "%s: a wait after %d HGMMA (waits after %s): ptxas serialized the MMA groups" % (KERNEL, min(runs), runs)


def test_build_log_has_no_wgmma_serialization_notes_for_the_coarse_kernel():
    if not os.path.exists(BUILD_LOG):
        pytest.skip("no build log")
    notes = [ln.strip() for ln in open(BUILD_LOG) if re.search(r"\(C75(10|17|18|19|20)\)", ln) and KERNEL in ln]
    assert not notes, "\n".join(notes)


def test_weight_gradient_kernels_keep_their_registers():
    """ptxas -v: both weight-gradient kernels within 255 registers and without spills (one CTA per SM is their design point)."""
    if not os.path.exists(BUILD_LOG):
        pytest.skip("no build log")
    log = open(BUILD_LOG).read()
    for k in ("render_bwd_wg_tile_kernel", KERNEL):
        m = re.search(r"Compiling entry function '_ZN3nsb\d+%sE\S*' for 'sm_90a'\n(.*?)Used (\d+) registers" % k, log, re.S)
        assert m is not None, k
        assert "0 bytes spill stores, 0 bytes spill loads" in m.group(1), (k, m.group(1))
        assert int(m.group(2)) <= 255, k
