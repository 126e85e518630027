"""The mesh-extraction kernels of nsb_mesh.cu keep everything in registers: no local-memory spills (ptxas -v output of the build).
CPU only: reads the build log."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD_LOG = os.path.join(ROOT, "nice_slam_b200", "csrc", "build.log")
KERNELS = ("mc_count_kernel", "mc_emit_kernel", "scan_blocks_kernel", "scan_add_kernel", "hull_support_kernel", "hull_outside_kernel",
           "hull_points_kernel", "depth_limits_kernel", "seen_kernel", "edge_union_kernel", "area_kernel", "keep_kernel", "compact_kernel",
           "colors_kernel")


def _ptxas_entries():
    if not os.path.exists(BUILD_LOG):
        pytest.skip("build log not available")
    out, cur = {}, None
    for line in open(BUILD_LOG):
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            cur = m.group(1)
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur:
            out[cur] = tuple(int(v) for v in m.groups())
    return out


@pytest.mark.parametrize("kernel", KERNELS)
def test_mesh_kernel_has_no_spills(kernel):
    ent = {k: v for k, v in _ptxas_entries().items() if "nsb_mesh_cu" in k and re.search(r"\d%s" % kernel, k)}
    assert ent, "%s not in %s" % (kernel, BUILD_LOG)
    for name, (stack, st, ld) in ent.items():
        assert st == 0 and ld == 0, (name, stack, st, ld)
