"""Option "deterministic": its kernels as compiled, and the option's refusals (CPU only: reads the built library and its build log, and calls
nsb_set_option / nsb_get_option, which touch no device).

  * the kDet instantiations of the tile backward exist, their MMA groups are not serialized (the rule of test_sass_wgmma) and they spill no
    more than the default kernels they mirror;
  * the option defaults to 0, round-trips, and is refused together with mlp_backend 1 / 2 or wgrad_tc 0 whichever is set second, with an
    error naming both options."""
import os
import re

import pytest

from test_sass_wgmma import BUILD_LOG, _wait_runs

import test_sass_wgmma as sw

DET = {"render_bwd_tile_det_kernel": "render_bwd_tile_kernel", "render_bwd_wg_tile_det_kernel": "render_bwd_wg_tile_kernel",
       "render_bwd_wg_coarse_tile_det_kernel": "render_bwd_wg_coarse_tile_kernel"}


def _sass(kernel):
    import subprocess
    tool = sw._cuobjdump()
    if not os.path.exists(sw.LIB) or tool is None:
        pytest.skip("libnsb.so or cuobjdump not available")
    sass = subprocess.run([tool, "-sass", sw.LIB], check=True, capture_output=True, text=True).stdout
    for m in re.finditer(r"Function : (\S+)\n(.*?)(?=\n\s*Function : |\Z)", sass, re.S):
        if re.search(r"\d%s[A-Z]" % kernel, m.group(1)):
            return m.group(2)
    return None


def _spills(kernel):
    if not os.path.exists(BUILD_LOG):
        pytest.skip("build log not available")
    log = open(BUILD_LOG).read()
    m = re.search(r"Compiling entry function '_ZN3nsb\d+%sE[^']*'.*?(\d+) bytes spill stores, (\d+) bytes spill loads" % kernel, log, re.S)
    assert m, kernel
    return int(m.group(1)) + int(m.group(2))


@pytest.mark.parametrize("kernel", sorted(DET))
def test_deterministic_kernels_mma_groups_not_serialized(kernel):
    body = _sass(kernel)
    assert body is not None, kernel
    runs = _wait_runs(body)
    assert body.count("HGMMA") > 0 and runs, kernel
    assert min(r for r in runs if r > 0) >= 3, (kernel, runs)


@pytest.mark.parametrize("kernel", sorted(DET))
def test_deterministic_kernels_spill_no_more_than_their_default_kernels(kernel):
    assert _spills(kernel) <= _spills(DET[kernel]), (kernel, _spills(kernel), DET[kernel], _spills(DET[kernel]))


def _lib():
    from nice_slam_b200 import _lib
    try:
        _lib.lib()
    except (RuntimeError, OSError) as e:
        pytest.skip("libnsb.so not loadable: %s" % e)
    return _lib


def test_option_defaults_off_and_round_trips():
    L = _lib()
    assert L.get_option("deterministic") == 0
    L.set_option("deterministic", 1)
    try:
        assert L.get_option("deterministic") == 1
    finally:
        L.set_option("deterministic", 0)


@pytest.mark.parametrize("other,value", [("mlp_backend", 1), ("mlp_backend", 2), ("wgrad_tc", 0)])
def test_refused_combinations_name_both_options(other, value):
    L = _lib()
    prev = L.get_option(other)
    try:
        L.set_option("deterministic", 1)
        with pytest.raises(RuntimeError, match=r"deterministic.*%s|%s.*deterministic" % (other, other)):
            L.set_option(other, value)
        assert L.get_option(other) == prev
        L.set_option("deterministic", 0)
        L.set_option(other, value)
        with pytest.raises(RuntimeError, match=r"deterministic.*%s|%s.*deterministic" % (other, other)):
            L.set_option("deterministic", 1)
        assert L.get_option("deterministic") == 0
    finally:
        L.set_option("deterministic", 0)
        L.set_option(other, prev)
