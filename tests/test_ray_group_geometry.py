"""CPU: which decoder kernel family serves a render call, and the launch geometry of the round-1 ray-group and FP32-FMA kernels
(nsb_render.cu kernel_family, choose_config, plan_split, nsb_eval_points), restated here.  The float64 checks of those families
(test_gpu_f64_backends.py) pick their batch sizes from this restatement for the SM count they run on, so that every case lands on the
geometry it names: decoder-parallel (split) CTAs of one or several rays, a ragged last ray group, CTAs of two tiles, a second wave of CTAs.
The tests below assert that at 132 SMs (H100 SXM) and 114 SMs (H100 PCIe)."""
import math
from collections import namedtuple

import pytest

K_MIN_SAMPLES = 8           # tl::kMinSamples
MAX_SAMPLES = 256           # NSB_MAX_SAMPLES
K_MAX_PTS_TC = 256          # kMaxPtsTc: points per ray-group CTA (2 tiles)
K_MAX_PTS_PER_BLOCK = 384   # kMaxPtsPerBlock
K_MAX_RAYS_PER_BLOCK = 24   # kMaxRaysPerBlock
K_CHUNK = 16                # kChunk: points per warp work item of the FP32-FMA kernels
TM = 128                    # tc::TM: points per tile
K_SPLIT_MAX_RAYS = 256      # kSplitMaxRays
N_DEC = {"coarse": 1, "middle": 1, "fine": 2, "color": 3}


def kernel_family(S, n_rays, points, mlp_backend, small_rays):
    """'tile', 'group' or 'fma' (nsb_render.cu kernel_family)."""
    tile_backend = mlp_backend in (0, 3)
    if points:
        return "tile" if tile_backend else "group" if mlp_backend == 2 else "fma"
    small = mlp_backend == 0 and n_rays <= small_rays and S <= K_MAX_PTS_TC
    if tile_backend and K_MIN_SAMPLES <= S <= MAX_SAMPLES and not small:
        return "tile"
    if mlp_backend in (0, 2) and S <= K_MAX_PTS_TC:
        return "group"
    return "fma"


def rays_per_cta(n_rays, S, sms, max_pts_cap):
    """choose_config's rays per CTA: fill every SM once before growing CTAs, up to max_pts_cap points and kMaxRaysPerBlock rays."""
    r_cap = min(max(max_pts_cap // S, 1), K_MAX_RAYS_PER_BLOCK)
    return min(max(-(-n_rays // sms), 1), r_cap)


def tiles(r, S):
    return -(-r * S // TM)


def plan_split(n_rays, S, nd, sms, r0):
    """plan_split: rays per CTA of decoder-parallel CTAs, or None when one CTA per ray group does all decoders (cost model: tiles a CTA
    walks through x decoders it evaluates x waves)."""
    if nd < 2 or n_rays > K_SPLIT_MAX_RAYS:
        return None
    r_cap = K_MAX_PTS_TC // S
    if r_cap < 1:
        return None
    r_cap = min(r_cap, K_MAX_RAYS_PER_BLOCK)
    r1 = next((r for r in range(1, r_cap + 1) if -(-n_rays // r) * nd <= sms), None)
    if r1 is None:
        return None
    groups0 = -(-n_rays // r0)
    cost0 = -(-groups0 // sms) * tiles(r0, S) * nd
    return r1 if tiles(r1, S) < cost0 else None


Geom = namedtuple("Geom", "split r tiles groups last ctas waves")


def group_geometry(n_rays, S, sms, stage="color"):
    """Launch geometry of the ray-group kernels (launch_group) for a render call: split (decoder-parallel CTAs per ray group), rays per
    CTA, tiles per CTA, ray groups, rays of the last group, CTAs and waves of them (one CTA per SM)."""
    nd = N_DEC[stage]
    r = rays_per_cta(n_rays, S, sms, K_MAX_PTS_TC)
    r1 = plan_split(n_rays, S, nd, sms, r)
    split = r1 is not None
    r = r1 if split else r
    groups = -(-n_rays // r)
    ctas = groups * (nd if split else 1)
    return Geom(split, r, tiles(r, S), groups, n_rays - (groups - 1) * r, ctas, -(-ctas // sms))


def fma_geometry(n_rays, S, sms):
    """Launch geometry of the FP32-FMA kernels (launch_fma): rays per CTA, the cap on it, CTAs and rays of the last CTA."""
    r = rays_per_cta(n_rays, S, sms, K_MAX_PTS_PER_BLOCK)
    r_cap = min(max(K_MAX_PTS_PER_BLOCK // S, 1), K_MAX_RAYS_PER_BLOCK)
    ctas = -(-n_rays // r)
    return dict(r=r, r_cap=r_cap, ctas=ctas, last=n_rays - (ctas - 1) * r)


def points_per_cta(n_points, sms):
    """nsb_eval_points: points per CTA of the ray-group and FP32-FMA kernels in points mode."""
    ppb = -(-n_points // sms)
    ppb = -(-ppb // K_CHUNK) * K_CHUNK
    return max(min(ppb, K_MAX_PTS_PER_BLOCK), K_CHUNK)


# -------------------------------------------------------------------------------- the cases of test_gpu_f64_backends.py
# (name, stage, S, the batch size at 132 SMs, predicate on group_geometry): on another SM count the case takes the batch size nearest
# the 132-SM one whose geometry satisfies the predicate.
GROUP_CASES = (
    ("split r=1", "color", 48, 16, lambda g, sms: g.split and g.r == 1 and g.ctas < sms),
    ("split r=1 every SM", "color", 48, 44, lambda g, sms: g.split and g.r == 1 and g.ctas == sms),
    ("split ragged last group", "color", 48, 45, lambda g, sms: g.split and 1 < g.r and g.tiles == 1 and g.last < g.r),
    ("split 2 tiles ragged last", "color", 48, 100, lambda g, sms: g.split and g.tiles == 2 and g.last < g.r),
    ("split at the ray cap", "color", 48, 200, lambda g, sms: g.split and g.r == K_MAX_PTS_TC // 48),
    ("no split r<=2", "color", 48, 257, lambda g, sms: not g.split and g.r <= 2),
    ("no split cap 2 waves ragged", "color", 48, 661, lambda g, sms: not g.split and g.r == 5 and g.tiles == 2 and g.waves == 2 and g.last < g.r),
    ("no split cap 2 waves", "color", 48, 1000, lambda g, sms: not g.split and g.r == 5 and g.waves == 2 and g.last == g.r and g.groups > sms + 16),
    ("S=129 split", "color", 129, 20, lambda g, sms: g.split and g.r == 1 and g.tiles == 2),
    ("S=129 no split", "color", 129, 60, lambda g, sms: not g.split and g.r == 1 and g.tiles == 2),
    ("S=256 split", "color", 256, 12, lambda g, sms: g.split and g.r == 1 and g.tiles == 2),
    ("S=256 no split", "color", 256, 50, lambda g, sms: not g.split and g.r == 1 and g.tiles == 2),
    ("stage fine split", "fine", 48, 100, lambda g, sms: g.split and g.r == 2),
    ("stage middle", "middle", 48, 100, lambda g, sms: not g.split),
    ("stage coarse", "coarse", 32, 100, lambda g, sms: not g.split),
)
# FP32-FMA kernels: (name, S, the batch size at 132 SMs, predicate on fma_geometry)
FMA_CASES = (
    ("r=1", 48, 24, lambda f, sms: f["r"] == 1),
    ("r=2 last CTA 1 ray", 48, 133, lambda f, sms: f["r"] == 2 and f["last"] == 1),
    ("ray cap ragged last", 48, 925, lambda f, sms: f["r"] == f["r_cap"] == 8 and f["last"] < f["r"]),
    ("S=33 ragged chunk", 33, 25, lambda f, sms: f["r"] == 1),
    ("S=47 ragged chunk", 47, 23, lambda f, sms: f["r"] == 1),
    ("S=256 r=1", 256, 40, lambda f, sms: f["r"] == f["r_cap"] == 1),
)


def pick(hint, ok, n_max=2000):
    """The batch size nearest `hint` (the smaller one on a tie) that satisfies ok(n)."""
    for d in range(n_max):
        for n in (hint - d, hint + d):
            if 1 <= n <= n_max and ok(n):
                return n
    raise AssertionError("no batch size near %d has the geometry" % hint)


def group_case_n(case, sms):
    name, stage, S, hint, pred = case
    return pick(hint, lambda n: pred(group_geometry(n, S, sms, stage), sms))


def fma_case_n(case, sms):
    name, S, hint, pred = case
    return pick(hint, lambda n: pred(fma_geometry(n, S, sms), sms))


def three_tile_points(sms):
    """A point count that gives the ray-group CTAs of points mode three tiles (more than 256 points each), with a ragged last CTA."""
    return 300 * sms + 77


SM_COUNTS = (132, 114)


# -------------------------------------------------------------------------------- tests
def test_issue_table_at_132_sms():
    """The geometry the measured small tracking batches take on an H100 SXM (S = 48, colour stage)."""
    g = {n: group_geometry(n, 48, 132) for n in (16, 44, 45, 64, 100, 200, 257, 661, 1000)}
    assert g[16] == Geom(True, 1, 1, 16, 1, 48, 1)
    assert g[44] == Geom(True, 1, 1, 44, 1, 132, 1)
    assert g[45] == Geom(True, 2, 1, 23, 1, 69, 1)
    assert g[64] == Geom(True, 2, 1, 32, 2, 96, 1)
    assert g[100] == Geom(True, 3, 2, 34, 1, 102, 1)
    assert g[200] == Geom(True, 5, 2, 40, 5, 120, 1)
    assert g[257] == Geom(False, 2, 1, 129, 1, 129, 1)
    assert g[661] == Geom(False, 5, 2, 133, 1, 133, 2)
    assert g[1000] == Geom(False, 5, 2, 200, 5, 200, 2)


@pytest.mark.parametrize("sms", SM_COUNTS)
def test_group_cases_land_on_their_geometry(sms):
    seen = set()
    for case in GROUP_CASES:
        name, stage, S, hint, pred = case
        n = group_case_n(case, sms)
        g = group_geometry(n, S, sms, stage)
        assert pred(g, sms), (name, n, g)
        if sms == 132:
            assert n == hint, (name, n, g)
        # every case runs on the ray-group kernels under mlp_backend 2, and not under the default dispatch
        assert kernel_family(S, n, False, 2, 0) == "group"
        assert kernel_family(S, n, False, 0, 0) == "tile"
        seen.add((stage, S, g))
    assert len(seen) == len(GROUP_CASES)


@pytest.mark.parametrize("sms", SM_COUNTS)
def test_fma_cases_land_on_their_geometry(sms):
    for case in FMA_CASES:
        name, S, hint, pred = case
        n = fma_case_n(case, sms)
        f = fma_geometry(n, S, sms)
        assert pred(f, sms), (name, n, f)
        if sms == 132:
            assert n == hint, (name, n, f)
        assert kernel_family(S, n, False, 1, 0) == "fma"
    assert 33 % K_CHUNK == 1 and 47 % K_CHUNK == 15


def test_auto_dispatch_below_the_tile_kernels_minimum():
    """S <= 7 goes to the ray-group kernels under the default dispatch, whatever the batch size; S >= 8 to the tile kernels."""
    for S in (1, 3, 6, 7):
        for n in (1, 40, 257, 5000):
            assert kernel_family(S, n, False, 0, 0) == "group"
    for S in (8, 48, 256):
        assert kernel_family(S, 40, False, 0, 0) == "tile"


def test_small_rays_dispatch():
    """small_rays = 64: batches of up to 64 rays go to the ray-group kernels, larger ones to the tile kernels."""
    assert [kernel_family(48, n, False, 0, 64) for n in (16, 64, 65)] == ["group", "group", "tile"]
    assert kernel_family(48, 64, False, 3, 64) == "tile"           # small_rays belongs to the auto dispatch only
    assert kernel_family(257, 16, False, 0, 64) == "fma"


@pytest.mark.parametrize("sms", SM_COUNTS)
def test_small_batches_take_the_split_path(sms):
    """The 16- and 64-ray tracking iterations (S = 48, colour) run decoder-parallel CTAs."""
    for n in (16, 64):
        assert group_geometry(n, 48, sms).split


@pytest.mark.parametrize("sms", SM_COUNTS)
def test_points_mode(sms):
    """Points mode sizes its CTAs by itself: up to kMaxPtsPerBlock = 384 points, which is three tiles for the ray-group kernels."""
    assert kernel_family(1, 0, True, 2, 0) == "group" and kernel_family(1, 0, True, 1, 0) == "fma"
    assert kernel_family(1, 0, True, 0, 64) == "tile"
    n = three_tile_points(sms)
    ppb = points_per_cta(n, sms)
    assert 2 * TM < ppb <= K_MAX_PTS_PER_BLOCK and n % ppb != 0
    assert points_per_cta(255, sms) == K_CHUNK
    assert math.ceil(n / ppb) <= sms
