"""The loss-seed kernels (nsb_tracking_seeds, nsb_mapping_seeds, nsb_tracking_residuals, and the same bodies run by the last CTA of the forward
launch), the batch depth maxima and the bbox pre-filter, against plain float64 torch on the CPU.

These kernels decide WHICH rays carry a loss: the tracker keeps a ray when its residual is below ten times the batch median (Tracker.py:113), and
the median is hand-written with five selection paths -- direct rank counting (pool <= 256), a bitonic sort of 512 padded keys (257 .. 512), an
8-bit radix select that hands the wanted bin to either of those once it has shrunk to <= 512 keys, and all eight radix passes when it never does.
A wrong choice drops or adds whole rays, which no tolerance on a loss over well-spread random residuals shows.  So the bars here are exact: the
seeds g_depth / g_rgb equal the reference bit for bit (sqrt, divide and abs are correctly rounded on both sides: ieee_sqrt below), which makes the set of
kept rays an exact assertion; only the loss, whose summation order is free, is compared at 1e-12 against math.fsum.

The reference below is written from the reference implementation's lines, not from the kernel, and is itself checked without a GPU against
autograd through oracle.torch_port and against the captured real tracker iteration."""
import ctypes as C
import math
import os

import numpy as np
import pytest
import torch

import scene_util as su
from gpu_util import LV, make_renderer
from oracle import torch_port as tp

DEV = "cuda"
gpu = pytest.mark.gpu
NSB_ERR_ARG = -1
F64, F32 = torch.float64, torch.float32
NAN, INF = float("nan"), float("inf")


# ------------------------------------------------------------------------------------ reference (float64 torch on the CPU)
def ieee_sqrt(x):
    """Correctly rounded square root.  torch.sqrt's vectorised CPU path is within one ulp but not correctly rounded on every machine (it
    differed from the IEEE result on 2 of 200 variances where this was written); the kernels' sqrt.rn.f64 is, and the bars here are exact."""
    with np.errstate(invalid="ignore"):
        return torch.from_numpy(np.sqrt(x.detach().numpy()))


def residuals_ref(depth, var, gt):
    return torch.abs(gt.double() - depth) / ieee_sqrt(var + 1e-10)                        # Tracker.py:112


def tracking_seeds_ref(depth, var, rgb, gt, gt_rgb, w_color=0.5, handle_dynamic=True, use_color=True, pool=None):
    """Tracker.py:108-123 -> dict(loss, g_depth f64 [n], g_rgb f32 [n,3], mask, median).  torch.median is the real one: lower median of an even
    count, NaN when the pool holds a NaN.  pool: the residuals the median is taken over when they are not this batch's own."""
    diff = gt.double() - depth
    den = ieee_sqrt(var + 1e-10)
    res = torch.abs(diff) / den
    mask = gt > 0
    med = None
    if handle_dynamic:
        med = (res if pool is None else pool).median()
        mask = (res < 10 * med) & mask
    g_depth = torch.where(mask, -torch.sign(diff) / den, torch.zeros_like(res))
    terms = [float(x) for x in res[mask]]
    g_rgb = torch.zeros(gt.numel(), 3, dtype=F32)
    if use_color:
        dc = gt_rgb - rgb.double()
        g_rgb = torch.where(mask[:, None], (-w_color * torch.sign(dc)).float(), g_rgb)
        terms += [w_color * float(x) for x in torch.abs(dc)[mask].reshape(-1)]
    return dict(loss=math.fsum(terms), g_depth=g_depth, g_rgb=g_rgb, mask=mask, median=med, res=res)


def mapping_seeds_ref(depth, rgb, gt, gt_rgb, w_color=0.2, use_color=True):
    """Mapper.py:487-493: depth term over gt > 0, colour term (a float32 difference) over all rays."""
    m = gt > 0
    diff = gt.double() - depth
    g_depth = torch.where(m, -torch.sign(diff), torch.zeros_like(diff))
    terms = [float(x) for x in torch.abs(diff)[m]]
    g_rgb = torch.zeros(gt.numel(), 3, dtype=F32)
    if use_color:
        dc = gt_rgb - rgb                                                                  # float32 - float32
        g_rgb = (-w_color * torch.sign(dc).double()).float()
        terms += [w_color * float(x) for x in torch.abs(dc).reshape(-1)]
    return dict(loss=math.fsum(terms), g_depth=g_depth, g_rgb=g_rgb)


def same_bits(a, b):
    a, b = a.detach().cpu().contiguous(), b.detach().cpu().contiguous()
    it = {F64: torch.int64, F32: torch.int32}[a.dtype]
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(a.view(it), b.view(it))


def loss_close(got, want):
    return got == want if (want == 0.0 or math.isinf(want)) else abs(got - want) <= 1e-12 * abs(want)


# ------------------------------------------------------------------------------------ inputs
def random_batch(n, seed=9):
    """The spread-out random batch: every 13th ray without sensor depth."""
    g = torch.Generator().manual_seed(seed)
    depth = torch.rand(n, generator=g, dtype=F64) * 3
    var = torch.rand(n, generator=g, dtype=F64) * 0.1
    rgb = torch.rand(n, 3, generator=g)
    gt = torch.rand(n, generator=g) * 3
    gt[::13] = 0
    gt_rgb = torch.rand(n, 3, generator=g, dtype=F64)
    return dict(depth=depth, var=var, rgb=rgb, gt=gt, gt_rgb=gt_rgb)


GT0 = 64.0                       # sensor depth of the constructed rays
QUANTUM = 2.0 ** -46             # 64 - r and 64 + r are exact for residuals r < 32 that are multiples of this
VAR_ONE = 1.0 - 1e-10            # sqrt(VAR_ONE + 1e-10) == 1.0 exactly


def batch_with_residuals(r, seed=3):
    """Rays whose residuals are exactly r (float64 multiples of QUANTUM below 32), on alternating sides of the sensor depth."""
    r = torch.as_tensor(r, dtype=F64)
    n = r.numel()
    g = torch.Generator().manual_seed(seed)
    side = torch.where(torch.arange(n) % 2 == 0, 1.0, -1.0).double()
    b = dict(depth=GT0 - side * r, var=torch.full((n,), VAR_ONE, dtype=F64), rgb=torch.rand(n, 3, generator=g),
             gt=torch.full((n,), GT0), gt_rgb=torch.rand(n, 3, generator=g, dtype=F64))
    assert same_bits(residuals_ref(b["depth"], b["var"], b["gt"]), r), "constructed residuals are not what they were meant to be"
    return b


def quantize(x):
    return torch.floor(x.double() / QUANTUM) * QUANTUM


def spread_residuals(n, seed):
    """Skewed over [0, 8): the median is near 0.5, so ten times the median falls inside the bulk and a wrong median changes the kept set."""
    u = torch.rand(n, generator=torch.Generator().manual_seed(seed), dtype=F64)
    return quantize(8 * u ** 4)


def lower_median_residuals(n):
    """Even n: lower median 1/16, upper median >= 3/4, and the upper half between 10/16 and 10 * 3/4 -- kept only under the upper-median rule."""
    g = torch.Generator().manual_seed(n)
    lo = torch.cat([quantize(torch.rand(n // 2 - 1, generator=g, dtype=F64) / 32), torch.tensor([1.0 / 16], dtype=F64)])
    hi = quantize(0.75 + 0.45 * torch.rand(n // 2, generator=g, dtype=F64))
    r = torch.cat([lo, hi])
    return r[torch.randperm(n, generator=g)]


def distribution(kind, n, seed=1):
    """Residuals that steer the median's selection code (n <= 256 direct, <= 512 bitonic, above: radix passes first)."""
    g = torch.Generator().manual_seed(seed * 7919 + n)
    if kind == "identical":                         # above 512: all eight radix passes, no direct step
        return torch.full((n,), 0.5, dtype=F64)
    if kind == "two_values":                        # the median is the last of the low value: one rank further and every high ray is kept
        k = (n - 1) // 2 + 1
        r = torch.cat([torch.full((k,), 1.0 / 16, dtype=F64), torch.full((n - k,), 1.0, dtype=F64)])
        return r[torch.randperm(n, generator=g)]
    if kind == "heavy_bin":                         # up to 600 copies of the median among spread values: its bin never shrinks to 512 keys
        copies = min(600, n - 100)
        rest = n - copies
        r = torch.cat([torch.full((copies,), 0.25, dtype=F64), quantize(torch.rand(rest // 2, generator=g, dtype=F64) * 0.2),
                       quantize(0.3 + 7.5 * torch.rand(rest - rest // 2, generator=g, dtype=F64) ** 2)])
        return r[torch.randperm(n, generator=g)]
    if kind == "shared_top_byte":                   # 400 keys in [0.5, 0.53) around the median, the rest in other top bytes: radix, then bitonic
        mid = min(400, n // 2)
        below = (n - mid) // 2
        r = torch.cat([quantize(0.5 + 0.03 * torch.rand(mid, generator=g, dtype=F64)),
                       quantize(2.0 ** -16 * torch.rand(below, generator=g, dtype=F64)),
                       quantize(2.0 + 5.9 * torch.rand(n - mid - below, generator=g, dtype=F64))])
        return r[torch.randperm(n, generator=g)]
    if kind == "narrow":                            # [1, 1 + 2^-30]: the keys share five bytes; 2 % probes around ten times the median
        probes = max(n // 50, 2)
        r = torch.cat([1.0 + torch.randint(0, 1 << 16, (n - probes,), generator=g).double() * QUANTUM,
                       10.0 + torch.randint(0, 10 << 16, (probes,), generator=g).double() * QUANTUM])
        return r[torch.randperm(n, generator=g)]
    raise ValueError(kind)


DISTRIBUTIONS = ["identical", "two_values", "heavy_bin", "shared_top_byte", "narrow"]
EDITS = ["zeros", "var0", "one_inf", "several_inf"]


def edited_batch(kind, n):
    """The random batch with rays whose residual is an exact zero, huge (var = 0) or +inf (var = -1e-10: a zero denominator)."""
    b = random_batch(n, seed=21)
    if kind == "zeros":
        b["depth"][::3] = b["gt"][::3].double()
        b["gt_rgb"][::5] = b["rgb"][::5].double()
    elif kind == "var0":
        b["var"][::4] = 0.0
    elif kind == "one_inf":
        b["var"][n // 2] = -1e-10
    elif kind == "several_inf":
        b["var"][1::7] = -1e-10
    return b


# ------------------------------------------------------------------------------------ the references themselves (no GPU)
def _autograd_tracking(b, **kw):
    d = b["depth"].clone().requires_grad_(True)
    c = b["rgb"].clone().requires_grad_(True)
    loss = tp.tracking_loss(d, b["var"], c, b["gt"], b["gt_rgb"], 0.5, **kw)
    loss.backward()
    return float(loss.detach()), d.grad, c.grad


@pytest.mark.parametrize("handle_dynamic,use_color", [(True, True), (False, True), (True, False)])
@pytest.mark.parametrize("n", [2, 200, 777])
def test_tracking_reference_is_autograd_of_the_ported_loss(n, handle_dynamic, use_color):
    b = random_batch(n)
    want = tracking_seeds_ref(b["depth"], b["var"], b["rgb"], b["gt"], b["gt_rgb"], 0.5, handle_dynamic, use_color)
    loss, gd, gc = _autograd_tracking(b, handle_dynamic=handle_dynamic, use_color=use_color)
    assert abs(want["loss"] - loss) <= 1e-12 * abs(loss)
    assert torch.equal(want["g_depth"] != 0, gd != 0)                                      # the same rays kept
    assert bool(((want["g_depth"] - gd).abs() <= 4e-16 * gd.abs()).all())                  # one ulp: autograd's denominator is torch.sqrt
    assert torch.equal(want["g_rgb"], gc if use_color else torch.zeros(n, 3))
    assert 0 < int(want["mask"].sum()) < n


@pytest.mark.parametrize("stage", ["middle", "color"])
def test_mapping_reference_is_autograd_of_the_ported_loss(stage):
    b = random_batch(777)
    gt_rgb = b["gt_rgb"].float()
    want = mapping_seeds_ref(b["depth"], b["rgb"], b["gt"], gt_rgb, 0.2, stage == "color")
    d = b["depth"].clone().requires_grad_(True)
    c = b["rgb"].clone().requires_grad_(True)
    loss = tp.mapping_loss(d, c, b["gt"], gt_rgb, stage, 0.2)
    loss.backward()
    assert abs(want["loss"] - float(loss.detach())) <= 1e-6 * abs(float(loss.detach()))                      # the ported colour sum is a float32 sum
    assert torch.equal(want["g_depth"], d.grad)
    assert torch.equal(want["g_rgb"], c.grad if stage == "color" else torch.zeros(777, 3))


def test_tracking_reference_on_the_captured_real_tracker_iteration():
    import glue
    case = torch.load(os.path.join(su.GOLDEN, "tracker_color.pt"), map_location="cpu", weights_only=False)
    sc = su.load_scenes()[case["scene"]]
    ro, rd, gd, gc = glue.tracking_rays(sc, case, case["camera_tensor"])
    keep = tp.bbox_prefilter(ro, rd, gd, su.scene_bound(sc))
    assert torch.equal(gd[keep], case["gt_depth"])
    want = tracking_seeds_ref(case["depth"], case["var"], case["rgb"], case["gt_depth"], gc[keep], sc["tracking"]["w_color_loss"])
    assert abs(want["loss"] - case["loss"]) <= 1e-12 * abs(case["loss"])


def test_reference_median_rules():
    r = torch.tensor([1.0, NAN, 2.0, 3.0], dtype=F64)
    b = dict(depth=4.0 - r, var=torch.full((4,), VAR_ONE, dtype=F64), rgb=torch.rand(4, 3), gt=torch.full((4,), 4.0), gt_rgb=torch.rand(4, 3, dtype=F64))
    w = tracking_seeds_ref(**b)
    assert math.isnan(float(w["median"])) and not bool(w["mask"].any()) and w["loss"] == 0.0
    assert not bool(w["g_depth"].any()) and not bool(w["g_rgb"].any())
    assert float(tracking_seeds_ref(**batch_with_residuals([4.0, 1.0, 3.0, 2.0]))["median"]) == 2.0     # lower median


@pytest.mark.parametrize("n", [2, 256, 512])
def test_lower_median_batches_tell_the_two_median_rules_apart(n):
    r = lower_median_residuals(n)
    s = torch.sort(r).values
    lower, upper = float(s[(n - 1) // 2]), float(s[n // 2])
    assert lower == 1.0 / 16 and upper >= 0.75
    w = tracking_seeds_ref(**batch_with_residuals(r))
    assert float(w["median"]) == lower
    assert int(w["mask"].sum()) == n // 2 and int((r < 10 * upper).sum()) == n


@pytest.mark.parametrize("n", [300, 512, 777, 2000, 5000])
@pytest.mark.parametrize("kind", DISTRIBUTIONS)
def test_distributions_are_what_they_claim(kind, n):
    r = distribution(kind, n)
    w = tracking_seeds_ref(**batch_with_residuals(r))
    med = float(w["median"])
    keys = r.view(torch.int64)
    if kind == "identical":
        assert int(w["mask"].sum()) == n
    if kind == "two_values":
        assert med == 1.0 / 16 and float(torch.sort(r).values[(n - 1) // 2 + 1]) == 1.0 and int(w["mask"].sum()) == (n - 1) // 2 + 1
    if kind == "heavy_bin":
        assert med == 0.25 and int((r == med).sum()) == min(600, n - 100) and 0 < int(w["mask"].sum()) < n
    if kind == "shared_top_byte" and n > 512:
        in_bin = int(((keys >> 56) == (torch.tensor(med, dtype=F64).view(torch.int64) >> 56)).sum())
        assert 256 < in_bin <= 512 and 0 < int(w["mask"].sum()) < n
    if kind == "narrow":
        bulk = keys[r < 2]
        assert int(((bulk >> 24) != (bulk[0] >> 24)).sum()) == 0                           # five bytes shared: six radix passes at least
        assert 1.0 <= med <= 1.0 + 2.0 ** -30 and int(w["mask"].sum()) < n


def strict_bound_case(m):
    """Three rays with residuals just below, at and just above ten times the pool median m."""
    t = float(torch.tensor(10.0, dtype=F64) * torch.tensor(m, dtype=F64))
    r = torch.tensor([math.nextafter(t, 0.0), t, math.nextafter(t, INF)], dtype=F64)
    b = dict(depth=4.0 - r, var=torch.full((3,), VAR_ONE, dtype=F64), rgb=torch.rand(3, 3, generator=torch.Generator().manual_seed(1)),
             gt=torch.full((3,), 4.0), gt_rgb=torch.rand(3, 3, generator=torch.Generator().manual_seed(2), dtype=F64))
    assert same_bits(residuals_ref(b["depth"], b["var"], b["gt"]), r)
    return b, torch.tensor([m], dtype=F64)


@pytest.mark.parametrize("m", [0.3, 0.25, 0.37])
def test_strict_bound_case_sits_on_the_bound(m):
    b, pool = strict_bound_case(m)
    assert tracking_seeds_ref(**b, pool=pool)["mask"].tolist() == [True, False, False]


# ------------------------------------------------------------------------------------ the C entry points
def _lib():
    from nice_slam_b200 import _lib as lib
    return lib, lib.lib()


CANARY = 12345.0


def run_tracking_seeds(b, w_color=0.5, handle_dynamic=1, use_color=1, pool=None, n=None):
    """nsb_tracking_seeds -> dict(loss, g_depth, g_rgb); the outputs and the workspace are followed by canaries that must survive."""
    lib, L = _lib()
    n = b["gt"].numel() if n is None else n
    d = {k: v.to(DEV) for k, v in b.items()}
    gD = torch.full((n + 8,), CANARY, dtype=F64, device=DEV)
    gC = torch.full((n + 8, 3), CANARY, dtype=F32, device=DEV)
    lo = torch.full((2,), CANARY, dtype=F64, device=DEV)
    nws = L.nsb_tracking_seeds_workspace(n)
    ws = torch.full((nws // 8 + 8,), CANARY, dtype=F64, device=DEV)
    pool_d = pool.to(DEV) if pool is not None else None
    lib.check(L.nsb_tracking_seeds(d["depth"].data_ptr(), d["var"].data_ptr(), d["rgb"].data_ptr(), d["gt"].data_ptr(),
                                   d["gt_rgb"].data_ptr() if use_color else None, n, w_color, handle_dynamic, use_color,
                                   pool_d.data_ptr() if pool is not None else None, pool.numel() if pool is not None else 0,
                                   gD.data_ptr(), gC.data_ptr(), lo.data_ptr(), ws.data_ptr(), nws, None), "nsb_tracking_seeds")
    torch.cuda.synchronize()
    assert bool((gD[n:] == CANARY).all()) and bool((gC[n:] == CANARY).all()) and float(lo[1]) == CANARY and bool((ws[(nws + 7) // 8:] == CANARY).all())
    return dict(loss=float(lo[0]), g_depth=gD[:n].cpu(), g_rgb=gC[:n].cpu())


def check_tracking(b, handle_dynamic=1, use_color=1, pool=None, w_color=0.5):
    want = tracking_seeds_ref(b["depth"], b["var"], b["rgb"], b["gt"], b["gt_rgb"], w_color, bool(handle_dynamic), bool(use_color), pool)
    got = run_tracking_seeds(b, w_color, handle_dynamic, use_color, pool)
    kept = got["g_depth"] != 0
    if not same_bits(got["g_depth"], want["g_depth"]):
        bad = torch.nonzero(got["g_depth"].view(torch.int64) != want["g_depth"].view(torch.int64)).reshape(-1)
        pytest.fail("g_depth differs on %d of %d rays (first %d: got %r, want %r); kept %d, reference keeps %d; reference median %r" % (
            bad.numel(), kept.numel(), int(bad[0]), float(got["g_depth"][bad[0]]), float(want["g_depth"][bad[0]]), int(kept.sum()),
            int(want["mask"].sum()), None if want["median"] is None else float(want["median"])))
    assert same_bits(got["g_rgb"], want["g_rgb"])
    assert loss_close(got["loss"], want["loss"]), (got["loss"], want["loss"])
    return want


@gpu
@pytest.mark.parametrize("n", [1, 2, 3, 255, 256, 257, 258, 511, 512, 513, 1023, 1024, 1025, 4097])
def test_tracking_seeds_at_every_entry_size(n):
    """Spread residuals at the sizes where the selection code changes path (256 | 257, 512 | 513) and the 1024-thread loop wraps."""
    want = check_tracking(batch_with_residuals(spread_residuals(n, seed=n)))
    assert int(want["mask"].sum()) >= 1 and (n < 255 or int(want["mask"].sum()) < n)


@gpu
@pytest.mark.parametrize("n", [200, 513, 777, 5000])
def test_tracking_seeds_on_random_batches_with_a_pool_and_mapping_seeds(n):
    """Random depth / variance / colour with missing sensor depths: own median, no median gate (handle_dynamic 0), the median over an external
    pool of 1601 residuals (what a sharded batch all-gathers), and the mapping seeds of the same batch."""
    b = random_batch(n)
    check_tracking(b)
    check_tracking(b, handle_dynamic=0)
    pool = torch.rand(1601, generator=torch.Generator().manual_seed(10), dtype=F64) * 2.0
    want = check_tracking(b, pool=pool)
    assert want["loss"] > 0
    check_mapping(b, 1)


@gpu
@pytest.mark.parametrize("n", [2, 256, 512])
def test_tracking_seeds_take_the_lower_median(n):
    want = check_tracking(batch_with_residuals(lower_median_residuals(n)))
    assert int(want["mask"].sum()) == n // 2


@gpu
@pytest.mark.parametrize("n", [300, 512, 777, 2000, 5000])
@pytest.mark.parametrize("kind", DISTRIBUTIONS)
def test_tracking_seeds_on_steering_distributions(kind, n):
    check_tracking(batch_with_residuals(distribution(kind, n)))


@gpu
@pytest.mark.parametrize("n", [300, 512, 777, 2000, 5000])
@pytest.mark.parametrize("kind", EDITS)
def test_tracking_seeds_with_zero_huge_and_infinite_residuals(kind, n):
    b = edited_batch(kind, n)
    res = residuals_ref(b["depth"], b["var"], b["gt"])
    if kind == "zeros":
        assert int((res == 0).sum()) >= n // 3
    if kind.endswith("inf"):
        assert int(torch.isinf(res).sum()) >= 1 and not bool(torch.isnan(res).any())
    check_tracking(b)
    if kind.endswith("inf"):
        check_tracking(b, handle_dynamic=0)           # then the infinite residual is kept: loss and its seed are +-inf on both sides


@gpu
@pytest.mark.parametrize("n_pool", [257, 2000])
def test_tracking_seeds_with_a_subnormal_pool(n_pool):
    """A pool of zeros (just under half) and subnormal residuals: the median is subnormal, and rays with residual exactly 0 are kept only if it is
    not mistaken for one of the zeros."""
    g = torch.Generator().manual_seed(n_pool)
    zeros = (n_pool - 1) // 2
    sub = torch.randint(1, 1 << 40, (n_pool - zeros,), generator=g).view(F64)               # bit patterns of subnormal doubles
    pool = torch.cat([torch.zeros(zeros, dtype=F64), sub])[torch.randperm(n_pool, generator=g)]
    assert 0.0 < float(pool.median()) < 2.3e-308
    b = random_batch(200, seed=5)
    b["depth"][::2] = b["gt"][::2].double()
    want = check_tracking(b, pool=pool)
    assert int(want["mask"].sum()) == int((b["gt"][::2] > 0).sum())


@gpu
@pytest.mark.parametrize("m", [0.3, 0.25, 0.37])
def test_tracking_seeds_mask_is_strictly_below_ten_medians(m):
    b, pool = strict_bound_case(m)
    want = check_tracking(b, pool=pool)
    assert want["mask"].tolist() == [True, False, False]


@gpu
@pytest.mark.parametrize("n_pool", [1, 2, 256, 257, 512, 513, 1601])
def test_tracking_seeds_with_pools_smaller_and_larger_than_the_batch(n_pool):
    """200 rays spread over [0, 8), pool over [0, 0.8): ten pool medians cut through the middle of the batch."""
    pool = torch.rand(n_pool, generator=torch.Generator().manual_seed(n_pool), dtype=F64) * 0.8
    r = quantize(8 * torch.rand(200, generator=torch.Generator().manual_seed(77), dtype=F64))
    want = check_tracking(batch_with_residuals(r), pool=pool)
    assert 0 < int(want["mask"].sum()) < 200


@gpu
@pytest.mark.parametrize("handle_dynamic", [0, 1])
@pytest.mark.parametrize("use_color", [0, 1])
def test_tracking_seeds_switches(handle_dynamic, use_color):
    """handle_dynamic x use_color (no gt_rgb pointer when colour is off); a batch without any sensor depth; an empty batch."""
    b = random_batch(300, seed=31)
    check_tracking(b, handle_dynamic, use_color)
    dark = dict(b, gt=torch.zeros(300))
    got = run_tracking_seeds(dark, 0.5, handle_dynamic, use_color)
    assert got["loss"] == 0.0 and same_bits(got["g_depth"], torch.zeros(300, dtype=F64)) and same_bits(got["g_rgb"], torch.zeros(300, 3))
    got = run_tracking_seeds(b, 0.5, handle_dynamic, use_color, n=0)                        # the canaries check that nothing but the loss is written
    assert got["loss"] == 0.0


@gpu
@pytest.mark.parametrize("n", [200, 400, 2000])
def test_tracking_seeds_with_a_nan_residual_keep_nothing(n):
    """torch.median of residuals that hold a NaN is NaN, so `tmp < 10 * tmp.median()` is False everywhere: the reference tracker's loss for such a
    batch is 0 with zero gradients.  (Direct, bitonic and radix entry.)"""
    b = random_batch(n, seed=41)
    b["depth"][n // 3] = NAN
    want = check_tracking(b)
    assert math.isnan(float(want["median"])) and want["loss"] == 0.0 and not bool(want["mask"].any())
    clean = random_batch(200, seed=42)
    pool = residuals_ref(b["depth"], b["var"], b["gt"])
    assert check_tracking(clean, pool=pool)["loss"] == 0.0                                  # ... and so is a pool with a NaN in it


@gpu
def test_tracking_residuals_bit_equal():
    lib, L = _lib()
    for n in (1, 255, 256, 257, 5000):
        b = edited_batch("several_inf", n) if n > 100 else random_batch(n)
        res = torch.full((n + 4,), CANARY, dtype=F64, device=DEV)
        d = {k: v.to(DEV) for k, v in b.items()}
        lib.check(L.nsb_tracking_residuals(d["depth"].data_ptr(), d["var"].data_ptr(), d["gt"].data_ptr(), n, res.data_ptr(), None), "nsb_tracking_residuals")
        torch.cuda.synchronize()
        assert same_bits(res[:n], residuals_ref(b["depth"], b["var"], b["gt"])) and bool((res[n:] == CANARY).all())


@gpu
def test_seed_entry_points_refuse_bad_arguments():
    lib, L = _lib()
    n = 100
    d = {k: v.to(DEV) for k, v in random_batch(n).items()}
    gD = torch.full((n,), CANARY, dtype=F64, device=DEV)
    gC = torch.full((n, 3), CANARY, dtype=F32, device=DEV)
    lo = torch.full((1,), CANARY, dtype=F64, device=DEV)
    nws = L.nsb_tracking_seeds_workspace(n)
    assert nws >= 8 * n
    ws = torch.empty(nws, dtype=torch.uint8, device=DEV)
    pool = torch.ones(4, dtype=F64, device=DEV)
    p = lambda k: d[k].data_ptr()

    def call(n=n, gt_rgb=p("gt_rgb"), use_color=1, pool_ptr=None, n_pool=0, ws_ptr=ws.data_ptr(), ws_bytes=nws):
        return L.nsb_tracking_seeds(p("depth"), p("var"), p("rgb"), p("gt"), gt_rgb, n, 0.5, 1, use_color, pool_ptr, n_pool,
                                    gD.data_ptr(), gC.data_ptr(), lo.data_ptr(), ws_ptr, ws_bytes, None)

    assert call(ws_bytes=nws - 1) == NSB_ERR_ARG and call(ws_ptr=None) == NSB_ERR_ARG
    assert call(pool_ptr=pool.data_ptr(), n_pool=0) == NSB_ERR_ARG and call(pool_ptr=pool.data_ptr(), n_pool=-3) == NSB_ERR_ARG
    assert call(gt_rgb=None) == NSB_ERR_ARG and call(n=-1) == NSB_ERR_ARG
    assert L.nsb_mapping_seeds(p("depth"), p("rgb"), p("gt"), None, n, 0.2, 1, gD.data_ptr(), gC.data_ptr(), lo.data_ptr(), None) == NSB_ERR_ARG
    assert L.nsb_mapping_seeds(p("depth"), p("rgb"), p("gt"), None, -1, 0.2, 0, gD.data_ptr(), gC.data_ptr(), lo.data_ptr(), None) == NSB_ERR_ARG
    torch.cuda.synchronize()
    assert float(lo[0]) == CANARY and bool((gD == CANARY).all()) and bool((gC == CANARY).all())     # a refusal launches nothing
    assert call(gt_rgb=None, use_color=0) == 0 and call() == 0
    torch.cuda.synchronize()


def check_mapping(b, use_color, w_color=0.2):
    lib, L = _lib()
    n = b["gt"].numel()
    gt_rgb = b["gt_rgb"].float()
    want = mapping_seeds_ref(b["depth"], b["rgb"], b["gt"], gt_rgb, w_color, bool(use_color))
    gD = torch.full((n + 8,), CANARY, dtype=F64, device=DEV)
    gC = torch.full((n + 8, 3), CANARY, dtype=F32, device=DEV)
    lo = torch.full((2,), CANARY, dtype=F64, device=DEV)
    t = [b["depth"].to(DEV), b["rgb"].to(DEV), b["gt"].to(DEV), gt_rgb.to(DEV)]
    lib.check(L.nsb_mapping_seeds(t[0].data_ptr(), t[1].data_ptr(), t[2].data_ptr(), t[3].data_ptr() if use_color else None, n, w_color, use_color,
                                  gD.data_ptr(), gC.data_ptr(), lo.data_ptr(), None), "nsb_mapping_seeds")
    torch.cuda.synchronize()
    assert bool((gD[n:] == CANARY).all()) and bool((gC[n:] == CANARY).all()) and float(lo[1]) == CANARY
    assert same_bits(gD[:n], want["g_depth"]) and same_bits(gC[:n], want["g_rgb"])
    assert loss_close(float(lo[0]), want["loss"]), (float(lo[0]), want["loss"])
    return want


@gpu
@pytest.mark.parametrize("use_color", [0, 1])
@pytest.mark.parametrize("n", [1, 1023, 1024, 1025, 5000])
def test_mapping_seeds(n, use_color):
    """Depth term over gt > 0 only, colour term over ALL rays (Mapper.py:487-493); rays whose colour or depth matches exactly get a zero seed."""
    b = random_batch(n, seed=n)
    if n == 1:
        b["gt"][0] = 1.5
    b["gt_rgb"][::5] = b["rgb"][::5].double()
    b["depth"][1::6] = b["gt"][1::6].double()
    want = check_mapping(b, use_color)
    if use_color and n > 13:
        assert bool(want["g_rgb"][b["gt"] == 0].any())                                     # rays without sensor depth still carry colour seeds


# ------------------------------------------------------------------------------------ fused: the last CTA of the forward launch
def _scene():
    sc = su.load_scenes()["room0"]
    grids, dec_state = su.make_grids(sc, "soft"), su.load_decoders("soft")
    renderer, c, dec = make_renderer(sc, grids, dec_state, DEV)
    return sc, renderer, c, dec


def disturbed_rays(sc, n, seed):
    """Rays of a synthetic frame after the bbox pre-filter, some without sensor depth and a block whose sensor depth is far off the surface
    (a moving object in front of the camera), which the median rule must remove."""
    ro, rd, gd, gc = su.make_rays(sc, 2 * n + 64, seed=seed)
    keep = tp.bbox_prefilter(ro, rd, gd, su.scene_bound(sc))
    ro, rd, gd, gc = (t[keep][:n].contiguous() for t in (ro, rd, gd, gc))
    assert ro.shape[0] == n
    gd = gd.clone()
    gd[5::17] = 0.0
    gd[n // 2: n // 2 + max(n // 10, 1)] *= 10.0
    return ro, rd, gd, gc


@gpu
@pytest.mark.parametrize("handle_dynamic", [1, 0])
@pytest.mark.parametrize("n", [255, 256, 257, 300, 511, 512, 513])
def test_tracking_iteration_seeds_match_the_reference_on_its_own_render(n, handle_dynamic):
    """nsb_tracking_iteration: up to 512 rays the seeds come from the forward's last CTA (256 threads, borrowed shared memory: direct counting and
    the bitonic sort), 513 takes the stand-alone kernel.  The reference is applied to the depth / variance / colour the iteration itself rendered."""
    from nice_slam_b200.steps import IterationContext
    sc, renderer, c, dec = _scene()
    ro, rd, gd, gc = disturbed_rays(sc, n, seed=300 + n)
    ctx = IterationContext(renderer, n, "color", DEV, kind="track", host_staging=False)
    dev_in = [t.to(DEV) for t in (ro, rd, gd, gc.double())]
    runs = []
    for rep in range(2):                    # second run: the arrival counter and the borrowed shared memory came back clean
        ctx.run(c, dec, *dev_in, handle_dynamic=bool(handle_dynamic))
        torch.cuda.synchronize()
        runs.append([t.cpu().clone() for t in (ctx.depth, ctx.var, ctx.rgb, ctx.g_depth, ctx.g_rgb, ctx.loss)])
    depth, var, rgb, g_depth, g_rgb, loss = runs[0]
    want = tracking_seeds_ref(depth, var, rgb, gd, gc.double(), 0.5, bool(handle_dynamic), True)
    n_valid = int((gd > 0).sum())
    if handle_dynamic:
        assert 1 <= int(want["mask"].sum()) < n_valid, "the median rule was meant to remove some rays and keep some"
    assert same_bits(g_depth, want["g_depth"]), (int((g_depth != 0).sum()), int(want["mask"].sum()))
    assert same_bits(g_rgb, want["g_rgb"])
    assert loss_close(float(loss), want["loss"]), (float(loss), want["loss"])
    assert all(same_bits(a, b) for a, b in zip(runs[0], runs[1]))


@gpu
@pytest.mark.parametrize("stage", ["middle", "color"])
@pytest.mark.parametrize("n", [1023, 1024, 1025])
def test_mapping_iteration_seeds_match_the_reference_on_its_own_render(n, stage):
    """nsb_mapping_iteration: up to 1024 rays fused into the forward launch, 1025 through the stand-alone kernel."""
    from nice_slam_b200.steps import IterationContext
    sc, renderer, c, dec = _scene()
    ro, rd, gd, gc = disturbed_rays(sc, n, seed=500 + n)
    gg = tuple("grid_" + l for l in LV[stage])
    ctx = IterationContext(renderer, n, stage, DEV, kind="map", grad_grids=gg, host_staging=False)
    dev_in = [t.to(DEV) for t in (ro, rd, gd, gc.float())]
    runs = []
    for rep in range(2):
        ctx.run(c, dec, *dev_in)
        torch.cuda.synchronize()
        runs.append([t.cpu().clone() for t in (ctx.depth, ctx.rgb, ctx.g_depth, ctx.g_rgb, ctx.loss)])
    depth, rgb, g_depth, g_rgb, loss = runs[0]
    want = mapping_seeds_ref(depth, rgb, gd, gc.float(), 0.2, stage == "color")
    assert same_bits(g_depth, want["g_depth"]) and same_bits(g_rgb, want["g_rgb"])
    assert loss_close(float(loss), want["loss"]), (float(loss), want["loss"])
    assert all(same_bits(a, b) for a, b in zip(runs[0], runs[1]))


# ------------------------------------------------------------------------------------ batch depth maxima and the bbox pre-filter
def run_batch_max(gt):
    lib, L = _lib()
    out = torch.full((3,), CANARY, device=DEV)
    g = gt.to(DEV)
    lib.check(L.nsb_batch_max_depth(g.data_ptr() if gt.numel() else None, gt.numel(), out.data_ptr(), None), "nsb_batch_max_depth")
    torch.cuda.synchronize()
    assert float(out[2]) == CANARY
    return out[:2].cpu()


@gpu
@pytest.mark.parametrize("n", [1, 31, 32, 33, 1023, 1024, 1025, 100000])
def test_batch_max_depth_wherever_the_maximum_sits(n):
    """out = [torch.max(gt), torch.max(gt * 1.2)] with the maximum first, last, at a warp seam and nowhere special; a batch of zeros."""
    base = torch.rand(n, generator=torch.Generator().manual_seed(n)) * 5
    for pos in sorted({0, n - 1, min(31, n - 1), min(32, n - 1), n // 2}):
        gt = base.clone()
        gt[pos] = 7.3
        assert same_bits(run_batch_max(gt), torch.stack([torch.max(gt), torch.max(gt * 1.2)])), pos
    assert same_bits(run_batch_max(base), torch.stack([torch.max(base), torch.max(base * 1.2)]))
    assert same_bits(run_batch_max(torch.zeros(n)), torch.zeros(2))


@gpu
def test_batch_max_depth_of_nothing_and_of_nan():
    """n = 0 gives zeros.  A NaN sensor depth is skipped by the maxima (torch.max would return NaN and the reference's sampler would make every
    sample of the batch NaN); a batch of nothing but NaN gives -inf.  include/nice_slam_b200.h states this at nsb_batch_max_depth."""
    assert same_bits(run_batch_max(torch.zeros(0)), torch.zeros(2))
    gt = torch.rand(777, generator=torch.Generator().manual_seed(3)) * 5
    clean = torch.stack([torch.max(gt), torch.max(gt * 1.2)])
    for pos in (0, 400, 776):
        bad = gt.clone()
        bad[pos] = NAN
        assert math.isnan(float(torch.max(bad)))
        keep = torch.ones(777, dtype=torch.bool)
        keep[pos] = False
        assert same_bits(run_batch_max(bad), torch.stack([torch.max(bad[keep]), torch.max(bad[keep] * 1.2)]))
    assert same_bits(run_batch_max(gt), clean)
    assert run_batch_max(torch.full((40,), NAN)).tolist() == [-INF, -INF]


def forward_z_vals(renderer, c, dec, ro, rd, gd, maxima, stage="color"):
    """z_vals of one nsb_render_forward with the batch maxima handed over as `maxima`: 'explicit' (depth_max from nsb_batch_max_depth), 'inline'
    (every CTA reduces gt_depth itself) or 'batch' (reduced from gt_depth_batch)."""
    from nice_slam_b200 import renderer as R
    lib, L = _lib()
    ro, rd, gd = ro.to(DEV), rd.to(DEV), gd.to(DEV)
    call, grids, _ = renderer._call(c, dec, stage, gd, torch.device(DEV))
    _, t_u, t_s, (depth, var, rgb, z_vals, raw, split), out = R._forward_setup(call, ro)
    dm = None
    if maxima == "explicit":
        dm = torch.empty(2, device=DEV)
        lib.check(L.nsb_batch_max_depth(gd.data_ptr(), gd.numel(), dm.data_ptr(), None), "nsb_batch_max_depth")
    inp = R._inputs(call, ro, rd, dm, t_u, t_s, [g.detach() for g in grids])
    if maxima == "batch":
        inp.gt_depth_batch, inp.n_batch = gd.data_ptr(), gd.numel()
    lib.check(L.nsb_render_forward(C.byref(inp), C.byref(out), None), "nsb_render_forward")
    torch.cuda.synchronize()
    return z_vals.cpu()


@gpu
@pytest.mark.parametrize("n", [1, 33, 1024])
def test_the_three_sources_of_the_batch_maxima_sample_the_same_depths(n):
    sc, renderer, c, dec = _scene()
    ro, rd, gd, _ = su.make_rays(sc, n, seed=40 + n)
    gd = gd.clone()
    gd[::7] = 0.0                                   # rays without sensor depth take their surface samples from the batch maximum
    if n > 1:
        gd[n - 1] = 9.0                             # the maximum, last
    z = [forward_z_vals(renderer, c, dec, ro, rd, gd, m) for m in ("explicit", "inline", "batch")]
    assert same_bits(z[0], z[1]) and same_bits(z[0], z[2])
    want = tp.sample_z_vals(ro, rd, gd, su.scene_bound(sc), renderer.N_samples, renderer.N_surface, "color")
    assert same_bits(z[0], want)


def edge_rays(bound):
    """Rays a random frame never contains, with their sensor depth at the exit distance bit for bit and one float32 step either side."""
    lo, hi = bound[:, 0], bound[:, 1]
    mid = ((lo + hi) / 2).float()
    rays = []
    for axis in range(3):                           # a zero direction component: both crossings of that axis are +-inf
        d = torch.tensor([0.3, -0.4, 0.5]); d[axis] = 0.0
        rays.append((mid.clone(), d))
        d2 = d.clone(); d2[axis] = -0.0
        rays.append((mid.clone(), d2))
    for axis in range(3):                           # origin exactly on a face with a zero component there: 0 / 0
        o = mid.clone(); o[axis] = lo[axis].float()
        if float(o[axis].double()) == float(lo[axis]):
            d = torch.tensor([0.2, 0.3, -0.6]); d[axis] = 0.0
            rays.append((o, d))
    rays.append((hi.float() + 1.0, torch.tensor([0.5, 0.4, 0.3])))          # origin outside, direction pointing away: negative exit distance
    rays.append((hi.float() + 1.0, torch.tensor([-0.5, -0.4, -0.3])))       # origin outside, pointing in
    rays.append((mid.clone(), torch.tensor([1e-30, 1.0, -1e-30])))          # nearly axis-parallel
    ro = torch.stack([r[0] for r in rays]); rd = torch.stack([r[1] for r in rays])
    t = (bound.unsqueeze(0) - ro.unsqueeze(-1)) / rd.unsqueeze(-1)
    far = torch.min(torch.max(t, dim=2)[0], dim=1)[0]                       # float64 exit distance, as Tracker.py:97-101
    out_o, out_d, out_g = [], [], []
    for i in range(ro.shape[0]):
        f = far[i]
        cands = [0.0, 1.0]
        if bool(torch.isfinite(f)) and float(f) > 0:
            g = f.float()
            cands += [float(g), float(torch.nextafter(g, torch.tensor(0.0))), float(torch.nextafter(g, torch.tensor(INF)))]
        for gval in cands:
            out_o.append(ro[i]); out_d.append(rd[i]); out_g.append(gval)
    return torch.stack(out_o), torch.stack(out_d), torch.tensor(out_g)


@gpu
def test_bbox_prefilter_on_random_and_on_edge_rays():
    """keep = (t_exit >= gt_depth) (Tracker.py:95-104) on 5000 random rays of a frame and on edge_rays()."""
    lib, L = _lib()
    sc = su.load_scenes()["room0"]
    bound = su.scene_bound(sc)
    b6 = (C.c_double * 6)(*bound.reshape(6).tolist())
    ro, rd, gd, _ = su.make_rays(sc, 5000, seed=1)
    eo, ed, eg = edge_rays(bound)
    want_edge = tp.bbox_prefilter(eo, ed, eg, bound)
    assert bool(want_edge.any()) and not bool(want_edge.all())
    for o, d, g in ((ro, rd, gd), (eo, ed, eg)):
        n = o.shape[0]
        k = torch.full((n + 16,), 77, dtype=torch.uint8, device=DEV)
        od, dd, gdv = o.to(DEV), d.to(DEV), g.to(DEV)
        lib.check(L.nsb_bbox_prefilter(od.data_ptr(), dd.data_ptr(), gdv.data_ptr(), n, b6, k.data_ptr(), None), "nsb_bbox_prefilter")
        torch.cuda.synchronize()
        want = tp.bbox_prefilter(o, d, g, bound)
        assert torch.equal(k[:n].cpu(), want.to(torch.uint8)), torch.nonzero(k[:n].cpu() != want.to(torch.uint8)).reshape(-1).tolist()
        assert bool((k[n:] == 77).all())
    out = run_batch_max(gd)
    assert same_bits(out, torch.stack([torch.max(gd), torch.max(gd * 1.2)]))


@gpu
def test_sampler_far_bound_on_edge_rays():
    """The sampler clamps its far bound with the same exit distance: z_vals of the edge rays, bit for bit."""
    sc, renderer, c, dec = _scene()
    bound = su.scene_bound(sc)
    eo, ed, eg = edge_rays(bound)
    want = tp.sample_z_vals(eo, ed, eg, bound, renderer.N_samples, renderer.N_surface, "color")
    got = forward_z_vals(renderer, c, dec, eo, ed, eg, "inline")
    assert same_bits(torch.nan_to_num(got, nan=-1.0), torch.nan_to_num(want, nan=-1.0)) and torch.equal(torch.isnan(got), torch.isnan(want))
