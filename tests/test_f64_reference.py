"""CPU: the float64 reference (oracle/f64_ref.py) that the GPU suite measures the kernels and the float32 port against.

Three things pin it: it agrees with the float32 port (itself bit-identical to the reference) within float32 noise on every render
fixture; its gradients match central differences of itself in float64; and its own ReLU decisions differ from the port's only at knife
edges, where nothing else changes.  Bars are set from a CPU run of these tests (figures in the comments)."""
import glob
import os

import pytest
import torch

import scene_util as su
from oracle import f64_ref as fr

RENDER_CASES = sorted(glob.glob(os.path.join(su.GOLDEN, "render_*.pt")))
IDS = [os.path.basename(p)[:-3] for p in RENDER_CASES]
LV = fr.STAGE_DECODERS


def load(path):
    case = torch.load(path, map_location="cpu", weights_only=False)
    sc = su.load_scenes()[case["scene"]]
    return case, sc, su.make_grids(sc, case["variant"]), su.load_decoders(case["variant"]), su.scene_bound(sc)


def both(path, masks_from_port=False):
    case, sc, grids, dec, bound = load(path)
    stage = case["stage"]
    gg = tuple("grid_" + lvl for lvl in LV[stage])
    args = (grids, dec, case["rays_o"], case["rays_d"], stage, case["gt_depth"], bound, case["g_depth"], case["g_var"], case["g_rgb"])
    port = fr.port_run(*args, grad_grids=gg, grad_decoders=LV[stage])
    f64 = fr.run(*args, grad_grids=gg, grad_decoders=LV[stage], coarse_enlarge=sc["coarse_bound_enlarge"],
                 masks=port["masks"] if masks_from_port else None)
    return case, port, f64, gg


@pytest.mark.parametrize("path", RENDER_CASES, ids=IDS)
def test_f64_reference_agrees_with_the_float32_port(path):
    """Measured (port vs f64, max-norm): soft grids, depth / var / rgb <= 1.2e-5 (room0 color: 1.7e-6 / 2.7e-6 / 8.3e-6), ray and voxel
    gradients <= 6.6e-5 (Apartment), decoder gradients <= 6.0e-5; init grids, var 1.8e-5, grid_fine gradient 3.0e-5 and the fine decoder's
    weight gradients 8.6e-4 (f32 rounding of 1 - alpha at alpha = 1)."""
    case, port, f64, gg = both(path)
    assert torch.equal(f64["z_vals"], case["z_vals"])
    lvl0 = LV[case["stage"]][0]
    assert torch.equal(f64["fixed"]["cells"][lvl0]["i0"].reshape(case["corner_idx"].shape).to(torch.int16), case["corner_idx"])
    assert torch.equal(port["depth"], case["depth"]) and torch.equal(port["d_rays_o"], case["d_rays_o"])     # the port is the pinned one
    init = case["variant"] == "init"
    inb = f64["fixed"]["inb"].reshape(f64["raw"].shape[:2])
    for k, x, t in (("depth", port["depth"], f64["depth"]), ("var", port["var"], f64["var"]), ("rgb", port["rgb"], f64["rgb"]),
                    ("occ", port["raw"][..., 3][inb], f64["raw"][..., 3][inb]), ("raw rgb", port["raw"][..., :3], f64["raw"][..., :3])):
        assert fr.errors(x, t)["max"] < 3e-5, (k, fr.errors(x, t))
    for k in ("d_rays_o", "d_rays_d") + tuple("d_" + g for g in gg):
        e = fr.errors(port[k], f64[k])
        assert e["max"] < 1.5e-4 and e["l2"] < 1e-4, (k, e)
    for lvl, grads in f64["d_dec"].items():
        for k, t in grads.items():
            e = fr.errors(port["d_dec"][lvl][k], t)
            assert e["max"] < (2e-3 if init and lvl != "color" else 1.5e-4), (lvl, k, e)


@pytest.mark.parametrize("path", RENDER_CASES, ids=IDS)
def test_own_relu_decisions_differ_from_the_ports_only_at_knife_edges(path):
    """The float64 reference on its own ReLU signs and on the port's: every unit where they disagree has |u| <= 1e-5 x (that layer's
    largest |u|) (measured: <= 2.1e-6, at most 3 units per fixture), and every point / ray without such a unit is bit-identical."""
    case, port, own, _ = both(path)
    _, _, on_port, _ = both(path, masks_from_port=True)
    flip = own["masks"] != port["masks"]
    n_flip = int(flip.sum())
    assert n_flip <= 4, n_flip
    if n_flip:
        scale = own["pre"].abs().amax(0, keepdim=True).expand_as(own["pre"])
        assert float((own["pre"][flip].abs() / scale[flip]).max()) < 1e-5
    pt = flip.reshape(flip.shape[0], -1).any(1).reshape(own["raw"].shape[:2])
    ray = pt.any(1)
    assert torch.equal(own["raw"][~pt], on_port["raw"][~pt])
    for k in ("depth", "var", "rgb", "d_rays_o", "d_rays_d"):
        assert torch.equal(own[k][~ray], on_port[k][~ray]), k
    if n_flip == 0:
        for k in own:
            if k.startswith("d_grid"):
                assert torch.equal(own[k], on_port[k]), k


def _loss(grids, dec, ro, rd, case, stage, bound, fixed, masks):
    d, u, c, _ = fr.render_batch_ray(grids, dec, rd, ro, stage, None, bound, masks=masks, fixed=fixed, round32=False)
    n = ro.shape[0]
    return (d * case["g_depth"][:n].double()).sum() + (u * case["g_var"][:n].double()).sum() + (c * case["g_rgb"][:n].double()).sum()


@pytest.mark.parametrize("stage", ["coarse", "middle", "fine", "color"])
def test_f64_gradients_match_central_differences(stage):
    """Hand-written trilinear gather, masked ReLU and compositing against central differences (Richardson-extrapolated) of the same float64 function (decisions and
    ReLU masks frozen, float32 rounding points off, so the function is smooth): along one random direction for the rays, for each stage grid
    (over the whole tensor) and for each decoder parameter tensor.  Measured worst relative difference per stage (CPU): coarse 1.5e-10,
    middle 8.3e-8, fine 9.4e-8, color 3.7e-8."""
    path = os.path.join(su.GOLDEN, "render_%s_soft.pt" % stage)
    case, sc, grids, dec, bound = load(path)
    n = 24
    ro, rd = case["rays_o"][:n].double(), case["rays_d"][:n].double()
    g64 = {k: v.double() for k, v in grids.items()}
    d64 = {lvl: {k: v.double() for k, v in W.items()} for lvl, W in dec.items()}
    gt = case["gt_depth"][:n] if case["gt_depth"] is not None else None
    shapes = {lvl: tuple(g64["grid_" + lvl].shape[2:]) for lvl in fr.STAGE_GRIDS[stage]}
    fixed = fr.decide(ro, rd, stage, gt, bound, shapes, coarse_enlarge=sc["coarse_bound_enlarge"])
    _, _, _, aux = fr.render_batch_ray(g64, d64, rd, ro, stage, None, bound, fixed=fixed, round32=False)
    masks = aux["masks"]
    if "middle" in fr.STAGE_GRIDS[stage]:              # the fine decoder's middle features carry no gradient: hold them still
        fixed["fine_mid"] = fr._trilinear(g64["grid_middle"], aux["points"], bound, fixed["cells"]["middle"], False)
    # analytic gradients of everything at once
    ro_l, rd_l = ro.clone().requires_grad_(True), rd.clone().requires_grad_(True)
    gl = {k: v.clone().requires_grad_(True) for k, v in g64.items()}
    dl = {lvl: {k: v.clone().requires_grad_(True) for k, v in W.items()} for lvl, W in d64.items()}
    _loss(gl, dl, ro_l, rd_l, case, stage, bound, fixed, masks).backward()
    gen = torch.Generator().manual_seed(2024)
    checks = [("rays", None, None)] + [("grid_" + lvl, None, None) for lvl in fr.STAGE_GRIDS[stage]] + \
             [(lvl, k, None) for lvl in LV[stage] for k in d64[lvl] if dl[lvl][k].grad is not None]
    for what, name, _ in checks:
        if what == "rays":
            do, dd = torch.randn(ro.shape, generator=gen, dtype=torch.float64), torch.randn(rd.shape, generator=gen, dtype=torch.float64)
            ana = float((ro_l.grad * do).sum() + (rd_l.grad * dd).sum())
            h = 1e-4
            f = lambda s: float(_loss(g64, d64, ro + s * do, rd + s * dd, case, stage, bound, fixed, masks))
        elif name is None:
            x = g64[what]
            dx = torch.randn(x.shape, generator=gen, dtype=torch.float64)
            ana = float((gl[what].grad * dx).sum())
            h = 1e-4 * float(x.abs().max())
            f = lambda s: float(_loss({**g64, what: x + s * dx}, d64, ro, rd, case, stage, bound, fixed, masks))
        else:
            x = d64[what][name]
            dx = torch.randn(x.shape, generator=gen, dtype=torch.float64)
            ana = float((dl[what][name].grad * dx).sum())
            h = (1e-6 if name == "embedder._B" else 1e-4) * max(float(x.abs().max()), 0.1)     # (sin(p B): B x p reaches ~1e2)
            f = lambda s: float(_loss(g64, {**d64, what: {**d64[what], name: x + s * dx}}, ro, rd, case, stage, bound, fixed, masks))
        cd = lambda h: (f(h) - f(-h)) / (2 * h)
        fd = (4 * cd(h / 2) - cd(h)) / 3                      # Richardson: O(h^4)
        err = abs(fd - ana) / max(abs(ana), 1e-12)
        assert abs(ana) > 0 and err < 2e-7, (what, name, ana, fd)
