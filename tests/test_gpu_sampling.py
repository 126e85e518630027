"""GPU: FusedRenderer with the reference's perturb, lindisp and N_importance settings (src/utils/Renderer.py:152-196) against the fixtures
of the unmodified reference (tests/golden/sampling/, tests/make_golden_sampling.py) and the sampling port (tests/sampling_port.py).

Bars as tests/test_gpu_parity.py: bit-exact z_vals and voxel-corner indices wherever the sample positions are fixed by the reference's
arithmetic (perturb, lindisp, and a second pass fed the reference's own sample list); 1e-4 relative (max-norm) on outputs and gradients."""
import os
from types import SimpleNamespace

import pytest
import torch

import sampling_port as spt
import scene_util as su
from gpu_util import LV, make_cfg, rel
from nice_slam_b200 import _lib
from nice_slam_b200.decoders import NICEDecoders
from nice_slam_b200.renderer import FusedRenderer, _RenderFn

pytestmark = pytest.mark.gpu
DEV = "cuda"
TOL = 1e-4
# mlp_backend 1 (FP32-FMA decoders) sums the decoder weight gradients over a ray group in another order than the tensor-core kernels: on
# render_color_perturb its fine.fc_c.4.bias gradient is 1.02e-4 from the reference (H100 80GB HBM3), everything else below 1e-4.  On the
# default sampler that back-end does not meet 1e-4 against the dense-grid oracle either (test_gpu_parity.py under NSB_MLP_BACKEND=1).
TOL_FMA_DEC = 2e-4
# Importance samples vs float64 sample_pdf on the kernel's own pass-1 weights, relative to the error of the reference's float32 torch
# sample_pdf on the same weights (max abs over the merged sample lists).  Measured on an H100 80GB HBM3 (render_color_importance, 96 rays):
# kernel 1.93e-6, torch float32 1.49e-3, ratio 1.3e-3 -- the kernel's float64 sum and running sum (rounded to f32 once) track the exact cdf
# more closely than torch's float32 sum, so its samples sit closer to the float64 ones.  K leaves a 40x margin over the measured ratio.
K_IMP = 0.05
# End-to-end importance sampling against the reference fixture.  The reference's own float32 samples are up to 1.5e-3 away from the float64
# sample_pdf (above) and the kernel's are not bit-identical to them, so the second pass sees slightly different sample depths and every
# output and gradient moves with them.  Measured on an H100 80GB HBM3, max over the three fixtures: z_vals 3.6e-4, depth 9.2e-6, variance
# 1.2e-5, rgb 1.5e-4, gradients 1.6e-3 (render_color_importance).  The bar is 3x the largest.
TOL_E2E = 5e-3


def load(name):
    case = torch.load(os.path.join(su.GOLDEN, "sampling", name + ".pt"), map_location="cpu", weights_only=False)
    sc = su.load_scenes()[case["scene"]]
    return case, sc, su.make_grids(sc, case["variant"]), su.load_decoders(case["variant"])


def renderer_for(case, sc, grids, dec_state, n_importance=None):
    cfg = make_cfg(sc)
    cfg["rendering"].update(perturb=case["perturb"], lindisp=case["lindisp"],
                            N_importance=case["n_importance"] if n_importance is None else n_importance)
    c = {k: v.to(DEV) for k, v in grids.items()}
    cam = sc["cam"]
    slam = SimpleNamespace(nice=True, bound=su.scene_bound(sc), shared_c=c, H=cam["H"], W=cam["W"], fx=cam["fx"], fy=cam["fy"],
                           cx=cam["cx"], cy=cam["cy"])
    r = FusedRenderer(cfg, SimpleNamespace(nice=True), slam)
    return r, slam.shared_c, NICEDecoders.from_state(dec_state, DEV)


def prepare(c, dec, case, stage):
    ro = case["rays_o"].to(DEV).requires_grad_(True)
    rd = case["rays_d"].to(DEV).requires_grad_(True)
    for k in c:
        c[k] = c[k].detach().requires_grad_(k[5:] in LV[stage])
    for p in dec.parameters():
        p.grad = None
        p.requires_grad_(True)
    gt = case["gt_depth"].to(DEV) if case["gt_depth"] is not None else None
    return ro, rd, gt


def backprop(case, d, u, col):
    ((d * case["g_depth"].to(DEV)).sum() + (u * case["g_var"].to(DEV)).sum() + (col * case["g_rgb"].to(DEV)).sum()).backward()


def check_grads(case, c, dec, ro, rd, tol, tol_dec=None):
    errs = dict(d_rays_o=rel(ro.grad, case["d_rays_o"]), d_rays_d=rel(rd.grad, case["d_rays_d"]))
    for k, summ in case["d_grid"].items():
        g = c[k].grad
        assert g is not None, k
        errs[k] = max(rel(g.reshape(-1).cpu()[summ["idx"]], summ["val"]), abs(float(g.double().norm()) - summ["norm"]) / summ["norm"])
    for lvl, gd in case["d_dec"].items():
        mine = dict(getattr(dec, lvl + "_decoder").named_parameters())
        for k, v in gd.items():
            errs["%s.%s" % (lvl, k)] = rel(mine[k].grad, v)
    dec_keys = {"%s.%s" % (lvl, k) for lvl, gd in case["d_dec"].items() for k in gd}
    bad = {k: v for k, v in errs.items() if not v < (tol_dec if (tol_dec is not None and k in dec_keys) else tol)}
    assert not bad, bad
    return max(errs.values())


@pytest.fixture
def backend():
    L = _lib.lib()
    keep = int(os.environ.get("NSB_MLP_BACKEND", "0"))

    def use(b):
        _lib.check(L.nsb_set_option(b"mlp_backend", b), "nsb_set_option")
    yield use
    use(keep)


@pytest.mark.parametrize("mlp_backend", [0, 1, 2])
@pytest.mark.parametrize("name", ["render_color_perturb", "render_coarse_perturb", "render_color_lindisp"])
def test_perturb_lindisp_against_reference_fixture(name, mlp_backend, backend):
    backend(mlp_backend)
    case, sc, grids, dec_state = load(name)
    stage = case["stage"]
    r, c, dec = renderer_for(case, sc, grids, dec_state)
    ro, rd, gt = prepare(c, dec, case, stage)
    aux = {}
    torch.manual_seed(case["seed"])
    d, u, col = r.render_batch_ray(c, dec, rd, ro, DEV, stage, gt_depth=gt, aux=aux)
    assert torch.equal(torch.rand(8), case["next_draw"])              # the caller's CPU random stream advanced as the reference's
    assert torch.equal(aux["z_vals"].cpu(), case["z_vals"])
    assert torch.equal(aux["corner_idx"].cpu().to(torch.int16), case["corner_idx"])
    assert rel(d, case["depth"]) < TOL and rel(u, case["var"]) < TOL
    if stage == "color":
        assert rel(col, case["rgb"]) < TOL
    backprop(case, d, u, col)
    check_grads(case, c, dec, ro, rd, TOL, TOL_FMA_DEC if mlp_backend == 1 else None)


def test_lindisp_zero_sensor_depth_gives_the_reference_nans():
    case, sc, grids, dec_state = load("render_color_lindisp")
    zd = case["zero_depth"]
    r, c, dec = renderer_for(case, sc, grids, dec_state)
    aux = {}
    with torch.no_grad():
        d, _, _ = r.render_batch_ray(c, dec, zd["rays_d"].to(DEV), zd["rays_o"].to(DEV), DEV, "color", gt_depth=zd["gt_depth"].to(DEV), aux=aux)
    z = aux["z_vals"].cpu()
    assert torch.equal(z.isnan(), zd["z_vals"].isnan()) and torch.equal(z[~z.isnan()], zd["z_vals"][~zd["z_vals"].isnan()])
    d = d.cpu()
    assert torch.equal(d.isnan(), zd["depth"].isnan()) and bool(d.isnan().any())
    assert rel(d[~d.isnan()], zd["depth"][~zd["depth"].isnan()]) < TOL


@pytest.mark.parametrize("name", ["render_color_importance", "render_color_importance_perturb", "render_coarse_importance"])
def test_second_pass_on_the_reference_samples(name):
    """Pass 2 fed the fixture's final sample list: outputs, gradients and voxel-corner indices as the reference's."""
    case, sc, grids, dec_state = load(name)
    stage = case["stage"]
    r, c, dec = renderer_for(case, sc, grids, dec_state)
    ro, rd, gt = prepare(c, dec, case, stage)
    aux = {}
    call, gl, plist = r._call(c, dec, stage, gt, ro.device, aux)
    call.lindisp, call.t_rand, call.z_given = False, None, case["z_vals"].to(DEV)
    d, u, col = _RenderFn.apply(call, ro, rd, *gl, *plist)
    assert torch.equal(aux["z_vals"].cpu(), case["z_vals"])
    assert torch.equal(aux["corner_idx"].cpu().to(torch.int16), case["corner_idx"])
    assert rel(d, case["depth"]) < TOL and rel(u, case["var"]) < TOL
    if stage == "color":
        assert rel(col, case["rgb"]) < TOL
    backprop(case, d, u, col)
    check_grads(case, c, dec, ro, rd, TOL)


def test_importance_samples_against_float64_sample_pdf():
    case, sc, grids, dec_state = load("render_color_importance")
    r, c, dec = renderer_for(case, sc, grids, dec_state)
    aux = {}
    with torch.no_grad():
        r.render_batch_ray(c, dec, case["rays_d"].to(DEV), case["rays_o"].to(DEV), DEV, "color", gt_depth=case["gt_depth"].to(DEV), aux=aux)
    z0, raw0, z = aux["z_vals0"].cpu(), aux["raw0"].cpu(), aux["z_vals"].cpu()
    n_imp = case["n_importance"]
    assert z.shape[1] == z0.shape[1] + n_imp
    mids = .5 * (z0[..., 1:] + z0[..., :-1])

    def weights(dtype):
        alpha = torch.sigmoid(10 * raw0[..., 3].to(dtype))
        T = torch.cumprod(torch.cat([torch.ones_like(alpha[:, :1]), 1. - alpha + 1e-10], -1), -1)[:, :-1]
        return alpha * T

    def merged(samples):
        return torch.sort(torch.cat([z0, samples.double()], -1), -1)[0]
    want = merged(spt.sample_pdf(mids, weights(torch.float64)[..., 1:-1], n_imp))
    torch32 = merged(spt.sample_pdf(mids, weights(torch.float32)[..., 1:-1], n_imp))
    err_kernel = float((z - want).abs().max())
    err_torch = float((torch32 - want).abs().max())
    print("importance samples: kernel %.3e, torch float32 %.3e vs float64 sample_pdf" % (err_kernel, err_torch))
    assert err_kernel <= K_IMP * max(err_torch, 1e-12), (err_kernel, err_torch)


@pytest.mark.parametrize("name", ["render_color_importance", "render_color_importance_perturb", "render_coarse_importance"])
def test_importance_end_to_end_against_reference_fixture(name):
    case, sc, grids, dec_state = load(name)
    stage = case["stage"]
    r, c, dec = renderer_for(case, sc, grids, dec_state)
    ro, rd, gt = prepare(c, dec, case, stage)
    aux = {}
    torch.manual_seed(case["seed"])
    d, u, col = r.render_batch_ray(c, dec, rd, ro, DEV, stage, gt_depth=gt, aux=aux)
    assert torch.equal(torch.rand(8), case["next_draw"])              # the caller's CPU random stream advanced as the reference's
    assert torch.equal(aux["z_vals0"].cpu(), case["z_vals0"])         # pass 1 is bit-exact
    errs = dict(z=rel(aux["z_vals"], case["z_vals"]), depth=rel(d, case["depth"]), var=rel(u, case["var"]))
    if stage == "color":
        errs["rgb"] = rel(col, case["rgb"])
    backprop(case, d, u, col)
    errs["grads"] = check_grads(case, c, dec, ro, rd, 1.0)
    print("%s end to end: %s" % (name, ", ".join("%s=%.1e" % kv for kv in errs.items())))
    assert all(v < TOL_E2E for v in errs.values()), errs


def test_fused_loop_classes_refuse_other_sampling_settings():
    from nice_slam_b200 import dist, mapping, steps
    case, sc, grids, dec_state = load("render_color_importance_perturb")
    r, c, dec = renderer_for(case, sc, grids, dec_state)
    ctx = SimpleNamespace(r=r, kind="map", n=8, dev=torch.device(DEV))
    with pytest.raises(RuntimeError, match="N_importance=0"):
        steps.IterationContext(r, 8, "color", DEV)
    with pytest.raises(RuntimeError, match="N_importance=0"):
        dist.ShardedTrackingIteration(ctx)
    with pytest.raises(RuntimeError, match="N_importance=0"):
        dist.ShardedMappingIteration(ctx)
    with pytest.raises(RuntimeError, match="N_importance=0"):
        mapping.FusedMappingLoop(r, c, dec, torch.eye(4), torch.ones(4, 4))
