"""GPU: option wgrad_all -- the weight gradients of every decoder of a stage on the tensor cores (render_bwd_wg_tile_kernel for the middle, fine
and colour decoders, render_bwd_wg_coarse_tile_kernel for the coarse one), as the reference's tracker and mapper ask for them through the
drop-in renderer: they leave every decoder parameter trainable, so autograd requests the gradients of all of the stage's decoders.

  * float64 yardstick of every stage with all its decoders graded, at ragged last tiles and on large features;
  * the reference fixtures (which carry every decoder's gradients) at the tolerances of test_gpu_parity;
  * kernel selection (profiler) of an unmodified drop-in tracking call and of the coarse mapper's call, with the option on and off;
  * the real tracker's iteration and the fused mapping iteration with every decoder graded;
  * render_img under no_grad keeps no layer outputs."""
import os

import pytest
import torch

import glue
import scene_util as su
from gpu_util import make_renderer, rel
from oracle import f64_ref as fr
from oracle import torch_port as tp
from test_gpu_f64 import FLOOR, GRIDS, K_FP32_PASS, METRICS, check_masks, cotangents, kernel_run, modes, options, scene, tensors

pytestmark = pytest.mark.gpu
DEV = "cuda"
TOL = 1e-4
# The coarse stage (MLP_no_xyz): the float32 port is at its most accurate there (2e-7 relative in max norm), so 3xTF32 -- which drops lo*lo and
# reads 10 mantissa bits of each part -- sits furthest above it (see K_COARSE in test_gpu_f64).  Worst kernel / port ratios measured on an H100
# 80GB HBM3 (700 W) over the ragged-tile and x30 cases below, bars about 1.5x above them:
#  * coarse-decoder weight gradients: max 33 (output_linear.bias, the sum of dL/d occupancy over the points: 1.0e-5 vs 3.0e-7, the forward's
#    error carried through the compositing backward), L2 36 (pts_linears.3.bias), per-element 69 (pts_linears.3.weight, 8.9e-4 vs 1.3e-5),
#    99.9th percentile 62 (output_linear.weight);
#  * the same launch's rays, voxels and outputs at S = 33: max 24 (var), L2 27 (var), per-element 39 (d_rays_d) -- just above K_COARSE,
#    which was measured at S = 32.
# Deterministic mode (render_bwd_wg_coarse_tile_det_kernel, the per-tile partials summed in tile order), same H100, (kernel - FLOOR) / port:
# max 32.7, L2 35.5, per-element 68.4, 99.9th percentile 59.8 -- the default mode's figures on the same cases.
K_COARSE_WG = {"max": 50.0, "l2": 54.0, "pe_max": 104.0, "pe_999": 92.0}
SOFT_FIXTURES = sorted(p for p in os.listdir(su.GOLDEN) if p.startswith("render_") and p.endswith(".pt") and "_soft" in p)


class wgrad_all:
    """Option wgrad_all for the duration of a block, restored afterwards."""

    def __init__(self, value=1):
        self.value = value

    def __enter__(self):
        from nice_slam_b200 import _lib
        self.prev = _lib.get_option("wgrad_all")
        _lib.check(_lib.lib().nsb_set_option(b"wgrad_all", int(self.value)), "nsb_set_option")

    def __exit__(self, *exc):
        from nice_slam_b200 import _lib
        _lib.check(_lib.lib().nsb_set_option(b"wgrad_all", int(self.prev)), "nsb_set_option")


def kernel_names(prof):
    return [e.name.split("(")[0].split("::")[-1].split("<")[0] for e in prof.events() if e.device_type.name == "CUDA"]


# ------------------------------------------------------------------------------------ float64 yardstick
def check_all_decoders(label, stage, variant="soft", scale=1.0, n_rays=96, n_samples=None, n_surface=None, seed=0, det=0, channels_last=True):
    """check_case of test_gpu_f64 with every decoder of the stage graded and option wgrad_all on: truth on the kernel's saved ReLU bits (the
    weight-gradient kernel reads them, as the input-gradient one does).  Bars: K_FP32_PASS, the bars every decoder's weight gradients are
    held to; in the coarse stage K_COARSE_WG.  det = 1: option deterministic instead of wgrad_all (it implies it), whose kDet kernels and
    ordered sums add the same products in another order, held to the same bars."""
    sc, grids, dec_state = scene(variant=variant, scale=scale)
    n_samples = sc["rendering"]["N_samples"] if n_samples is None else n_samples
    n_surface = sc["rendering"]["N_surface"] if n_surface is None else n_surface
    ro, rd, gd, _ = su.make_rays(sc, n_rays, seed=1600 + n_rays)
    decs = fr.STAGE_DECODERS[stage]
    cot = cotangents(n_rays, seed)
    renderer, c, dec = make_renderer(sc, grids, dec_state, DEV, n_samples=n_samples, n_surface=n_surface, channels_last=channels_last)
    with options(wgrad_all=1 - det, deterministic=det):
        kern = kernel_run(renderer, c, dec, ro, rd, gd, stage, cot, GRIDS[stage], decs)
    args = (grids, dec_state, ro, rd, stage, gd if stage != "coarse" else None, su.scene_bound(sc)) + cot
    kw = dict(grad_grids=GRIDS[stage], grad_decoders=decs, n_samples=n_samples, n_surface=n_surface)
    port = fr.port_run(*args, **kw)
    tk = fr.run(*args, **kw, coarse_enlarge=sc["coarse_bound_enlarge"], masks=kern["masks"])
    tpt = fr.run(*args, **kw, coarse_enlarge=sc["coarse_bound_enlarge"], masks=port["masks"])
    assert torch.equal(kern["z_vals"], tk["z_vals"])
    inb_k = tk["fixed"]["inb"].reshape(tk["raw"].shape[:2])
    inb_p = tpt["fixed"]["inb"].reshape(tpt["raw"].shape[:2])
    truth_k, truth_p = dict(tensors(tk, inb_k, stage)), dict(tensors(tpt, inb_p, stage))
    mine, ports = dict(tensors(kern, inb_k, stage)), dict(tensors(port, inb_p, stage))
    failures = []
    for name, t in truth_k.items():
        bar = K_COARSE_WG if stage == "coarse" else K_FP32_PASS
        ek, ep = fr.errors(mine[name], t), fr.errors(ports[name], truth_p[name])
        print("f64 %-28s %-26s kernel %s port %s" % (label, name, " ".join("%.1e" % ek[m] for m in METRICS), " ".join("%.1e" % ep[m] for m in METRICS)))
        for m in METRICS:
            if not ek[m] <= bar[m] * ep[m] + FLOOR[m]:
                failures.append("%s %s %s: kernel %.2e > %.1f x port %.2e + %.0e" % (label, name, m, ek[m], bar[m], ep[m], FLOOR[m]))
    failures += check_masks(label, kern["masks"], tk["pre"], tk["fixed"]["inb"])
    assert not failures, "\n".join(failures)


@pytest.mark.parametrize("n_rays,stage,det", modes([(n, st) for n in (97, 95, 64, 31) for st in ("coarse", "middle", "fine", "color")], layout=False))
def test_all_decoder_weight_gradients_at_ragged_tiles_against_f64(n_rays, stage, det):
    """S = 33 (17 + 16; the coarse stage, rendered without depth: 33 uniform samples): N * S mod 128 = 1, 63, 64, 127."""
    ns, nsurf = (33, 16) if stage == "coarse" else (17, 16)
    check_all_decoders("wg all %s N=%d det=%d" % (stage, n_rays, det), stage, n_rays=n_rays, n_samples=ns, n_surface=nsurf, seed=n_rays, det=det)


@pytest.mark.parametrize("det", [0, 1])
@pytest.mark.parametrize("stage", ["coarse", "middle", "fine", "color"])
def test_all_decoder_weight_gradients_on_ncdhw_grids_against_f64(stage, det):
    """The reference's NCDHW grids (FusedRenderer(convert_grids=False)): the weight-gradient kernels gather the grid features through
    gather_tile_kt's strided branch, the scatter through grid_load4's scalar loads; N * S = 97 * 33 (mod 128 = 1)."""
    ns, nsurf = (33, 16) if stage == "coarse" else (17, 16)
    check_all_decoders("wg all %s ncdhw det=%d" % (stage, det), stage, n_rays=97, n_samples=ns, n_surface=nsurf, seed=97, det=det,
                       channels_last=False)


@pytest.mark.parametrize("stage,det", modes(["coarse", "middle", "fine", "color"], layout=False))
def test_all_decoder_weight_gradients_on_large_features_against_f64(stage, det):
    """Soft grids x 30 (activations in the tens)."""
    check_all_decoders("wg all %s soft x30 det=%d" % (stage, det), stage, scale=30.0, seed=16, det=det)


@pytest.mark.parametrize("stage,det", modes(["coarse", "middle"], layout=False))
def test_all_decoder_weight_gradients_in_the_saturated_scene_against_f64(stage, det):
    """Init grids (alpha = 1 at the first sample).  Stages fine and colour are not claimed there: their decoders' weight gradients sit at the
    float32 noise floor, and one bias element each goes past K_FP32_PASS (measured on an H100: fine fc_c.0.bias 1.9e-3 in max norm against
    the port's 1.8e-4, 10.6x; colour fc_c.0.bias 2.4e-4 per element against 1.6e-5, 14x) -- the fine and colour decoders' kernel code is the
    one option wgrad_all does not change (test_gpu_mapper_settings does not claim this scene for the fine decoder either)."""
    check_all_decoders("wg all %s init det=%d" % (stage, det), stage, variant="init", seed=17, det=det)


# ------------------------------------------------------------------------------------ reference fixtures
@pytest.mark.parametrize("layout", ["channels_last", "ncdhw"])
@pytest.mark.parametrize("name", SOFT_FIXTURES)
def test_reference_fixtures_with_every_decoder_on_tensor_cores(name, layout):
    """Every soft-scene render fixture (the real reference's outputs and all decoder gradients) at the tolerances of
    test_gpu_parity.test_render_against_reference_fixture, with wgrad_all on."""
    from test_gpu_parity import test_render_against_reference_fixture
    with wgrad_all(1):
        test_render_against_reference_fixture(os.path.join(su.GOLDEN, name), layout)


# ------------------------------------------------------------------------------------ kernel selection
def _trainable_scene():
    sc, grids, dec_state = scene()
    renderer, c, dec = make_renderer(sc, grids, dec_state, DEV)
    for p in dec.parameters():
        p.requires_grad_(True)                  # as the tracker's deep copy and the mapper's shared decoders leave them
    return sc, renderer, c, dec


def _profiled(fn, attempts=3):
    """Kernel names of one call of fn (after a warm-up call), from a trace that holds the call's device work.  A trace without both a render
    forward and a render backward kernel has lost device records, and the call is traced again: late in a long suite run, the trace of a
    whole fused mapping iteration once held its pack_kernel alone, with neither the render kernels nor the input copies around it."""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    for _ in range(attempts):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        names = kernel_names(prof)
        if any(n.startswith("render_fwd") for n in names) and any(n.startswith("render_bwd") for n in names):
            break
    return names


def test_dropin_tracking_call_takes_the_tensor_core_weight_gradients():
    """render_batch_ray + the torch tracking loss + backward(), 200 rays, stage color, every NICEDecoders parameter trainable: with wgrad_all
    the backward is render_bwd_wg_tile_kernel alone (no FP32-FMA render_bwd_kernel); without it, today's render_bwd_kernel."""
    sc, renderer, c, dec = _trainable_scene()
    ro, rd, gd, gc = (t.to(DEV) for t in su.make_rays(sc, 200, seed=1700))
    cam_ro = ro.clone().requires_grad_(True)

    def track():
        cam_ro.grad = None
        for p in dec.parameters():
            p.grad = None
        depth, var, color = renderer.render_batch_ray(c, dec, rd, cam_ro, DEV, "color", gt_depth=gd)
        tp.tracking_loss(depth, var, color, gd, gc.double(), sc["tracking"]["w_color_loss"]).backward()

    for on, want, not_want in ((1, "render_bwd_wg_tile_kernel", "render_bwd_kernel"), (0, "render_bwd_kernel", "render_bwd_wg_tile_kernel")):
        with wgrad_all(on):
            names = _profiled(track)
        assert want in names and not_want not in names, (on, names)
        assert all(p.grad is not None for lvl in ("fine", "color", "middle") for p in getattr(dec, lvl + "_decoder").parameters())


def test_coarse_mapper_call_takes_the_tensor_core_weight_gradients():
    """The coarse mapper's call (stage coarse, rendered without depth, the torch mapping loss): render_bwd_wg_coarse_tile_kernel with wgrad_all,
    render_bwd_kernel without it."""
    sc, renderer, c, dec = _trainable_scene()
    ro, rd, gd, gc = (t.to(DEV) for t in su.make_rays(sc, 996, seed=1800))
    c = {k: v.detach().requires_grad_(k == "grid_coarse") for k, v in c.items()}

    def coarse_map():
        c["grid_coarse"].grad = None
        for p in dec.parameters():
            p.grad = None
        depth, var, color = renderer.render_batch_ray(c, dec, rd, ro, DEV, "coarse", gt_depth=None)
        tp.mapping_loss(depth, color, gd, gc.float(), "coarse").backward()

    for on, want, not_want in ((1, "render_bwd_wg_coarse_tile_kernel", "render_bwd_kernel"),
                               (0, "render_bwd_kernel", "render_bwd_wg_coarse_tile_kernel")):
        with wgrad_all(on):
            names = _profiled(coarse_map)
        assert want in names and not_want not in names, (on, names)
        assert all(p.grad is not None for p in dec.coarse_decoder.parameters())


# ------------------------------------------------------------------------------------ real tracker, fused iteration
def test_real_tracker_iteration_with_trainable_decoders():
    """The tracker_color fixture (one real Tracker.optimize_cam_in_batch iteration) replayed through the drop-in with every decoder parameter
    trainable and wgrad_all on: the camera-tensor gradient, loss and depth as the reference's."""
    case = torch.load(os.path.join(su.GOLDEN, "tracker_color.pt"), map_location="cpu", weights_only=False)
    sc = su.load_scenes()[case["scene"]]
    renderer, c, dec = make_renderer(sc, su.make_grids(sc, case["variant"]), su.load_decoders(case["variant"]), DEV)
    assert all(p.requires_grad for p in dec.parameters())
    with wgrad_all(1):
        out = glue.tracking_iteration(sc, case, lambda rd, ro, stage, gd: renderer.render_batch_ray(c, dec, rd, ro, DEV, stage, gt_depth=gd),
                                      su.scene_bound(sc), device=DEV)
    assert torch.equal(out["rays_o"], case["rays_o"])
    assert rel(out["depth"], case["depth"]) < TOL
    assert abs(out["loss"] - case["loss"]) < TOL * abs(case["loss"])
    assert rel(out["d_camera"], case["d_camera"]) < TOL, (out["d_camera"], case["d_camera"])
    assert all(p.grad is not None for lvl in ("fine", "color", "middle") for p in getattr(dec, lvl + "_decoder").parameters())


@pytest.mark.parametrize("stage,gdec", [("middle", ("middle",)), ("color", ("fine", "color", "middle"))])
def test_fused_mapping_iteration_with_every_decoder_graded(stage, gdec):
    """IterationContext(grad_decoders=...) with wgrad_all: the kept layer outputs cover every graded decoder, the backward takes
    render_bwd_wg_tile_kernel, and loss, ray, voxel and decoder gradients match the oracle."""
    from nice_slam_b200._lib import LEVELS
    from nice_slam_b200.steps import IterationContext
    from test_gpu_parity import _flat_named
    sc = su.load_scenes()["room0"]
    grids, dec_state = su.make_grids(sc, "soft"), su.load_decoders("soft")
    renderer, c, dec = make_renderer(sc, grids, dec_state, DEV)
    n_rays = 300
    ro, rd, gd, gc = su.make_rays(sc, n_rays, seed=99)
    gg = GRIDS[stage]
    out = tp.iteration("map", grids, dec_state, ro, rd, gd, gc.float(), stage, su.scene_bound(sc), grad_grids=gg, grad_decoders=gdec)
    with wgrad_all(1):
        ctx = IterationContext(renderer, n_rays, stage, DEV, kind="map", grad_grids=gg, grad_decoders=gdec, host_staging=False)
        assert ctx.acts is not None and ctx.acts.shape[0] == len(gdec)
        names = _profiled(lambda: ctx.run(c, dec, ro.to(DEV), rd.to(DEV), gd.to(DEV), gc.float().to(DEV)))
    assert "render_bwd_wg_tile_kernel" in names and "render_bwd_kernel" not in names, names
    assert abs(float(ctx.loss) - float(out["loss"])) < TOL * abs(float(out["loss"]))
    assert rel(ctx.d_rays_o, out["d_rays_o"]) < TOL and rel(ctx.d_rays_d, out["d_rays_d"]) < TOL
    for k in gg:
        assert rel(ctx.d_grid[k], out["d_" + k]) < TOL, k
    for lvl in gdec:
        mine = _flat_named(LEVELS.index(lvl), ctx.d_flat[lvl])
        for k, v in out["d_dec"][lvl].items():
            assert rel(mine[k], v.reshape(-1)) < TOL, (lvl, k)


# ------------------------------------------------------------------------------------ no layer outputs under no_grad
def test_render_img_under_no_grad_keeps_no_layer_outputs():
    """render_img (no_grad, 100 000-ray chunks) with every decoder trainable: the same peak device memory with wgrad_all on as with it off
    (kept layer outputs would add ~9 GB per chunk).  The same batch rendered with grad enabled does keep them (the measurement sees them)."""
    sc, renderer, c, dec = _trainable_scene()
    depth, _ = su.make_frame(sc, 3)
    c2w, gtd = su.make_pose(sc, 3).to(DEV), depth.to(DEV)
    peak = {}
    for on in (0, 1):
        with wgrad_all(on):
            renderer.render_img(c, dec, c2w, DEV, "color", gt_depth=gtd)
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            renderer.render_img(c, dec, c2w, DEV, "color", gt_depth=gtd)
            torch.cuda.synchronize()
            peak[on] = torch.cuda.max_memory_allocated() - base
    print("render_img peak above the resident set: wgrad_all 0 %.1f MB, 1 %.1f MB" % (peak[0] / 2 ** 20, peak[1] / 2 ** 20))
    assert peak[1] == peak[0], peak
    n = 2000
    ro, rd, gd, _ = (t.to(DEV) for t in su.make_rays(sc, n, seed=1900))
    kept = {}
    for grad in (False, True):
        with wgrad_all(1), torch.set_grad_enabled(grad):
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            out = renderer.render_batch_ray(c, dec, rd, ro, DEV, "color", gt_depth=gd)
            torch.cuda.synchronize()
            kept[grad] = torch.cuda.max_memory_allocated() - base
            del out
    acts_bytes = 3 * n * 48 * 5 * 32 * 4
    assert kept[True] - kept[False] >= acts_bytes, (kept, acts_bytes)
