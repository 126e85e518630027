"""GPU: the mapper's fix_fine / fix_color / frustum_feature_selection settings in the native loop (mapping.FusedMappingLoop) against real
Mapper.optimize_map runs (tests/make_golden_mapper_settings.py), the two-decoder fused Adam step against torch.optim.Adam, and the fine
decoder's weight gradients -- alone in stage fine, beside the colour decoder's in stage colour -- against the float64 reference."""
import os

import pytest
import torch

import scene_util as su
from gpu_util import make_renderer, rel
from oracle import f64_ref as fr
from test_gpu_f64 import GRIDS, K_FP32_PASS, check_case, check_masks, cotangents, kernel_run, options, scene, yardstick

pytestmark = pytest.mark.gpu
DEV = "cuda"
GOLD = os.path.join(su.GOLDEN, "mapper_settings")


def test_two_decoder_adam_matches_torch_adam_over_one_group():
    """nsb_adam_mapper_step_decoders against torch.optim.Adam with the fine and colour decoders in ONE parameter group (fix_fine = False,
    Mapper.py:336-341, :368) beside a voxel group, through middle -> fine -> color -> color: in stage middle neither decoder has a gradient
    (Adam skips both), in stage fine the fine decoder steps at decoders_lr = 0 (its state advances, its values stay), the colour decoder's
    first step is in stage color."""
    from nice_slam_b200._lib import LEVELS, flat_layout
    from nice_slam_b200.masked import MaskedVoxels
    from nice_slam_b200.optim import FusedMapperAdam
    sc = su.load_scenes()["room0"]
    grids, dec_state = su.make_grids(sc, "soft"), su.load_decoders("soft")
    renderer, c, dec = make_renderer(sc, grids, dec_state, DEV)
    key = "grid_fine"
    g = torch.Generator(device=DEV).manual_seed(5)
    vm = torch.rand(c[key].shape[2:], device=DEV, generator=g) < 0.4
    mv = MaskedVoxels(c[key], vm)
    mask5 = vm.unsqueeze(0).unsqueeze(0).expand_as(c[key])
    val_ref = c[key].clone()
    val_grad = val_ref[mask5].clone().requires_grad_(True)
    levels = ("fine", "color")
    ref = {lvl: {k: v.detach().clone().requires_grad_(True) for k, v in getattr(dec, lvl + "_decoder").named_parameters()} for lvl in levels}
    opt = torch.optim.Adam([{"params": list(ref["fine"].values()) + list(ref["color"].values()), "lr": 0.0}, {"params": [val_grad], "lr": 0.0}])
    lay = {lvl: flat_layout(LEVELS.index(lvl)) for lvl in levels}
    fused = FusedMapperAdam()
    fine0 = {k: v.detach().clone() for k, v in ref["fine"].items()}
    schedule = [("middle", 0.0, 0.1), ("fine", 0.0, 0.005), ("color", 0.005, 0.005), ("color", 0.005, 0.005)]
    for step, (stage, lr_d, lr_v) in enumerate(schedule):
        graded = [lvl for lvl in levels if (lvl == "fine" and stage != "middle") or (lvl == "color" and stage == "color")]
        gv = torch.randn(mv.count, 32, device=DEV, generator=g) * (10.0 ** (-step))
        opt.param_groups[0]["lr"], opt.param_groups[1]["lr"] = lr_d, lr_v
        val_grad.grad = mv.to_reference(gv)
        items = []
        for lvl in levels:
            if lvl in graded:
                gflat = torch.randn(sum(n for _, _, n in lay[lvl]), device=DEV, generator=g) * 0.1
                for name, off, cnt in lay[lvl]:
                    ref[lvl][name].grad = gflat[off:off + cnt].view_as(ref[lvl][name]).clone()
                items.append((lvl, dec, gflat, lr_d))
            else:
                for p in ref[lvl].values():
                    p.grad = None
        opt.step()
        fused.step_all([(key, c[key], mv, gv, lr_v)], items, renderer=renderer)
        want = val_ref.clone()
        want[mask5] = val_grad.detach()
        assert rel(c[key], want) < 1e-6, step
        assert torch.equal(c[key][~mask5], val_ref[~mask5])
        for lvl in levels:
            mine = dict(getattr(dec, lvl + "_decoder").named_parameters())
            for name, p in ref[lvl].items():
                assert rel(mine[name], p) < 1e-6, (step, lvl, name)
            st = fused.state.get("dec_" + lvl)
            want_steps = max((opt.state[p]["step"] for p in ref[lvl].values() if p in opt.state), default=0)
            assert (st["step"] if st else 0) == int(want_steps), (step, lvl)
        if stage == "fine":
            assert all(torch.equal(dict(dec.fine_decoder.named_parameters())[k].detach(), v) for k, v in fine0.items())


def test_fused_mapping_loop_with_fix_fine_false_against_real_mapper():
    """Five real joint iterations (3 x middle, fine, color) with fix_fine = False and the real torch Adam against FusedMappingLoop(fix_fine=False):
    the fine decoder gets weight gradients in stages fine and color and shares the fused Adam launch with the colour decoder.  The closeness rules
    of the default-settings loop test (sign-like first Adam steps: the bulk tight, outliers few)."""
    from nice_slam_b200.mapping import FusedMappingLoop
    case = torch.load(os.path.join(GOLD, "joint_fix_fine_false.pt"), map_location="cpu", weights_only=False)
    sc = su.load_scenes()[case["scene"]]
    dec_state = su.load_decoders(case["variant"])
    renderer, c, dec = make_renderer(sc, su.make_grids(sc, case["variant"]), dec_state, DEV)
    depth, _ = su.make_frame(sc, case["frame_seed"])
    c2w = su.make_pose(sc, case["pose_seed"])
    start = {k: v.clone() for k, v in c.items()}
    loop = FusedMappingLoop(renderer, c, dec, c2w, depth.to(DEV), w_color=case["w_color_loss"], fix_fine=False)
    assert [loop.grad_decoders(s) for s in ("middle", "fine", "color")] == [(), ("fine",), ("fine", "color")]
    for it in case["iterations"]:
        loss = loop.iteration(it["stage"], it["rays_o"].to(DEV), it["rays_d"].to(DEV), it["gt_depth"].to(DEV), it["gt_color"].to(DEV), it["lr"])
        assert bool(torch.isfinite(loss).all())
    for key, fin in case["final"].items():
        mv = loop.masked[key]
        after = mv.to_reference(mv.gather(c[key])).cpu()
        before = mv.to_reference(mv.gather(start[key])).cpu()
        got, want = after[fin["idx"]], fin["val"]
        close = (got - want).abs() <= 1e-3 * (1 + want.abs())
        assert float(close.float().mean()) > 0.995, (key, float(close.float().mean()))
        dn = float((after - before).double().norm())
        assert abs(dn - fin["delta_norm"]) < 0.02 * fin["delta_norm"], (key, dn, fin["delta_norm"])
        m5 = (mv.slot_map.view(c[key].shape[2:]) >= 0).unsqueeze(0).unsqueeze(0).expand_as(c[key])
        assert torch.equal(c[key][~m5], start[key][~m5])
    for lvl in ("fine", "color"):
        mine = dict(getattr(dec, lvl + "_decoder").named_parameters())
        for k, v in case[lvl + "_decoder"].items():
            close = (mine[k].detach().cpu() - v).abs() <= 1e-3 * (1 + v.abs())
            assert float(close.float().mean()) > 0.99, (lvl, k, float(close.float().mean()))
        assert any(not torch.equal(mine[k].detach().cpu(), dec_state[lvl][k]) for k in dec_state[lvl]), lvl


def test_color_refinement_loop_with_ba_against_real_mapper():
    """Real colour-refinement iterations with BA (fix_color = True, frustum_feature_selection = False; the reference's schedule with ratios 0
    makes the first iteration 'middle', the rest 'color') against FusedMappingLoop(fix_color=True, frustum_feature_selection=False) +
    enable_ba + iteration_ba: every voxel of each grid is a parameter, so voxels outside the current frustum move too; no decoder moves; the
    fixed frame stays and the other poses land within a fifth of the reference's update (four sign-like first Adam steps on L1 losses, with
    every voxel of three grids moving under them)."""
    from nice_slam_b200.mapping import FusedMappingLoop
    from nice_slam_b200.masked import frustum_voxel_mask
    case = torch.load(os.path.join(GOLD, "color_refine_ba.pt"), map_location="cpu", weights_only=False)
    sc = su.load_scenes()[case["scene"]]
    dec_state = su.load_decoders(case["variant"])
    renderer, c, dec = make_renderer(sc, su.make_grids(sc, case["variant"]), dec_state, DEV)
    depth, _ = su.make_frame(sc, case["frame_seed"])
    c2w_cur = su.make_pose(sc, case["pose_seed"])
    start = {k: v.clone() for k, v in c.items()}
    win = case["window_keyframes"]
    fixed = win.index(min(k for k in win if k >= 0))
    loop = FusedMappingLoop(renderer, c, dec, None, None, w_color=case["w_color_loss"], fix_color=True, frustum_feature_selection=False)
    assert all(loop.masked[k].count == c[k][0, 0].numel() for k in loop.masked)
    loop.enable_ba(case["window_c2w"], fixed, case["BA_cam_lr"], camera_tensors=case["camera_tensors"])
    for stage, lr, dr in zip(case["stages"], case["lrs"], case["draws"]):
        assert loop.grad_decoders(stage) == ()
        loss = loop.iteration_ba(stage, dr["i"].to(DEV), dr["j"].to(DEV), dr["depth"].to(DEV), dr["color"].to(DEV), lr)
        assert bool(torch.isfinite(loss).all())
    got = loop.window_c2w().cpu()
    want, s0 = case["final_c2w"], case["window_c2w"]
    assert torch.equal(got[fixed], s0[fixed])
    failures = []
    for r in range(6):
        if r != fixed:
            upd, off = float((want[r] - s0[r]).norm()), float((got[r] - want[r]).norm())
            print("refine pose row %d: off %.2e of the reference's update %.2e" % (r, off, upd))
            if not off < 0.2 * upd:
                failures.append("pose row %d: %.2e >= 0.2 x %.2e" % (r, off, upd))
    for key, fin in case["final"].items():
        after = c[key].detach().cpu().reshape(-1)
        got_v, want_v = after[fin["idx"]], fin["val"]
        close = float(((got_v - want_v).abs() <= 2e-3 * (1 + want_v.abs())).float().mean())
        dn = float((after - start[key].cpu().reshape(-1)).double().norm())
        outside = ~frustum_voxel_mask(renderer, c2w_cur, key, c[key], depth.to(DEV))
        o5 = outside.unsqueeze(0).unsqueeze(0).expand_as(c[key])
        moved_out = int((c[key][o5] != start[key][o5]).sum())
        print("refine %s: close %.4f, delta norm %.4e (reference %.4e), moved outside the frustum %d (reference %d)" %
              (key, close, dn, fin["delta_norm"], moved_out, case["moved_outside_frustum"][key]))
        if not close > 0.99:
            failures.append("%s: close %.4f" % (key, close))
        if not abs(dn - fin["delta_norm"]) < 0.03 * fin["delta_norm"]:
            failures.append("%s: delta norm %.4e vs %.4e" % (key, dn, fin["delta_norm"]))
        if moved_out == 0:
            failures.append("%s: no voxel outside the frustum moved" % key)
    assert not failures, failures
    for lvl in ("fine", "color", "middle", "coarse"):
        mine = dict(getattr(dec, lvl + "_decoder").named_parameters())
        assert all(torch.equal(mine[k].detach().cpu(), v) for k, v in dec_state[lvl].items()), lvl


# ------------------------------------------------------------------------------------ fine-decoder weight gradients against float64
# (stage, decoders with weight gradients): what FusedMappingLoop(fix_fine=False) asks for in stages fine and color.  Both sets are served by the
# tensor-core weight-gradient kernel (render_bwd_wg_tile_kernel) from the forward's kept layer outputs and saved ReLU bits: the float64 truth runs
# on those bits.  The bars are those every occupancy decoder's weight gradients are held to (K_FP32_PASS): the fine decoder's bias gradients are
# sums over the points of dL/d occupancy, whose signs vary, and the kernel adds its per-warp partial sums with float atomics, so on a single bias
# element it sits up to 11x the float32 port's error (measured on an H100: fine fc_c.0.bias on the x30 grids, 2.6e-3 against 2.4e-4).
CASES = {"fine": ("fine",), "color": ("fine", "color")}


@pytest.mark.parametrize("stage", ["fine", "color"])
@pytest.mark.parametrize("n_rays", [97, 95, 64, 31])
def test_fine_decoder_weight_gradients_on_tensor_cores_at_ragged_tiles_against_f64(n_rays, stage):
    """S = 33 (17 + 16): N * S mod 128 = 1, 63, 64, 127."""
    sc, grids, dec = scene()
    ro, rd, gd, _ = su.make_rays(sc, n_rays, seed=1300 + n_rays)
    check_case("wg %s N=%d" % ("+".join(CASES[stage]), n_rays), sc, grids, dec, stage, ro, rd, gd, GRIDS[stage], CASES[stage],
               n_samples=17, n_surface=16, seed=n_rays, k_bar=K_FP32_PASS, opts=dict(wgrad_tc=1))


@pytest.mark.parametrize("stage", ["fine", "color"])
@pytest.mark.parametrize("variant,scale", [("soft", 30.0)])
def test_fine_decoder_weight_gradients_on_tensor_cores_value_ranges_against_f64(variant, scale, stage):
    """Large features (soft grids x 30).  The saturated scene (init grids) is not claimed: there the fine decoder's weight gradients are at the
    float32 noise floor (alpha = 1 at the first sample) and the kernel's per-element errors reach 12-19x the port's (measured)."""
    sc, grids, dec = scene(variant=variant, scale=scale)
    ro, rd, gd, _ = su.make_rays(sc, 96, seed=1400)
    check_case("wg %s %s x%g" % ("+".join(CASES[stage]), variant, scale), sc, grids, dec, stage, ro, rd, gd, GRIDS[stage], CASES[stage],
               seed=14, k_bar=K_FP32_PASS, opts=dict(wgrad_tc=1))


@pytest.mark.parametrize("stage", ["fine", "color"])
@pytest.mark.parametrize("variant,scale", [("init", 1.0), ("soft", 30.0)])
def test_fine_decoder_weight_gradients_fp32_pass_against_f64(variant, scale, stage):
    """Option wgrad_tc = 0: the same sets through the FP32-FMA weight-gradient pass, beside the tile input-gradient launch of the middle decoder.
    The two launches decide their ReLUs in different places -- the tile launch on the forward's saved bits, the FP32-FMA pass on its own float32
    recomputation -- so the float64 truth follows each: the saved bits for the middle decoder, its own signs for the others; the bars are the
    FP32-FMA pass's (test_gpu_f64.test_all_decoder_gradients_against_f64)."""
    sc, grids, dec_state = scene(variant=variant, scale=scale)
    ro, rd, gd, _ = su.make_rays(sc, 96, seed=1400)
    label = "wg fp32 %s %s x%g" % ("+".join(CASES[stage]), variant, scale)
    cot = cotangents(96, 14)
    renderer, c, dec = make_renderer(sc, grids, dec_state, DEV)
    with options(wgrad_tc=0):
        kern = kernel_run(renderer, c, dec, ro, rd, gd, stage, cot, GRIDS[stage], CASES[stage])
    args = (grids, dec_state, ro, rd, stage, gd, su.scene_bound(sc)) + cot
    kw = dict(grad_grids=GRIDS[stage], grad_decoders=CASES[stage], n_samples=sc["rendering"]["N_samples"], n_surface=sc["rendering"]["N_surface"])
    port = fr.port_run(*args, **kw)
    own = fr.run(*args, **kw, coarse_enlarge=sc["coarse_bound_enlarge"])
    mixed = kern["masks"].clone()
    for j, lvl in enumerate(fr.STAGE_DECODERS[stage]):
        if lvl in CASES[stage]:
            mixed[:, j] = own["masks"][:, j]
    tk = fr.run(*args, **kw, coarse_enlarge=sc["coarse_bound_enlarge"], masks=mixed)
    tpt = fr.run(*args, **kw, coarse_enlarge=sc["coarse_bound_enlarge"], masks=port["masks"])
    assert torch.equal(kern["z_vals"], tk["z_vals"])
    failures = yardstick(label, kern, tk, port, tpt, stage, K_FP32_PASS) + check_masks(label, kern["masks"], tk["pre"], tk["fixed"]["inb"])
    assert not failures, "\n".join(failures)


@pytest.mark.parametrize("stage", ["fine", "color"])
def test_fine_decoder_weight_gradients_take_the_tensor_core_kernel(stage):
    """Profiler: a mapping iteration with the fine decoder's weight gradients (stage fine: fine; stage color: fine + colour) launches
    render_bwd_wg_tile_kernel and not the FP32-FMA render_bwd_kernel; with wgrad_tc = 0 the reverse."""
    from torch.profiler import ProfilerActivity, profile
    from nice_slam_b200.steps import IterationContext
    sc, grids, dec_state = scene()
    renderer, c, dec = make_renderer(sc, grids, dec_state, DEV)
    ro, rd, gd, gc = (t.to(DEV) for t in su.make_rays(sc, 200, seed=1500))
    ctx = IterationContext(renderer, 200, stage, DEV, kind="map", grad_grids=GRIDS[stage], grad_decoders=CASES[stage], host_staging=False)
    assert ctx.acts is not None and ctx.acts.shape[0] == len(CASES[stage])
    for tc, want, not_want in ((1, "render_bwd_wg_tile_kernel", "render_bwd_kernel"), (0, "render_bwd_kernel", "render_bwd_wg_tile_kernel")):
        with options(wgrad_tc=tc):
            ctx.run(c, dec, ro, rd, gd, gc.float())
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                ctx.run(c, dec, ro, rd, gd, gc.float())
                torch.cuda.synchronize()
        names = [e.name for e in prof.events() if e.device_type.name == "CUDA"]
        assert any(want in nm for nm in names), (tc, names)
        assert not any(nm.split("(")[0].split("::")[-1].split("<")[0] == not_want for nm in names), (tc, names)
