"""CPU: the oracle port replays the real Mapper.optimize_map runs with the `mapping:` settings the default leaves off
(tests/make_golden_mapper_settings.py): fix_fine = False, and the colour-refinement pass (fix_color = True, frustum_feature_selection =
False) with bundle adjustment.  Pins the chains that FusedMappingLoop's settings replace."""
import os

import torch

import scene_util as su
from oracle import frustum as fr
from oracle import torch_port as tp

GOLD = os.path.join(su.GOLDEN, "mapper_settings")
KEYS = ("grid_middle", "grid_fine", "grid_color")


def rel(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return float((a - b).abs().max() / (b.abs().max() + 1e-30))


def test_oracle_reproduces_joint_iterations_with_fix_fine_false():
    """Five real joint iterations (3 x middle, fine, color) with fix_fine = False: the fine decoder's parameters are in parameter group 0 beside
    the colour decoder's.  Adam skips the fine decoder in stage middle (it is not evaluated), steps it with decoders_lr = 0 in stage fine
    (state advances, values stay) and for real in stage color."""
    case = torch.load(os.path.join(GOLD, "joint_fix_fine_false.pt"), map_location="cpu", weights_only=False)
    sc = su.load_scenes()[case["scene"]]
    grids, dec = su.make_grids(sc, case["variant"]), su.load_decoders(case["variant"])
    depth, _ = su.make_frame(sc, case["frame_seed"])
    c2w = su.make_pose(sc, case["pose_seed"])
    bound = su.scene_bound(sc)
    m5 = {k: fr.frustum_mask(c2w, k, tuple(grids[k].shape[2:]), depth.numpy(), bound, sc["cam"]).unsqueeze(0).unsqueeze(0).expand_as(grids[k])
          for k in KEYS}
    val_grad = {k: grids[k][m5[k]].clone().requires_grad_(True) for k in KEYS}
    dw = {n: {k: v.clone().requires_grad_(n in ("fine", "color")) for k, v in W.items()} for n, W in dec.items()}
    opt = torch.optim.Adam([{"params": list(dw["fine"].values()) + list(dw["color"].values()), "lr": 0}] +
                           [{"params": [val_grad[k]], "lr": 0} for k in KEYS])
    fine0 = {k: v.detach().clone() for k, v in dw["fine"].items()}
    for it in case["iterations"]:
        opt.param_groups[0]["lr"] = it["lr"]["decoders"]
        for gi, k in enumerate(KEYS):
            opt.param_groups[1 + gi]["lr"] = it["lr"][k[5:]]
        g = {k: v.clone() for k, v in grids.items()}
        for k in KEYS:
            g[k][m5[k]] = val_grad[k]
        opt.zero_grad()
        d, _, col = tp.render_batch_ray(g, dw, it["rays_d"], it["rays_o"], it["stage"], it["gt_depth"], bound)
        tp.mapping_loss(d, col, it["gt_depth_loss"], it["gt_color"], it["stage"], case["w_color_loss"]).backward()
        fine_grad = any(p.grad is not None for p in dw["fine"].values())
        assert fine_grad == (it["stage"] != "middle"), it["stage"]
        opt.step()
        if it["stage"] == "fine":                                       # decoders_lr = 0: the state advances, the values do not
            assert all(torch.equal(dw["fine"][k].detach(), fine0[k]) for k in fine0)
            assert all(opt.state[p]["step"] == 1 for p in dw["fine"].values())
        for k in KEYS:
            grids[k][m5[k]] = val_grad[k].detach()
    for k, fin in case["final"].items():
        got = val_grad[k].detach()[fin["idx"]]
        assert torch.allclose(got, fin["val"], rtol=1e-5, atol=1e-6), (k, float((got - fin["val"]).abs().max()))
    for lvl in ("fine", "color"):
        for k, v in case[lvl + "_decoder"].items():
            assert torch.allclose(dw[lvl][k].detach(), v, rtol=1e-5, atol=1e-6), (lvl, k)
        assert any(not torch.equal(dw[lvl][k].detach(), dec[lvl][k]) for k in dec[lvl]), lvl


def test_oracle_reproduces_color_refinement_with_ba():
    """Real colour-refinement iterations with bundle adjustment (fix_color = True, frustum_feature_selection = False, middle / fine ratios 0):
    every voxel of every grid is a leaf parameter (Mapper.py:302-312), parameter group 0 is empty, the poses move in the 'color' iterations.
    With both ratios 0 the reference's schedule makes the first iteration a 'middle' one (Mapper.py:403-409)."""
    case = torch.load(os.path.join(GOLD, "color_refine_ba.pt"), map_location="cpu", weights_only=False)
    sc = su.load_scenes()[case["scene"]]
    cam = sc["cam"]
    grids, dec = su.make_grids(sc, case["variant"]), su.load_decoders(case["variant"])
    bound = su.scene_bound(sc)
    assert case["stages"][0] == "middle" and set(case["stages"][1:]) == {"color"}
    start = {k: grids[k].clone() for k in KEYS}
    leaf = {k: grids[k].clone().requires_grad_(True) for k in KEYS}
    win = case["window_keyframes"]
    fixed = win.index(min(k for k in win if k >= 0))
    cams = [case["camera_tensors"][k].clone().requires_grad_(True) for k in range(5)]
    opt = torch.optim.Adam([{"params": [], "lr": 0}, {"params": [], "lr": 0}] + [{"params": [leaf[k]], "lr": 0} for k in KEYS]
                           + [{"params": cams, "lr": 0}])
    for it, (stage, lr, dr) in enumerate(zip(case["stages"], case["lrs"], case["draws"])):
        for gi, k in enumerate(KEYS):
            opt.param_groups[2 + gi]["lr"] = lr[k[5:]]
        if stage == "color":
            opt.param_groups[5]["lr"] = case["BA_cam_lr"]
        g = dict(grids, **leaf)
        opt.zero_grad()
        n = dr["i"].shape[1]
        fid = torch.arange(6).repeat_interleave(n)
        ro, rd = tp.ba_window_rays(torch.stack(cams), case["window_c2w"][fixed], fixed, dr["i"].reshape(-1), dr["j"].reshape(-1), fid,
                                   cam["fx"], cam["fy"], cam["cx"], cam["cy"])
        gd, gc = dr["depth"].reshape(-1), dr["color"].reshape(-1, 3)
        keep = tp.bbox_prefilter(ro, rd, gd, bound)
        d, _, col = tp.render_batch_ray(g, dec, rd[keep], ro[keep], stage, gd[keep], bound)
        tp.mapping_loss(d, col, gd[keep], gc[keep], stage, case["w_color_loss"]).backward()
        hist = case["camera_history"][it]
        assert rel(torch.stack([c.detach() for c in cams]), hist["cam"]) < 1e-6 and rel(torch.stack([c.grad for c in cams]), hist["grad"]) < 1e-4, it
        opt.step()
    got = tp.camera_from_tensor(torch.stack([c.detach() for c in cams]))
    want = torch.stack([case["final_c2w"][r] for r in range(6) if r != fixed])
    assert float((got - want).abs().max()) < 2e-5, float((got - want).abs().max())
    for k, fin in case["final"].items():
        after = leaf[k].detach().reshape(-1)
        gotv = after[fin["idx"]]
        assert torch.allclose(gotv, fin["val"], rtol=1e-4, atol=2e-5), (k, float((gotv - fin["val"]).abs().max()))
        dn = float((after - start[k].reshape(-1)).double().norm())
        assert abs(dn - fin["delta_norm"]) < 1e-3 * fin["delta_norm"], (k, dn, fin["delta_norm"])
        assert case["moved_outside_frustum"][k] > 0
