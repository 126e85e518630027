"""CPU: the real Mapper.optimize_map calls of tests/make_golden_mapper_frames.py against the oracle port and against mapping.FusedMapper's
host-side logic.  The oracle replays each call's first iteration from its recorded draws (per-row get_samples under the window's poses,
torch.cat, the bbox pre-filter, the render and the mapping loss); the window, its fixed row, pixs_per_image, the stage schedule and the
learning rates FusedMapper derives must be the reference's, the overlap pick under the recorded numpy seed and the global pick included."""
import os

import numpy as np
import pytest
import torch

import scene_util as su
from nice_slam_b200.keyframes import pick_overlap
from nice_slam_b200.mapping import map_stage, random_select, stage_lrs, tensor_from_c2w, window_rows
from oracle import keyframes as okf
from oracle import torch_port as tp

GOLD = os.path.join(su.GOLDEN, "mapper_frames")
CASES = ("ba_overlap", "no_ba", "first_frame", "coarse")


def load(name):
    return torch.load(os.path.join(GOLD, name + ".pt"), map_location="cpu", weights_only=False)


def selection_of(case, sc):
    """The keyframes FusedMapper.select_window picks for the case, with the overlap counts from the oracle's restatement of
    keyframe_selection_overlap on the recorded draw."""
    s, cam = case["settings"], sc["cam"]
    K = len(case["keyframe_seeds"])
    np.random.seed(case["seed"])
    if K == 0:
        return []
    if s["keyframe_selection_method"] == "global":
        return random_select(K - 1, s["mapping_window_size"] - 2)
    k = case["overlap_draw"].long()
    i, j = (k % cam["W"]).float(), (k // cam["W"]).float()
    depth, _ = su.make_frame(sc, case["frame_seed"])
    ro, rd = tp.rays_from_uv(i, j, su.make_pose(sc, case["frame_seed"]), cam["fx"], cam["fy"], cam["cx"], cam["cy"])
    pts = okf.overlap_points(ro, rd, depth.reshape(-1)[k])
    counts = [okf.percent_inside(pts, su.make_pose(sc, seed), cam["H"], cam["W"], cam["fx"], cam["fy"], cam["cx"], cam["cy"])[1]
              for seed in case["keyframe_seeds"][:K - 1]]
    return pick_overlap(counts, pts.shape[0], s["mapping_window_size"] - 2)


@pytest.mark.parametrize("name", CASES)
def test_host_logic_reproduces_the_reference_call(name):
    case = load(name)
    sc = su.load_scenes()[case["scene"]]
    s = case["settings"]
    assert [int(x) for x in selection_of(case, sc)] == case["selection"]
    K = len(case["keyframe_seeds"])
    rows, fixed = window_rows(case["selection"], K)
    F = case["draws"].shape[1]
    assert len(rows) == F and rows[-1] == -1 and (K == 0 or rows[-2] == K - 1)
    assert fixed == (None if K == 0 else rows.index(min(rows[:-1])))
    assert case["draws"].shape[2] == s["pixels"] // F
    stages = [map_stage(it, case["iters"], s["middle_iter_ratio"], s["fine_iter_ratio"], case["coarse_mapper"]) for it in range(case["iters"])]
    assert stages == case["stages"]
    lr = stage_lrs(s["stage"], stages[0], case["lr_factor"])
    assert lr["middle"] == s["stage"][stages[0]]["middle_lr"] * case["lr_factor"] and set(lr) == {"decoders", "coarse", "middle", "fine", "color"}


def test_cases_cover_every_stage_and_both_selections():
    cases = {n: load(n) for n in CASES}
    assert {"middle", "fine", "color"} <= set(cases["ba_overlap"]["stages"]) and set(cases["coarse"]["stages"]) == {"coarse"}
    assert cases["ba_overlap"]["settings"]["keyframe_selection_method"] == "overlap" and len(cases["ba_overlap"]["selection"]) > 1
    assert cases["coarse"]["settings"]["keyframe_selection_method"] == "global" and cases["first_frame"]["draws"].shape[1] == 1
    assert cases["ba_overlap"]["cur_c2w"] is not None and cases["no_ba"]["cur_c2w"] is None


@pytest.mark.parametrize("name", CASES)
def test_oracle_reproduces_the_first_iteration(name):
    """The first iteration's inputs are the reference's own: its loss, replayed through the oracle port from the recorded draws."""
    case = load(name)
    sc = su.load_scenes()[case["scene"]]
    cam = sc["cam"]
    grids, dec, bound = su.make_grids(sc, case["variant"]), su.load_decoders(case["variant"]), su.scene_bound(sc)
    K = len(case["keyframe_seeds"])
    rows, fixed = window_rows(case["selection"], K)
    frames = [su.make_frame(sc, case["keyframe_seeds"][k] if k >= 0 else case["frame_seed"]) for k in rows]
    poses = [su.make_pose(sc, case["keyframe_seeds"][k] if k >= 0 else case["frame_seed"]) for k in rows]
    ro, rd, gd, gc = [], [], [], []
    for r, k in enumerate(case["draws"][0].long()):
        pose = tp.camera_from_tensor(tensor_from_c2w(poses[r])) if case["ba"] and r != fixed else poses[r]
        o, d = tp.rays_from_uv((k % cam["W"]).float(), (k // cam["W"]).float(), pose, cam["fx"], cam["fy"], cam["cx"], cam["cy"])
        ro.append(o.float()); rd.append(d.float())
        gd.append(frames[r][0].reshape(-1)[k].float()); gc.append(frames[r][1].reshape(-1, 3)[k].float())
    ro, rd, gd, gc = (torch.cat(x) for x in (ro, rd, gd, gc))
    keep = tp.bbox_prefilter(ro, rd, gd, bound)
    stage = case["stages"][0]
    d, _, col = tp.render_batch_ray(grids, dec, rd[keep], ro[keep], stage, None if case["coarse_mapper"] else gd[keep], bound)
    loss = float(tp.mapping_loss(d, col, gd[keep], gc[keep], stage, case["settings"]["w_color_loss"]))
    want = float(case["losses"][0])
    assert abs(loss - want) <= 1e-5 * abs(want), (loss, want)
