"""CPU: the oracle port replays the real multi-frame Tracker.run executions of tests/make_golden_tracker_frames.py -- recorded pixel draws,
get_camera_from_tensor + get_rays_from_uv, the bbox pre-filter, the median-gated loss, torch.optim.Adam (one group, or translation at lr and
quaternion at 0.2 lr) and the best-pose rule of each learning-rate mode, restated here.  Pins the fixtures and the chain that
tracking.FusedTrackingLoop replaces."""
import os

import pytest
import torch

import scene_util as su
from nice_slam_b200.mapping import tensor_from_c2w
from oracle import torch_port as tp

GOLD = os.path.join(su.GOLDEN, "tracker_frames")
CASES = ("shipped", "seperate_lr", "pixels1000")


def load(name):
    return torch.load(os.path.join(GOLD, name + ".pt"), map_location="cpu", weights_only=False)


def replay_frame(case, f, sc, grids, dec, bound):
    """Frame f (>= 1) of the case as Tracker.run optimises it.  Returns (losses, chosen iteration, c2w [4,4])."""
    s, cam = case["settings"], sc["cam"]
    depth, color = su.make_frame(sc, case["frame_seeds"][f])
    H0, W0 = s["ignore_edge_H"], s["ignore_edge_W"]
    Wr = cam["W"] - 2 * W0
    start = case["initial_tensors"][f - 1].clone()
    if s["seperate_LR"]:
        quad, T = start[:4].clone().requires_grad_(True), start[4:].clone().requires_grad_(True)
        opt = torch.optim.Adam([{"params": [T], "lr": s["lr"]}, {"params": [quad], "lr": s["lr"] * 0.2}])
    else:
        leaf = start.clone().requires_grad_(True)
        opt = torch.optim.Adam([leaf], lr=s["lr"])
    losses, best, candidate = [], 1e10, None
    for it in range(s["iters"]):
        cam_t = torch.cat([quad, T], 0) if s["seperate_LR"] else leaf
        assert torch.equal(cam_t.detach(), case["cams"][f - 1, it]), (f, it)
        k = case["draws"][f - 1, it].long()
        i, j = (W0 + k % Wr).float(), (H0 + k // Wr).float()
        ro, rd = tp.rays_from_uv(i, j, tp.camera_from_tensor(cam_t), cam["fx"], cam["fy"], cam["cx"], cam["cy"])
        gd, gc = depth[j.long(), i.long()], color[j.long(), i.long()]
        keep = tp.bbox_prefilter(ro, rd, gd, bound)
        opt.zero_grad()
        d, v, col = tp.render_batch_ray(grids, dec, rd[keep], ro[keep], "color", gd[keep], bound)
        loss = tp.tracking_loss(d, v, col, gd[keep], gc[keep], s["w_color_loss"], s["handle_dynamic"], s["use_color_in_tracking"])
        loss.backward()
        opt.step()
        losses.append(loss.item())
        if losses[-1] < best:                   # Tracker.py:245-247: camera_tensor after the step (one tensor), before it (torch.cat copy)
            best, candidate = losses[-1], (it, cam_t.detach().clone())
    c2w = torch.cat([tp.camera_from_tensor(candidate[1]), torch.tensor([[0, 0, 0, 1.0]])], 0)
    return torch.tensor(losses, dtype=torch.float64), candidate[0], c2w


@pytest.mark.parametrize("name", CASES)
def test_oracle_reproduces_real_tracker_runs(name):
    case = load(name)
    sc = su.load_scenes()[case["scene"]]
    grids, dec, bound = su.make_grids(sc, case["variant"]), su.load_decoders(case["variant"]), su.scene_bound(sc)
    est = case["estimate_c2w_list"]
    assert torch.equal(est[0], su.make_pose(sc, case["frame_seeds"][0]))          # frame 0 keeps its ground-truth pose
    for f in range(1, est.shape[0]):
        losses, chosen, c2w = replay_frame(case, f, sc, grids, dec, bound)
        want = case["losses"][f - 1]
        assert float(((losses - want).abs() / want.abs()).max()) < 1e-6, (f, losses, want)
        assert chosen == int(torch.argmin(want)), (f, chosen)
        assert float((c2w - est[f]).abs().max()) < 1e-6, (f, float((c2w - est[f]).abs().max()))


@pytest.mark.parametrize("name", CASES)
def test_start_poses_follow_the_constant_speed_rule(name):
    """The recorded start tensor of every frame is mapping.tensor_from_c2w of the previous estimate (frame 1), or of
    (est[f-1] @ est[f-2]^-1) @ est[f-1] (Tracker.py:190-200), up to the quaternion's sign."""
    case = load(name)
    est = case["estimate_c2w_list"]
    for f in range(1, est.shape[0]):
        pose = est[f - 1] @ est[f - 2].inverse() @ est[f - 1] if f >= 2 else est[f - 1]
        got, want = tensor_from_c2w(pose), case["initial_tensors"][f - 1]
        if float(got[:4] @ want[:4]) < 0:
            got[:4] = -got[:4]
        assert float((got - want).abs().max()) < 1e-5, (f, got, want)


def test_cases_cover_both_selection_rules_and_large_batches():
    """The fixtures exercise what they are for: a chosen iteration other than the last, an ungated depth-only loss, > 1024 draws."""
    cases = {n: load(n) for n in CASES}
    assert cases["seperate_lr"]["settings"]["seperate_LR"] and not cases["shipped"]["settings"]["seperate_LR"]
    assert cases["pixels1000"]["draws"].shape[-1] == 1000
    chosen = [int(torch.argmin(c["losses"][f])) for c in cases.values() for f in range(c["losses"].shape[0])]
    assert any(ci < len(c) - 1 for ci, c in zip(chosen, [c["losses"][f] for c in cases.values() for f in range(c["losses"].shape[0])]))
