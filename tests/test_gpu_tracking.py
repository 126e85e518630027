"""GPU: the tracker's per-frame loop (tracking.FusedTrackingLoop) -- its frame sampler against the reference's get_samples + bbox pre-filter
restated, its pose step against autograd through quad2rotation + torch.optim.Adam with both best-pose rules, and whole frames against the
real multi-frame Tracker.run executions of tests/make_golden_tracker_frames.py."""
import ctypes as C
import os

import pytest
import torch

import scene_util as su
from gpu_util import make_renderer, rel
from oracle import torch_port as tp

pytestmark = pytest.mark.gpu
DEV = "cuda"
VP = C.c_void_p
GOLD = os.path.join(su.GOLDEN, "tracker_frames")


@pytest.fixture(scope="module")
def room0():
    sc = su.load_scenes()["room0"]
    renderer, c, dec = make_renderer(sc, su.make_grids(sc, "soft"), su.load_decoders("soft"), DEV)
    return sc, renderer, c, dec


def loop_for(room0, settings):
    from nice_slam_b200.tracking import FusedTrackingLoop
    sc, renderer, c, dec = room0
    return FusedTrackingLoop(renderer, c, dec, settings["pixels"], **settings)


def test_frame_sampler_matches_get_samples_and_prefilter(room0):
    """nsb_track_samples on 3000 draws (three rounds of the one-CTA compaction) of a region with unequal, non-zero edges: kept mask, order and
    count exact, gathered depth / colour bit-exact, rays within the nsb_window_rays bars, dirs exact.  A band of far sensor depths makes
    the pre-filter drop rays."""
    from nice_slam_b200 import _lib
    L = _lib.lib()
    sc, renderer, _, _ = room0
    cam = sc["cam"]
    H, W = cam["H"], cam["W"]
    H0, H1, W0, W1 = 30, H - 45, 70, W - 10
    depth, color = su.make_frame(sc, 3)
    depth[200:260] = 40.0                                          # beyond every ray's bound exit
    from nice_slam_b200.mapping import tensor_from_c2w
    camera = tensor_from_c2w(su.make_pose(sc, 3))
    camera[:4] *= 1.03                                             # quad2rotation normalises: a non-unit quaternion is legal
    n, n_region = 3000, (H1 - H0) * (W1 - W0)
    draws = torch.randint(n_region, (n,), generator=torch.Generator().manual_seed(8))
    d = dict(cam=camera.to(DEV), draws=draws.to(DEV), depth=depth.to(DEV), color=color.to(DEV))
    out = {k: torch.full((n, 3), float("nan"), device=DEV) for k in ("ro", "rd", "dirs")}
    gd = torch.full((n,), float("nan"), device=DEV)
    gc = torch.full((n, 3), float("nan"), dtype=torch.float64, device=DEV)
    kept = torch.full((n,), -1, dtype=torch.int32, device=DEV)
    count = torch.zeros(1, dtype=torch.int32, device=DEV)
    b6 = (C.c_double * 6)(*su.scene_bound(sc).reshape(6).tolist())
    _lib.check(L.nsb_track_samples(VP(d["cam"].data_ptr()), VP(d["draws"].data_ptr()), n, VP(d["depth"].data_ptr()), VP(d["color"].data_ptr()), H, W,
                                   H0, H1, W0, W1, cam["fx"], cam["fy"], cam["cx"], cam["cy"], b6, VP(out["ro"].data_ptr()), VP(out["rd"].data_ptr()),
                                   VP(out["dirs"].data_ptr()), VP(gd.data_ptr()), VP(gc.data_ptr()), VP(kept.data_ptr()), VP(count.data_ptr()), None),
               "nsb_track_samples")
    # restatement: get_sample_uv's region indexing (common.py:110-122) + get_rays_from_uv + Tracker.py:95-104
    i, j = (W0 + draws % (W1 - W0)).float(), (H0 + draws // (W1 - W0)).float()
    wro, wrd = tp.rays_from_uv(i, j, tp.camera_from_tensor(camera), cam["fx"], cam["fy"], cam["cx"], cam["cy"])
    wgd = depth[H0:H1, W0:W1].reshape(-1)[draws]
    wgc = color[H0:H1, W0:W1].reshape(-1, 3)[draws]
    keep = tp.bbox_prefilter(wro, wrd, wgd, su.scene_bound(sc))
    k = int(count.item())
    assert 0 < k < n and k == int(keep.sum()), (k, int(keep.sum()))
    assert torch.equal(kept[:k].cpu().long(), torch.nonzero(keep).reshape(-1))
    assert torch.equal(gd[:k].cpu(), wgd[keep]) and torch.equal(gc[:k].cpu(), wgc[keep])
    assert float((out["ro"][:k].cpu() - wro[keep]).abs().max()) <= 1e-6 and float((out["rd"][:k].cpu() - wrd[keep]).abs().max()) <= 2e-6
    want_dirs = torch.stack([(i - cam["cx"]) / cam["fx"], -(j - cam["cy"]) / cam["fy"], -torch.ones_like(i)], -1)
    assert torch.equal(out["dirs"][:k].cpu(), want_dirs[keep])


@pytest.mark.parametrize("seperate_lr", [False, True])
def test_pose_step_matches_torch_adam_and_the_selection_rule(seperate_lr):
    """nsb_track_pose_step over six steps with gradients of mixed scale against autograd through get_camera_from_tensor + torch.optim.Adam
    (one group at lr, or translation at lr and quaternion at 0.2 lr), and the best-pose rule of Tracker.py:223-247: strict `<` from 1e10 (a tie
    keeps the first), a NaN loss never wins; the candidate is the tensor after the step (one tensor) or before it (seperate_LR)."""
    from nice_slam_b200 import _lib
    L = _lib.lib()
    g = torch.Generator().manual_seed(17)
    start = torch.tensor([0.9, 0.1, -0.3, 0.2, 0.4, -1.1, 2.0])
    lr = 1e-3
    if seperate_lr:
        quad, T = start[:4].clone().requires_grad_(True), start[4:].clone().requires_grad_(True)
        opt = torch.optim.Adam([{"params": [T], "lr": lr}, {"params": [quad], "lr": lr * 0.2}])
    else:
        leaf = start.clone().requires_grad_(True)
        opt = torch.optim.Adam([leaf], lr=lr)
    cam = start.clone().to(DEV)
    m, v, cand = torch.zeros(7, device=DEV), torch.zeros(7, device=DEV), torch.zeros(7, device=DEV)
    c2w16 = torch.zeros(16, device=DEV)
    losses = torch.zeros(6, dtype=torch.float64, device=DEV)
    best = torch.tensor([1e10, -1.0], dtype=torch.float64, device=DEV)
    seq = [5.0, 3.0, 3.0, float("nan"), 2.5, 4.0]
    want_best, want_cand = 1e10, None
    for step, lv in enumerate(seq, start=1):
        G = (torch.randn(3, 4, generator=g, dtype=torch.float64) * (300.0 if step % 2 else 0.01)).contiguous()
        cam_t = torch.cat([quad, T], 0) if seperate_lr else leaf
        before = cam_t.detach().clone()
        opt.zero_grad()
        (tp.camera_from_tensor(cam_t) * G.float()).sum().backward()
        opt.step()
        if lv < want_best:
            want_best, want_cand = lv, (step - 1, before if seperate_lr else leaf.detach().clone())
        loss_d = torch.tensor([lv], dtype=torch.float64, device=DEV)
        Gd = G.to(DEV)
        _lib.check(L.nsb_track_pose_step(VP(cam.data_ptr()), VP(loss_d.data_ptr()), VP(Gd.data_ptr()), VP(m.data_ptr()), VP(v.data_ptr()),
                                         lr, lr * 0.2 if seperate_lr else lr, 0.9, 0.999, 1e-8, step, 0 if seperate_lr else 1,
                                         VP(losses.data_ptr()), VP(best.data_ptr()), VP(cand.data_ptr()), VP(c2w16.data_ptr()), None),
                   "nsb_track_pose_step")
        now = torch.cat([quad, T]).detach() if seperate_lr else leaf.detach()
        assert float((cam.cpu() - now).abs().max()) < 2e-6, step
        assert float(best[0]) == want_best and int(best[1]) == want_cand[0], (step, best.tolist())
        assert float((cand.cpu() - want_cand[1]).abs().max()) < 2e-6, step
        want_c2w = torch.cat([tp.camera_from_tensor(want_cand[1]), torch.tensor([[0, 0, 0, 1.0]])], 0)
        assert float((c2w16.view(4, 4).cpu() - want_c2w).abs().max()) < 2e-6, step
    got = losses.cpu()
    assert torch.equal(got[~torch.isnan(got)], torch.tensor([x for x in seq if x == x], dtype=torch.float64)) and bool(torch.isnan(got[3]))


def flipped_rays(loop, case, f, upto, sc):
    """Rays whose gradient takes the other branch of the L1 loss on the GPU than in the reference, over iterations 0..upto of frame f: each
    iteration is sampled and rendered at the REFERENCE's recorded camera tensor, and the per-ray gradients are compared with the oracle's
    on the same rays (as test_gpu_ba.py counts them).  A residual |gt - depth| within rounding of zero makes such a ray's gradient change sign."""
    s = case["settings"]
    grids, dec, bound = su.make_grids(sc, "soft"), su.load_decoders("soft"), su.scene_bound(sc)
    flips = 0
    for it in range(upto + 1):
        loop.cam.copy_(case["cams"][f - 1, it])
        n = loop.sample(case["draws"][f - 1, it].to(DEV, torch.int64))
        loop.iterate(n)
        ro, rd = loop.rays_o[:n].cpu().requires_grad_(True), loop.rays_d[:n].cpu().requires_grad_(True)
        gd, gc = loop.gt_depth[:n].cpu(), loop.gt_color[:n].cpu()
        d, v, col = tp.render_batch_ray(grids, dec, rd, ro, "color", gd, bound)
        tp.tracking_loss(d, v, col, gd, gc, s["w_color_loss"], s["handle_dynamic"], s["use_color_in_tracking"]).backward()
        want = torch.cat([ro.grad, rd.grad], 1)
        got = torch.cat([loop.ctx.d_rays_o[:n], loop.ctx.d_rays_d[:n]], 1).cpu()
        flips += int(((got - want).abs().amax(1) > 1e-4 * float(want.abs().max())).sum())
    return flips


@pytest.mark.parametrize("name", ["shipped", "seperate_lr", "pixels1000"])
def test_whole_frames_against_real_tracker_run(room0, name):
    """Frames 1-3 of a real Tracker.run with its recorded draws: per-iteration losses within 1e-4 relative, the same chosen iteration, the final
    c2w within 1e-5 (as matrices: the quaternion's sign is free); the constant-speed start pose from the previous estimates.
    The tracking loss is an L1: a ray whose rendered depth is within rounding of its sensor depth can take the other sign on the GPU, which
    moves that iteration's pose gradient by ~2/n and, through Adam's normalised step, the pose by up to one learning rate.  A frame whose pose
    misses 1e-5 must show such rays in the per-ray comparison (flipped_rays), and gets one learning rate of slack per flipped ray."""
    from nice_slam_b200.mapping import tensor_from_c2w
    case = torch.load(os.path.join(GOLD, name + ".pt"), map_location="cpu", weights_only=False)
    sc = room0[0]
    loop = loop_for(room0, case["settings"])
    est = case["estimate_c2w_list"]
    for f in range(1, est.shape[0]):
        start = loop.initial_pose(est[f - 1], est[f - 2] if f >= 2 else None)
        got_t, want_t = tensor_from_c2w(start), case["initial_tensors"][f - 1]
        if float(got_t[:4] @ want_t[:4]) < 0:
            got_t[:4] = -got_t[:4]
        assert float((got_t - want_t).abs().max()) < 1e-5, (f, got_t, want_t)
        depth, color = su.make_frame(sc, case["frame_seeds"][f])
        c2w = loop.track_frame(color, depth, want_t, draws=case["draws"][f - 1])
        want = case["losses"][f - 1]
        losses = loop.losses.cpu()
        assert float(((losses - want).abs() / want.abs()).max()) < 1e-4, (f, losses, want)
        assert loop.best_iter == int(torch.argmin(want)), (f, loop.best_iter, want)
        err = float((c2w.cpu() - est[f]).abs().max())
        if err >= 1e-5:
            flips = flipped_rays(loop, case, f, loop.best_iter, sc)
            assert 0 < flips <= 3 and err < 1e-5 + flips * case["settings"]["lr"], (f, err, flips)


def test_default_draws_follow_torch_randint(room0):
    """Without recorded draws every iteration calls torch.randint(n_region, (pixels,), device) as select_uv does: after the same seed, the
    loop leaves the CUDA generator where as many direct calls leave it, and replaying those calls' draws gives the same frame."""
    s = dict(ignore_edge_W=20, ignore_edge_H=20, pixels=200, iters=4, lr=0.001, seperate_LR=False, handle_dynamic=True,
             use_color_in_tracking=True, w_color_loss=0.5, const_speed_assumption=True)
    sc = room0[0]
    loop = loop_for(room0, s)
    depth, color = su.make_frame(sc, 21)
    start = su.make_pose(sc, 20)
    torch.cuda.manual_seed(99)
    c2w = loop.track_frame(color, depth, start)
    losses, state = loop.losses.clone(), torch.cuda.get_rng_state()
    torch.cuda.manual_seed(99)
    draws = torch.stack([torch.randint(loop.n_region, (s["pixels"],), device=DEV) for _ in range(s["iters"])])
    assert torch.equal(torch.cuda.get_rng_state(), state)
    c2w2 = loop.track_frame(color, depth, start, draws=draws)
    assert rel(loop.losses, losses) < 1e-6 and rel(c2w2, c2w) < 1e-6


def test_errors(room0):
    """A batch the pre-filter empties raises (the reference fails in median()); a renderer configured for perturbed sampling is refused."""
    from nice_slam_b200.tracking import FusedTrackingLoop
    sc, renderer, c, dec = room0
    s = dict(ignore_edge_W=20, ignore_edge_H=20, pixels=64, iters=2)
    loop = loop_for(room0, s)
    depth, color = su.make_frame(sc, 2)
    with pytest.raises(RuntimeError, match="kept no ray"):
        loop.track_frame(color, torch.full_like(depth, 1e6), su.make_pose(sc, 2))
    with pytest.raises(RuntimeError, match="draws must lie"):
        loop.track_frame(color, depth, su.make_pose(sc, 2), draws=torch.full((2, 64), loop.n_region))
    perturb, renderer.perturb = renderer.perturb, 1.0
    try:
        with pytest.raises(RuntimeError, match="perturb"):
            FusedTrackingLoop(renderer, c, dec, 64, **s)
    finally:
        renderer.perturb = perturb
