"""Generate tests/golden/tracker_frames/*.pt: the UNMODIFIED reference Tracker.run (imported from the reference checkout through
tests/ref_harness.py) tracking four synthetic frames on CPU, room0 geometry, 'soft' grids.

    python tests/make_golden_tracker_frames.py        # needs the reference checkout

Each fixture stores seeds, not images (frames: scene_util.make_frame / make_pose), the tracking settings, and what the run produced:
every torch.randint draw of select_uv (int32, [frame][iteration][pixels]), the camera tensor every optimize_cam_in_batch call received and
the loss it returned, the initial camera tensor of each tracked frame, and estimate_c2w_list.  Frame 0 takes its ground-truth pose
(Tracker.py:180-185); frames 1-3 are optimised.

    shipped.pt          the shipped configs/nice_slam.yaml tracking settings (ignore_edge 20, 200 px x 10 iterations, seperate_LR False,
                        handle_dynamic and colour on, constant-speed start)
    seperate_lr.pt      room0's ignore_edge 100, seperate_LR True (the other best-pose rule, quaternion at 0.2 lr), handle_dynamic False,
                        use_color_in_tracking False (the ungated depth-only loss)
    pixels1000.pt       the shipped settings with 1000 px x 3 iterations: batches above 1024 rays before the pre-filter, and the render's
                        batch depth maxima outside the forward kernel when more than 1024 survive
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import make_golden as mg        # noqa: E402
import ref_harness as rh        # noqa: E402
import scene_util as su         # noqa: E402

OUT = os.path.join(su.GOLDEN, "tracker_frames")
N_FRAMES = 4
FRAME_SEEDS = [20, 21, 22, 23]
TORCH_SEED = 2024
SHIPPED = dict(ignore_edge_W=20, ignore_edge_H=20, pixels=200, iters=10, lr=0.001, seperate_LR=False, handle_dynamic=True,
               use_color_in_tracking=True, w_color_loss=0.5, const_speed_assumption=True)
CASES = {
    "shipped": SHIPPED,
    "seperate_lr": dict(SHIPPED, ignore_edge_W=100, ignore_edge_H=100, seperate_LR=True, handle_dynamic=False, use_color_in_tracking=False),
    "pixels1000": dict(SHIPPED, pixels=1000, iters=3),
}


class _NoVisualizer:
    def vis(self, *a, **k):
        pass


def tracker_for_run(cfg, slam, renderer, frames, device="cpu"):
    """A reference Tracker whose own run() can be driven (Tracker.py:130-253): ref_harness.make_tracker's attributes plus the loop's --
    `frames` is the frame loader (an iterable of (idx [1], gt_color [1,H,W,3], gt_depth [1,H,W], gt_c2w [1,4,4]) batches, as a DataLoader of
    batch size 1 yields them), sync_method 'free', a visualiser that draws nothing, verbose and low_gpu_mem off.  Grids and decoders are
    taken from slam.shared_c / shared_decoders by run()'s own update_para_from_mapping."""
    t = rh.make_tracker(cfg, slam, renderer, device=device)
    tr = cfg["tracking"]
    t.sync_method = "free"
    t.verbose = False
    t.low_gpu_mem = False
    t.frame_loader = frames
    t.n_img = len(frames)
    t.visualizer = _NoVisualizer()
    t.shared_c, t.shared_decoders = slam.shared_c, slam.shared_decoders
    t.mapping_idx = torch.zeros(1).int()
    t.prev_mapping_idx = -1
    t.idx = torch.zeros(1).int()
    t.estimate_c2w_list = torch.zeros(len(frames), 4, 4)
    t.gt_c2w_list = torch.zeros(len(frames), 4, 4)
    t.cam_lr, t.num_cam_iters, t.tracking_pixels = tr["lr"], tr["iters"], tr["pixels"]
    t.gt_camera, t.seperate_LR, t.const_speed_assumption = tr["gt_camera"], tr["seperate_LR"], tr["const_speed_assumption"]
    t.every_frame = cfg["mapping"]["every_frame"]
    t.no_vis_on_first_frame = cfg["mapping"]["no_vis_on_first_frame"]
    return t


def frames(sc):
    out = []
    for k, s in enumerate(FRAME_SEEDS):
        depth, color = su.make_frame(sc, s)
        out.append((torch.tensor([k]), color.unsqueeze(0), depth.unsqueeze(0), su.make_pose(sc, s).unsqueeze(0)))
    return out


def gen_case(name, settings):
    rh.import_reference()
    import src.Tracker as tracker_mod
    sc, cfg, slam, renderer = mg.ref_scene("room0", "soft")
    cfg = dict(cfg)
    cfg["tracking"] = dict(cfg["tracking"], **settings, gt_camera=False)
    tracker = tracker_for_run(cfg, slam, renderer, frames(sc))
    draws, cams, losses, tensors = [], [], [], []
    _ri, _gtc = torch.randint, tracker_mod.get_tensor_from_camera
    _opt = tracker.optimize_cam_in_batch

    def randint_rec(*a, **k):
        r = _ri(*a, **k)
        draws.append(r.clone())
        return r

    def gtc_rec(*a, **k):
        r = _gtc(*a, **k)
        tensors.append(r.clone())
        return r

    def opt_rec(camera_tensor, *a, **k):
        cams.append(camera_tensor.detach().clone())
        loss = _opt(camera_tensor, *a, **k)
        losses.append(loss)
        return loss
    torch.randint, tracker_mod.get_tensor_from_camera, tracker.optimize_cam_in_batch = randint_rec, gtc_rec, opt_rec
    try:
        torch.manual_seed(TORCH_SEED); np.random.seed(TORCH_SEED)
        tracker.run()
    finally:
        torch.randint, tracker_mod.get_tensor_from_camera = _ri, _gtc
    it, n = settings["iters"], settings["pixels"]
    tracked = N_FRAMES - 1
    assert len(draws) == len(losses) == len(cams) == tracked * it and len(tensors) == 2 * tracked
    H, W = sc["cam"]["H"], sc["cam"]["W"]
    n_region = (H - 2 * settings["ignore_edge_H"]) * (W - 2 * settings["ignore_edge_W"])
    assert all(tuple(d.shape) == (n,) and int(d.max()) < n_region for d in draws)
    obj = dict(scene="room0", variant="soft", frame_seeds=FRAME_SEEDS, torch_seed=TORCH_SEED, settings=settings,
               draws=torch.stack(draws).to(torch.int32).view(tracked, it, n),
               cams=torch.stack(cams).view(tracked, it, 7),
               losses=torch.tensor(losses, dtype=torch.float64).view(tracked, it),
               initial_tensors=torch.stack(tensors[1::2]),                   # get_tensor_from_camera(gt_c2w) comes first in each frame
               estimate_c2w_list=tracker.estimate_c2w_list.clone())
    os.makedirs(OUT, exist_ok=True)
    path = os.path.join(OUT, name + ".pt")
    torch.save(obj, path)
    print("wrote %-16s %8.1f KB  losses %s" % (name + ".pt", os.path.getsize(path) / 1024, [round(float(v), 3) for v in obj["losses"][:, -1]]))


if __name__ == "__main__":
    import warnings
    warnings.filterwarnings("ignore")
    for name in (sys.argv[1:] or CASES):
        gen_case(name, CASES[name])
