"""Time a whole RGB-D sequence through slam.FusedSLAM on the GPU and report its ATE.

    python tools/bench_slam_sequence.py [--frames 51] [--rounds 2] [--out DIR]

Frames are rendered on the GPU with FusedRenderer.render_img (depth and colour, stage 'color') from the room0 'soft' scene along a known
trajectory (tests/slam_sequences.path_pose), so tracking has a consistent scene to follow.  Each round then runs the shipped Replica
settings from the same start (the 'soft' grids and decoders): 1500 first-frame iterations, every_frame 5, 60 iterations per mapped frame,
BA once there are more than 4 keyframes, colour refinement on the last frame, the coarse mapper on.  A short warm-up run loads every
module and shape first.  No L2 flush: a run is one long stream of work.  Reports the wall time per phase (host clock up to a device
synchronise at the end of each phase), frames per second, the ATE of the run, the card, its power limit and the spread over the rounds.
Needs a CUDA device; there is no CPU fallback."""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402

import scene_util as su  # noqa: E402
from gpu_util import make_renderer  # noqa: E402
from measure import card  # noqa: E402
from nice_slam_b200 import FusedSLAM, ate_rmse  # noqa: E402
from slam_sequences import path_pose  # noqa: E402

STAGE = {"coarse": dict(decoders_lr=0.0, coarse_lr=0.001, middle_lr=0.0, fine_lr=0.0, color_lr=0.0),
         "middle": dict(decoders_lr=0.0, coarse_lr=0.0, middle_lr=0.1, fine_lr=0.0, color_lr=0.0),
         "fine": dict(decoders_lr=0.0, coarse_lr=0.0, middle_lr=0.005, fine_lr=0.005, color_lr=0.0),
         "color": dict(decoders_lr=0.005, coarse_lr=0.0, middle_lr=0.005, fine_lr=0.005, color_lr=0.005)}
TRACKING = dict(ignore_edge_W=20, ignore_edge_H=20, iters=10, lr=0.001, pixels=200, seperate_LR=False, handle_dynamic=True,
                use_color_in_tracking=True, w_color_loss=0.5, const_speed_assumption=True, gt_camera=False)
MAPPING = dict(pixels=1000, mapping_window_size=5, middle_iter_ratio=0.4, fine_iter_ratio=0.6, stage=STAGE, BA_cam_lr=0.001, w_color_loss=0.2,
               keyframe_selection_method="overlap", fix_fine=True, fix_color=False, frustum_feature_selection=True, every_frame=5,
               keyframe_every=50, ckpt_freq=500, no_log_on_first_frame=True, iters=60, iters_first=1500, lr_factor=1.0, lr_first_factor=5.0,
               color_refine=True, BA=True, save_selected_keyframes_info=False)
CFG = dict(tracking=TRACKING, mapping=MAPPING, coarse=True, sync_method="strict")


def frames_for(sc, n):
    renderer, c, dec = make_renderer(sc, su.make_grids(sc, "soft"), su.load_decoders("soft"), "cuda")
    out = []
    for k in range(n):
        pose = path_pose(sc, k)
        depth, _, color = renderer.render_img(c, dec, pose, "cuda", "color")
        out.append((k, color.float().clamp(0, 1).cpu(), depth.float().cpu(), pose))
    return out


def one_run(sc, frames, ckpt_dir=None, cfg=CFG):
    renderer, c, dec = make_renderer(sc, su.make_grids(sc, "soft"), su.load_decoders("soft"), "cuda")
    slam = FusedSLAM(renderer, c, dec, cfg, seed=0, ckpt_dir=ckpt_dir)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    est, gt = slam.run(frames)
    torch.cuda.synchronize()
    return time.perf_counter() - t0, dict(slam.times), ate_rmse(est, gt)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=51)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_slam_sequence: needs a CUDA device")
    gpu = card()
    sc = su.load_scenes()["room0"]
    frames = frames_for(sc, a.frames)
    warm = dict(CFG, mapping=dict(MAPPING, iters_first=20, iters=10))
    one_run(sc, frames[:7], cfg=warm)
    rounds = []
    for r in range(a.rounds):
        import tempfile
        with tempfile.TemporaryDirectory() as d:
            total, phases, ate = one_run(sc, frames, ckpt_dir=d)
        rounds.append(dict(total_s=total, phases_s=phases, fps=a.frames / total, ate_m=ate))
        print("round %d: %.3f s  %.2f frames/s  ATE %.4f m  %s" % (r, total, a.frames / total, ate,
                                                                 {k: round(v, 3) for k, v in phases.items()}), flush=True)
    # baseline for the ATE: the same frames with the mapping cut to one iteration per call, so the map stays (nearly) the one the frames
    # were rendered from; the difference to the rounds above is what mapping on these frames does to the trajectory
    base = dict(CFG, mapping=dict(MAPPING, iters_first=1, iters=1))
    b_total, _, b_ate = one_run(sc, frames, cfg=base)
    print("baseline (1 mapping iteration per call): %.3f s  ATE %.4f m" % (b_total, b_ate), flush=True)
    tot = [x["total_s"] for x in rounds]
    res = dict(card=gpu, frames=a.frames, rounds=rounds, total_s_min=min(tot), total_s_max=max(tot),
               spread=(max(tot) - min(tot)) / min(tot), fps=a.frames / min(tot), ate_m=rounds[0]["ate_m"],
               baseline_one_mapping_iteration=dict(total_s=b_total, ate_m=b_ate))
    print(json.dumps(res))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_slam_sequence.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
