"""Time the 2D reconstruction metric (recon.eval_depth_l1) on synthetic rooms of about 0.5 M and 2 M faces: tests/cull_scene.box_room with
24 closed boxes inside it (furniture: occlusion, faces behind the camera), 1000 views x 2 meshes at 500 x 500.

  kernel  nsb_depth_render of the 1000 views of one mesh, in launches of the batch render_depth picks, bracketed by CUDA events after
          one warm-up; the median of --rounds
  views   depth.sample_views of 1000 views against an unseen-region cloud (the vertices 16 poses inside the room do not see,
          cull.cull_mesh), host clock
  e2e     recon.eval_depth_l1 of a moved copy against the room (ICP, views, 2 x 1000 renders, view errors), host clock

The render runs --rounds times, the view sampling and the metric --host-rounds times.  Medians and spreads (max - min) are printed as
one JSON line, with the card's name, power limit and SM clocks read with nvidia-smi in the same run.

python tools/bench_depth_l1.py [--rounds 5] [--host-rounds 2] [--views 1000] [--steps 0.022 0.011]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

from measure import card, log, median_spread, time_call                        # noqa: E402


def furnished_room(step, n_boxes=24, seed=0):
    """box_room(step) with n_boxes closed boxes of 0.3-1.0 m standing on its floor, all sides at about `step`."""
    from cull_scene import ROOM, box_room
    rs = np.random.RandomState(seed)
    v, f = box_room(step)
    vs, fs, base = [v], [f], len(v)
    for _ in range(n_boxes):
        size = rs.uniform(0.3, 1.0, 3)
        bv, bf = box_room(step, tuple(size))
        lo = np.array([rs.uniform(0.1, ROOM[0] - size[0] - 0.1), rs.uniform(0.1, ROOM[1] - size[1] - 0.1), 0.0])
        vs.append(bv + lo)
        fs.append(bf + base)
        base += len(bv)
    return np.concatenate(vs), np.concatenate(fs)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--host-rounds", type=int, default=2, help="rounds of the view sampling and of the end-to-end metric")
    ap.add_argument("--views", type=int, default=1000)
    ap.add_argument("--steps", type=float, nargs="+", default=[0.022, 0.011], help="box_room steps (0.022: 0.5 M faces, 0.011: 2 M)")
    a = ap.parse_args()
    from cull_scene import room_poses
    from nice_slam_b200 import depth as dp
    from nice_slam_b200.cull import cull_mesh
    from nice_slam_b200.recon import eval_depth_l1
    from oracle.recon import rigid, transform_points
    res = dict(card=card(), views=a.views, H=500, W=500, sizes=[])
    for step in a.steps:
        v, f = furnished_room(step)
        case = dict(faces=int(len(f)), vertices=int(len(v)))
        log("room: %d faces, %d vertices" % (len(f), len(v)))
        seen, _ = cull_mesh(v, f, room_poses(16, 1, max_pitch_deg=40.0))
        unseen = v[seen.cpu().numpy() == 0]
        t0 = time.perf_counter()
        c2w, drawn, rejected = dp.sample_views(v, unseen, a.views, seed=0)
        t_views = [time.perf_counter() - t0]
        for _ in range(a.host_rounds - 1):
            t0 = time.perf_counter()
            dp.sample_views(v, unseen, a.views, seed=0)
            t_views.append(time.perf_counter() - t0)
        case["views"] = dict(median_spread([1e3 * t for t in t_views]), candidates=int(drawn), rejected=int(rejected), unseen_points=int(len(unseen)))
        dp.render_depth(v, f, c2w)                                     # warm-up
        ms = [time_call(lambda: dp.render_depth(v, f, c2w))[1] for _ in range(a.rounds)]
        case["kernel_ms_per_mesh"] = median_spread(ms)
        mv = transform_points(v, rigid(0.01, (0.0, 0.0, 1.0), (0.02, -0.01, 0.01)))
        eval_depth_l1((mv, f), (v, f), unseen, n_views=a.views)      # warm-up
        e2e, val = [], None
        for _ in range(a.host_rounds):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            val = eval_depth_l1((mv, f), (v, f), unseen, n_views=a.views)["depth_l1"]
            torch.cuda.synchronize()
            e2e.append(1e3 * (time.perf_counter() - t0))
        case["e2e_ms"] = median_spread(e2e)
        case["depth_l1_cm"] = val
        log("  " + json.dumps(case))
        res["sizes"].append(case)
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
