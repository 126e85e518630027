"""Time ground-truth culling (nice_slam_b200.cull) on synthetic box rooms of about 0.5 M and 2 M vertices (tests/cull_scene.py) with 200
and 2000 camera poses inside them (pitch within +-25 degrees: about 1 % of the vertices stay unseen and run every pose).

  kernel     nsb_cull_seen and nsb_cull_faces + emit, each bracketed by CUDA events after an L2 flush (a 256 MB write)
  cli        python -m nice_slam_b200.cull's main() in this process (PLY read, poses, culling, PLY write), host clock
  reference  cull_mesh.py's per-pose loop restated in torch on the same GPU: per pose an upload of the vertices, a float32 projection
             and the .cpu() copies of uv and z (its host round trip), host clock

Each size runs one warm-up and --rounds timed rounds (--ref-rounds for the reference loop); medians and spreads (max - min) are
reported with the card's name, power limit and SM clocks, read with nvidia-smi in the same run.

python tools/bench_cull.py [--rounds 5] [--ref-rounds 2] [--out results/bench_cull.json]
"""
import argparse
import contextlib
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

from cull_scene import box_room, room_poses, write_ply_with_extras, write_traj   # noqa: E402
from measure import Flush, card, log, median_spread, time_call                # noqa: E402

STEPS = {"0.5M": 0.0109, "2M": 0.0054}                        # box_room grid steps: 0.50 M and 2.03 M vertices
POSES = (200, 2000)


def kernel_round(v, f, w2c, flush):
    from nice_slam_b200.cull import cull_faces, cull_seen
    seen, seen_ms, _ = time_call(lambda: cull_seen(v, w2c), flush)
    kept, faces_ms, _ = time_call(lambda: cull_faces(f, seen), flush)
    return dict(seen_ms=seen_ms, faces_ms=faces_ms), seen, kept


def reference_loop(pc, poses):
    """cull_mesh.py:47-70 restated in torch (float32 on the GPU, the mask on the host)."""
    H, W, fx, fy, cx, cy = 680, 1200, 600.0, 600.0, 599.5, 339.5
    whole_mask = np.ones(pc.shape[0]).astype(bool)
    for c2w in poses:
        points = torch.from_numpy(pc.copy()).cuda()
        w2c = torch.from_numpy(np.linalg.inv(c2w)).cuda().float()
        K = torch.from_numpy(np.array([[fx, .0, cx], [.0, fy, cy], [.0, .0, 1.0]]).reshape(3, 3)).cuda()
        ones = torch.ones_like(points[:, 0]).reshape(-1, 1).cuda()
        homo_points = torch.cat([points, ones], dim=1).reshape(-1, 4, 1).cuda().float()
        cam_cord = (w2c @ homo_points)[:, :3]
        cam_cord[:, 0] *= -1
        uv = K.float() @ cam_cord.float()
        z = uv[:, -1:] + 1e-5
        uv = (uv[:, :2] / z).float().squeeze(-1).cpu().numpy()
        mask = (0 <= -z[:, 0, 0].cpu().numpy()) & (uv[:, 0] < W) & (uv[:, 0] > 0) & (uv[:, 1] < H) & (uv[:, 1] > 0)
        whole_mask &= ~mask
    return ~whole_mask


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--ref-rounds", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_cull.py measures on the GPU"
    from nice_slam_b200 import cull
    res = dict(card=card(), rounds=a.rounds, ref_rounds=a.ref_rounds, cases=[])
    flush = Flush()
    with tempfile.TemporaryDirectory() as tmp:
        for vname, step in STEPS.items():
            v, f = box_room(step)
            gt = os.path.join(tmp, "room.ply")
            write_ply_with_extras(gt, v, f)
            v = v.astype(np.float32).astype(np.float64)                       # the vertices the CLI reads back
            vd, fd = torch.from_numpy(v).cuda(), torch.from_numpy(f).int().cuda()
            for P in POSES:
                c2w = room_poses(P, 1, 25.0)
                traj, out = os.path.join(tmp, "traj.txt"), os.path.join(tmp, "out.ply")
                write_traj(traj, c2w)
                w2c = torch.from_numpy(cull.w2c_of(cull.load_poses(traj))).cuda()
                log("%s vertices (%d), %d faces, %d poses" % (vname, len(v), len(f), P))
                kernel_round(vd, fd, w2c, flush)                                # warm-up
                rounds = [kernel_round(vd, fd, w2c, flush) for _ in range(a.rounds)]
                seen, kept = rounds[0][1].cpu().numpy(), rounds[0][2].cpu().numpy()
                assert all(torch.equal(r[1], rounds[0][1]) and torch.equal(r[2], rounds[0][2]) for r in rounds)
                argv = ["--input_mesh", gt, "--traj", traj, "--output_mesh", out]
                cli = []
                for i in range(a.rounds):
                    h0 = time.perf_counter()
                    with contextlib.redirect_stdout(sys.stderr):
                        cull.main(argv)
                    torch.cuda.synchronize()
                    cli.append((time.perf_counter() - h0) * 1e3)
                ref, ref_seen = [], None
                for i in range(a.ref_rounds):
                    torch.cuda.synchronize()
                    h0 = time.perf_counter()
                    ref_seen = reference_loop(v, list(cull.load_poses(traj)))
                    torch.cuda.synchronize()
                    ref.append((time.perf_counter() - h0) * 1e3)
                case = dict(vertices=int(len(v)), faces=int(len(f)), poses=P, unseen=float(1 - seen.mean()), kept_faces=int(len(kept)),
                            seen_kernel_ms=median_spread([r[0]["seen_ms"] for r in rounds]),
                            faces_kernel_ms=median_spread([r[0]["faces_ms"] for r in rounds]),
                            cli_ms=median_spread(cli), reference_loop_ms=median_spread(ref) if ref else None,
                            reference_mask_differs=int((ref_seen != seen.astype(bool)).sum()) if ref_seen is not None else None)
                log("  " + json.dumps(case))
                res["cases"].append(case)
    res["card_after"] = card()
    print("card: %s" % res["card"])
    print("%9s %6s %8s | %16s %16s %16s %18s" % ("vertices", "poses", "unseen", "seen kernel ms", "faces kernel ms", "CLI ms", "per-pose loop ms"))
    for c in res["cases"]:
        ms = lambda d: "%9.3f +- %-5.3f" % (d["median"], d["spread"]) if d else "not run"
        print("%9d %6d %7.2f%% | %16s %16s %16s %18s" % (c["vertices"], c["poses"], 100 * c["unseen"], ms(c["seen_kernel_ms"]),
                                                          ms(c["faces_kernel_ms"]), ms(c["cli_ms"]), ms(c["reference_loop_ms"])))
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
