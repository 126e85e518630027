"""Generate tests/golden/mesh/room0.pt from the UNMODIFIED reference Mesher (src/utils/Mesher.py, imported through tests/ref_harness.py,
which stubs open3d / skimage / trimesh) on CPU, room0 geometry, 'soft' grids.

    python tests/make_golden_mesh.py        # needs the reference checkout

Mesher.__init__ opens the dataset, so the methods run on an instance whose attributes are set as __init__ sets them.  Recorded:
  grid_points  Mesher.get_grid_uniform(24)['grid_points'] (float32, the reference's meshgrid('xy') order) and its axes
  z            Mesher.eval_points(grid_points, stage 'fine')[:, 3]
  edge_points  float32 points between float32(bound) and bound (and on either side of it), with eval_points' occupancy
  probe        float32 points: the lattice and 2000 points near lattice points
  seen_kf / seen_all  point_masks' seen output of the probe points for 5 keyframes (keyframe mode, depth maxima) and for estimate_c2w_list[0..4]
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

OUT = os.path.join(su.GOLDEN, "mesh")
RES = 24
KEYFRAME_SEEDS = [40, 41, 42, 43, 44]


def edge_points(bound):
    """For each axis and side: the float32 values just inside / at / just outside float32(bound), other coordinates at the centre."""
    b = bound.numpy()
    ctr = b.mean(1).astype(np.float32)
    pts = []
    for a in range(3):
        for side in (0, 1):
            f = np.float32(b[a][side])
            for v in (np.nextafter(f, np.float32(-np.inf)), f, np.nextafter(f, np.float32(np.inf))):
                p = ctr.copy(); p[a] = v; pts.append(p)
    return torch.from_numpy(np.stack(pts))


def main():
    rh.import_reference()
    from src.utils.Mesher import Mesher
    sc, cfg, slam, renderer = mg.ref_scene("room0", "soft")
    m = Mesher.__new__(Mesher)                     # the attributes Mesher.__init__ sets (Mesher.py:26-51), without the dataset
    m.points_batch_size, m.ray_batch_size, m.renderer = 500000, 100000, renderer
    m.coarse, m.scale, m.occupancy = cfg["coarse"], cfg["scale"], cfg["occupancy"]
    for k in ("resolution", "level_set", "clean_mesh_bound_scale", "remove_small_geometry_threshold", "color_mesh_extraction_method",
              "get_largest_components", "depth_test"):
        setattr(m, k, cfg["meshing"][k])
    m.bound, m.nice, m.verbose = slam.bound, True, False
    m.marching_cubes_bound = torch.from_numpy(np.array(cfg["mapping"]["marching_cubes_bound"]) * m.scale)
    m.H, m.W, m.fx, m.fy, m.cx, m.cy = slam.H, slam.W, slam.fx, slam.fy, slam.cx, slam.cy
    grid = m.get_grid_uniform(RES)
    with torch.no_grad():
        z = m.eval_points(grid["grid_points"], slam.shared_decoders, slam.shared_c, "fine", "cpu")[:, 3].clone()
        ep = edge_points(slam.bound)
        ez = m.eval_points(ep.clone(), slam.shared_decoders, slam.shared_c, "fine", "cpu")[:, 3].clone()
    kf = []
    for s in KEYFRAME_SEEDS:
        depth, color = su.make_frame(sc, s)
        kf.append(dict(est_c2w=su.make_pose(sc, s), depth=depth, color=color))
    est = torch.stack([k["est_c2w"] for k in kf])
    rng = np.random.RandomState(5)
    pts = grid["grid_points"].numpy().astype(np.float64)
    near = pts[rng.choice(len(pts), 2000, replace=False)] + rng.normal(0, 0.02, (2000, 3))
    probe = np.concatenate([pts, near]).astype(np.float32).astype(np.float64)
    seen_kf = m.point_masks(probe, kf, est, len(kf) - 1, "cpu", get_mask_use_all_frames=False)[0]
    seen_all = m.point_masks(probe, kf, est, len(kf) - 1, "cpu", get_mask_use_all_frames=True)[0]
    os.makedirs(OUT, exist_ok=True)
    torch.save(dict(resolution=RES, marching_cubes_bound=cfg["mapping"]["marching_cubes_bound"], scale=cfg["scale"],
                    axes=[torch.as_tensor(x).clone() for x in grid["xyz"]], grid_points=grid["grid_points"], z=z, edge_points=ep, edge_z=ez,
                    keyframe_seeds=KEYFRAME_SEEDS, probe=torch.from_numpy(probe.astype(np.float32)), seen_kf=torch.from_numpy(seen_kf),
                    seen_all=torch.from_numpy(seen_all)),
               os.path.join(OUT, "room0.pt"))


if __name__ == "__main__":
    main()
