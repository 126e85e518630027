"""Time each phase of the reconstruction metric (nice_slam_b200.recon.eval_recon) on FusedMesher meshes of room0's 'soft' grids (10
synthetic keyframes, as tools/bench_mesh.py) at marching-cubes resolutions 256 and 512 as ground truth, with a rigidly moved copy
(2 degrees about the centroid, 3 cm) as the reconstruction.

GPU phases are bracketed by CUDA events after an L2 flush (a 256 MB write); ICP also by the host clock (it reads 17 sums back per
iteration).  Each resolution runs one warm-up and --rounds timed rounds; medians and spreads (max - min) are reported with the card's
name and power limit, read in the same run.  The host arm times the same workload through oracle/recon.py's cKDTree path: that is
the reference's own method for the metric queries (eval_recon.py builds cKDTrees); for ICP it stands in for open3d, which is not used.

python tools/bench_recon.py [--rounds 5] [--host-rounds 1] [--out results/bench_recon.json]
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

import scene_util as su                                       # noqa: E402
from gpu_util import make_renderer                            # noqa: E402
from measure import Flush, card, log, median_spread, time_call  # noqa: E402
from oracle import recon as orc                               # noqa: E402

MC_BOUND = [[-2.9, 8.9], [-3.2, 5.5], [-3.5, 3.3]]          # configs/Replica/room0.yaml
N_SAMPLES = 200000


def meshes(resolutions, keyframes=10):
    """FusedMesher.get_mesh of room0's 'soft' grids with the synthetic keyframe set of tools/bench_mesh.py: {R: (vertices, faces)}."""
    from nice_slam_b200.keyframes import KeyframeStore
    from nice_slam_b200.mesh import FusedMesher
    sc = su.load_scenes()["room0"]
    renderer, c, dec = make_renderer(sc, su.make_grids(sc, "soft"), su.load_decoders("soft"), "cuda")
    cam = sc["cam"]
    store = KeyframeStore(cam["H"], cam["W"], cam["fx"], cam["fy"], cam["cx"], cam["cy"], "cuda")
    for k in range(keyframes):
        depth, color = su.make_frame(sc, 500 + k)
        store.append(k, color, depth, su.make_pose(sc, 500 + k))
    est = torch.stack(store.est_c2w)
    out = {}
    for R in resolutions:
        cfg = dict(meshing=dict(resolution=R, level_set=0, clean_mesh_bound_scale=1.02, remove_small_geometry_threshold=0.2,
                                get_largest_components=False, color_mesh_extraction_method="direct_point_query", depth_test=False),
                   mapping=dict(marching_cubes_bound=MC_BOUND), scale=1)
        v, f, _ = FusedMesher(renderer, cfg).get_mesh(None, c, dec, store, est, keyframes - 1, color=False)
        out[R] = (v, f)
    return out


def moved(v):
    ctr = np.eye(4)
    ctr[:3, 3] = v.mean(0)
    M = ctr @ orc.rigid(2.0, (0.2, -0.3, 1.0), (0.03, 0.0, 0.0)) @ np.linalg.inv(ctr)
    return orc.transform_points(v, M)


def gpu_round(rv, rf, gv, gf, flush):
    from nice_slam_b200.recon import NearestNeighbours, icp_align, sample_surface
    t = {}

    def timed(name, fn):
        out, events_ms, host_ms = time_call(fn, flush)
        t[name] = dict(events_ms=events_ms, host_ms=host_ms)
        return out

    dev = torch.device("cuda")
    rvd, rfd = torch.from_numpy(rv).to(dev), torch.from_numpy(rf).to(dev)
    gvd, gfd = torch.from_numpy(gv).to(dev), torch.from_numpy(gf).to(dev)
    nn_v = timed("grid_build_vertices", lambda: NearestNeighbours(gvd))
    T, fit, rmse, it = timed("icp", lambda: icp_align(rvd, nn_v, 0.1))
    rva = torch.from_numpy(rv @ T[:3, :3].T + T[:3, 3]).to(dev)
    g = torch.Generator(device=dev)
    g.manual_seed(0)
    rec = timed("sampling", lambda: (sample_surface(rva, rfd, N_SAMPLES, g)[0], sample_surface(gvd, gfd, N_SAMPLES, g)[0]))
    nn_g = timed("grid_build_samples", lambda: (NearestNeighbours(rec[1]), NearestNeighbours(rec[0])))
    d = timed("metric_queries", lambda: (nn_g[0].query(rec[0])[0], nn_g[1].query(rec[1])[0]))
    acc, comp = float(d[0].mean()) * 100, float(d[1].mean()) * 100
    t["icp"]["iterations"] = it
    t["icp"]["per_iteration_ms"] = t["icp"]["events_ms"] / max(it, 1)
    return t, dict(accuracy_cm=acc, completion_cm=comp, ratio_pct=float((d[1] < 0.05).double().mean()) * 100, icp_iterations=it,
                   fitness=fit, rmse=rmse)


def host_round(rv, rf, gv, gf):
    from scipy.spatial import cKDTree
    t = {}
    h0 = time.perf_counter()
    T, fit, rmse, it = orc.icp_align(rv, gv, 0.1)
    t["icp"] = dict(host_ms=(time.perf_counter() - h0) * 1e3, iterations=it)
    log("  host icp: %.0f ms, %d iterations" % (t["icp"]["host_ms"], it))
    rs = np.random.default_rng(0)
    rva = orc.transform_points(rv, T)
    h0 = time.perf_counter()
    rec, _ = orc.sample_surface(rva, rf, rs.random((N_SAMPLES, 3)))
    gt, _ = orc.sample_surface(gv, gf, rs.random((N_SAMPLES, 3)))
    t["sampling"] = dict(host_ms=(time.perf_counter() - h0) * 1e3)
    h0 = time.perf_counter()
    tg, tr = cKDTree(gt), cKDTree(rec)
    t["grid_build_samples"] = dict(host_ms=(time.perf_counter() - h0) * 1e3)
    h0 = time.perf_counter()
    tg.query(rec)
    tr.query(gt)
    t["metric_queries"] = dict(host_ms=(time.perf_counter() - h0) * 1e3)
    return t


def summarise(rounds):
    out = {}
    for ph in rounds[0]:
        for k, v0 in rounds[0][ph].items():
            vals = [r[ph][k] for r in rounds]
            out.setdefault(ph, {})[k] = v0 if k == "iterations" else median_spread(vals)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--host-rounds", type=int, default=1)
    ap.add_argument("--resolutions", type=int, nargs="+", default=[256, 512])
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_recon.py measures on the GPU"
    res = dict(card=card(), n_samples=N_SAMPLES, rounds=a.rounds, host_rounds=a.host_rounds, resolutions={})
    flush = Flush()
    for R, (gv, gf) in meshes(a.resolutions).items():
        rv = moved(gv)
        log("resolution %d: %d vertices, %d faces" % (R, len(gv), len(gf)))
        gpu_round(rv, gf, gv, gf, flush)                                             # warm-up
        rounds = []
        for i in range(a.rounds):
            rounds.append(gpu_round(rv, gf, gv, gf, flush))
            log("  gpu round %d: %s" % (i, json.dumps(rounds[-1][0])))
        host = []
        for i in range(a.host_rounds):
            host.append(host_round(rv, gf, gv, gf))
            log("  host round %d: %s" % (i, json.dumps(host[-1])))
        res["resolutions"][R] = dict(vertices=int(len(gv)), faces=int(len(gf)), gpu=summarise([r[0] for r in rounds]), result=rounds[0][1],
                                     host_ckdtree=summarise(host) if host else None)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
