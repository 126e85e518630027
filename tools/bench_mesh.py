"""Time each phase of FusedMesher.get_mesh on room0's 'soft' grids with a synthetic keyframe set, at marching-cubes resolutions 256 and 512.

Every phase is bracketed by CUDA events after an L2 flush (a 256 MB write); phases with host work (the hull's scipy step, the count
read-backs, the PLY write) are also timed with the host clock around a device synchronise.  Each resolution runs one warm-up and
--rounds timed rounds; the median and the spread (max - min) over the rounds are reported, with the card's name and power limit.

python tools/bench_mesh.py [--rounds 5] [--keyframes 10] [--out results/bench_mesh.json]
"""
import argparse
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

import scene_util as su                                       # noqa: E402
from gpu_util import make_renderer                            # noqa: E402
from measure import Flush, card, median_spread, time_call     # noqa: E402

PHASES = ("hull", "lattice", "marching_cubes", "masks", "components", "colors", "ply_write")
MC_BOUND = [[-2.9, 8.9], [-3.2, 5.5], [-3.5, 3.3]]          # configs/Replica/room0.yaml


def one_round(mesher, c, dec, store, est, flush, tmpdir):
    t = {}

    def timed(name, fn):
        out, events_ms, host_ms = time_call(fn, flush)
        t[name] = dict(events_ms=events_ms, host_ms=host_ms)
        return out

    with torch.no_grad():
        planes = timed("hull", lambda: mesher.hull(store))
        z = timed("lattice", lambda: mesher.lattice(c, dec, planes))
        verts, faces, _ = timed("marching_cubes", lambda: mesher.marching_cubes(z))
        seen = timed("masks", lambda: mesher.seen(verts, store, est, len(store) - 1))
        cv, cf = timed("components", lambda: mesher.clean(verts, faces, seen))
        col = timed("colors", lambda: mesher.colors(cv, c, dec))
        v, f, cc = cv.cpu().numpy() / mesher.scale, cf.cpu().numpy().astype(np.int64), col.cpu().numpy()
    from nice_slam_b200.mesh import write_ply
    h0 = time.perf_counter()
    write_ply(os.path.join(tmpdir, "bench.ply"), v, f, cc)
    t["ply_write"] = dict(events_ms=None, host_ms=(time.perf_counter() - h0) * 1e3)
    sizes = dict(lattice_points=int(z.numel()), mc_vertices=int(verts.shape[0]), mc_faces=int(faces.shape[0]), vertices=int(len(v)), faces=int(len(f)))
    return t, sizes


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--keyframes", type=int, default=10)
    ap.add_argument("--resolutions", type=int, nargs="+", default=[256, 512])
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_mesh.py measures on the GPU"
    from nice_slam_b200.keyframes import KeyframeStore
    from nice_slam_b200.mesh import FusedMesher
    sc = su.load_scenes()["room0"]
    renderer, c, dec = make_renderer(sc, su.make_grids(sc, "soft"), su.load_decoders("soft"), "cuda")
    cam = sc["cam"]
    store = KeyframeStore(cam["H"], cam["W"], cam["fx"], cam["fy"], cam["cx"], cam["cy"], "cuda")
    for k in range(a.keyframes):
        depth, color = su.make_frame(sc, 500 + k)
        store.append(k, color, depth, su.make_pose(sc, 500 + k))
    est = torch.stack(store.est_c2w)
    flush = Flush()
    res = dict(card=card(), keyframes=a.keyframes, rounds=a.rounds, resolutions={})
    with tempfile.TemporaryDirectory() as tmpdir:
        for R in a.resolutions:
            cfg = dict(meshing=dict(resolution=R, level_set=0, clean_mesh_bound_scale=1.02, remove_small_geometry_threshold=0.2,
                                    get_largest_components=False, color_mesh_extraction_method="direct_point_query", depth_test=False),
                       mapping=dict(marching_cubes_bound=MC_BOUND), scale=1)
            mesher = FusedMesher(renderer, cfg)
            one_round(mesher, c, dec, store, est, flush, tmpdir)                      # warm-up
            rounds = [one_round(mesher, c, dec, store, est, flush, tmpdir) for _ in range(a.rounds)]
            summary = {}
            for ph in PHASES:
                for kind in ("events_ms", "host_ms"):
                    vals = [r[0][ph][kind] for r in rounds if r[0][ph][kind] is not None]
                    if vals:
                        summary.setdefault(ph, {})[kind] = median_spread(vals)
            total = [sum(r[0][ph]["host_ms"] for ph in PHASES) for r in rounds]
            res["resolutions"][R] = dict(phases=summary, total_host_ms=median_spread(total), sizes=rounds[0][1])
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
