#!/usr/bin/env python
"""Time the decoder back-ends that option mlp_backend selects against each other, on the iterations bench.py and the mapper run.

    python tools/bench_mlp_backends.py [--backends 2 0] [--steps 200] [--rounds 3]

mlp_backend 0 = auto (the tile kernels here), 1 = FP32-FMA decoders, 2 = round-1 ray-group tensor-core kernels, 3 = tile kernels.

Workloads (room0 'soft' grids, stage color, 48 samples per ray, bench.make_batch rays):
  * the tracking iteration of bench.py (forward + loss + input-gradient backward + pose gradient) at 16, 64, 200 and 1000 rays;
  * the BASELINE configs[1] mapping iteration: 996 rays, dense voxel gradients of the middle, fine and colour grids + colour-decoder gradients.
Every iteration is one IterationContext CUDA-graph replay, captured under its back-end (a graph keeps the kernels it captured, so the
back-ends' graphs can alternate).  L2 is flushed before every step; mean ms per step from CUDA events.  Rounds alternate the back-ends
in the order given.  Prints the card name and its power limit with the numbers.  Needs a CUDA device; there is no CPU fallback."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402

import bench  # noqa: E402
from measure import Flush, alternate, card, stats, time_events  # noqa: E402
from nice_slam_b200 import _lib  # noqa: E402
from nice_slam_b200.steps import IterationContext  # noqa: E402

TRACK_RAYS = (16, 64, 200, 1000)
MAP_RAYS = 996


def set_backend(b):
    _lib.check(_lib.lib().nsb_set_option(b"mlp_backend", b), "nsb_set_option(mlp_backend)")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--backends", type=int, nargs="+", default=[2, 0])
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda", 0)
    gpu = card()
    sc, renderer, c, dec = bench.build_scene(dev)
    flush = Flush(dev)

    # (workload, backend) -> graph; the contexts stay alive as long as their graphs
    graphs, keep = {}, []
    work = [("track_%d" % n, n) for n in TRACK_RAYS] + [("map_%d" % MAP_RAYS, MAP_RAYS)]
    for name, n in work:
        ro, rd, dirs, gd, gc = [t.to(dev) for t in bench.make_batch(sc, n, 0 if name.startswith("track") else 101)]
        for b in args.backends:
            set_backend(b)
            if name.startswith("track"):
                ctx = IterationContext(renderer, n, "color", dev, kind="track")
                ctx.load_device_inputs(ro, rd, gd, gc)
                g = ctx.build_graph(c, dec, dirs=dirs)
            else:
                ctx = IterationContext(renderer, n, "color", dev, kind="map", grad_grids=("grid_middle", "grid_fine", "grid_color"),
                                       grad_decoders=("color",))
                ctx.load_device_inputs(ro, rd, gd, gc.float())
                g = ctx.build_graph(c, dec)
            graphs[name, b] = g
            keep.append(ctx)
    set_backend(0)

    ms = alternate(tuple(graphs), args.rounds, lambda k: sum(time_events(graphs[k].replay, args.steps, warmup=20, flush=flush)) / args.steps,
                   reverse=False)
    rows = []
    for name, _n in work:
        row = {"workload": name}
        for b in args.backends:
            v = ms[name, b]
            row["mlp_backend_%d" % b] = {**{k + "_ms": x for k, x in stats(v).items()}, "rounds": [round(x, 4) for x in v]}
        rows.append(row)
    print(json.dumps({"card": gpu, "steps": args.steps, "rounds": args.rounds, "results": rows}, indent=1))
    print("card: %s" % gpu)
    print("%-10s" % "workload" + "".join("  backend %d: mean [min, max] ms" % b for b in args.backends))
    for row in rows:
        print("%-10s" % row["workload"] + "".join("  %8.4f [%.4f, %.4f]" % (row["mlp_backend_%d" % b]["mean_ms"], row["mlp_backend_%d" % b]["min_ms"],
                                                                            row["mlp_backend_%d" % b]["max_ms"]) for b in args.backends))


if __name__ == "__main__":
    main()
