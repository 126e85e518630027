"""Cost of option "deterministic": default against deterministic mode, CUDA events around each call, L2 flushed before every timed call,
the two modes alternating round by round.  Workloads: the 996-ray mapping iteration (stage colour, dense voxel grads, every decoder
graded), the coarse mapper's iteration (996 rays, stage coarse) and the 200-ray tracking iteration (no voxel / decoder grads: unchanged
by the mode).  Also prints each context's workspace bytes in both modes.

    python tools/bench_deterministic.py [--rounds 20] [--iters 20]"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import scene_util as su                                       # noqa: E402
from gpu_util import make_renderer                            # noqa: E402
from measure import Flush, alternate, card, time_events       # noqa: E402
from nice_slam_b200 import _lib                               # noqa: E402
from nice_slam_b200.steps import IterationContext             # noqa: E402

DEV = "cuda"


def workloads(sc, renderer):
    ro, rd, gd, gc = (t.to(DEV).contiguous() for t in su.make_rays(sc, 996, seed=3000))
    tro, trd, tgd, tgc = (t.to(DEV).contiguous() for t in su.make_rays(sc, 200, seed=3001))
    return {
        "mapping 996 rays, stage color": (dict(n_rays=996, stage="color", kind="map", grad_grids=("grid_middle", "grid_fine", "grid_color"),
                                               grad_decoders=("middle", "fine", "color")), (ro, rd, gd, gc.float().contiguous())),
        "coarse mapper 996 rays": (dict(n_rays=996, stage="coarse", kind="map", grad_grids=("grid_coarse",), grad_decoders=("coarse",),
                                        coarse_mapper=True), (ro, rd, gd, gc.float().contiguous())),
        "tracking 200 rays": (dict(n_rays=200, stage="color", kind="track"), (tro, trd, tgd, tgc.double().contiguous())),
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=20)
    ap.add_argument("--iters", type=int, default=20)
    a = ap.parse_args()
    print("card: %s" % card(), flush=True)
    sc = su.load_scenes()["room0"]
    renderer, c, dec = make_renderer(sc, su.make_grids(sc, "soft"), su.load_decoders("soft"), DEV)
    for p in dec.parameters():
        p.requires_grad_(True)
    flush = Flush(DEV)
    props = torch.cuda.get_device_properties(0)
    out = {"gpu": props.name, "results": {}}
    for name, (kw, inputs) in workloads(sc, renderer).items():
        kw = dict(kw)
        n = kw.pop("n_rays")
        stage = kw.pop("stage")
        ctxs = {}
        for det in (0, 1):
            _lib.set_option("deterministic", det)
            ctxs[det] = IterationContext(renderer, n, stage, DEV, **kw)
            for _ in range(3):
                ctxs[det].run(c, dec, *inputs)

        def run(det):
            _lib.set_option("deterministic", det)
            # one synchronize per call: the host enqueues each call on an idle device
            return [time_events(lambda: ctxs[det].run(c, dec, *inputs), 1, flush=flush)[0] for _ in range(a.iters)]
        times = {d: sum(r, []) for d, r in alternate((0, 1), a.rounds, run).items()}
        _lib.set_option("deterministic", 0)
        med = {d: sorted(t)[len(t) // 2] for d, t in times.items()}
        out["results"][name] = dict(default_ms=med[0], deterministic_ms=med[1], ratio=med[1] / med[0],
                                    workspace_mb={"default": ctxs[0].ws.numel() / 2 ** 20, "deterministic": ctxs[1].ws.numel() / 2 ** 20})
        print("%-32s default %.3f ms  deterministic %.3f ms  (x%.2f)  workspace %.0f / %.0f MiB" %
              (name, med[0], med[1], med[1] / med[0], ctxs[0].ws.numel() / 2 ** 20, ctxs[1].ws.numel() / 2 ** 20), flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
