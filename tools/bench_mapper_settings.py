"""Time the mapping iteration under the mapper settings FusedMappingLoop takes (fix_fine, fix_color, frustum_feature_selection).

    python tools/bench_mapper_settings.py [--steps 100] [--rounds 3]

BASELINE configs[1] batch (996 rays, room0 'soft' grids), L2 flushed before every step, CUDA events, mean ms per step:
  * the mapping iteration (IterationContext.run) in stage fine with the fine decoder's weight gradients, in stage color with the fine + colour
    decoders' (fix_fine = False), and in stage color with the colour decoder's alone (the default settings), each with option wgrad_tc = 1
    and 0 -- rounds alternate the two;
  * one native loop step (iteration + fused Adam) with the default settings and with fix_fine = False, stage color;
  * one colour-refinement loop step: fix_color = True, frustum_feature_selection = False, bundle adjustment over a window of six frames
    x 166 rays, stage color.
Prints the card name and its power limit with the numbers.  Needs a CUDA device; there is no CPU fallback."""
import argparse
import copy
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402

import bench  # noqa: E402
import scene_util as su  # noqa: E402
from gpu_util import make_renderer  # noqa: E402
from measure import Flush, alternate, card, stats, time_events  # noqa: E402
from nice_slam_b200 import _lib  # noqa: E402
from nice_slam_b200.mapping import FusedMappingLoop  # noqa: E402
from nice_slam_b200.steps import IterationContext  # noqa: E402

GRIDS = {"fine": ("grid_fine", "grid_middle"), "color": ("grid_middle", "grid_fine", "grid_color")}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_mapper_settings: needs a CUDA device")
    print("card: %s" % card(), flush=True)
    dev = torch.device("cuda")
    flush = Flush(dev)

    def time_steps(fn):
        return sum(time_events(fn, a.steps, warmup=3, flush=flush)) / a.steps

    sc = su.load_scenes()["room0"]
    renderer, c, dec = make_renderer(sc, su.make_grids(sc, "soft"), su.load_decoders("soft"), dev)
    n = 996
    ro, rd, dirs, gd, gc = [t.to(dev) for t in bench.make_batch(sc, n, 101)]
    gcf = gc.float()
    L = _lib.lib()
    iters = [("fine", ("fine",)), ("color", ("fine", "color")), ("color", ("color",))]
    ctxs = {(s, d): IterationContext(renderer, n, s, dev, kind="map", grad_grids=GRIDS[s], grad_decoders=d, host_staging=False) for s, d in iters}

    def run(tc):
        _lib.check(L.nsb_set_option(b"wgrad_tc", tc), "nsb_set_option")
        return [time_steps(lambda: ctx.run(c, dec, ro, rd, gd, gcf)) for ctx in ctxs.values()]
    per_tc = alternate((1, 0), a.rounds, run, reverse=False)
    rows = {"iteration stage %-5s grad_decoders=%-15s wgrad_tc=%d" % (s, "+".join(d), tc): [r[i] for r in per_tc[tc]]
            for tc in (1, 0) for i, (s, d) in enumerate(ctxs)}
    _lib.check(L.nsb_set_option(b"wgrad_tc", 1), "nsb_set_option")
    depth1, color1 = su.make_frame(sc, 1)
    lr = dict(decoders=0.005, middle=0.005, fine=0.005, color=0.005)
    for label, kw in (("loop step stage color, default settings", {}), ("loop step stage color, fix_fine=False", dict(fix_fine=False))):
        loop = FusedMappingLoop(renderer, {k: v.clone() for k, v in c.items()}, copy.deepcopy(dec), su.make_pose(sc, 1), depth1.to(dev), **kw)
        rows[label] = [time_steps(lambda: loop.iteration("color", ro, rd, gd, gcf, lr)) for _ in range(a.rounds)]
    # colour refinement: six window rows (five keyframes + the current frame), 166 pixel draws each
    loop = FusedMappingLoop(renderer, {k: v.clone() for k, v in c.items()}, copy.deepcopy(dec), None, None, fix_color=True,
                            frustum_feature_selection=False)
    loop.enable_ba(torch.stack([su.make_pose(sc, 10 + k) for k in range(5)] + [su.make_pose(sc, 1)]), 0, 0.001)
    g = torch.Generator().manual_seed(5)
    F, m = 6, 166
    pi = torch.randint(0, sc["cam"]["W"], (F, m), generator=g).float().to(dev)
    pj = torch.randint(0, sc["cam"]["H"], (F, m), generator=g).float().to(dev)
    pd = depth1[pj.long().cpu(), pi.long().cpu()].to(dev)
    pc = color1[pj.long().cpu(), pi.long().cpu()].float().to(dev)
    rows["colour-refinement loop step (BA, 6 x 166 rays)"] = [time_steps(lambda: loop.iteration_ba("color", pi, pj, pd, pc, lr))
                                                               for _ in range(a.rounds)]
    print("996 rays, room0 soft, L2 flushed, CUDA events, %d steps x %d rounds: mean ms per step (min .. max over rounds)" % (a.steps, a.rounds))
    for label, v in rows.items():
        print("  %-62s %.4f  (%.4f .. %.4f)" % (label, *stats(v).values()))


if __name__ == "__main__":
    main()
