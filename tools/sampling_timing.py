"""Forward + backward time of FusedRenderer.render_batch_ray under the reference's sampling settings (src/utils/Renderer.py:152-196):
the default sampler, perturb, lindisp and N_importance = 12, at 200 and 1000 rays in stage color (room0 'soft', gradients for the rays,
the colour / fine / middle grids and the colour decoder, as in a colour mapping iteration).  CUDA events around `iters` calls after
`warmup` calls; prints the card name and power limit, then one JSON line per case.

    python tools/sampling_timing.py [--iters 200] [--warmup 20]
"""
import argparse
import json
import os
import subprocess
import sys
from types import SimpleNamespace

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import scene_util as su                                   # noqa: E402
from gpu_util import make_cfg                             # noqa: E402
from nice_slam_b200.decoders import NICEDecoders           # noqa: E402
from nice_slam_b200.renderer import FusedRenderer          # noqa: E402

CASES = {"default": {}, "perturb": dict(perturb=1.0), "lindisp": dict(lindisp=True), "importance12": dict(N_importance=12)}


def card():
    try:
        q = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], text=True)
        return q.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return torch.cuda.get_device_name(0) + ", power limit unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sampling_timing needs a CUDA device")
    dev = "cuda"
    print("card: %s" % card())
    sc = su.load_scenes()["room0"]
    grids, dec_state = su.make_grids(sc, "soft"), su.load_decoders("soft")
    cam = sc["cam"]
    for n in (200, 1000):
        ro, rd, gd, _ = su.make_rays(sc, n, seed=7)
        ro, rd, gd = ro.to(dev), rd.to(dev), gd.to(dev)
        for name, over in CASES.items():
            cfg = make_cfg(sc)
            cfg["rendering"].update(over)
            c = {k: v.to(dev) for k, v in grids.items()}
            slam = SimpleNamespace(nice=True, bound=su.scene_bound(sc), shared_c=c, H=cam["H"], W=cam["W"], fx=cam["fx"], fy=cam["fy"],
                                   cx=cam["cx"], cy=cam["cy"])
            r = FusedRenderer(cfg, SimpleNamespace(nice=True), slam)
            c = slam.shared_c
            dec = NICEDecoders.from_state(dec_state, dev)
            for k in c:
                c[k].requires_grad_(k != "grid_coarse")
            for nm, p in dec.named_parameters():
                p.requires_grad_(nm.startswith("color_decoder"))
            o, d = ro.clone().requires_grad_(True), rd.clone().requires_grad_(True)

            def step():
                depth, var, rgb = r.render_batch_ray(c, dec, d, o, dev, "color", gt_depth=gd)
                (depth.sum() + var.sum() + rgb.sum()).backward()
            for _ in range(a.warmup):
                step()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.iters):
                step()
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / a.iters
            print(json.dumps(dict(rays=n, sampling=name, ms_fwd_bwd=round(ms, 4), iters=a.iters)))


if __name__ == "__main__":
    main()
