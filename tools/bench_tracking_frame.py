"""Time one tracked frame (Tracker.run's camera optimisation of one frame, src/Tracker.py:188-253) two ways on room0 'soft' grids:

  * loop:    tracking.FusedTrackingLoop.track_frame -- one sampler launch, the fused tracking iteration and one pose-step launch per iteration,
             one 4-byte kept-count read per iteration and one read at the end of the frame;
  * drop-in: optimize_cam_in_batch restated on FusedRenderer (Tracker.py:71-128) -- get_camera_from_tensor with autograd, get_samples' full
             region meshgrid + torch.randint, the torch bbox pre-filter and boolean indexing, render_batch_ray, the median-gated torch loss,
             loss.backward(), torch.optim.Adam, loss.item() and the best-pose clone, every iteration.  Decoders frozen (no weight gradients):
             the cheapest backward the drop-in can take, so the comparison does not favour the loop.

    python tools/bench_tracking_frame.py [--rounds 3] [--frames 5]

Shapes: 10 iterations x 200 px (Replica) and 200 x 5000 px (TUM).  Both arms alternate within every round; the L2 is flushed (256 MiB memset)
before every frame; each frame is timed with CUDA events and with the host clock up to a synchronise.  Prints the card, its power limit and
SM clocks with the numbers.  Needs a CUDA device; there is no CPU fallback."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402

import scene_util as su  # noqa: E402
from bench_dropin_decoder_grads import quad2rot  # noqa: E402
from gpu_util import make_renderer  # noqa: E402
from measure import Flush, alternate, card, stats, time_call  # noqa: E402
from nice_slam_b200.mapping import tensor_from_c2w  # noqa: E402
from nice_slam_b200.tracking import FusedTrackingLoop  # noqa: E402
from oracle import torch_port as tp  # noqa: E402

SHAPES = ((10, 200), (200, 5000))
SETTINGS = dict(ignore_edge_W=20, ignore_edge_H=20, lr=0.001, seperate_LR=False, handle_dynamic=True, use_color_in_tracking=True,
                w_color_loss=0.5, const_speed_assumption=True)


def dropin_frame(renderer, c, dec, depth, color, cam0, iters, pixels, s):
    """optimize_cam_in_batch x iters + the best-pose bookkeeping of Tracker.run, as the reference calls them, on FusedRenderer."""
    dev = depth.device
    H, W = depth.shape
    H0, H1, W0, W1 = s["ignore_edge_H"], H - s["ignore_edge_H"], s["ignore_edge_W"], W - s["ignore_edge_W"]
    bound = renderer.bound.to(dev)
    cam = cam0.clone().requires_grad_(True)
    opt = torch.optim.Adam([cam], lr=s["lr"])
    best, cand = 1e10, None
    for _ in range(iters):
        opt.zero_grad()
        c2w = torch.cat([quad2rot(cam[:4]), cam[4:, None]], 1)
        i, j = torch.meshgrid(torch.linspace(W0, W1 - 1, W1 - W0, device=dev), torch.linspace(H0, H1 - 1, H1 - H0, device=dev), indexing="ij")
        i, j = i.t().reshape(-1), j.t().reshape(-1)
        idx = torch.randint(i.shape[0], (pixels,), device=dev)
        i, j = i[idx], j[idx]
        gd, gc = depth[H0:H1, W0:W1].reshape(-1)[idx], color[H0:H1, W0:W1].reshape(-1, 3)[idx]
        dirs = torch.stack([(i - renderer.cx) / renderer.fx, -(j - renderer.cy) / renderer.fy, -torch.ones_like(i)], -1)
        rd = torch.sum(dirs.reshape(-1, 1, 3) * c2w[:3, :3], -1)
        ro = c2w[:3, -1].expand(rd.shape)
        with torch.no_grad():
            t = (bound.unsqueeze(0) - ro.detach().unsqueeze(-1)) / rd.detach().unsqueeze(-1)
            keep = torch.min(torch.max(t, dim=2)[0], dim=1)[0] >= gd
        rd, ro, gd, gc = rd[keep], ro[keep], gd[keep], gc[keep]
        d, u, col = renderer.render_batch_ray(c, dec, rd, ro, dev, "color", gt_depth=gd)
        loss = tp.tracking_loss(d, u, col, gd, gc, s["w_color_loss"], s["handle_dynamic"], s["use_color_in_tracking"])
        loss.backward()
        opt.step()
        opt.zero_grad()
        lv = loss.item()
        if lv < best:
            best, cand = lv, cam.clone().detach()
    return torch.cat([torch.cat([quad2rot(cand[:4]), cand[4:, None]], 1), torch.tensor([[0, 0, 0, 1.0]], device=dev)], 0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--frames", type=int, default=5, help="frames per arm and round (the 200 x 5000 shape uses a third of them, at least 1)")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_tracking_frame: needs a CUDA device")
    dev = torch.device("cuda")
    flush = Flush(dev)
    sc = su.load_scenes()["room0"]
    renderer, c, dec = make_renderer(sc, su.make_grids(sc, "soft"), su.load_decoders("soft"), dev)
    for p in dec.parameters():
        p.requires_grad_(False)
    depth, color = su.make_frame(sc, 21)
    depth_d, color_d = depth.to(dev), color.to(dev)
    cam0 = tensor_from_c2w(su.make_pose(sc, 20)).to(dev)
    print("card: %s" % card())
    results = []
    for iters, pixels in SHAPES:
        s = dict(SETTINGS, iters=iters, pixels=pixels)
        loop = FusedTrackingLoop(renderer, c, dec, pixels, **s)
        arms = {"loop": lambda: loop.track_frame(color, depth, cam0),
                "drop-in": lambda: dropin_frame(renderer, c, dec, depth_d, color_d, cam0, iters, pixels, s)}
        n_frames = a.frames if iters <= 10 else max(1, a.frames // 3)
        for fn in arms.values():                                        # warm-up: module loads, allocator, autograd
            fn(); fn()
        torch.cuda.synchronize()
        per_round = alternate(tuple(arms), a.rounds, lambda arm: [time_call(arms[arm], flush)[1:] for _ in range(n_frames)], reverse=False)
        times = {k: dict(event=[e for r in v for e, _ in r], wall=[w for r in v for _, w in r]) for k, v in per_round.items()}
        row = dict(iters=iters, pixels=pixels, frames_per_arm=a.rounds * n_frames)
        for name, t in times.items():
            for kind, v in t.items():
                row["%s_%s_ms" % (name, kind)] = {k: round(x, 3) for k, x in stats(v).items()}
        row["speedup_wall"] = round(row["drop-in_wall_ms"]["mean"] / row["loop_wall_ms"]["mean"], 2)
        results.append(row)
        print(json.dumps(row))
    return results


if __name__ == "__main__":
    main()
