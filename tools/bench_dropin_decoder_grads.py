"""Time the drop-in call patterns (FusedRenderer.render_batch_ray + a torch loss + loss.backward()) as the reference's tracker and mapper make
them: every decoder parameter requires grad (the tracker deep-copies the shared decoders, src/Tracker.py:138; the mapper uses them as they
are), so autograd asks the backward for the weight gradients of every decoder of the stage.

    python tools/bench_dropin_decoder_grads.py [--steps 100] [--rounds 3]

Rows (room0 'soft' grids, bench.make_batch rays):
  * tracking iteration: 200 rays, stage color, camera tensor -> rays, the torch tracking loss (Tracker.py:108-123), backward();
  * mapping iteration: 996 rays, stages middle, fine and color, dense leaf grids of the stage, the torch mapping loss (Mapper.py:487-493);
  * coarse mapper: 996 rays, stage coarse rendered without depth, the coarse grid as leaf.
Each under three settings, alternated within every round: decoders frozen (requires_grad False on every decoder parameter, the pattern
bench.py's extra.dropin times -- the floor), every decoder trainable with option wgrad_all = 0 (their weight gradients by the FP32-FMA pass,
which recomputes the forward) and with wgrad_all = 1 (on the tensor cores from the kept layer outputs).  L2 flushed before every step (256 MiB
memset outside the event pair), CUDA events, mean ms per step over the rounds (min .. max): what the caller waits for, host-side autograd
glue included.  A separate torch.profiler pass (--profile-steps per case and setting) gives the device time per step of the render kernels
(forward + backward) and of the backward launches alone, and names the backward kernels.  Prints the card, its power limit and SM clocks
with the numbers.  Needs a CUDA device; there is no CPU fallback."""
import argparse
import collections
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
from nice_slam_b200.mapping import tensor_from_c2w  # noqa: E402
from oracle import torch_port as tp  # noqa: E402

STAGE_GRIDS = {"coarse": ("grid_coarse",), "middle": ("grid_middle",), "fine": ("grid_fine", "grid_middle"),
               "color": ("grid_fine", "grid_color", "grid_middle")}
SETTINGS = (("frozen decoders", False, 0), ("trainable, wgrad_all=0", True, 0), ("trainable, wgrad_all=1", True, 1))


def quad2rot(q):
    two_s = 2.0 / (q * q).sum()
    qr, qi, qj, qk = q[0], q[1], q[2], q[3]
    return torch.stack([1 - two_s * (qj ** 2 + qk ** 2), two_s * (qi * qj - qk * qr), two_s * (qi * qk + qj * qr),
                        two_s * (qi * qj + qk * qr), 1 - two_s * (qi ** 2 + qk ** 2), two_s * (qj * qk - qi * qr),
                        two_s * (qi * qk - qj * qr), two_s * (qj * qk + qi * qr), 1 - two_s * (qi ** 2 + qj ** 2)]).reshape(3, 3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--profile-steps", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_dropin_decoder_grads: needs a CUDA device")
    print("card: %s" % card(), flush=True)
    dev = torch.device("cuda")
    flush = Flush(dev)
    L = _lib.lib()

    def kernel_time(fn):
        """(render-kernel device ms per step, backward-launch device ms per step, backward kernel names) over a profiled run of its own"""
        from torch.profiler import ProfilerActivity, profile
        fn()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(a.profile_steps):
                fn()
            torch.cuda.synchronize()
        tot = collections.Counter()
        for e in prof.events():
            if e.device_type.name == "CUDA":
                tot[e.name.split("(")[0].split("::")[-1].split("<")[0]] += e.time_range.elapsed_us()
        render = sum(v for k, v in tot.items() if k.startswith("render_")) / a.profile_steps / 1e3
        bwd = {k: v for k, v in tot.items() if k.startswith("render_bwd")}
        return render, sum(bwd.values()) / a.profile_steps / 1e3, "+".join(sorted(bwd))

    sc = su.load_scenes()["room0"]
    renderer, c, dec = make_renderer(sc, su.make_grids(sc, "soft"), su.load_decoders("soft"), dev)
    w_track, w_map = sc["tracking"]["w_color_loss"], sc["mapping"]["w_color_loss"]

    # tracking: camera tensor -> c2w -> rays (get_rays_from_uv) -> render -> tracking loss -> backward to the camera tensor
    ro_t, rd_t, dirs_t, gd_t, gc_t = [t.to(dev) for t in bench.make_batch(sc, 200, 0)]
    cam = tensor_from_c2w(su.make_pose(sc, 0)).to(dev).requires_grad_(True)
    ct = {k: v.detach() for k, v in c.items()}

    def track():
        cam.grad = None
        for p in dec.parameters():
            p.grad = None
        rays_d = torch.sum(dirs_t.reshape(-1, 1, 3) * quad2rot(cam[:4]), -1)
        rays_o = cam[4:].expand(rays_d.shape)
        depth, var, color = renderer.render_batch_ray(ct, dec, rays_d, rays_o, dev, "color", gt_depth=gd_t)
        tp.tracking_loss(depth, var, color, gd_t, gc_t, w_track).backward()

    # mapping: dense leaf grids of the stage + the decoders as the mapper leaves them
    n = 996
    ro, rd, _, gd, gc = [t.to(dev) for t in bench.make_batch(sc, n, 101)]
    gcf = gc.float()

    def mapper(stage):
        cm = {k: v.detach().clone().requires_grad_(k in STAGE_GRIDS[stage]) for k, v in c.items()}

        def it():
            for k in STAGE_GRIDS[stage]:
                cm[k].grad = None
            for p in dec.parameters():
                p.grad = None
            depth, var, color = renderer.render_batch_ray(cm, dec, rd, ro, dev, stage, gt_depth=None if stage == "coarse" else gd)
            tp.mapping_loss(depth, color, gd, gcf, stage, w_map).backward()
        return it

    cases = [("tracking iteration, 200 rays, stage color", track)]
    cases += [("mapping iteration, 996 rays, stage %s" % s, mapper(s)) for s in ("middle", "fine", "color")]
    cases += [("coarse mapper, 996 rays, stage coarse (no depth)", mapper("coarse"))]

    def run(setting):
        label, trainable, wa = setting
        for p in dec.parameters():
            p.requires_grad_(trainable)
        _lib.check(L.nsb_set_option(b"wgrad_all", wa), "nsb_set_option")
        return [sum(time_events(fn, a.steps, warmup=5, flush=flush)) / a.steps for _, fn in cases]
    per_setting = alternate(SETTINGS, a.rounds, run, reverse=False)
    rows = {(name, s[0]): [r[i] for r in per_setting[s]] for s in SETTINGS for i, (name, _) in enumerate(cases)}
    kt = {}
    for label, trainable, wa in SETTINGS:
        for p in dec.parameters():
            p.requires_grad_(trainable)
        _lib.check(L.nsb_set_option(b"wgrad_all", wa), "nsb_set_option")
        for name, fn in cases:
            kt[(name, label)] = kernel_time(fn)
    _lib.check(L.nsb_set_option(b"wgrad_all", 0), "nsb_set_option")
    for p in dec.parameters():
        p.requires_grad_(True)
    print("room0 soft, L2 flushed, CUDA events, %d steps x %d rounds: mean ms per step (min .. max over rounds) | device ms per step of the "
          "render kernels / of the backward launches (torch.profiler, %d steps, L2 not flushed) and the backward kernels" % (a.steps, a.rounds, a.profile_steps))
    for (name, label), v in rows.items():
        r, b, names = kt[(name, label)]
        print("  %-52s %-24s %.4f  (%.4f .. %.4f) | %.4f / %.4f  %s" % (name, label, *stats(v).values(), r, b, names))


if __name__ == "__main__":
    main()
