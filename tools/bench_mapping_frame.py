"""Time one Mapper.optimize_map call (src/Mapper.py:230-540) two ways on room0 'soft' grids:

  * fused:   mapping.FusedMapper.map_frame -- keyframe images resident on the device, per iteration the reference's per-row torch.randint
             draws, one sampler launch (nsb_map_samples), one 4-byte kept-count read, the fused mapping iteration and the fused Adam steps;
  * drop-in: optimize_map restated on FusedRenderer -- keyframe images kept on the host and copied to the device for every row of every
             iteration (Mapper.py:439-440), get_samples' full-image meshgrid + torch.randint per row, get_camera_from_tensor with autograd
             under bundle adjustment, torch.cat, the torch bbox pre-filter and boolean indexing, the frustum-selected voxels scattered into the
             grids and back (Mapper.py:393-401, :510-519), render_batch_ray, the torch loss, loss.backward() and torch.optim.Adam.  The drop-in
             takes its frustum masks from the device kernel (the reference computes them on the host), which does not favour the fused path.

    python tools/bench_mapping_frame.py [--rounds 3] [--calls 2]

Workloads: 60 iterations x 1000 px with a window of 5 keyframes + the current frame under bundle adjustment (the shipped mapper, a frame
once BA is on), and the coarse mapper's call (60 iterations, global selection, stage 'coarse').  Both arms alternate within every round; the
L2 is flushed (256 MiB memset) before every call; each call is timed with CUDA events and with the host clock up to a synchronise.  Prints
the card, its power limit and SM clocks with the numbers.  Needs a CUDA device; there is no CPU fallback."""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import scene_util as su  # noqa: E402
from bench_dropin_decoder_grads import card, quad2rot  # noqa: E402
from gpu_util import make_renderer  # noqa: E402
from nice_slam_b200 import FusedMapper  # noqa: E402
from nice_slam_b200.keyframes import KeyframeStore  # noqa: E402
from nice_slam_b200.mapping import map_stage, stage_lrs, tensor_from_c2w, window_rows  # noqa: E402
from nice_slam_b200.masked import frustum_voxel_mask  # noqa: E402
from oracle import torch_port as tp  # noqa: E402

STAGE = {"coarse": dict(decoders_lr=0.0, coarse_lr=0.001, middle_lr=0.0, fine_lr=0.0, color_lr=0.0),
         "middle": dict(decoders_lr=0.0, coarse_lr=0.0, middle_lr=0.1, fine_lr=0.0, color_lr=0.0),
         "fine": dict(decoders_lr=0.0, coarse_lr=0.0, middle_lr=0.005, fine_lr=0.005, color_lr=0.0),
         "color": dict(decoders_lr=0.005, coarse_lr=0.0, middle_lr=0.005, fine_lr=0.005, color_lr=0.005)}
SETTINGS = dict(pixels=1000, mapping_window_size=5, middle_iter_ratio=0.4, fine_iter_ratio=0.6, stage=STAGE, BA_cam_lr=0.001, w_color_loss=0.2,
                keyframe_selection_method="overlap", fix_fine=True, fix_color=False, frustum_feature_selection=True)
KEYFRAMES = [10, 11, 12, 13, 14]


def dropin_call(renderer, c, dec, host_kf, cur, iters, selection, ba, coarse_mapper, s):
    """optimize_map as the reference runs it, on FusedRenderer, for the window selection + last keyframe + current frame."""
    dev = c["grid_middle"].device
    depth_c, color_c, c2w_c = cur
    H, W = depth_c.shape
    rows, fixed = window_rows(selection, len(host_kf))
    keys = ("grid_coarse",) if coarse_mapper else ("grid_middle", "grid_fine", "grid_color")
    masks, paras = {}, {}
    for key in keys:
        m = frustum_voxel_mask(renderer, c2w_c, key, c[key], depth_c)
        masks[key] = m.view(1, 1, *m.shape).expand_as(c[key])
        paras[key] = c[key][masks[key]].clone().requires_grad_(True)
    dec_params = [] if coarse_mapper else list(dec.color_decoder.parameters())
    cams = [tensor_from_c2w(host_kf[k][2] if k >= 0 else c2w_c).to(dev).requires_grad_(True) for r, k in enumerate(rows) if r != fixed] if ba else []
    groups = [dict(params=dec_params, lr=0)] + [dict(params=[paras[k]] if k in paras else [], lr=0) for k in
                                                 ("grid_coarse", "grid_middle", "grid_fine", "grid_color")]
    if ba:
        groups.append(dict(params=cams, lr=0))
    opt = torch.optim.Adam(groups)
    ppi = s["pixels"] // len(rows)
    bound = renderer.bound.to(dev)
    for it in range(iters):
        stage = map_stage(it, iters, s["middle_iter_ratio"], s["fine_iter_ratio"], coarse_mapper)
        lr = stage_lrs(STAGE, stage, 1.0)
        for g, name in zip(opt.param_groups, ("decoders", "coarse", "middle", "fine", "color")):
            g["lr"] = lr[name]
        if ba and stage == "color":
            opt.param_groups[5]["lr"] = s["BA_cam_lr"]
        grids = dict(c)
        for key in keys:
            val = c[key].clone()
            val[masks[key]] = paras[key]
            grids[key] = val
        opt.zero_grad()
        ro_l, rd_l, gd_l, gc_l = [], [], [], []
        cam_id = 0
        for r, k in enumerate(rows):
            depth, color = (host_kf[k][0].to(dev), host_kf[k][1].to(dev)) if k >= 0 else (depth_c, color_c)
            if ba and r != fixed:
                q = cams[cam_id]; cam_id += 1
                c2w = torch.cat([quad2rot(q[:4]), q[4:, None]], 1)
            else:
                c2w = (host_kf[k][2] if k >= 0 else c2w_c).to(dev)
            i, j = torch.meshgrid(torch.linspace(0, W - 1, W, device=dev), torch.linspace(0, H - 1, H, device=dev), indexing="ij")
            i, j = i.t().reshape(-1), j.t().reshape(-1)
            idx = torch.randint(i.shape[0], (ppi,), device=dev)
            i, j = i[idx], j[idx]
            dirs = torch.stack([(i - renderer.cx) / renderer.fx, -(j - renderer.cy) / renderer.fy, -torch.ones_like(i)], -1)
            rd = torch.sum(dirs.reshape(-1, 1, 3) * c2w[:3, :3], -1)
            ro_l.append(c2w[:3, -1].expand(rd.shape)); rd_l.append(rd)
            gd_l.append(depth.reshape(-1)[idx].float()); gc_l.append(color.reshape(-1, 3)[idx].float())
        ro, rd, gd, gc = torch.cat(ro_l), torch.cat(rd_l), torch.cat(gd_l), torch.cat(gc_l)
        with torch.no_grad():
            t = (bound.unsqueeze(0) - ro.detach().unsqueeze(-1)) / rd.detach().unsqueeze(-1)
            keep = torch.min(torch.max(t, dim=2)[0], dim=1)[0] >= gd
        ro, rd, gd, gc = ro[keep], rd[keep], gd[keep], gc[keep]
        d, _, col = renderer.render_batch_ray(grids, dec, rd, ro, dev, stage, gt_depth=None if coarse_mapper else gd)
        loss = tp.mapping_loss(d, col, gd, gc, stage, s["w_color_loss"])
        loss.backward()
        opt.step()
        opt.zero_grad()
    for key in keys:
        with torch.no_grad():
            c[key][masks[key]] = paras[key].detach()
    return [torch.cat([quad2rot(q[:4]), q[4:, None]], 1).detach() for q in cams]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--calls", type=int, default=2, help="calls per arm and round")
    ap.add_argument("--iters", type=int, default=60)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_mapping_frame: needs a CUDA device")
    dev = torch.device("cuda")
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    sc = su.load_scenes()["room0"]
    cam = sc["cam"]
    renderer, c, dec = make_renderer(sc, su.make_grids(sc, "soft"), su.load_decoders("soft"), dev)
    for p in dec.parameters():
        p.requires_grad_(False)
    for p in dec.color_decoder.parameters():
        p.requires_grad_(True)
    host_kf = []
    store = KeyframeStore(cam["H"], cam["W"], cam["fx"], cam["fy"], cam["cx"], cam["cy"], dev)
    for k, seed in enumerate(KEYFRAMES):
        depth, color = su.make_frame(sc, seed)
        host_kf.append((depth, color, su.make_pose(sc, seed)))
        store.append(5 * k, color, depth, su.make_pose(sc, seed))
    depth, color = su.make_frame(sc, 1)
    c2w = su.make_pose(sc, 1)
    cur = (depth.to(dev), color.to(dev), c2w.to(dev))
    print("card: %s" % card())
    results = []
    for name, ba, coarse_mapper in (("ba_window", True, False), ("coarse_mapper", False, True)):
        s = dict(SETTINGS, mapping_window_size=6 if ba else 5)
        mapper = FusedMapper(renderer, c, dec, store, coarse_mapper=coarse_mapper, **s)
        selection = [0, 1, 2, 3] if ba else [0, 1, 2]
        arms = {"fused": lambda: mapper.map_frame(a.iters, 1.0, color, depth, c2w, ba, selection=selection),
                "drop-in": lambda: dropin_call(renderer, c, dec, host_kf, cur, a.iters, selection, ba, coarse_mapper, s)}
        np.random.seed(0)
        for fn in arms.values():                                        # warm-up: module loads, allocator, autograd
            fn(); fn()
        torch.cuda.synchronize()
        times = {k: dict(event=[], wall=[]) for k in arms}
        for _ in range(a.rounds):
            for arm, fn in arms.items():
                for _ in range(a.calls):
                    flush.zero_()
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    e0.record(); fn(); e1.record()
                    torch.cuda.synchronize()
                    times[arm]["wall"].append((time.perf_counter() - t0) * 1e3)
                    times[arm]["event"].append(e0.elapsed_time(e1))
        row = dict(workload=name, iters=a.iters, pixels=s["pixels"], window_rows=len(selection) + 2, calls_per_arm=a.rounds * a.calls)
        for arm, t in times.items():
            for kind, v in t.items():
                row["%s_%s_ms" % (arm, kind)] = dict(mean=round(sum(v) / len(v), 3), min=round(min(v), 3), max=round(max(v), 3))
        row["speedup_wall"] = round(row["drop-in_wall_ms"]["mean"] / row["fused_wall_ms"]["mean"], 2)
        results.append(row)
        print(json.dumps(row))
    return results


if __name__ == "__main__":
    main()
