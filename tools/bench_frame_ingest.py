"""Time frame ingest: the reference's host chain against decode + raw upload + nsb_frame_prepare, and what ingest costs a whole run.

    python tools/bench_frame_ingest.py [--frames 20] [--rounds 3] [--seq 51] [--out DIR]

1. Per format -- Replica (680x1200 JPEG colour), TUM (480x640 PNG colour, freiburg1 distortion, crop_size [384,512], crop_edge 8) and
   ScanNet (1296x968 JPEG colour against 640x480 depth, crop_edge 10) -- synthetic frames are written to a temporary directory and each
   frame is timed on the host clock up to a device synchronise:
   - host path: BaseDataset.__getitem__'s chain restated (cv2.imread, cv2.undistort, cvtColor, / 255., depth / png_depth_scale,
     cv2.resize, torch interpolate, crop) and the float64 colour / float32 depth .to(device);
   - GPU path: cv2.imread, pinned copy, raw upload and nsb_frame_prepare (FrameReader's steps, in the caller's thread);
   - the kernel alone: CUDA events around nsb_frame_prepare.
2. A --seq-frame room0 sequence rendered from the 'soft' scene is written as a Replica folder and run with the shipped Replica settings
   through nice_slam_b200.run.main from disk with --prefetch 0 and 2, and through FusedSLAM.run over the same frames preloaded on the
   device (the same scene, seed, checkpoints and meshes).  The wall time of the run is compared.
Reports the card, its power limit and the spread over rounds.  Needs a CUDA device; there is no CPU fallback."""
import argparse
import json
import os
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import cv2  # noqa: E402
import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402
import yaml  # noqa: E402

from measure import card  # noqa: E402
from nice_slam_b200 import datasets as ds  # noqa: E402

TUM_DIST = [0.2624, -0.9531, -0.0054, 0.0026, 1.1633]
FORMATS = {
    "replica": dict(color=(680, 1200), depth=(680, 1200), ext="jpg",
                    cam=dict(fx=600.0, fy=600.0, cx=599.5, cy=339.5, png_depth_scale=6553.5, crop_edge=0)),
    "tum": dict(color=(480, 640), depth=(480, 640), ext="png",
                cam=dict(fx=517.3, fy=516.5, cx=318.6, cy=255.3, png_depth_scale=5000.0, crop_edge=8, crop_size=[384, 512], distortion=TUM_DIST)),
    "scannet": dict(color=(968, 1296), depth=(480, 640), ext="jpg",
                    cam=dict(fx=577.59, fy=578.73, cx=318.91, cy=242.68, png_depth_scale=1000.0, crop_edge=10)),
}


def write_frames(folder, fmt, n):
    rng = np.random.default_rng(0)
    (hc, wc), (hd, wd) = fmt["color"], fmt["depth"]
    y, x = np.mgrid[0:hc, 0:wc]
    paths = []
    for k in range(n):
        base = np.stack([128 + 100 * np.sin(x / 37.0 + k + c) * np.cos(y / 29.0 - c) for c in range(3)], -1)
        img = np.clip(base + rng.normal(0, 6, (hc, wc, 3)), 0, 255).astype(np.uint8)
        yd, xd = np.mgrid[0:hd, 0:wd]
        dep = (3000 + 7 * xd + 5 * yd + rng.integers(0, 50, (hd, wd))).astype(np.uint16)
        cp, dp = os.path.join(folder, "c%04d.%s" % (k, fmt["ext"])), os.path.join(folder, "d%04d.png" % k)
        cv2.imwrite(cp, img)
        cv2.imwrite(dp, dep)
        paths.append((cp, dp))
    return paths


def host_path(cp, dp, cam, dev):
    """src/utils/datasets.py:78-113 on the host, then to the device."""
    color = cv2.imread(cp)
    depth = cv2.imread(dp, cv2.IMREAD_UNCHANGED)
    if cam.get("distortion") is not None:
        K = np.array([[cam["fx"], 0, cam["cx"]], [0, cam["fy"], cam["cy"]], [0, 0, 1.0]])
        color = cv2.undistort(color, K, np.array(cam["distortion"]))
    color = cv2.cvtColor(color, cv2.COLOR_BGR2RGB) / 255.
    depth = depth.astype(np.float32) / cam["png_depth_scale"]
    H, W = depth.shape
    color = torch.from_numpy(cv2.resize(color, (W, H)))
    depth = torch.from_numpy(depth) * 1
    if cam.get("crop_size") is not None:
        color = F.interpolate(color.permute(2, 0, 1)[None], cam["crop_size"], mode="bilinear", align_corners=True)[0].permute(1, 2, 0).contiguous()
        depth = F.interpolate(depth[None, None], cam["crop_size"], mode="nearest")[0, 0]
    e = cam["crop_edge"]
    if e > 0:
        color, depth = color[e:-e, e:-e], depth[e:-e, e:-e]
    return color.to(dev), depth.to(dev)


def gpu_path(cp, dp, cam, dev, events=None):
    color, depth = ds.decode(cp, dp)
    c = torch.from_numpy(color).pin_memory().to(dev, non_blocking=True)
    d = torch.from_numpy(depth.view(np.int16)).pin_memory().to(dev, non_blocking=True)
    p = ds.frame_params(dict(cam=cam, scale=1), color.shape, depth.shape)
    if events is not None:
        events[0].record()
    out = ds.prepare_frame(p, c, d)
    if events is not None:
        events[1].record()
    return out


def time_formats(n, rounds, dev):
    res = {}
    with tempfile.TemporaryDirectory() as tmp:
        for name, fmt in FORMATS.items():
            folder = os.path.join(tmp, name)
            os.makedirs(folder)
            paths = write_frames(folder, fmt, n)
            cam = fmt["cam"]
            for cp, dp in paths[:2]:                                        # warm-up: module load, allocator, cv2 codecs
                host_path(cp, dp, cam, dev)
                gpu_path(cp, dp, cam, dev)
            torch.cuda.synchronize()
            per = {"host_ms": [], "gpu_ms": [], "kernel_ms": []}
            for _ in range(rounds):
                for key, fn in (("host_ms", host_path), ("gpu_ms", gpu_path)):
                    t0 = time.perf_counter()
                    for cp, dp in paths:
                        fn(cp, dp, cam, dev)
                        torch.cuda.synchronize()
                    per[key].append((time.perf_counter() - t0) * 1e3 / n)
                ks = []
                for cp, dp in paths:
                    ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
                    gpu_path(cp, dp, cam, dev, ev)
                    torch.cuda.synchronize()
                    ks.append(ev[0].elapsed_time(ev[1]))
                per["kernel_ms"].append(float(np.mean(ks)))
            res[name] = {k: dict(min=min(v), max=max(v), rounds=v) for k, v in per.items()}
            print("%-8s host %.2f-%.2f ms/frame  gpu path %.2f-%.2f ms/frame  kernel %.3f-%.3f ms" % (
                name, min(per["host_ms"]), max(per["host_ms"]), min(per["gpu_ms"]), max(per["gpu_ms"]), min(per["kernel_ms"]),
                max(per["kernel_ms"])), flush=True)
    return res


def write_sequence(folder, n):
    import scene_util as su
    from gpu_util import make_renderer
    from slam_sequences import path_pose
    sc = su.load_scenes()["room0"]
    renderer, c, dec = make_renderer(sc, su.make_grids(sc, "soft"), su.load_decoders("soft"), "cuda")
    os.makedirs(os.path.join(folder, "results"))
    with open(os.path.join(folder, "traj.txt"), "w") as f:
        for k in range(n):
            pose = path_pose(sc, k)
            depth, _, color = renderer.render_img(c, dec, pose, "cuda", "color")
            bgr = (color.float().clamp(0, 1).cpu().numpy()[..., ::-1] * 255).round().astype(np.uint8)
            cv2.imwrite(os.path.join(folder, "results", "frame%06d.jpg" % k), bgr)
            cv2.imwrite(os.path.join(folder, "results", "depth%06d.png" % k), (depth.cpu().numpy() * 6553.5).round().astype(np.uint16))
            traj = pose.detach().double().cpu().numpy().copy()
            traj[:3, 1] *= -1
            traj[:3, 2] *= -1
            f.write(" ".join(repr(float(v)) for v in traj.reshape(-1)) + "\n")
    return sc


def time_sequence(n, rounds, dev):
    """run.main from disk (prefetch 0 and 2) against FusedSLAM.run over the same frames preloaded on the device."""
    import scene_util as su
    from make_golden_datasets import OUT, convonet_checkpoints
    from nice_slam_b200 import FusedSLAM, build_scene, run
    from nice_slam_b200.config import load_config
    cwd = os.getcwd()
    res = {"prefetch0_s": [], "prefetch2_s": [], "preloaded_s": []}
    with tempfile.TemporaryDirectory() as tmp:
        data = os.path.join(tmp, "room")
        sc = write_sequence(data, n)
        ck = convonet_checkpoints(tmp)
        os.makedirs(os.path.join(tmp, "configs"))
        base = torch.load(os.path.join(OUT, "scenes.pt"), weights_only=False)["room0"]["cfg"]      # the merged room0 config
        with open(os.path.join(tmp, "configs", "nice_slam.yaml"), "w") as f:
            yaml.safe_dump(base, f)
        cam, bound = sc["cam"], su.scene_bound(sc).tolist()
        cfg_path = os.path.join(tmp, "run.yaml")
        with open(cfg_path, "w") as f:
            yaml.safe_dump(dict(pretrained_decoders=ck, cam=dict(H=cam["H"], W=cam["W"], fx=cam["fx"], fy=cam["fy"], cx=cam["cx"], cy=cam["cy"],
                                                                 png_depth_scale=6553.5, crop_edge=0),
                                mapping=dict(bound=bound, marching_cubes_bound=bound), meshing=dict(eval_rec=False)), f)
        os.chdir(tmp)
        try:
            cfg = load_config(cfg_path, "configs/nice_slam.yaml")
            frames = list(ds.FrameReader(cfg, data, dev, prefetch=0))
            short = dict(cfg, mapping=dict(cfg["mapping"], iters_first=20, iters=5))                    # warm-up of every shape
            slam = build_scene(short, dev, seed=0)
            FusedSLAM(slam.renderer, slam.shared_c, slam.shared_decoders, short, seed=0).run(frames[:7])
            for r in range(rounds):
                for pf in (0, 2):
                    out = run.main([cfg_path, "--input_folder", data, "--output", os.path.join(tmp, "out%d_%d" % (pf, r)), "--seed", "0",
                                    "--prefetch", str(pf)])
                    res["prefetch%d_s" % pf].append(out["wall_s"])
                slam = build_scene(cfg, dev, seed=0)
                outp = os.path.join(tmp, "pre%d" % r)
                os.makedirs(os.path.join(outp, "mesh"))
                fused = FusedSLAM(slam.renderer, slam.shared_c, slam.shared_decoders, cfg, seed=0, ckpt_dir=os.path.join(outp, "ckpts"),
                                  mesh_dir=os.path.join(outp, "mesh"))
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fused.run(frames)
                torch.cuda.synchronize()
                res["preloaded_s"].append(time.perf_counter() - t0)
                print("sequence round %d: prefetch 0 %.3f s, prefetch 2 %.3f s, preloaded %.3f s" % (
                    r, res["prefetch0_s"][-1], res["prefetch2_s"][-1], res["preloaded_s"][-1]), flush=True)
        finally:
            os.chdir(cwd)
    return {k: dict(min=min(v), max=max(v), rounds=v) for k, v in res.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--seq", type=int, default=51)
    ap.add_argument("--seq_rounds", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_frame_ingest: needs a CUDA device")
    dev = torch.device("cuda", 0)
    res = dict(card=card(), per_frame=time_formats(a.frames, a.rounds, dev), frames_per_format=a.frames)
    if a.seq > 0:
        res["sequence"] = dict(frames=a.seq, **time_sequence(a.seq, a.seq_rounds, dev))
    res["card_after"] = card()
    print(json.dumps(res))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_frame_ingest.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
