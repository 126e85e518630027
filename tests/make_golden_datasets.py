"""Writes tests/golden/datasets/: tiny datasets in the replica, scannet, azure and tumrgbd layouts (a few ~64x48 frames each; ScanNet's
colour at another size than its depth, TUM with distortion and crop_size) and what the reference computes from them -- get_dataset's
file lists, poses and fingerprints of every prepared frame (reference.pt), and NICE_SLAM's initial state (update_cam, bound, grid
shapes and the bits of the grids and decoders under a fixed seed) for the room0, scene0000, apartment and freiburg1_desk configs, with pretrained checkpoints in
the ConvONet layout built from decoders.pt (scenes.pt).

    python tests/make_golden_datasets.py          (needs the reference tree; see ref_harness.py)"""
import hashlib
import os
import sys
import tempfile
from types import SimpleNamespace

import cv2
import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_harness as rh  # noqa: E402

OUT = os.path.join(HERE, "golden", "datasets")
CONFIGS = {"room0": "configs/Replica/room0.yaml", "scene0000": "configs/ScanNet/scene0000.yaml",
           "apartment": "configs/Apartment/apartment.yaml", "freiburg1_desk": "configs/TUM_RGBD/freiburg1_desk.yaml"}
SEED = 7


# cam settings of the fixtures (the real cameras scaled down to ~64x48; TUM keeps the shipped freiburg1 distortion)
CAMS = {
    "replica": dict(H=48, W=64, fx=40.0, fy=40.0, cx=31.5, cy=23.5, png_depth_scale=6553.5, crop_edge=0),
    "scannet": dict(H=48, W=64, fx=57.7, fy=57.8, cx=31.9, cy=24.3, png_depth_scale=1000.0, crop_edge=2),
    "azure": dict(H=45, W=80, fx=38.0, fy=38.0, cx=39.8, cy=23.1, png_depth_scale=1000.0, crop_edge=0),
    "tumrgbd": dict(H=48, W=64, fx=51.73, fy=51.65, cx=31.86, cy=25.53, png_depth_scale=5000.0, crop_edge=2, crop_size=[40, 52],
                    distortion=[0.2624, -0.9531, -0.0054, 0.0026, 1.1633]),
}


def fixture_cfg(name):
    return dict(dataset=name, cam=dict(CAMS[name]), data=dict(input_folder=os.path.join(OUT, name)))


def _img(rng, h, w):
    """Smooth colour with noise, so resampling has something to do and JPEG keeps it small."""
    y, x = np.mgrid[0:h, 0:w]
    base = np.stack([128 + 100 * np.sin(x / 7.0 + k) * np.cos(y / 5.0 - k) for k in range(3)], -1)
    return np.clip(base + rng.normal(0, 3, (h, w, 3)), 0, 255).astype(np.uint8)


def _depth(rng, h, w):
    """A smooth ramp (small PNGs) with holes (0) and one saturated pixel (65535)."""
    y, x = np.mgrid[0:h, 0:w]
    d = (3000 + 80 * x + 50 * y + rng.integers(0, 4, (h, w))).astype(np.uint16)
    d[rng.random((h, w)) < 0.05] = 0
    d[0, 0] = 65535
    return d


def _pose(rng):
    from scipy.spatial.transform import Rotation
    p = np.eye(4)
    p[:3, :3] = Rotation.from_rotvec(rng.normal(0, 0.3, 3)).as_matrix()
    p[:3, 3] = rng.normal(0, 1.0, 3)
    return p


def write_fixtures():
    rng = np.random.default_rng(20)
    # replica: results/frame%06d.jpg, depth%06d.png, traj.txt
    d = os.path.join(OUT, "replica")
    os.makedirs(os.path.join(d, "results"), exist_ok=True)
    with open(os.path.join(d, "traj.txt"), "w") as f:
        for i in range(4):
            cv2.imwrite(os.path.join(d, "results", "frame%06d.jpg" % i), _img(rng, 48, 64))
            cv2.imwrite(os.path.join(d, "results", "depth%06d.png" % i), _depth(rng, 48, 64))
            f.write(" ".join("%.18e" % v for v in _pose(rng).reshape(-1)) + "\n")
    # scannet: frames/{color,depth,pose}/<int>.{jpg,png,txt}, colour 81x61 against depth 64x48, stems that sort differently as strings
    d = os.path.join(OUT, "scannet", "frames")
    for sub in ("color", "depth", "pose"):
        os.makedirs(os.path.join(d, sub), exist_ok=True)
    for i in (0, 1, 2, 10):
        cv2.imwrite(os.path.join(d, "color", "%d.jpg" % i), _img(rng, 61, 81))
        cv2.imwrite(os.path.join(d, "depth", "%d.png" % i), _depth(rng, 48, 64))
        np.savetxt(os.path.join(d, "pose", "%d.txt" % i), _pose(rng), fmt="%.9f", delimiter=" ")
    # azure: color/*.jpg, depth/*.png, scene/trajectory.log (blocks of 5 lines)
    d = os.path.join(OUT, "azure")
    for sub in ("color", "depth", "scene"):
        os.makedirs(os.path.join(d, sub), exist_ok=True)
    with open(os.path.join(d, "scene", "trajectory.log"), "w") as f:
        for i in range(3):
            cv2.imwrite(os.path.join(d, "color", "%05d.jpg" % i), _img(rng, 45, 80))
            cv2.imwrite(os.path.join(d, "depth", "%05d.png" % i), _depth(rng, 45, 80))
            f.write("%d %d %d\n" % (i, i, i + 1))
            for row in _pose(rng):
                f.write(" ".join("%.9f" % v for v in row) + "\n")
    # tumrgbd: rgb.txt, depth.txt, groundtruth.txt (one header line) with unaligned stamps.  Image 1 lies 0.0197 s after image 0, under
    # 1/32 s, so frame_rate 32 drops it; image 5 has no depth within max_dt 0.08 (its own is 0.09 s away, the others farther), so the
    # association drops it.  Five frames remain: images 0, 2, 3, 4 and 6.
    d = os.path.join(OUT, "tumrgbd")
    for sub in ("rgb", "depth"):
        os.makedirs(os.path.join(d, sub), exist_ok=True)
    t_img = [1305031102.175304, 1305031102.195000, 1305031102.243211, 1305031102.275326, 1305031102.311267, 1305031102.450000,
             1305031102.600000]
    t_dep = [t + (0.09 if k == 5 else 0.004) for k, t in enumerate(t_img)]
    t_pose = np.arange(1305031102.17, 1305031102.62, 0.01)
    with open(os.path.join(d, "rgb.txt"), "w") as fr, open(os.path.join(d, "depth.txt"), "w") as fd:
        for k, (ti, td) in enumerate(zip(t_img, t_dep)):
            cv2.imwrite(os.path.join(d, "rgb", "%.6f.png" % ti), _img(rng, 48, 64))
            cv2.imwrite(os.path.join(d, "depth", "%.6f.png" % td), _depth(rng, 48, 64))
            fr.write("%.6f rgb/%.6f.png\n" % (ti, ti))
            fd.write("%.6f depth/%.6f.png\n" % (td, td))
    from scipy.spatial.transform import Rotation
    with open(os.path.join(d, "groundtruth.txt"), "w") as f:
        f.write("# timestamp tx ty tz qx qy qz qw\n")
        for t in t_pose:
            q = Rotation.from_rotvec(rng.normal(0, 0.2, 3)).as_quat()
            f.write("%.4f %s %s\n" % (t, " ".join("%.4f" % v for v in rng.normal(0, 1, 3)), " ".join("%.4f" % v for v in q)))


def reference_readers():
    ref = rh.import_reference()
    if not hasattr(np, "unicode_"):
        np.unicode_ = np.str_
    from src.utils import datasets as ds
    out = {}
    for name in CAMS:
        cfg = fixture_cfg(name)
        r = ds.get_dataset(cfg, SimpleNamespace(input_folder=None), 1, device="cpu")
        items = [r[i] for i in range(len(r))]
        out[name] = dict(color_paths=[os.path.relpath(p, OUT) for p in r.color_paths], depth_paths=[os.path.relpath(p, OUT) for p in r.depth_paths],
                         poses=torch.stack([it[3] for it in items]), frames=[frame_print(it[1], it[2]) for it in items])
    del ref
    return out


def frame_print(color, depth):
    """Fingerprint of a prepared frame: shapes, the depth's and the colour's bytes (sha256), and float64 sums of the colour -- its sum and
    three fixed random projections -- that a colour within a tolerance of this one reproduces to that tolerance times its size."""
    c = color.detach().cpu().double().contiguous()
    g = torch.Generator().manual_seed(77)
    proj = [float((c * torch.rand(c.shape, generator=g, dtype=torch.float64)).sum()) for _ in range(3)]
    return dict(color_shape=list(c.shape), depth_shape=list(depth.shape), depth=digest(depth.float()), color=digest(c),
                color_sum=float(c.sum()), color_proj=proj)


def check_frame(color, depth, want, tol):
    """Assert that a prepared frame matches its reference fingerprint: depth bit-exact, colour bit-exact or within tol per element
    (its sum and projections within tol times the element count)."""
    c = color.detach().cpu().double().contiguous()
    assert list(c.shape) == want["color_shape"] and list(depth.shape) == want["depth_shape"]
    assert digest(depth.detach().cpu().float()) == want["depth"]
    if digest(c) == want["color"]:
        return
    got = frame_print(c, depth)
    bound = tol * c.numel()
    assert abs(got["color_sum"] - want["color_sum"]) <= bound, (got["color_sum"], want["color_sum"])
    assert all(abs(a - b) <= bound for a, b in zip(got["color_proj"], want["color_proj"])), (got["color_proj"], want["color_proj"])


def convonet_checkpoints(folder):
    """ConvONet-layout checkpoints of tests/golden/decoders.pt: coarse.pt ('decoder.' + key) and middle_fine.pt ('decoder.coarse_' +
    middle key, 'decoder.fine_' + fine key), each with an encoder entry that must be skipped."""
    st = torch.load(os.path.join(HERE, "golden", "decoders.pt"), map_location="cpu", weights_only=True)
    enc = torch.zeros(3)
    coarse = dict({"decoder." + k: v for k, v in st["coarse"].items()}, **{"encoder.fc.weight": enc})
    mf = {"decoder.coarse_" + k: v for k, v in st["middle"].items()}
    mf.update({"decoder.fine_" + k: v for k, v in st["fine"].items()})
    mf["encoder.decoder_like.weight"] = enc
    paths = dict(coarse=os.path.join(folder, "coarse.pt"), middle_fine=os.path.join(folder, "middle_fine.pt"))
    torch.save({"model": coarse}, paths["coarse"])
    torch.save({"model": mf}, paths["middle_fine"])
    return paths


def digest(t):
    return hashlib.sha256(t.detach().cpu().contiguous().numpy().tobytes()).hexdigest()


def reference_scenes(ckpts):
    out = {}
    for name, rel in CONFIGS.items():
        cfg = rh.load_cfg(rel)
        cfg["pretrained_decoders"] = dict(ckpts)
        slam = rh.build_slam(cfg, seed=SEED)
        out[name] = dict(config=rel, cfg={k: v for k, v in cfg.items() if k != "pretrained_decoders"}, cam=(slam.H, slam.W, slam.fx, slam.fy, slam.cx, slam.cy), bound=slam.bound.clone(),
                         shapes={k: list(v.shape) for k, v in slam.shared_c.items()},
                         grids={k: digest(v) for k, v in slam.shared_c.items()},
                         decoders={k: digest(v) for k, v in slam.shared_decoders.state_dict().items()},
                         rng_after=digest(torch.get_rng_state()))
    return out


def main():
    write_fixtures()
    torch.save(reference_readers(), os.path.join(OUT, "reference.pt"))
    with tempfile.TemporaryDirectory() as d:
        torch.save(reference_scenes(convonet_checkpoints(d)), os.path.join(OUT, "scenes.pt"))
    print("wrote", OUT)


if __name__ == "__main__":
    main()
