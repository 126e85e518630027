"""Run a NICE-SLAM sequence from its config on the fused path: the counterpart of the reference's run.py, without the reference package.

    python -m nice_slam_b200.run CONFIG [--input_folder DIR] [--output DIR] [--seed S] [--prefetch N] [--deterministic]

Run from a NICE-SLAM checkout (or a tree with its layout): CONFIG's inherit_from chain, configs/nice_slam.yaml and the pretrained decoders
are opened relative to the current directory, as the reference opens them.  Checkpoints go to {output}/ckpts (Logger.log's format),
meshes to {output}/mesh (Mapper.run's), and the per-phase times, frames per second and ATE to stdout and {output}/run.json.  Only
sync_method 'strict' is supported; iMAP* (--imap) is not.  --deterministic turns on the library's deterministic mode (INTEGRATION.md):
two runs of the same build on the same GPU model then optimise to the same bits (trajectory, grids, decoders, checkpoints); mesh
extraction is not covered (its component areas are still summed with atomics)."""
import argparse
import json
import os
import sys
import time

import torch

from .config import load_config
from .datasets import FrameReader
from .scene import build_scene
from .slam import FusedSLAM, ate_rmse


def parse(argv):
    ap = argparse.ArgumentParser(description="Run NICE-SLAM on the fused path.")
    ap.add_argument("config", type=str, help="path to the config file")
    ap.add_argument("--input_folder", type=str, help="input folder; overrides the config's data.input_folder")
    ap.add_argument("--output", type=str, help="output folder; overrides the config's data.output")
    ap.add_argument("--seed", type=int, default=None, help="torch.manual_seed before the scene is built, and the run's seed (default 0)")
    ap.add_argument("--prefetch", type=int, default=2, help="frames decoded ahead by the reader's thread (0: none)")
    ap.add_argument("--deterministic", action="store_true", help="voxel and decoder gradients summed in a fixed order: repeatable optimisation (meshes excepted)")
    grp = ap.add_mutually_exclusive_group(required=False)
    grp.add_argument("--nice", dest="nice", action="store_true")
    grp.add_argument("--imap", dest="nice", action="store_false")
    ap.set_defaults(nice=True)
    return ap.parse_args(argv)


def main(argv=None):
    """Returns the figures written to run.json."""
    a = parse(argv)
    if not a.nice:
        raise SystemExit("nice_slam_b200.run: --imap (iMAP*) is not supported; only NICE-SLAM runs on the fused path")
    cfg = load_config(a.config, "configs/nice_slam.yaml")
    if cfg["sync_method"] != "strict":
        raise SystemExit("nice_slam_b200.run: sync_method %r is not supported; only 'strict' (set sync_method: strict)" % cfg["sync_method"])
    if not torch.cuda.is_available():
        raise SystemExit("nice_slam_b200.run: needs a CUDA device")
    out = a.output if a.output is not None else cfg["data"]["output"]
    ckpt_dir, mesh_dir = os.path.join(out, "ckpts"), os.path.join(out, "mesh")
    os.makedirs(ckpt_dir, exist_ok=True)
    os.makedirs(mesh_dir, exist_ok=True)
    dev = torch.device("cuda", torch.cuda.current_device())
    if a.deterministic:
        from ._lib import set_option
        set_option("deterministic", 1)                     # before any fused context sizes its workspaces
    slam = build_scene(cfg, dev, seed=a.seed)
    reader = FrameReader(cfg, a.input_folder, dev, prefetch=a.prefetch)
    fused = FusedSLAM(slam.renderer, slam.shared_c, slam.shared_decoders, cfg, seed=a.seed if a.seed is not None else 0,
                      ckpt_dir=ckpt_dir, mesh_dir=mesh_dir)
    print("nice_slam_b200.run: %d frames of %s, output %s" % (len(reader), reader.input_folder, out), flush=True)
    torch.cuda.synchronize(dev)
    t0 = time.perf_counter()
    est, gt = fused.run(reader)
    torch.cuda.synchronize(dev)
    wall = time.perf_counter() - t0
    from ._lib import get_option
    res = dict(deterministic=bool(get_option("deterministic")), frames=len(reader), wall_s=wall, fps=len(reader) / wall, phases_s=dict(fused.times), ate_rmse=ate_rmse(est, gt))
    for k, v in res["phases_s"].items():
        print("  %-12s %8.3f s" % (k, v))
    print("wall %.3f s, %.2f frames/s, ATE RMSE %.6f m" % (wall, res["fps"], res["ate_rmse"]), flush=True)
    with open(os.path.join(out, "run.json"), "w") as f:
        json.dump(res, f, indent=1)
    return res


if __name__ == "__main__":
    main(sys.argv[1:])
