"""Measure how far whole-sequence replays through slam.FusedSLAM drift, frame by frame, from the reference's CPU run
(tests/golden/slam_sequences, tests/make_golden_slam_sequences.py) and from each other.

    python tools/slam_replay_drift.py [--out DIR]

Per fixture: two replays A and B of the same recorded draws and windows (coarse off) and one replay C with the coarse mapper on.
Reported per frame: the pose (m, rad) and relative loss deviation of A and of B from the reference, of A from B (same inputs: what the
non-deterministic order of the backward's atomic gradient sums alone makes of the sequence), and of C from A.  Per run: the largest
|x - y| / (1 + |y|) over the fixture's voxel sample and trained decoders (A, B against the reference), and over the whole middle / fine /
colour grids and every decoder (A against B, C against A); whether grid_coarse moved.  These are the measurements the bars of
tests/test_gpu_slam.py come from.  Needs a CUDA device."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402

import scene_util as su  # noqa: E402
from gpu_util import make_renderer  # noqa: E402
from nice_slam_b200 import FusedSLAM  # noqa: E402
from slam_sequences import per_frame, rel_dev, sequence  # noqa: E402

FINE_GRIDS = ("grid_middle", "grid_fine", "grid_color")


def load(name):
    return torch.load(os.path.join(su.GOLDEN, "slam_sequences", name + ".pt"), map_location="cpu", weights_only=False)


def cfg_of(case, coarse=None):
    s = case["settings"]
    return dict(tracking=dict(s["tracking"]), mapping=dict(s["mapping"]), coarse=s["coarse"] if coarse is None else coarse,
                sync_method=s["sync_method"])


def replay(sc, case, coarse=False):
    """One replay: (estimate_c2w_list, run_log without coarse calls, grids, decoder state, grid_coarse before)."""
    renderer, c, dec = make_renderer(sc, su.make_grids(sc, "soft"), su.load_decoders("soft"), "cuda")
    slam = FusedSLAM(renderer, c, dec, cfg_of(case, coarse))
    start_coarse = c["grid_coarse"].clone()
    est, _ = slam.run(sequence(sc, case["n"]), replay=case["replay"])
    log = [e for e in slam.run_log if e["kind"] != "coarse"]
    return dict(est=est, log=log, full_log=slam.run_log, c={k: v.detach().clone() for k, v in c.items()},
                dec={k: v.detach().clone() for k, v in dec.state_dict().items()}, start_coarse=start_coarse)


def against_reference(run, case):
    vox = max(rel_dev(run["c"][k].reshape(-1).cpu()[fin["idx"].long()], fin["val"]) for k, fin in case["final"].items())
    dec = max(rel_dev(run["dec"]["%s_decoder.%s" % (lvl, k)].reshape(v.shape), v) for lvl, want in case["decoders"].items() for k, v in want.items())
    return vox, dec


def run_vs_run(x, y):
    grids = {k: rel_dev(x["c"][k], y["c"][k]) for k in FINE_GRIDS}
    dec = max(rel_dev(x["dec"][k], y["dec"][k]) for k in y["dec"])
    return grids, dec


def measure(sc, name):
    case = load(name)
    n = case["n"]
    a, b, c = replay(sc, case), replay(sc, case), replay(sc, case, coarse=True)
    res = dict(frames={k: {} for k in range(n)})
    for tag, (x_est, x_log, y_est, y_log) in dict(ref_a=(a["est"], a["log"], case["estimate_c2w_list"], case["run_log"]),
                                                 ref_b=(b["est"], b["log"], case["estimate_c2w_list"], case["run_log"]),
                                                 a_b=(a["est"], a["log"], b["est"], b["log"]),
                                                 a_c=(c["est"], c["log"], a["est"], a["log"])).items():
        for k, d in per_frame(x_est, x_log, y_est, y_log, n).items():
            res["frames"][k][tag] = d
    res["ref_a_voxel"], res["ref_a_decoder"] = against_reference(a, case)
    res["ref_b_voxel"], res["ref_b_decoder"] = against_reference(b, case)
    res["a_b_grids"], res["a_b_decoder"] = run_vs_run(a, b)
    res["a_c_grids"], res["a_c_decoder"] = run_vs_run(c, a)
    res["coarse_moved_without_coarse"] = not torch.equal(a["c"]["grid_coarse"], a["start_coarse"])
    res["coarse_moved_with_coarse"] = not torch.equal(c["c"]["grid_coarse"], c["start_coarse"])
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("slam_replay_drift: needs a CUDA device")
    sc = su.load_scenes()["room0"]
    out = {}
    for name in ("every1", "blocks"):
        r = measure(sc, name)
        out[name] = r
        print(name)
        for k, d in r["frames"].items():
            print("  %2d " % k + "  ".join("%s t %.1e r %.1e ml %.1e tl %.1e" % (tag, v["t"], v["r"], v["map_loss"], v["track_loss"]) for tag, v in d.items()))
        print("  " + json.dumps({k: v for k, v in r.items() if k != "frames"}))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "slam_replay_drift.json"), "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
