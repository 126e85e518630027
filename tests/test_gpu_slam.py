"""GPU: whole sequences through slam.FusedSLAM -- replays of the real runs of tests/make_golden_slam_sequences.py, the random streams of
the default draws, checkpoints, the coarse mapper and errors."""
import json
import os

import numpy as np
import pytest
import torch

import scene_util as su
from gpu_util import make_renderer
from slam_sequences import per_frame, rel_dev, sequence

pytestmark = pytest.mark.gpu
DEV = "cuda"
GOLD = os.path.join(su.GOLDEN, "slam_sequences")
FIELDS = ("idx", "num_joint_iters", "lr_factor", "ba", "refine", "window", "fixed_row", "stages", "keyframes", "mapping_window_size", "fix_color",
          "frustum_feature_selection")
# Per-frame bars, each 4x the largest deviation measured on an H100 80GB HBM3 (700 W) by tools/slam_replay_drift.py and rounded up:
# (translation m, rotation rad, relative mapping loss, relative tracking loss) of estimate_c2w_list[k] and of frame k's calls.
# REF: a replay against the reference's CPU run (four replays measured).  FUSED: two replays of the same draws against each other, and
# a replay with the coarse mapper against one without (five pairs per fixture measured in all).  Fused replays with identical inputs drift:
# blocks frame 1 by 2.3e-5 m, frame 11 by 5.7e-2 m; every1 frame 1 by 2.1e-4 m, frame 7 by 0.10 m.  The reduction order of the backward's
# atomic gradient sums is the only difference between them, and the sequence amplifies it: the frames are independent random images,
# so no pose fits them well, and the constant-speed start carries each frame's error into the next.  Against the reference, frame 0's call
# (5x rates under lr_first_factor) already differs by 3e-4 in its losses where two fused runs differ by 1.3e-6 (blocks), the first-frame
# divergence test_gpu_mapping_frames admits (voxels to 1e-2 (1 + |v|)); every later frame is tracked or mapped on that map.  Frame 1's
# first tracking loss (same start pose, same draws: only the map differs) is 5358.4-5359.7 in fused runs against the reference's 5008.9
# (every1) and 4434.1-4434.6 against 4430.8 (blocks).
REF = {"every1": [(0.0, 0.0, 0.0026, 0.0), (0.0014, 0.0032, 0.022, 0.29), (0.022, 0.038, 0.034, 0.97), (0.082, 0.15, 0.13, 2.7),
                  (0.17, 0.35, 0.11, 4.4), (0.3, 0.65, 0.15, 5.4), (0.45, 0.91, 0.31, 8.5), (0.55, 1.1, 0.3, 9.6)],
       "blocks": [(0.0, 0.0, 0.0013, 0.0), (0.0019, 0.0029, 0.0, 0.38), (0.029, 0.042, 0.0, 0.58), (0.05, 0.11, 0.0, 1.4), (0.064, 0.15, 0.0, 1.8),
                  (0.12, 0.24, 0.06, 1.5), (0.15, 0.34, 0.0, 2.2), (0.22, 0.51, 0.0, 2.0), (0.32, 0.69, 0.0, 3.0), (0.43, 0.88, 0.0, 2.7),
                  (0.52, 1.1, 0.21, 3.2), (0.6, 1.3, 0.29, 4.2)]}
REF_RUN = {"every1": dict(voxel=5.4, decoder=0.52), "blocks": dict(voxel=2.7, decoder=0.34)}     # |x - ref| / (1 + |ref|), voxel sample / decoders
FUSED = {"every1": [(0.0, 0.0, 0.00065, 0.0), (0.0016, 0.0041, 0.018, 0.54), (0.03, 0.059, 0.038, 2.4), (0.072, 0.14, 0.16, 3.2),
                    (0.13, 0.22, 0.14, 3.3), (0.22, 0.39, 0.14, 4.2), (0.34, 0.58, 0.51, 4.9), (0.42, 0.78, 0.4, 8.6)],
         "blocks": [(0.0, 0.0, 8.6e-05, 0.0), (9.1e-05, 0.00088, 0.0, 0.24), (0.00019, 0.00082, 0.0, 0.3),
                    (0.003, 0.023, 0.0, 0.54), (0.014, 0.043, 0.0, 0.6), (0.043, 0.12, 0.065, 1.3), (0.066, 0.19, 0.0, 1.4),
                    (0.094, 0.24, 0.0, 1.3), (0.15, 0.32, 0.0, 1.6), (0.22, 0.42, 0.0, 1.7), (0.28, 0.54, 0.19, 2.1),
                    (0.34, 0.7, 0.2, 2.4)]}
FUSED_RUN = {"every1": dict(grid_middle=7.5, grid_fine=0.72, grid_color=0.63, decoder=0.23),       # whole grids / every decoder
             "blocks": dict(grid_middle=6.1, grid_fine=0.59, grid_color=0.56, decoder=0.081)}
QS = ("t", "r", "map_loss", "track_loss")


@pytest.fixture(scope="module")
def room0():
    return su.load_scenes()["room0"]


def load(name):
    return torch.load(os.path.join(GOLD, name + ".pt"), map_location="cpu", weights_only=False)


def cfg_of(case, **mapping):
    s = case["settings"]
    return dict(tracking=dict(s["tracking"]), mapping=dict(s["mapping"], **mapping), coarse=s["coarse"], sync_method=s["sync_method"])


def slam_for(sc, cfg, **kw):
    from nice_slam_b200 import FusedSLAM
    renderer, c, dec = make_renderer(sc, su.make_grids(sc, "soft"), su.load_decoders("soft"), DEV)
    return FusedSLAM(renderer, c, dec, cfg, **kw)


def replay(sc, case, coarse=None):
    cfg = cfg_of(case)
    if coarse is not None:
        cfg["coarse"] = coarse
    slam = slam_for(sc, cfg)
    est, gt = slam.run(sequence(sc, case["n"]), replay=case["replay"])
    return slam, est, gt


def within(dev, bars, what):
    for k, d in dev.items():
        for q, bar in zip(QS, bars[k]):
            assert d[q] <= bar, (what, k, q, d[q], bar)


def against_reference(slam, case):
    vox = max(rel_dev(slam.c[k].detach().reshape(-1).cpu()[fin["idx"].long()], fin["val"]) for k, fin in case["final"].items())
    st = slam.dec.state_dict()
    dec = max(rel_dev(st["%s_decoder.%s" % (lvl, k)].reshape(v.shape), v) for lvl, want in case["decoders"].items() for k, v in want.items())
    return vox, dec


@pytest.mark.parametrize("name", ("every1", "blocks"))
def test_replay_of_the_reference_sequence(room0, name):
    """Two replays of the reference's draws and selections: the call log is the reference's exactly; no component draws from its
    generator (the replayed draws are used); the first mapping call keeps test_gpu_mapping_frames' first-frame rule (first loss within
    1e-4, every loss within 5 %); every frame is within its measured bar against the reference (REF) and against the other replay (FUSED)."""
    case = load(name)
    sc = room0
    n = case["n"]
    slam, est, gt = replay(sc, case)
    ref_log = case["run_log"]
    assert [(e["kind"], e["idx"]) for e in slam.run_log] == [(e["kind"], e["idx"]) for e in ref_log]
    for got, ref in zip(slam.run_log, ref_log):
        if ref["kind"] == "track":
            assert (got["start_from"], got["speed_from"]) == (ref["start_from"], ref["speed_from"])
        else:
            for f in FIELDS:
                assert got[f] == ref[f], (ref["idx"], f, got[f], ref[f])
    assert slam.store.idx == case["keyframe_list"] and torch.equal(gt, case["gt_c2w_list"])
    for k, g in slam.generators.items():
        assert torch.equal(g.get_state(), torch.Generator(device=DEV).manual_seed(slam.seeds[k]).get_state()), k
    first, want = slam.run_log[0]["losses"], ref_log[0]["losses"]
    assert abs(float(first[0]) - float(want[0])) <= 1e-4 * abs(float(want[0]))
    assert float(((first - want).abs() / want.abs()).max()) < 0.05
    other, est_b, _ = replay(sc, case)
    dev_ref = per_frame(est, slam.run_log, case["estimate_c2w_list"], ref_log, n)
    dev_fused = per_frame(est, slam.run_log, est_b, other.run_log, n)
    vox, dec = against_reference(slam, case)
    t1 = next(i for i, e in enumerate(ref_log) if e["kind"] == "track")       # frame 1: same start pose and draws, so only the map differs
    report = dict(reference=dev_ref, fused=dev_fused, voxel=vox, decoder=dec,
                  frame1_first_tracking_loss=[float(slam.run_log[t1]["losses"][0]), float(ref_log[t1]["losses"][0]),
                                              float(other.run_log[t1]["losses"][0])])
    out = os.environ.get("NSB_SLAM_DRIFT_OUT")
    if out:
        os.makedirs(out, exist_ok=True)
        with open(os.path.join(out, "drift_%s.json" % name), "w") as f:
            json.dump(report, f, indent=1)
    print(name, json.dumps(report))
    within(dev_ref, REF[name], "reference")
    within(dev_fused, FUSED[name], "fused")
    assert vox <= REF_RUN[name]["voxel"] and dec <= REF_RUN[name]["decoder"], (vox, dec)


def small_cfg(case, **mapping):
    cfg = cfg_of(case, **dict(dict(every_frame=3, iters=4, iters_first=6, ckpt_freq=3), **mapping))
    cfg["tracking"] = dict(cfg["tracking"], iters=3)
    return cfg


def test_default_draws_follow_per_component_generators(room0):
    """Without replay: two runs from the same seed make the same calls with the same window sizes, so the same draws; each component's generator ends where the
    reference's calls, made directly on a generator with the same seed, leave it (tracker: per iteration randint(n_region, (pixels,));
    mapper: the overlap selection's randint(H*W, (100,)) when it has keyframes, then per iteration one randint(H*W, (ppi,)) per row;
    the coarse mapper: per iteration per row).  The numpy RandomStates likewise: the mapper's overlap selection permutes its candidates
    (all of them are selected while the window has room for them), the coarse mapper's random_select permutes range(K - 1).  Keyframes
    every mapped frame (every 2nd) and a 10-frame window make both selections run on growing keyframe lists."""
    sc = room0
    case = load("blocks")
    cfg = small_cfg(case, every_frame=2, keyframe_every=1, mapping_window_size=10)
    cfg["coarse"] = True
    runs = []
    for _ in range(2):
        slam = slam_for(sc, cfg, seed=7)
        slam.run(sequence(sc, 10))
        runs.append(slam)
    a, b = runs
    # the windows' sizes, which fix the draws; their order follows overlap counts under poses that differ in the last bits between runs
    assert [(e["kind"], e["idx"], len(e.get("window", ()))) for e in a.run_log] == [(e["kind"], e["idx"], len(e.get("window", ()))) for e in b.run_log]
    for k in a.generators:
        assert torch.equal(a.generators[k].get_state(), b.generators[k].get_state()), k
    H, W = sc["cam"]["H"], sc["cam"]["W"]
    tr = cfg["tracking"]
    n_region = (H - 2 * tr["ignore_edge_H"]) * (W - 2 * tr["ignore_edge_W"])
    g = {k: torch.Generator(device=DEV).manual_seed(s) for k, s in a.seeds.items()}
    for e in a.run_log:
        if e["kind"] == "track":
            for _ in range(tr["iters"]):
                torch.randint(n_region, (tr["pixels"],), device=DEV, generator=g["tracker"])
            continue
        gen = g["mapper" if e["kind"] == "map" else "coarse"]
        if e["kind"] == "map" and e["keyframes"] and cfg["mapping"]["keyframe_selection_method"] == "overlap":
            torch.randint(H * W, (100,), device=DEV, generator=gen)
        F = len(e["window"])
        for _ in range(e["num_joint_iters"]):
            for _ in range(F):
                torch.randint(H * W, (cfg["mapping"]["pixels"] // F,), device=DEV, generator=gen)
    for k in g:
        assert torch.equal(g[k].get_state(), a.generators[k].get_state()), k
    for k in a.rngs:
        sa, sb = a.rngs[k].get_state(), b.rngs[k].get_state()
        assert np.array_equal(sa[1], sb[1]) and sa[2:] == sb[2:], k
    rs = {k: np.random.RandomState(a.seeds[k]) for k in a.rngs}
    window = cfg["mapping"]["mapping_window_size"]
    for e in a.run_log:
        K = len(e.get("keyframes", ()))
        if e["kind"] == "map" and K:
            assert K - 1 <= window - 2                    # every candidate fits the window, so the permutation is of len(window) - 2
            rs["mapper"].permutation(len(e["window"]) - 2)
        elif e["kind"] == "coarse" and K:
            rs["coarse"].permutation(K - 1)
    assert sum(len(e["window"]) - 2 for e in a.run_log if e["kind"] == "map") > 0
    for k in rs:
        want, got = rs[k].get_state(), a.rngs[k].get_state()
        assert np.array_equal(want[1], got[1]) and want[2:] == got[2:], k
    # the first call of each kind saw the same first loss to the bit (same draws, same inputs)
    assert float(a.run_log[0]["losses"][0]) == float(b.run_log[0]["losses"][0])


def test_checkpoints_load_with_the_logger_keys(room0, tmp_path):
    sc = room0
    case = load("blocks")
    cfg = small_cfg(case)
    slam = slam_for(sc, cfg, ckpt_dir=str(tmp_path))
    est, gt = slam.run(sequence(sc, 8))
    files = sorted(os.listdir(tmp_path))
    assert files == ["00003.tar", "00006.tar", "00007.tar"]          # no_log_on_first_frame, ckpt_freq 3, the last frame
    for f in files:
        ck = torch.load(os.path.join(tmp_path, f), map_location="cpu", weights_only=False)
        assert set(ck) == {"c", "decoder_state_dict", "gt_c2w_list", "estimate_c2w_list", "keyframe_list", "selected_keyframes", "idx"}
        k = int(ck["idx"])
        assert f == "%05d.tar" % k
        assert ck["estimate_c2w_list"].shape == (8, 4, 4) and ck["gt_c2w_list"].shape == (8, 4, 4)
        assert torch.equal(ck["estimate_c2w_list"][:k + 1], est[:k + 1]) and torch.equal(ck["gt_c2w_list"][:k + 1], gt[:k + 1])
        assert set(ck["c"]) == set(slam.c) and all(ck["c"][g].shape == slam.c[g].shape for g in slam.c)
        assert set(ck["decoder_state_dict"]) == set(slam.dec.state_dict())
    assert torch.equal(ck["estimate_c2w_list"], est) and [int(x) for x in ck["keyframe_list"]] == slam.store.idx
    assert all(torch.equal(ck["c"][g].cpu(), slam.c[g].cpu()) for g in slam.c)


def test_coarse_mapper_changes_only_grid_coarse(room0):
    """The same replayed sequence with and without the coarse mapper: grid_coarse moves only with it, and the coarse mapper maps each
    mapped frame once.  Everything else agrees with the run without it to the bars measured between two fused replays (FUSED /
    FUSED_RUN): per-frame poses and losses, the middle, fine and colour grids and every decoder -- not bit-equal, since the backward
    sums gradients atomically."""
    sc = room0
    case = load("blocks")
    off, e0, _ = replay(sc, case, coarse=False)
    start = su.make_grids(sc, "soft")["grid_coarse"].to(DEV)
    on, e1, _ = replay(sc, case, coarse=True)
    assert torch.equal(off.c["grid_coarse"], start) and not torch.equal(on.c["grid_coarse"], start)
    assert [e["idx"] for e in on.run_log if e["kind"] == "coarse"] == sorted({e["idx"] for e in case["run_log"] if e["kind"] == "map"})
    fine_log = [e for e in on.run_log if e["kind"] != "coarse"]
    within(per_frame(e1, fine_log, e0, off.run_log, case["n"]), FUSED["blocks"], "coarse on / off")
    for k in ("grid_middle", "grid_fine", "grid_color"):
        assert rel_dev(on.c[k], off.c[k]) <= FUSED_RUN["blocks"][k], k
    a, b = on.dec.state_dict(), off.dec.state_dict()
    assert max(rel_dev(a[k], b[k]) for k in b) <= FUSED_RUN["blocks"]["decoder"]
    assert all(torch.equal(a[k], b[k]) for k in b if k.startswith("coarse_decoder."))


def test_a_frame_without_rays_in_the_bound_names_the_frame(room0):
    sc = room0
    cfg = small_cfg(load("blocks"))
    frames = sequence(sc, 4)
    k, color, depth, c2w = frames[2]
    frames[2] = (k, color, torch.full_like(depth, 1e6), c2w)
    slam = slam_for(sc, cfg)
    with pytest.raises(RuntimeError, match="frame 2"):
        slam.run(frames)
