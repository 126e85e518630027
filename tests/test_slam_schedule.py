"""CPU: slam.FusedSLAM's schedule -- which frames are tracked and mapped, with which settings, from which poses, and what becomes a keyframe
or a checkpoint -- driven through stand-in tracker and mapper objects.  Against the real runs of tests/make_golden_slam_sequences.py the
stand-ins return the recorded outputs and the driver's call log must equal the reference's; further cases check the stated rules.  Also
slam.ate_rmse against closed-form cases."""
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import scene_util as su
from nice_slam_b200.mapping import map_stage, tensor_from_c2w, window_rows
from nice_slam_b200.slam import MAPPER_KEYS, FusedSLAM, ate_rmse
from nice_slam_b200.tracking import FusedTrackingLoop

GOLD = os.path.join(su.GOLDEN, "slam_sequences")
H, W = 4, 5                                     # the stand-ins never look at the images


def load(name):
    return torch.load(os.path.join(GOLD, name + ".pt"), map_location="cpu", weights_only=False)


class StandInTracker:
    """Records what the driver asks for; returns the next pose of `poses` (a callable idx, start -> pose)."""
    initial_pose = FusedTrackingLoop.initial_pose

    def __init__(self, pose_of, const_speed_assumption=True, iters=10):
        self.dev, self.const_speed_assumption, self.pose_of, self.iters = torch.device("cpu"), const_speed_assumption, pose_of, iters
        self.calls = []

    def track_frame(self, gt_color, gt_depth, init_c2w, draws=None):
        idx = len(self.calls) + 1
        self.calls.append(dict(init=init_c2w.clone(), draws=draws))
        out = self.pose_of(idx, init_c2w)
        self.losses = torch.arange(self.iters, dtype=torch.float64)
        self.best_iter = self.iters - 1
        return out.clone()


class StandInMapper:
    """Computes the window and stage schedule from its settings (mapping.window_rows / map_stage), checks the replayed draws' shape, and
    returns the next recorded result of `results` (dict(returned=, keyframe_est_c2w=)) or, without one, the start pose moved 1 cm along z."""

    def __init__(self, store, settings, coarse, results):
        self.store, self.coarse_mapper, self.results = store, coarse, results
        self.window_size, self.middle_iter_ratio, self.fine_iter_ratio = settings["mapping_window_size"], settings["middle_iter_ratio"], settings["fine_iter_ratio"]
        self.fix_color, self.frustum_feature_selection, self.pixels = settings["fix_color"], settings["frustum_feature_selection"], settings["pixels"]
        self.calls = []

    def map_frame(self, num_joint_iters, lr_factor, cur_gt_color, cur_gt_depth, cur_c2w, ba, draws=None, selection=None):
        assert not (ba and self.coarse_mapper)
        self.window, self.fixed_row = window_rows(list(selection) if selection is not None else [], len(self.store))
        F = len(self.window)
        if draws is not None:
            assert tuple(draws.shape) == (num_joint_iters, F, self.pixels // F)
        self.stages = [map_stage(it, num_joint_iters, self.middle_iter_ratio, self.fine_iter_ratio, self.coarse_mapper) for it in range(num_joint_iters)]
        self.losses = torch.zeros(num_joint_iters, dtype=torch.float64)
        self.calls.append(dict(cur=torch.as_tensor(cur_c2w).clone(), ba=ba))
        res = self.results.pop(0) if self.results else None
        if not ba:
            return None
        if res is None:
            out = torch.as_tensor(cur_c2w).float().clone()
            out[2, 3] += 0.01
            return out
        for k in range(len(self.store)):
            self.store.update_pose(k, res["keyframe_est_c2w"][k])
        return res["returned"].clone()


class Driver(FusedSLAM):
    """FusedSLAM with stand-in components."""

    def __init__(self, cfg, tracker_pose=None, results=None, **kw):
        self._tracker_pose = tracker_pose or (lambda idx, start: start.float() + 0.001)
        self._results = list(results or [])
        renderer = SimpleNamespace(H=H, W=W, fx=1.0, fy=1.0, cx=2.0, cy=2.0)
        super().__init__(renderer, {"grid_middle": torch.zeros(1)}, torch.nn.Linear(1, 1), cfg, **kw)

    def _tracker(self):
        return StandInTracker(self._tracker_pose, self.cfg["tracking"]["const_speed_assumption"], self.cfg["tracking"]["iters"])

    def _mapper(self, store, overrides, coarse=False):
        settings = dict({k: self.cfg["mapping"][k] for k in MAPPER_KEYS}, **overrides)
        return StandInMapper(store, settings, coarse, [] if coarse else self._results)


def frames_of(gt):
    return [(k, torch.zeros(H, W, 3), torch.zeros(H, W), gt[k]) for k in range(gt.shape[0])]


def cfg_of(case, **mapping):
    s = case["settings"]
    return dict(tracking=dict(s["tracking"]), mapping=dict(s["mapping"], **mapping), coarse=s["coarse"], sync_method=s["sync_method"])


def fixture_run(case, cfg=None, **kw):
    """Run the driver on a fixture: the tracker returns the recorded tracked pose (the start pose of the frame's first mapping call when
    the frame was mapped -- the list entry holds the BA pose then), the mapper the recorded BA results."""
    log = case["run_log"]
    maps = [e for e in log if e["kind"] == "map"]
    first_map = {}
    for e in maps:
        first_map.setdefault(e["idx"], e)

    def tracked(idx, start):
        return first_map[idx]["start_c2w"] if idx in first_map else case["estimate_c2w_list"][idx]
    d = Driver(cfg or cfg_of(case), tracker_pose=tracked, results=[dict(returned=e["returned"], keyframe_est_c2w=e["keyframe_est_c2w"]) for e in maps],
               **kw)
    est, gt = d.run(frames_of(case["gt_c2w_list"]), replay=case["replay"])
    return d, est, gt


FIELDS = ("idx", "num_joint_iters", "lr_factor", "ba", "refine", "window", "fixed_row", "stages", "keyframes", "mapping_window_size", "fix_color",
          "frustum_feature_selection")


@pytest.mark.parametrize("name", ("every1", "blocks"))
def test_call_log_matches_the_reference_run(name, tmp_path):
    """Frames, iteration counts, lr_factors, BA flags, windows, refinement settings, start poses and the list entries that feed them,
    keyframe appends with their poses, estimate_c2w_list and the checkpointed frames are the reference run's."""
    case = load(name)
    d, est, gt = fixture_run(case, ckpt_dir=str(tmp_path))
    want = case["run_log"]
    assert [(e["kind"], e["idx"]) for e in d.run_log] == [(e["kind"], e["idx"]) for e in want]
    for got, ref in zip(d.run_log, want):
        if ref["kind"] == "track":
            assert (got["start_from"], got["speed_from"]) == (ref["start_from"], ref["speed_from"]), ref["idx"]
            assert torch.allclose(tensor_from_c2w(got["start_c2w"]), ref["start_tensor"], atol=1e-6, rtol=0), ref["idx"]
        else:
            for f in FIELDS:
                assert got[f] == ref[f], (ref["idx"], f, got[f], ref[f])
            assert torch.equal(got["start_c2w"].float(), ref["start_c2w"]), ref["idx"]
    assert torch.equal(est, case["estimate_c2w_list"]) and torch.equal(gt, case["gt_c2w_list"])
    assert d.store.idx == case["keyframe_list"]
    assert torch.equal(torch.stack(d.store.est_c2w), case["keyframe_est_c2w"])
    assert sorted(int(f[:5]) for f in os.listdir(tmp_path)) == case["logged"]
    # the replayed draws reached the components in order
    assert [int(c["draws"].shape[0]) for c in d.tracker.calls] == [case["settings"]["tracking"]["iters"]] * (case["n"] - 1)
    assert all(torch.equal(c["draws"], case["replay"]["track"][k + 1]) for k, c in enumerate(d.tracker.calls))


def test_every1_reaches_ba_the_n_img_minus_2_keyframe_and_refinement():
    """The every1 fixture covers what it is meant to: BA switches on partway, frame n-2 is a keyframe, the last frame is refined over 5
    outer iterations with a doubled window; blocks maps 0, 5, 10, 11 with keyframes 0 and 10 and no BA."""
    log = [e for e in load("every1")["run_log"] if e["kind"] == "map"]
    bas = [e["ba"] for e in log]
    assert not bas[0] and bas[-1] and bas.index(True) > 1
    refine = [e for e in log if e["refine"]]
    assert len(refine) == 5 and all(e["idx"] == 7 and e["mapping_window_size"] == 2 * log[1]["mapping_window_size"] for e in refine)
    assert load("every1")["keyframe_list"][-2:] == [6, 7]
    b = load("blocks")
    assert [e["idx"] for e in b["run_log"] if e["kind"] == "map"] == [0, 5, 10] + [11] * 5 and b["keyframe_list"] == [0, 10]
    assert not any(e["ba"] for e in b["run_log"] if e["kind"] == "map")


def test_gt_camera_takes_every_ground_truth_pose():
    case = load("blocks")
    cfg = cfg_of(case)
    cfg["tracking"]["gt_camera"] = True
    d = Driver(cfg)
    est, gt = d.run(frames_of(case["gt_c2w_list"]))
    assert torch.equal(est, case["gt_c2w_list"]) and not d.tracker.calls
    assert [e["idx"] for e in d.run_log] == [0, 5, 10] + [11] * 5 and all(e["kind"] == "map" for e in d.run_log)
    assert all(torch.equal(e["start_c2w"], gt[e["idx"]]) for e in d.run_log)


def test_coarse_mapper_on_the_fine_frames_from_pre_ba_poses():
    """coarse: True -- after each fine call of a mapped frame one coarse call on the same frame, from the tracked pose (before the fine
    mapper's BA writes back), never with BA, at iters_first / lr_first_factor on frame 0 and iters / lr_factor (no refinement) after;
    the coarse keyframes are the fine ones' frames with the tracked poses."""
    case = load("every1")
    cfg = cfg_of(case)
    cfg["coarse"] = True
    d, est, _ = fixture_run(case, cfg)
    fine_log = [e for e in d.run_log if e["kind"] != "coarse"]
    assert [(e["kind"], e["idx"]) for e in fine_log] == [(e["kind"], e["idx"]) for e in case["run_log"]]
    coarse = [e for e in d.run_log if e["kind"] == "coarse"]
    mapped = sorted({e["idx"] for e in d.run_log if e["kind"] == "map"})
    assert [e["idx"] for e in coarse] == mapped
    for e in coarse:
        pos = d.run_log.index(e)
        assert d.run_log[pos - 1]["kind"] == "map" and d.run_log[pos - 1]["idx"] == e["idx"]         # after the fine mapper's last call
        first_fine = next(f for f in d.run_log if f["kind"] == "map" and f["idx"] == e["idx"])
        assert torch.equal(e["start_c2w"], first_fine["start_c2w"]) and not e["ba"] and not e["refine"]
        mp = cfg["mapping"]
        assert (e["num_joint_iters"], e["lr_factor"]) == ((mp["iters_first"], mp["lr_first_factor"]) if e["idx"] == 0 else (mp["iters"], mp["lr_factor"]))
        assert set(e["stages"]) == {"coarse"}
    assert d.coarse_store.idx == d.store.idx
    tracked = {e["idx"]: e["start_c2w"] for e in coarse}
    assert all(torch.equal(p, tracked[k]) for k, p in zip(d.coarse_store.idx, d.coarse_store.est_c2w))
    assert not all(torch.equal(a, b) for a, b in zip(d.coarse_store.est_c2w, d.store.est_c2w))      # BA moved the fine ones
    assert torch.equal(est, case["estimate_c2w_list"])


@pytest.mark.parametrize("no_log_first, freq, want", [(True, 2, [2, 4, 6, 8, 9]), (False, 2, [0, 2, 4, 6, 8, 9]), (True, 500, [9]),
                                                       (False, 3, [0, 3, 6, 9])])
def test_checkpoint_rule(tmp_path, no_log_first, freq, want):
    """Logger.log's rule (Mapper.py:627-631): mapped frames with idx % ckpt_freq == 0, frame 0 only without no_log_on_first_frame, and
    the last frame; the files carry the Logger's keys."""
    case = load("every1")
    cfg = cfg_of(case, ckpt_freq=freq, no_log_on_first_frame=no_log_first, color_refine=False, BA=False)
    gt = torch.stack([su.make_pose(su.load_scenes()["room0"], k) for k in range(10)])
    d = Driver(cfg, ckpt_dir=str(tmp_path))
    est, _ = d.run(frames_of(gt))
    files = sorted(os.listdir(tmp_path))
    assert files == ["%05d.tar" % k for k in want]
    ck = torch.load(os.path.join(tmp_path, files[-1]), weights_only=False)
    assert set(ck) == {"c", "decoder_state_dict", "gt_c2w_list", "estimate_c2w_list", "keyframe_list", "selected_keyframes", "idx"}
    assert int(ck["idx"]) == 9 and torch.equal(ck["estimate_c2w_list"], est) and [int(k) for k in ck["keyframe_list"]] == d.store.idx


def test_start_poses_follow_the_list_entries():
    """Without fixtures: frame idx starts from estimate_c2w_list[idx-1] -- the BA pose after a mapped frame -- with the constant-speed
    delta through [idx-2]; without const_speed_assumption from [idx-1] alone."""
    sc = su.load_scenes()["room0"]
    gt = torch.stack([su.make_pose(sc, k) for k in range(8)])
    for const in (True, False):
        cfg = dict(tracking=dict(gt_camera=False, const_speed_assumption=const, iters=3),
                   mapping=dict(every_frame=1, keyframe_every=1, ckpt_freq=500, color_refine=False, no_log_on_first_frame=True, BA=True,
                                iters=4, iters_first=6, lr_factor=1.0, lr_first_factor=5.0, pixels=100, mapping_window_size=5,
                                middle_iter_ratio=0.4, fine_iter_ratio=0.6, stage=None, BA_cam_lr=0.001, w_color_loss=0.2,
                                keyframe_selection_method="overlap", fix_fine=True, fix_color=False, frustum_feature_selection=True),
                   coarse=False, sync_method="strict")
        d = Driver(cfg)
        est, _ = d.run(frames_of(gt))
        tracks = [e for e in d.run_log if e["kind"] == "track"]
        for e in tracks:
            k = e["idx"]
            pre = est[k - 1]
            want = pre @ est[k - 2].inverse() @ pre if const and k >= 2 else pre
            assert torch.allclose(e["start_c2w"], want, atol=1e-6), k
        # BA on once 5 keyframes exist (frame 5): the stand-in's BA moved frames 5-7, and frames 6-7 started from the moved poses (above)
        maps = [e for e in d.run_log if e["kind"] == "map"]
        assert [e["ba"] for e in maps] == [False] * 5 + [True] * 3
        assert all(float(est[e["idx"]][2, 3] - e["start_c2w"][2, 3]) > 0.009 for e in maps[5:])


@pytest.mark.parametrize("method", ("loose", "free"))
def test_timing_dependent_sync_methods_raise(method):
    cfg = cfg_of(load("blocks"))
    cfg["sync_method"] = method
    with pytest.raises(RuntimeError, match="strict"):
        Driver(cfg)


def test_errors_name_the_frame():
    case = load("blocks")

    def failing(idx, start):
        if idx == 3:
            raise RuntimeError("FusedTrackingLoop: the bbox pre-filter kept no ray in iteration 0")
        return start.float()
    with pytest.raises(RuntimeError, match="frame 3"):
        Driver(cfg_of(case), tracker_pose=failing).run(frames_of(case["gt_c2w_list"]))


def rot(a, b, c):
    from scipy.spatial.transform import Rotation
    return Rotation.from_euler("xyz", [a, b, c]).as_matrix()


def test_ate_rmse_closed_form():
    """A rigid transform of a trajectory has ATE 0; noise orthogonal to what any rigid motion can absorb gives exactly its RMS."""
    g = np.random.RandomState(3)
    n = 40
    t = np.cumsum(g.randn(n, 3) * 0.1, 0)
    gt = np.tile(np.eye(4), (n, 1, 1))
    gt[:, :3, 3] = t
    R, off = rot(0.3, -0.2, 1.1), np.array([1.0, -2.0, 0.5])
    est = gt.copy()
    est[:, :3, 3] = t @ R.T + off
    est[:, :3, :3] = R @ gt[:, :3, :3]
    assert ate_rmse(torch.from_numpy(est), torch.from_numpy(gt)) < 1e-12
    # noise that no rigid motion can absorb: zero mean and uncorrelated with the centred positions in every axis pair, so the cross-
    # covariance is the positions' own (symmetric, positive definite), the best rotation is the identity and the ATE is the noise's RMS
    pos = gt[:, :3, 3]
    basis = np.concatenate([np.ones((n, 1)), pos - pos.mean(0)], 1)
    noise = g.randn(n, 3) * 0.01
    noise -= basis @ np.linalg.lstsq(basis, noise, rcond=None)[0]
    assert np.abs(noise.mean(0)).max() < 1e-15 and np.abs((pos - pos.mean(0)).T @ noise).max() < 1e-12
    rms = np.sqrt((noise ** 2).sum(1).mean())
    assert abs(ate_rmse(pos + noise, pos) - rms) < 1e-12, (ate_rmse(pos + noise, pos), rms)
    moved = (pos + noise) @ R.T + off
    assert abs(ate_rmse(moved, pos) - rms) < 1e-12
