"""A whole RGB-D sequence on the fused path, in one process: the order NICE_SLAM.run's tracker, mapper and coarse-mapper processes
(src/NICE_SLAM.py:298-318, src/Tracker.py:144-259, src/Mapper.py:542-657) follow under sync_method 'strict', where they never run at the
same time.  Per frame: tracking.FusedTrackingLoop.track_frame; every `every_frame` frames and on the last one: mapping.FusedMapper.map_frame
(and the coarse mapper's).  Checkpoints follow the reference's Logger.log, so its eval_ate.py, mesher and visualiser read a fused run."""
import os
import shutil
import time

import numpy as np
import torch

from .keyframes import KeyframeStore
from .mapping import FusedMapper
from .mesh import FusedMesher
from .tracking import FusedTrackingLoop

MAPPER_KEYS = ("pixels", "mapping_window_size", "middle_iter_ratio", "fine_iter_ratio", "stage", "BA_cam_lr", "w_color_loss",
               "keyframe_selection_method", "fix_fine", "fix_color", "frustum_feature_selection")
TRACKER_KEYS = ("ignore_edge_W", "ignore_edge_H", "iters", "lr", "seperate_LR", "handle_dynamic", "use_color_in_tracking", "w_color_loss",
                "const_speed_assumption")
PHASES = ("tracking", "mapping", "coarse", "refinement", "checkpoints")


class FusedSLAM:
    """NICE_SLAM.run under sync_method 'strict' (the only one whose result does not depend on timing):

    - frame 0 is mapped first, from its ground-truth pose, with iters_first and lr_first_factor; frame 0, and every frame under
      tracking.gt_camera, takes its ground-truth pose;
    - every other frame is tracked from estimate_c2w_list[idx-1] -- after a mapped frame the pose bundle adjustment refined
      (Tracker.py:164-167), else the tracker's own estimate -- with the constant-speed start through estimate_c2w_list[idx-2];
    - frames that are multiples of every_frame, and the last frame, are mapped after they are tracked: per outer iteration of
      Mapper.py:598-617 bundle adjustment is re-evaluated (more than 4 keyframes), the current pose is written back after it, and the
      keyframe is appended after the last outer iteration (idx % keyframe_every == 0 or idx == n_img - 2).  The last frame gets the
      colour-refinement pass when color_refine is set (Mapper.py:578-586: window x 2, both ratios 0, iterations x 5 over 5 outer iterations,
      fix_color, no frustum selection);
    - with cfg['coarse'] the coarse mapper maps the same frames, after the fine mapper, from the tracked (pre-BA) pose -- the reference's
      coarse process reads estimate_c2w_list[idx] before the fine mapper writes the BA pose back -- and keeps a keyframe list of its own with
      those poses.  Which frames the reference's coarse process maps depends on timing; nothing in tracking or fine mapping reads
      grid_coarse, so that choice cannot move a pose.

    Each component draws from its own torch.Generator on the device and its own numpy RandomState, seeded from `seed` (self.seeds), as the
    reference's three processes each have their own random state.

    With mesh_dir, the fine mapper's frames are meshed as Mapper.py:636-653 meshes them (mesh.FusedMesher, after the checkpoint):
    {idx:05d}_mesh.ply when idx % mesh_freq == 0 (not frame 0 under no_mesh_on_first_frame); on the last frame final_mesh.ply and a copy
    as {idx:05d}_mesh.ply, and with meshing.eval_rec final_mesh_eval_rec.ply culled with every frame's pose.  The scene hull is the
    convex hull of the keyframes' depth points rather than of open3d's TSDF surface (see mesh.py).  Meshing reads the grids only and
    draws no random numbers; its wall time goes to times['meshing']."""

    def __init__(self, renderer, c, decoders, cfg, seed=0, ckpt_dir=None, mesh_dir=None):
        """renderer / c / decoders: a FusedRenderer, the shared grids (updated in place) and decoders; cfg: the reference's loaded config
        (cfg['tracking'], cfg['mapping'], cfg['coarse'], cfg['sync_method']; with mesh_dir also cfg['meshing'], cfg['scale'] and
        mapping.marching_cubes_bound / mesh_freq / no_mesh_on_first_frame).  ckpt_dir: where the checkpoints go (none without it);
        mesh_dir: where the meshes go (no meshing without it)."""
        if cfg["sync_method"] != "strict":
            raise RuntimeError("FusedSLAM: sync_method %r is not supported; only 'strict' gives a result that does not depend on timing"
                               % cfg["sync_method"])
        self.r, self.c, self.dec, self.cfg, self.ckpt_dir, self.mesh_dir = renderer, c, decoders, cfg, ckpt_dir, mesh_dir
        self.mesher = FusedMesher(renderer, cfg) if mesh_dir is not None else None
        mp = cfg["mapping"]
        self.every_frame, self.keyframe_every, self.ckpt_freq = int(mp["every_frame"]), int(mp["keyframe_every"]), int(mp["ckpt_freq"])
        self.color_refine, self.no_log_on_first_frame = bool(mp["color_refine"]), bool(mp["no_log_on_first_frame"])
        self.save_selected = bool(mp.get("save_selected_keyframes_info", False))
        self.coarse = bool(cfg["coarse"])
        self.gt_camera = bool(cfg["tracking"]["gt_camera"])
        self.seeds = {"tracker": int(seed), "mapper": int(seed) + 1, "coarse": int(seed) + 2}
        self.dev = next(iter(c.values())).device
        self.run_log, self.times = [], self._phases()
        self.estimate_c2w_list = self.gt_c2w_list = None
        self._build()

    # ------------------------------------------------------------------------------------------ components
    def _build(self):
        """The tracker, the mapper(s) and their keyframe stores, each with its own random streams."""
        dev = self.dev
        self.generators = {k: torch.Generator(device=dev).manual_seed(s) for k, s in self.seeds.items()}
        self.rngs = {k: np.random.RandomState(self.seeds[k]) for k in ("mapper", "coarse")}      # the tracker draws nothing from numpy
        self.tracker = self._tracker()
        self.store = self._store()
        self.mapper = self._mapper(self.store, {})
        self.refiner = None                      # the last frame's colour-refinement settings: a mapper of their own, made when needed
        self.coarse_store = self._store() if self.coarse else None
        self.coarse_mapper = self._mapper(self.coarse_store, {}, coarse=True) if self.coarse else None

    def _tracker(self):
        tr = self.cfg["tracking"]
        return FusedTrackingLoop(self.r, self.c, self.dec, tr["pixels"], generator=self.generators["tracker"], **{k: tr[k] for k in TRACKER_KEYS})

    def _store(self):
        r = self.r
        return KeyframeStore(r.H, r.W, r.fx, r.fy, r.cx, r.cy, self.dev)

    def _mapper(self, store, overrides, coarse=False):
        mp = self.cfg["mapping"]
        kind = "coarse" if coarse else "mapper"
        settings = dict({k: mp[k] for k in MAPPER_KEYS}, **overrides)
        return FusedMapper(self.r, self.c, self.dec, store, coarse_mapper=coarse, generator=self.generators[kind], rng=self.rngs[kind], **settings)

    def _refiner(self):
        """Mapper.py:578-586, which the reference applies to its mapper's attributes for the last frame."""
        if self.refiner is None:
            mp = self.cfg["mapping"]
            self.refiner = self._mapper(self.store, dict(mapping_window_size=2 * mp["mapping_window_size"], middle_iter_ratio=0.0,
                                                         fine_iter_ratio=0.0, fix_color=True, frustum_feature_selection=False))
        return self.refiner

    # ------------------------------------------------------------------------------------------ the run
    def run(self, frames, replay=None):
        """Run the sequence `frames`: frame-reader items (idx, gt_color [H,W,3], gt_depth [H,W], gt_c2w [4,4]) in order, idx = 0, 1, ...
        (a leading batch dimension of 1 is accepted).  replay: optional recorded draws, dict(track={idx: [iters, pixels]}, map=[...],
        coarse=[...]), the mapping lists holding one dict(draws=, selection=) per call in call order (either key may be absent).
        Returns (estimate_c2w_list, gt_c2w_list), [N,4,4] float32 host tensors; self.run_log records every tracked frame and mapping call."""
        replay = replay or {}
        n = len(frames)
        self.n_img = n
        self.estimate_c2w_list = torch.zeros(n, 4, 4)
        self.gt_c2w_list = torch.zeros(n, 4, 4)
        self.selected_keyframes = {} if self.save_selected else None
        self.run_log, self.times = [], self._phases()
        self._replay = {k: list(replay.get(k, ())) for k in ("map", "coarse")}
        self._replay_track = replay.get("track", {})
        H, W = int(self.r.H), int(self.r.W)
        for pos, (idx, gt_color, gt_depth, gt_c2w) in enumerate(frames):
            idx = int(idx)
            if idx != pos:
                raise RuntimeError("FusedSLAM: frame %d arrived at position %d; frames must come in order from 0" % (idx, pos))
            color = torch.as_tensor(gt_color).to(self.dev).reshape(H, W, 3)      # the frame's one host -> device copy
            depth = torch.as_tensor(gt_depth).to(self.dev).reshape(H, W)
            gt_c2w = torch.as_tensor(gt_c2w).detach().float().cpu().reshape(4, 4)
            self.gt_c2w_list[idx] = gt_c2w
            if idx == 0:                                                       # Mapper.run maps frame 0 first, from its ground truth
                self.estimate_c2w_list[0] = gt_c2w
                self._map_frame(0, color, depth, gt_c2w)
            else:
                if self.gt_camera:
                    self.estimate_c2w_list[idx] = gt_c2w
                else:
                    self.estimate_c2w_list[idx] = self._track(idx, color, depth)
                if idx % self.every_frame == 0 or idx == n - 1:
                    self._map_frame(idx, color, depth, gt_c2w)
        return self.estimate_c2w_list.clone(), self.gt_c2w_list.clone()

    def _phases(self):
        return dict.fromkeys(PHASES + (("meshing",) if self.mesher is not None else ()), 0.0)

    def _timed(self, phase, t0):
        if self.dev.type == "cuda":
            torch.cuda.synchronize(self.dev)
        self.times[phase] += time.perf_counter() - t0

    def _track(self, idx, color, depth):
        """Tracker.py:184-253 for frame idx > 0: start from estimate_c2w_list[idx-1] (constant speed through [idx-2])."""
        t0 = time.perf_counter()
        pre = self.estimate_c2w_list[idx - 1]
        prev_prev = self.estimate_c2w_list[idx - 2] if idx >= 2 else None
        try:
            start = self.tracker.initial_pose(pre, prev_prev)
            c2w = self.tracker.track_frame(color, depth, start, draws=self._replay_track.get(idx))
        except RuntimeError as e:
            raise RuntimeError("FusedSLAM: tracking frame %d: %s" % (idx, e)) from e
        c2w = c2w.cpu()
        self.run_log.append(dict(kind="track", idx=idx, start_c2w=torch.as_tensor(start).detach().float().cpu().clone(),
                                 start_from=idx - 1, speed_from=idx - 2 if prev_prev is not None and self.tracker.const_speed_assumption else None,
                                 losses=self.tracker.losses.cpu(), best_iter=self.tracker.best_iter))
        self._timed("tracking", t0)
        return c2w

    def _map_frame(self, idx, color, depth, gt_c2w):
        """Mapper.run's body (Mapper.py:572-634) for the fine mapper, then the coarse mapper's, then the checkpoint."""
        mp = self.cfg["mapping"]
        tracked = self.estimate_c2w_list[idx].clone()                          # what the coarse process reads, before BA writes back
        first = idx == 0
        refine = not first and idx == self.n_img - 1 and self.color_refine
        if first:
            outer, lr_factor, iters = 1, mp["lr_first_factor"], mp["iters_first"]
        elif refine:
            outer, lr_factor, iters = 5, mp["lr_factor"], mp["iters"] * 5
        else:
            outer, lr_factor, iters = 1, mp["lr_factor"], mp["iters"]
        t0 = time.perf_counter()
        mapper = self._refiner() if refine else self.mapper
        cur = tracked
        for o in range(outer):
            ba = len(self.store) > 4 and bool(mp["BA"])
            new = self._call(mapper, "map", idx, iters // outer, lr_factor, color, depth, cur, gt_c2w, ba, refine)
            if ba:
                cur = new.cpu()
                self.estimate_c2w_list[idx] = cur
            if o == outer - 1:
                self._keyframe(self.store, idx, color, depth, cur, gt_c2w)
        self._timed("refinement" if refine else "mapping", t0)
        if self.coarse:
            t0 = time.perf_counter()
            c_iters, c_lr = (mp["iters_first"], mp["lr_first_factor"]) if first else (mp["iters"], mp["lr_factor"])
            self._call(self.coarse_mapper, "coarse", idx, c_iters, c_lr, color, depth, tracked, gt_c2w, False, False)
            self._keyframe(self.coarse_store, idx, color, depth, tracked, gt_c2w)
            self._timed("coarse", t0)
        if self.ckpt_dir is not None and (((not (first and self.no_log_on_first_frame)) and idx % self.ckpt_freq == 0) or idx == self.n_img - 1):
            t0 = time.perf_counter()
            self.log(idx)
            self._timed("checkpoints", t0)
        if self.mesher is not None:
            t0 = time.perf_counter()
            self._mesh(idx)
            self._timed("meshing", t0)

    def _mesh(self, idx):
        """Mapper.py:636-653 with the fine mapper's keyframes and estimate_c2w_list."""
        mp, ms = self.cfg["mapping"], self.cfg["meshing"]
        clean = bool(ms.get("clean_mesh", True))
        state = (self.c, self.dec, self.store, self.estimate_c2w_list, idx)
        if idx % int(mp["mesh_freq"]) == 0 and not (idx == 0 and mp["no_mesh_on_first_frame"]):
            self.mesher.get_mesh(os.path.join(self.mesh_dir, "{:05d}_mesh.ply".format(idx)), *state, clean_mesh=clean)
        if idx == self.n_img - 1:
            final = os.path.join(self.mesh_dir, "final_mesh.ply")
            if self.mesher.get_mesh(final, *state, clean_mesh=clean) is not None:
                shutil.copyfile(final, os.path.join(self.mesh_dir, "{:05d}_mesh.ply".format(idx)))
            if ms.get("eval_rec"):
                self.mesher.get_mesh(os.path.join(self.mesh_dir, "final_mesh_eval_rec.ply"), *state, clean_mesh=clean, get_mask_use_all_frames=True)

    def _call(self, mapper, kind, idx, iters, lr_factor, color, depth, cur, gt_c2w, ba, refine):
        """One optimize_map call, recorded in run_log."""
        store = mapper.store
        keyframes = list(store.idx)
        kf_poses = list(store.est_c2w)                                          # update_pose replaces entries: this keeps the pre-call poses
        rep = self._replay[kind].pop(0) if self._replay[kind] else {}
        try:
            new = mapper.map_frame(iters, lr_factor, color, depth, cur, ba, draws=rep.get("draws"), selection=rep.get("selection"))
        except RuntimeError as e:
            raise RuntimeError("FusedSLAM: %s mapping of frame %d: %s" % ("coarse" if kind == "coarse" else "fine", idx, e)) from e
        self.run_log.append(dict(kind=kind, idx=idx, num_joint_iters=int(iters), lr_factor=float(lr_factor), ba=bool(ba), refine=bool(refine),
                                 start_c2w=cur.clone(), window=list(mapper.window), fixed_row=mapper.fixed_row, stages=list(mapper.stages),
                                 losses=mapper.losses.cpu(), keyframes=keyframes, mapping_window_size=mapper.window_size,
                                 fix_color=mapper.fix_color, frustum_feature_selection=mapper.frustum_feature_selection))
        if kind == "map" and self.save_selected:                                # Mapper.py:274-287
            self.selected_keyframes[idx] = [dict(idx=keyframes[k], gt_c2w=store.gt_c2w[k], est_c2w=kf_poses[k]) if k >= 0 else
                                            dict(idx=idx, gt_c2w=gt_c2w, est_c2w=cur.clone()) for k in mapper.window]
        return new

    def _keyframe(self, store, idx, color, depth, c2w, gt_c2w):
        """Mapper.py:612-617: after the last outer iteration, frames idx % keyframe_every == 0 and idx == n_img - 2 become keyframes."""
        if (idx % self.keyframe_every == 0 or idx == self.n_img - 2) and idx not in store.idx:
            store.append(idx, color, depth, c2w, gt_c2w)

    # ------------------------------------------------------------------------------------------ checkpoints
    def log(self, idx):
        """Logger.log (src/utils/Logger.py): {ckpt_dir}/{idx:05d}.tar with the Logger's keys and formats (frame indices as int32 0-d tensors,
        as the reference's shared idx produces them)."""
        os.makedirs(self.ckpt_dir, exist_ok=True)
        path = os.path.join(self.ckpt_dir, "{:05d}.tar".format(idx))
        torch.save({
            "c": self.c,
            "decoder_state_dict": self.dec.state_dict(),
            "gt_c2w_list": self.gt_c2w_list,
            "estimate_c2w_list": self.estimate_c2w_list,
            "keyframe_list": [torch.tensor(k, dtype=torch.int32) for k in self.store.idx],
            "selected_keyframes": self.selected_keyframes,
            "idx": torch.tensor(idx, dtype=torch.int32),
        }, path, _use_new_zipfile_serialization=False)
        return path


def ate_rmse(est, gt):
    """Absolute trajectory error (TUM definition, as eval_ate.py reports it): RMSE of the translations after the rigid alignment (rotation
    and translation, no scale) of the estimate onto the ground truth that minimises it (Horn's method, closed form through the SVD of the
    cross-covariance).  est / gt: [N,4,4] poses or [N,3] positions.  float64 numpy."""
    p = np.asarray(torch.as_tensor(est).detach().cpu().double())
    q = np.asarray(torch.as_tensor(gt).detach().cpu().double())
    p = p[:, :3, 3] if p.ndim == 3 else p
    q = q[:, :3, 3] if q.ndim == 3 else q
    mp, mq = p.mean(0), q.mean(0)
    u, _, vt = np.linalg.svd((q - mq).T @ (p - mp))
    s = np.diag([1.0, 1.0, np.sign(np.linalg.det(u @ vt))])               # a rotation, not a reflection
    rot = u @ s @ vt
    res = (q - mq) - (p - mp) @ rot.T
    return float(np.sqrt((res ** 2).sum(1).mean()))
