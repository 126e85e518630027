"""Generate tests/golden/slam_sequences/*.pt: whole sequences through the UNMODIFIED reference Tracker.run and Mapper.run (imported from the
reference checkout through tests/ref_harness.py) on CPU, room0 geometry, 'soft' grids.

    python tests/make_golden_slam_sequences.py        # needs the reference checkout

The two run() loops are wired as NICE_SLAM.run wires its processes (src/NICE_SLAM.py:267-318): shared idx, mapping_idx,
mapping_first_frame, estimate_c2w_list and gt_c2w_list, the tracker starting once the first frame is mapped.  Here they are two threads of
one process; under sync_method 'strict' they never compute at the same time, so one recorder on torch.randint / get_sample_uv / the
keyframe selections / Tensor.backward, tagged by thread, captures both random streams.  Logger, mesher and visualiser are stubbed (the
logger records the frames it is asked to log).  coarse: False.

Frames are scene_util.make_frame images; the ground-truth poses lie on a smooth path near the room0 bound centre (slam_sequences.path_pose).  Mapping
`iters` / `iters_first` are cut (MAPPING) so the run finishes in minutes on CPU.  Each fixture stores the seeds and settings, every draw and
selection (the replay of FusedSLAM.run), the call log in FusedSLAM.run_log's form with per-iteration losses, estimate_c2w_list, the keyframe
list and its final est_c2w, a sample of the final voxels (mg_samples) and the trained decoders.

    every1.pt    8 frames, every_frame = keyframe_every = 1: BA switches on at frame 5, frame 6 is the n_img - 2 keyframe, frame 7 gets
                 colour refinement
    blocks.pt    12 frames, the shipped every_frame 5 / keyframe_every 50: frames 0, 5, 10, 11 are mapped, keyframes 0 and 10, no BA
"""
import os
import sys
import threading
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import make_golden as mg        # noqa: E402
import make_golden_mapper_frames as mgf     # noqa: E402
import make_golden_tracker_frames as mgt    # noqa: E402
import ref_harness as rh        # noqa: E402
import scene_util as su         # noqa: E402
from slam_sequences import FRAME_SEED0, sequence   # noqa: E402

OUT = os.path.join(su.GOLDEN, "slam_sequences")
MAPPING = dict(iters=5, iters_first=10)             # shipped Replica: 60 / 1500
CASES = {
    "every1": dict(n=8, every_frame=1, keyframe_every=1, ckpt_freq=4, seed=1201),
    "blocks": dict(n=12, every_frame=5, keyframe_every=50, ckpt_freq=500, seed=1202),
}


class _Stub:
    def __init__(self):
        self.logged = []

    def log(self, idx, *a, **k):
        self.logged.append(int(idx))

    def get_mesh(self, *a, **k):
        pass

    def vis(self, *a, **k):
        pass


def gen_case(name, spec):
    ref = rh.import_reference()
    import src.common as common_mod
    import src.Mapper as mapper_mod
    import src.Tracker as tracker_mod
    sc, cfg, slam, renderer = mg.ref_scene("room0", "soft")
    cfg = dict(cfg)
    cfg["sync_method"], cfg["coarse"] = "strict", False
    cfg["mapping"] = dict(cfg["mapping"], every_frame=spec["every_frame"], keyframe_every=spec["keyframe_every"], ckpt_freq=spec["ckpt_freq"],
                          **MAPPING)
    cfg["tracking"] = dict(cfg["tracking"], gt_camera=False)
    frames = sequence(sc, spec["n"])
    n = spec["n"]
    H, W = sc["cam"]["H"], sc["cam"]["W"]
    start_c = {k: v.detach().clone() for k, v in slam.shared_c.items()}

    # shared state of NICE_SLAM.__init__ (src/NICE_SLAM.py:67-85)
    estimate_c2w_list, gt_c2w_list = torch.zeros(n, 4, 4), torch.zeros(n, 4, 4)
    shared_idx, mapping_idx, mapping_first_frame, mapping_cnt = (torch.zeros(1).int() for _ in range(4))
    stub = _Stub()

    loader = [(torch.tensor([k]), c.unsqueeze(0), d.unsqueeze(0), p.unsqueeze(0)) for k, c, d, p in frames]
    tracker = mgt.tracker_for_run(cfg, slam, renderer, loader)
    tracker.sync_method = "strict"
    tracker.idx, tracker.mapping_idx = shared_idx, mapping_idx
    tracker.estimate_c2w_list, tracker.gt_c2w_list = estimate_c2w_list, gt_c2w_list
    tracker.visualizer = stub

    mapper = rh.make_mapper(cfg, slam, renderer)
    mp = cfg["mapping"]
    for k in ("every_frame", "keyframe_every", "ckpt_freq", "color_refine", "no_log_on_first_frame", "mesh_freq", "no_mesh_on_first_frame"):
        setattr(mapper, k, mp[k])
    mapper.num_joint_iters = mp["iters"]
    mapper.cfg, mapper.sync_method, mapper.coarse, mapper.scale = cfg, "strict", False, cfg["scale"]
    mapper.idx, mapper.mapping_idx, mapper.mapping_first_frame, mapper.mapping_cnt = shared_idx, mapping_idx, mapping_first_frame, mapping_cnt
    mapper.estimate_c2w_list = estimate_c2w_list
    mapper.frame_reader, mapper.n_img = frames, n
    mapper.logger, mapper.mesher, mapper.visualizer = stub, stub, stub
    mapper.low_gpu_mem, mapper.eval_rec, mapper.clean_mesh, mapper.mesh_coarse_level, mapper.args = False, False, False, False, None

    # recorders, tagged by thread
    track = {}                          # idx -> dict(draws=[...], losses=[...], tensors=[...])
    calls = []                          # one dict per optimize_map call
    cur_track = [None]
    _ri, _guv, _gtc, _bw = torch.randint, common_mod.get_sample_uv, tracker_mod.get_tensor_from_camera, torch.Tensor.backward
    _sel, _rs, _opt, _om = mapper.keyframe_selection_overlap, mapper_mod.random_select, tracker.optimize_cam_in_batch, mapper.optimize_map
    _system = mapper_mod.os.system

    def role():
        return threading.current_thread().name

    def randint_rec(*a, **k):
        r = _ri(*a, **k)
        if role() == "tracker":
            cur_track[0]["draws"].append(r.clone())
        return r

    def guv_rec(*a, **k):
        r = _guv(*a, **k)
        if role() == "mapper":
            calls[-1]["uv"].append((r[1].long() * W + r[0].long()).int())
        return r

    def gtc_rec(*a, **k):
        r = _gtc(*a, **k)
        if role() == "tracker":
            cur_track[0]["tensors"].append(r.clone())
        return r

    def bw_rec(self, *a, **k):
        if role() == "mapper":
            calls[-1]["losses"].append(float(self.detach()))
        return _bw(self, *a, **k)

    def sel_rec(*a, **k):
        r = _sel(*a, **k)
        calls[-1]["selection"] = [int(x) for x in r]
        return r

    def rs_rec(*a, **k):
        r = _rs(*a, **k)
        calls[-1]["selection"] = [int(x) for x in r]
        return r

    def opt_rec(camera_tensor, *a, **k):
        loss = _opt(camera_tensor, *a, **k)
        cur_track[0]["losses"].append(loss)
        return loss

    def om_rec(num_joint_iters, lr_factor, idx, cur_gt_color, cur_gt_depth, gt_cur_c2w, keyframe_dict, keyframe_list, cur_c2w):
        calls.append(dict(idx=int(idx), num_joint_iters=int(num_joint_iters), lr_factor=float(lr_factor), ba=bool(mapper.BA),
                          start_c2w=cur_c2w.detach().clone().float(), keyframes=[int(k) for k in keyframe_list],
                          mapping_window_size=mapper.mapping_window_size, middle_iter_ratio=mapper.middle_iter_ratio,
                          fine_iter_ratio=mapper.fine_iter_ratio, fix_color=mapper.fix_color,
                          frustum_feature_selection=mapper.frustum_feature_selection, uv=[], losses=[], selection=[]))
        r = _om(num_joint_iters, lr_factor, idx, cur_gt_color, cur_gt_depth, gt_cur_c2w, keyframe_dict, keyframe_list, cur_c2w)
        c = calls[-1]
        c["returned"] = None if r is None else r.detach().clone().float()
        c["keyframe_est_c2w"] = torch.stack([d["est_c2w"].detach().clone().float() for d in keyframe_dict]) if keyframe_dict else torch.zeros(0, 4, 4)
        return r

    # the tracker's per-frame boundaries: wrap the frame loader
    class _Frames:
        def __len__(self):
            return n

        def __iter__(self):
            for item in loader:
                cur_track[0] = track.setdefault(int(item[0][0]), dict(draws=[], losses=[], tensors=[]))
                yield item
    tracker.frame_loader = _Frames()

    torch.randint, common_mod.get_sample_uv, tracker_mod.get_tensor_from_camera, torch.Tensor.backward = randint_rec, guv_rec, gtc_rec, bw_rec
    mapper.keyframe_selection_overlap, mapper_mod.random_select, tracker.optimize_cam_in_batch, mapper.optimize_map = sel_rec, rs_rec, opt_rec, om_rec
    mapper_mod.os.system = lambda *a, **k: 0                   # the final `cp` of the mesh the stubbed mesher never wrote
    errors = []

    def guarded(fn):
        def body():
            try:
                fn()
            except BaseException as e:               # noqa: BLE001
                errors.append(e)
                raise
        return body

    def tracking():
        while int(mapping_first_frame[0]) != 1:      # NICE_SLAM.tracking
            if errors:
                return
            time.sleep(0.1)
        tracker.run()
    try:
        torch.manual_seed(spec["seed"]); np.random.seed(spec["seed"])
        threads = [threading.Thread(target=guarded(mapper.run), name="mapper"), threading.Thread(target=guarded(tracking), name="tracker")]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
    finally:
        torch.randint, common_mod.get_sample_uv, tracker_mod.get_tensor_from_camera, torch.Tensor.backward = _ri, _guv, _gtc, _bw
        mapper_mod.random_select, mapper_mod.os.system = _rs, _system
    assert not errors, errors

    # per tracked frame: draws [iters, pixels], losses, start camera tensor (get_tensor_from_camera(gt) comes first), chosen iteration
    it_t = cfg["tracking"]["iters"]
    log, replay_track, replay_map = [], {}, []
    tracked = {}
    for idx, t in sorted(track.items()):
        if idx == 0:
            continue
        losses = torch.tensor(t["losses"], dtype=torch.float64)
        assert len(t["draws"]) == it_t and len(t["tensors"]) == 2
        best, cur_min = -1, 1e10
        for i, v in enumerate(t["losses"]):           # Tracker.py:245-247
            if v < cur_min:
                best, cur_min = i, v
        tracked[idx] = dict(kind="track", idx=idx, start_tensor=t["tensors"][1], start_from=idx - 1,
                            speed_from=idx - 2 if idx >= 2 and cfg["tracking"]["const_speed_assumption"] else None, losses=losses, best_iter=best)
        replay_track[idx] = torch.stack(t["draws"]).int()
    # interleave in the order of the strict schedule: frame 0 mapped, then per frame tracked, then (if mapped) its calls
    by_frame = {}
    for c in calls:
        sel = c.pop("selection")
        overlap = mapper.keyframe_selection_method == "overlap" and len(c["keyframes"]) > 0
        uv = c.pop("uv")
        if overlap:
            uv.pop(0)
        rows = sel + ([len(c["keyframes"]) - 1] if c["keyframes"] else []) + [-1]
        F, iters = len(rows), c["num_joint_iters"]
        assert len(uv) == iters * F and len(c["losses"]) == iters, (len(uv), F, iters, len(c["losses"]))
        draws = torch.stack([torch.stack(uv[i * F:(i + 1) * F]) for i in range(iters)])
        replay_map.append(dict(draws=draws, selection=sel))
        stages = [("middle" if i <= int(iters * c["middle_iter_ratio"]) else ("fine" if i <= int(iters * c["fine_iter_ratio"]) else "color"))
                  for i in range(iters)]
        entry = dict(kind="map", idx=c["idx"], num_joint_iters=iters, lr_factor=c["lr_factor"], ba=c["ba"],
                     refine=bool(c["fix_color"] and not c["frustum_feature_selection"]), start_c2w=c["start_c2w"], window=rows,
                     fixed_row=rows.index(min(rows[:-1])) if len(rows) > 1 else None, stages=stages,
                     losses=torch.tensor(c["losses"], dtype=torch.float64), keyframes=c["keyframes"],
                     mapping_window_size=c["mapping_window_size"], fix_color=c["fix_color"],
                     frustum_feature_selection=c["frustum_feature_selection"], returned=c["returned"], keyframe_est_c2w=c["keyframe_est_c2w"])
        by_frame.setdefault(c["idx"], []).append(entry)
    for idx in range(n):
        if idx in tracked:
            log.append(tracked[idx])
        log.extend(by_frame.get(idx, []))
    st = cfg["mapping"]
    final = {k: mgf.mg_samples(slam.shared_c[k].detach().reshape(-1).clone(), start_c[k].reshape(-1)) for k in ("grid_middle", "grid_fine", "grid_color")}
    trained = [lvl for lvl, fixed in (("fine", st["fix_fine"]), ("color", st["fix_color"])) if not fixed]
    decs = {lvl: {k: v.detach().clone() for k, v in getattr(slam.shared_decoders, lvl + "_decoder").state_dict().items()} for lvl in trained}
    settings = dict(tracking={k: cfg["tracking"][k] for k in ("ignore_edge_W", "ignore_edge_H", "iters", "lr", "pixels", "seperate_LR", "handle_dynamic",
                                                              "use_color_in_tracking", "w_color_loss", "const_speed_assumption", "gt_camera")},
                    mapping={k: st[k] for k in (*mgf.SETTING_KEYS, "every_frame", "keyframe_every", "ckpt_freq", "no_log_on_first_frame", "iters",
                                                "iters_first", "lr_factor", "lr_first_factor", "color_refine", "BA", "save_selected_keyframes_info")},
                    coarse=False, sync_method="strict")
    obj = dict(scene="room0", variant="soft", n=n, frame_seed0=FRAME_SEED0, seed=spec["seed"], settings=settings,
               gt_c2w_list=gt_c2w_list.clone(), estimate_c2w_list=estimate_c2w_list.clone(),
               replay=dict(track=replay_track, map=replay_map), run_log=log, logged=list(stub.logged),
               keyframe_list=[int(k) for k in mapper.keyframe_list],
               keyframe_est_c2w=torch.stack([d["est_c2w"].detach().clone().float() for d in mapper.keyframe_dict]),
               final=final, decoders=decs)
    os.makedirs(OUT, exist_ok=True)
    path = os.path.join(OUT, name + ".pt")
    torch.save(obj, path)
    print("wrote %-12s %8.1f KB  mapped %s  keyframes %s  logged %s" % (name + ".pt", os.path.getsize(path) / 1024,
                                                                      [e["idx"] for e in log if e["kind"] == "map"], obj["keyframe_list"], stub.logged))


if __name__ == "__main__":
    import warnings
    warnings.filterwarnings("ignore")
    for nm in (sys.argv[1:] or CASES):
        gen_case(nm, CASES[nm])
