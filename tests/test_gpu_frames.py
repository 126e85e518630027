"""nsb_frame_prepare and the frame readers on the GPU: the kernel against oracle/frames.py and cv2 / torch at real frame sizes, the
readers against the reference's golden outputs, the decoder thread's life cycle, and a whole run through nice_slam_b200.run."""
import json
import os
import threading

import cv2
import numpy as np
import pytest
import torch
import torch.nn.functional as F
import yaml

from make_golden_datasets import CAMS, OUT, check_frame, convonet_checkpoints, fixture_cfg
from nice_slam_b200 import datasets as ds
from oracle import frames as fr

pytestmark = pytest.mark.gpu
REF = torch.load(os.path.join(OUT, "reference.pt"), weights_only=False)
TUM1 = [0.2624, -0.9531, -0.0054, 0.0026, 1.1633]
TUM2 = [0.2312, -0.7849, -0.0033, -0.0001, 0.9172]


def _gpu(cam, bgr, raw, scale=1.0):
    p = ds.frame_params(dict(cam=cam, scale=scale), bgr.shape, raw.shape)
    c, d = ds.prepare_frame(p, torch.from_numpy(bgr).cuda(), torch.from_numpy(raw.view(np.int16)).cuda())
    torch.cuda.synchronize()
    return c.cpu().numpy(), d.cpu().numpy()


def _frame(hc, wc, hd, wd, seed=0):
    rng = np.random.default_rng(seed)
    bgr = rng.integers(0, 256, (hc, wc, 3), dtype=np.uint8)
    raw = rng.integers(0, 65536, (hd, wd), dtype=np.uint16)
    raw[0, :8] = 0
    raw[-1, -8:] = 65535
    return bgr, raw


CASES = {
    "replica": ((680, 1200, 680, 1200), dict(fx=600.0, fy=600.0, cx=599.5, cy=339.5, png_depth_scale=6553.5, crop_edge=0)),
    "apartment": ((720, 1280, 720, 1280), dict(fx=607.47, fy=607.45, cx=637.0, cy=369.27, png_depth_scale=1000.0, crop_edge=0)),
    "tum1": ((480, 640, 480, 640), dict(fx=517.3, fy=516.5, cx=318.6, cy=255.3, png_depth_scale=5000.0, crop_edge=8, crop_size=[384, 512],
                                        distortion=TUM1)),
    "tum2": ((480, 640, 480, 640), dict(fx=520.9, fy=521.0, cx=325.1, cy=249.7, png_depth_scale=5000.0, crop_edge=8, crop_size=[384, 512],
                                        distortion=TUM2)),
    "scannet": ((968, 1296, 480, 640), dict(fx=577.59, fy=578.73, cx=318.91, cy=242.68, png_depth_scale=1000.0, crop_edge=10)),
    "odd": ((37, 53, 29, 41), dict(fx=40.3, fy=41.1, cx=26.2, cy=18.7, png_depth_scale=1000.0, crop_edge=1, crop_size=[31, 47],
                                   distortion=TUM1)),
    "downscale_2x2": ((96, 128, 48, 64), dict(fx=51.7, fy=51.6, cx=31.9, cy=25.5, png_depth_scale=5000.0, crop_edge=2)),
    "downscale_3x3": ((144, 192, 48, 64), dict(fx=51.7, fy=51.6, cx=31.9, cy=25.5, png_depth_scale=5000.0, crop_edge=0)),
    "off_image": ((480, 640, 480, 640), dict(fx=301.7, fy=299.3, cx=322.9, cy=238.1, png_depth_scale=5000.0, crop_edge=0,
                                             distortion=[-0.9, 0.6, 0.02, -0.01, 0.4])),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_kernel_against_oracle(case):
    sizes, cam = CASES[case]
    bgr, raw = _frame(*sizes, seed=len(case))
    c, d = _gpu(cam, bgr, raw)
    wc, wd = fr.prepare(bgr, raw, cam)
    assert c.shape == wc.shape and d.shape == wd.shape
    assert np.array_equal(d, wd)                                                   # depth: bit-exact
    if sizes[:2] == sizes[2:]:
        assert np.abs(c - wc).max() <= 1e-12
    else:
        assert np.array_equal(c, wc)                                               # same arithmetic as the oracle's cv2.resize
    # the reference's own operations, directly
    col = bgr
    if cam.get("distortion") is not None:
        K = np.array([[cam["fx"], 0, cam["cx"]], [0, cam["fy"], cam["cy"]], [0, 0, 1.0]])
        col = cv2.undistort(col, K, np.array(cam["distortion"]))
        assert np.array_equal(fr.undistort(bgr, cam["fx"], cam["fy"], cam["cx"], cam["cy"], cam["distortion"]), col)
    col = cv2.cvtColor(col, cv2.COLOR_BGR2RGB) / 255.
    dep = raw.astype(np.float32) / cam["png_depth_scale"]
    col = torch.from_numpy(cv2.resize(col, (dep.shape[1], dep.shape[0])))
    dep = torch.from_numpy(dep) * 1
    if cam.get("crop_size") is not None:
        col = F.interpolate(col.permute(2, 0, 1)[None], cam["crop_size"], mode="bilinear", align_corners=True)[0].permute(1, 2, 0)
        dep = F.interpolate(dep[None, None], cam["crop_size"], mode="nearest")[0, 0]
    e = cam["crop_edge"]
    if e > 0:
        col, dep = col[e:-e, e:-e], dep[e:-e, e:-e]
    assert np.array_equal(d, dep.numpy())
    assert np.abs(c - col.numpy()).max() <= (1e-6 if sizes[:2] != sizes[2:] else 1e-12)


def test_undistorted_bytes_bit_exact():
    bgr, raw = _frame(480, 640, 480, 640, seed=5)
    for dist in (TUM1, TUM2):
        cam = dict(fx=517.3, fy=516.5, cx=318.6, cy=255.3, png_depth_scale=5000.0, crop_edge=0, distortion=dist)
        c, _ = _gpu(cam, bgr, raw)
        K = np.array([[517.3, 0, 318.6], [0, 516.5, 255.3], [0, 0, 1.0]])
        want = cv2.cvtColor(cv2.undistort(bgr, K, np.array(dist)), cv2.COLOR_BGR2RGB) / 255.
        assert np.array_equal(c, want)


def _reader(name, prefetch=2):
    cfg = fixture_cfg(name)
    cfg["scale"] = 1
    return ds.FrameReader(cfg, device="cuda", prefetch=prefetch)


@pytest.mark.parametrize("name", sorted(CAMS))
def test_reader_against_reference(name):
    items = list(_reader(name))
    g = REF[name]
    assert [i[0] for i in items] == list(range(len(g["color_paths"])))
    assert torch.equal(torch.stack([i[3] for i in items]), g["poses"])
    assert len(items) == len(g["frames"])
    for (_, c, d, _), want in zip(items, g["frames"]):
        assert c.is_cuda and c.dtype == torch.float64 and d.is_cuda and d.dtype == torch.float32
        check_frame(c, d, want, 1e-12)


def test_prefetch_iterations_and_thread_exit():
    a = list(_reader("tumrgbd", prefetch=0))
    r = _reader("tumrgbd", prefetch=2)
    for _ in range(2):                                                      # a reader can be iterated twice
        b = list(r)
        assert len(a) == len(b) and all(torch.equal(x[1], y[1]) and torch.equal(x[2], y[2]) for x, y in zip(a, b))
    before = threading.active_count()
    bad = _reader("replica", prefetch=2)
    bad.depth_paths = list(bad.depth_paths)
    bad.depth_paths[2] = os.path.join(OUT, "missing.png")
    with pytest.raises(RuntimeError, match="cannot read"):
        for _ in bad:
            pass
    it = iter(_reader("replica", prefetch=2))
    next(it)
    it.close()                                                              # abandoned mid-sequence
    assert threading.active_count() == before
    assert not [t for t in threading.enumerate() if t.name == "nsb-frame-decoder"]


def test_run_end_to_end(tmp_path, capsys, monkeypatch):
    import scene_util as su
    from gpu_util import make_renderer
    from slam_sequences import path_pose
    from nice_slam_b200 import run
    from nice_slam_b200.slam import ate_rmse
    sc = su.load_scenes()["room0"]
    renderer, c, dec = make_renderer(sc, su.make_grids(sc, "soft"), su.load_decoders("soft"), "cuda")
    data = tmp_path / "room"
    (data / "results").mkdir(parents=True)
    n = 12
    with open(data / "traj.txt", "w") as f:
        for k in range(n):
            pose = path_pose(sc, k)
            depth, _, color = renderer.render_img(c, dec, pose, "cuda", "color")
            bgr = (color.float().clamp(0, 1).cpu().numpy()[..., ::-1] * 255).round().astype(np.uint8)
            cv2.imwrite(str(data / "results" / ("frame%06d.jpg" % k)), bgr)
            cv2.imwrite(str(data / "results" / ("depth%06d.png" % k)), (depth.cpu().numpy() * 6553.5).round().astype(np.uint16))
            traj = pose.detach().double().cpu().numpy().copy()
            traj[:3, 1] *= -1
            traj[:3, 2] *= -1
            f.write(" ".join(repr(float(v)) for v in traj.reshape(-1)) + "\n")
    ck = convonet_checkpoints(str(tmp_path))
    cam = sc["cam"]
    bound = su.scene_bound(sc)
    # the defaults: the merged room0 config recorded with the golden data, where run.main looks for configs/nice_slam.yaml
    (tmp_path / "configs").mkdir()
    base = torch.load(os.path.join(OUT, "scenes.pt"), weights_only=False)["room0"]["cfg"]
    (tmp_path / "configs" / "nice_slam.yaml").write_text(yaml.safe_dump(base))
    monkeypatch.chdir(tmp_path)
    cfg_text = ("pretrained_decoders: {coarse: %s, middle_fine: %s}\n"
                "cam: {H: %d, W: %d, fx: %r, fy: %r, cx: %r, cy: %r, png_depth_scale: 6553.5, crop_edge: 0}\n"
                "mapping: {bound: %s, marching_cubes_bound: %s, iters_first: 30, iters: 5}\n"
                "tracking: {iters: 5}\nmeshing: {resolution: 64, eval_rec: false}\n"
                % (ck["coarse"], ck["middle_fine"], cam["H"], cam["W"], cam["fx"], cam["fy"], cam["cx"], cam["cy"],
                   json.dumps(bound.tolist()), json.dumps(bound.tolist())))
    cfg_path = tmp_path / "run.yaml"
    cfg_path.write_text(cfg_text)
    out = tmp_path / "out"
    res = run.main([str(cfg_path), "--input_folder", str(data), "--output", str(out), "--seed", "1"])
    printed = capsys.readouterr().out
    ck_last = torch.load(out / "ckpts" / ("%05d.tar" % (n - 1)), weights_only=False)
    assert set(ck_last) == {"c", "decoder_state_dict", "gt_c2w_list", "estimate_c2w_list", "keyframe_list", "selected_keyframes", "idx"}
    want_gt = torch.stack(ds.replica_files(str(data))[2])
    assert torch.equal(ck_last["gt_c2w_list"], want_gt)
    assert torch.equal(ck_last["estimate_c2w_list"][0], want_gt[0])
    assert (out / "mesh" / "final_mesh.ply").exists()
    ate = ate_rmse(ck_last["estimate_c2w_list"], ck_last["gt_c2w_list"])
    assert res["ate_rmse"] == ate and ("ATE RMSE %.6f" % ate) in printed
    assert json.loads((out / "run.json").read_text())["ate_rmse"] == ate
    # the same run through the API: the same seed reaches build_scene and FusedSLAM, so the keyframes agree and the trajectory stays
    # within the drift that two fused runs of a 12-frame room0 sequence show (test_gpu_slam's FUSED bars, blocks)
    from nice_slam_b200 import FusedSLAM, build_scene
    from nice_slam_b200.config import load_config
    from slam_sequences import pose_dev
    from test_gpu_slam import FUSED
    cfg = load_config(str(cfg_path), "configs/nice_slam.yaml")
    slam = build_scene(cfg, torch.device("cuda"), seed=1)
    direct = FusedSLAM(slam.renderer, slam.shared_c, slam.shared_decoders, cfg, seed=1)
    est, gt = direct.run(ds.FrameReader(cfg, str(data), "cuda", prefetch=0))
    assert torch.equal(gt, ck_last["gt_c2w_list"])
    assert [int(k) for k in ck_last["keyframe_list"]] == list(direct.store.idx)
    for k in range(n):
        t, r = pose_dev(est[k], ck_last["estimate_c2w_list"][k])
        assert t <= FUSED["blocks"][k][0] and r <= FUSED["blocks"][k][1], (k, t, r)
