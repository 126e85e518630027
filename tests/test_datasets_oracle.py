"""CPU checks of running from a config: load_config's merge rules, build_scene's initial state against the reference's (golden), the
readers' file lists and poses, and oracle/frames.py against cv2 and torch."""
import os

import cv2
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from make_golden_datasets import CAMS, CONFIGS, OUT, SEED, check_frame, convonet_checkpoints, digest, fixture_cfg
from nice_slam_b200 import datasets as ds
from nice_slam_b200 import scene
from nice_slam_b200.config import load_config
from oracle import frames as fr

REF = torch.load(os.path.join(OUT, "reference.pt"), weights_only=False)
SCENES = torch.load(os.path.join(OUT, "scenes.pt"), weights_only=False)


def _w(path, text):
    with open(path, "w") as f:
        f.write(text)


def test_load_config_chain_and_merges(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    os.makedirs("configs/sub")
    _w("configs/default.yaml", "a: 1\nb: {x: 1, y: 2}\nc: {deep: {k: 1}}\nd: 5\n")
    _w("configs/base.yaml", "b: {y: 3}\nc: 7\n")                              # scalar over dict
    _w("configs/sub/mid.yaml", "inherit_from: configs/base.yaml\nd: {n: 1}\n")  # dict over scalar
    _w("configs/sub/top.yaml", "inherit_from: configs/sub/mid.yaml\nb: {z: 4}\n")
    cfg = load_config("configs/sub/top.yaml", "configs/default.yaml")
    assert cfg == {"a": 1, "b": {"x": 1, "y": 3, "z": 4}, "c": 7, "d": {"n": 1}, "inherit_from": "configs/sub/mid.yaml"}
    assert load_config("configs/base.yaml") == {"b": {"y": 3}, "c": 7}           # no default: nothing below


@pytest.fixture(scope="module")
def ckpts(tmp_path_factory):
    return convonet_checkpoints(str(tmp_path_factory.mktemp("pre")))


def _scene_cfg(name, ckpts):
    """The merged config the golden run used (recorded with it), with the test's ConvONet checkpoints."""
    cfg = dict(SCENES[name]["cfg"])
    cfg["pretrained_decoders"] = dict(ckpts)
    return cfg


@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_initial_state_bit_identical(name, ckpts):
    cfg = _scene_cfg(name, ckpts)
    g = SCENES[name]
    slam = scene.build_scene(cfg, "cpu", seed=SEED)
    assert torch.get_rng_state().numel() and digest(torch.get_rng_state()) == g["rng_after"]
    assert (slam.H, slam.W, slam.fx, slam.fy, slam.cx, slam.cy) == tuple(g["cam"])
    assert slam.bound.dtype == torch.float64 and torch.equal(slam.bound, g["bound"])
    assert {k: list(v.shape) for k, v in slam.shared_c.items()} == g["shapes"]
    assert {k: digest(v.contiguous()) for k, v in slam.shared_c.items()} == g["grids"]
    assert {k: digest(v) for k, v in slam.shared_decoders.state_dict().items()} == g["decoders"]


def test_pretrained_key_remapping(ckpts):
    st = torch.load(os.path.join(os.path.dirname(OUT), "decoders.pt"), weights_only=True)
    from nice_slam_b200.decoders import NICEDecoders
    dec = NICEDecoders()
    scene.load_pretrain(dict(coarse=True, pretrained_decoders=ckpts), dec)
    for lvl in ("coarse", "middle", "fine"):
        sd = getattr(dec, lvl + "_decoder").state_dict()
        assert set(sd) == set(st[lvl]) and all(torch.equal(sd[k], v) for k, v in st[lvl].items())


def test_model_settings_refused():
    for key, val in (("c_dim", 16), ("pos_embedding_method", "nerf")):
        m = dict(c_dim=32, pos_embedding_method="fourier")
        m[key] = val
        with pytest.raises(RuntimeError, match=key):
            scene.check_model(dict(model=m))


@pytest.mark.parametrize("name", sorted(CAMS))
def test_file_lists_and_poses(name):
    color, depth, poses = ds.FILES[name](os.path.join(OUT, name))
    g = REF[name]
    assert [os.path.relpath(p, OUT) for p in color] == g["color_paths"]
    assert [os.path.relpath(p, OUT) for p in depth][:len(color)] == g["depth_paths"][:len(color)]
    got = torch.stack(poses[:len(color)])
    assert got.dtype == torch.float32 and torch.equal(got, g["poses"])


def test_unsupported_dataset():
    with pytest.raises(RuntimeError, match="cofusion"):
        ds.FrameReader(dict(dataset="cofusion", scale=1, cam={}, data=dict(input_folder=".")))


@pytest.mark.parametrize("name", sorted(CAMS))
def test_oracle_against_reference_reader(name):
    """Every frame of every fixture: depth bit-exact, colour bit-exact or within 1e-12 per element."""
    cfg = fixture_cfg(name)
    color, depth, _ = ds.FILES[name](cfg["data"]["input_folder"])
    g = REF[name]
    assert len(g["frames"]) == len(color)
    for k, want in enumerate(g["frames"]):
        c, d = fr.prepare(*ds.decode(color[k], depth[k]), cfg["cam"])
        check_frame(torch.from_numpy(c), torch.from_numpy(d), want, 1e-12)


def test_tum_association_and_subsampling():
    """The TUM fixture drops one image to frame_rate 32 (0.0197 s after the first) and one to max_dt (no depth within 0.08 s)."""
    color, depth, poses = ds.tum_files(os.path.join(OUT, "tumrgbd"))
    stamps = [os.path.basename(p)[:-4] for p in color]
    assert stamps == ["1305031102.175304", "1305031102.243211", "1305031102.275326", "1305031102.311267", "1305031102.600000"]
    assert [os.path.basename(p)[:-4] for p in depth][-1] == "1305031102.604000"
    assert torch.equal(poses[0], torch.diag(torch.tensor([1.0, -1.0, -1.0, 1.0])))


TUM1 = (517.3, 516.5, 318.6, 255.3, [0.2624, -0.9531, -0.0054, 0.0026, 1.1633])
TUM2 = (520.9, 521.0, 325.1, 249.7, [0.2312, -0.7849, -0.0033, -0.0001, 0.9172])
OFF = (301.7, 299.3, 322.9, 238.1, [-0.9, 0.6, 0.02, -0.01, 0.4])           # strong barrel: the corners map off the image


@pytest.mark.parametrize("H,W,cam", [(480, 640, TUM1), (480, 640, TUM2), (480, 640, OFF), (37, 53, (40.3, 41.1, 26.2, 18.7, TUM1[4]))])
def test_oracle_undistort_matches_cv2(H, W, cam):
    fx, fy, cx, cy, dist = cam
    img = np.random.default_rng(H + W).integers(0, 256, (H, W, 3), dtype=np.uint8)
    K = np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1.0]])
    assert np.array_equal(fr.undistort(img, fx, fy, cx, cy, dist), cv2.undistort(img, K, np.array(dist)))


# includes integer downscales: 2x2 (where cv::resize computes INTER_AREA, the same 4-pixel average up to rounding), 3x3 and 2x3
@pytest.mark.parametrize("src,dst", [((968, 1296), (480, 640)), ((50, 70), (37, 53)), ((30, 40), (61, 77)), ((96, 128), (48, 64)),
                                     ((144, 192), (48, 64)), ((96, 192), (48, 64))])
def test_oracle_resize_matches_cv2(src, dst):
    img = np.random.default_rng(1).random(src + (3,))
    assert np.abs(fr.cv_resize_linear(img, *dst) - cv2.resize(img, dst[::-1])).max() < 1e-13


@pytest.mark.parametrize("src,dst", [((480, 640), (384, 512)), ((37, 53), (61, 77)), ((48, 64), (48, 30)), ((45, 80), (90, 160))])
def test_oracle_interpolate_matches_torch(src, dst):
    rng = np.random.default_rng(2)
    img = rng.random(src + (3,))
    want = F.interpolate(torch.from_numpy(img).permute(2, 0, 1)[None], dst, mode="bilinear", align_corners=True)[0].permute(1, 2, 0).numpy()
    assert np.abs(fr.interp_bilinear_ac(img, *dst) - want).max() < 1e-15
    d = rng.random(src).astype(np.float32)
    assert np.array_equal(fr.interp_nearest(d, *dst), F.interpolate(torch.from_numpy(d)[None, None], dst, mode="nearest")[0, 0].numpy())
