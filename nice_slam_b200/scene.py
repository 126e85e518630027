"""Scene setup: what NICE_SLAM.__init__ (src/NICE_SLAM.py:26-250) builds before a run, without the reference package.  build_scene
follows its order -- update_cam, the decoders (get_model's draws), load_bound, load_pretrain, grid_init on the CPU -- so that under one
seed the bound, the grids and the decoders are bit-identical to a reference run's initial state."""
from types import SimpleNamespace

import numpy as np
import torch

from .decoders import NICEDecoders
from .renderer import FusedRenderer


def update_cam(cfg):
    """NICE_SLAM.update_cam: (H, W, fx, fy, cx, cy) after crop_size (a resize) and crop_edge."""
    cam = cfg["cam"]
    H, W, fx, fy, cx, cy = cam["H"], cam["W"], cam["fx"], cam["fy"], cam["cx"], cam["cy"]
    if "crop_size" in cam:
        crop_size = cam["crop_size"]
        sx = crop_size[1] / W
        sy = crop_size[0] / H
        fx, fy, cx, cy = sx * fx, sy * fy, sx * cx, sy * cy
        W, H = crop_size[1], crop_size[0]
    if cam["crop_edge"] > 0:
        H -= cam["crop_edge"] * 2
        W -= cam["crop_edge"] * 2
        cx -= cam["crop_edge"]
        cy -= cam["crop_edge"]
    return H, W, fx, fy, cx, cy


def load_bound(cfg):
    """NICE_SLAM.load_bound: float64 [3,2], bound * scale with the upper end enlarged to a multiple of bound_divisible (through .int(),
    with the reference's float32 intermediate)."""
    bound = torch.from_numpy(np.array(cfg["mapping"]["bound"]) * cfg["scale"])
    bd = cfg["grid_len"]["bound_divisible"]
    bound[:, 1] = (((bound[:, 1] - bound[:, 0]) / bd).int() + 1) * bd + bound[:, 0]
    return bound


def _decoder_keys(ckpt, strip):
    return {key[strip:]: val for key, val in ckpt["model"].items() if "decoder" in key and "encoder" not in key}


def load_pretrain(cfg, decoders):
    """NICE_SLAM.load_pretrain: ConvONet checkpoints -> coarse ('decoder.' stripped), middle ('decoder.coarse_'), fine ('decoder.fine_')."""
    pre = cfg["pretrained_decoders"]
    if cfg["coarse"]:
        ckpt = torch.load(pre["coarse"], map_location="cpu", weights_only=False)
        decoders.coarse_decoder.load_state_dict(_decoder_keys(ckpt, 8))
    ckpt = torch.load(pre["middle_fine"], map_location="cpu", weights_only=False)
    middle, fine = {}, {}
    for key, val in ckpt["model"].items():
        if "decoder" in key and "encoder" not in key:
            if "coarse" in key:
                middle[key[8 + 7:]] = val
            elif "fine" in key:
                fine[key[8 + 5:]] = val
    decoders.middle_decoder.load_state_dict(middle)
    decoders.fine_decoder.load_state_dict(fine)


def grid_shapes(cfg, bound):
    """{key: [D, H, W]} of NICE_SLAM.grid_init (int() of xyz_len / grid_len, axes 0 and 2 swapped), in its order."""
    gl = cfg["grid_len"]
    xyz_len = bound[:, 1] - bound[:, 0]
    out = {}
    for key, length, enlarge in (("grid_coarse", gl["coarse"], cfg["model"]["coarse_bound_enlarge"]), ("grid_middle", gl["middle"], None),
                                 ("grid_fine", gl["fine"], None), ("grid_color", gl["color"], None)):
        if key == "grid_coarse" and not cfg["coarse"]:
            continue
        shape = list(map(int, ((xyz_len * enlarge if enlarge is not None else xyz_len) / length).tolist()))
        shape[0], shape[2] = shape[2], shape[0]
        out[key] = shape
    return out


def grid_init(cfg, bound):
    """NICE_SLAM.grid_init: torch.zeros(shape).normal_(0, std) on the CPU from the global generator, std 0.01 (fine: 1e-4)."""
    c_dim = cfg["model"]["c_dim"]
    return {key: torch.zeros([1, c_dim, *shape]).normal_(mean=0, std=0.0001 if key == "grid_fine" else 0.01)
            for key, shape in grid_shapes(cfg, bound).items()}


def check_model(cfg):
    m = cfg["model"]
    if m["c_dim"] != 32:
        raise RuntimeError("build_scene: model.c_dim %r is not supported; the fused kernels take c_dim 32" % (m["c_dim"],))
    if m.get("pos_embedding_method", "fourier") != "fourier":
        raise RuntimeError("build_scene: model.pos_embedding_method %r is not supported; the fused kernels take 'fourier'"
                           % (m["pos_embedding_method"],))


def build_scene(cfg, device, seed=None):
    """The initial state of a NICE-SLAM run on `device`.  seed: torch.manual_seed(seed) first (None: draw from the global generator as it
    stands).  Returns a namespace with cfg, nice, coarse, scale, H, W, fx, fy, cx, cy, bound (float64 [3,2], CPU), shared_c (the grids on
    the device, channels-last after the renderer's conversion), shared_decoders (NICEDecoders on the device) and renderer (FusedRenderer)
    -- the `slam` namespace FusedRenderer, FusedSLAM and FusedMesher read."""
    check_model(cfg)
    if seed is not None:
        torch.manual_seed(seed)
    slam = SimpleNamespace(cfg=cfg, nice=True, coarse=bool(cfg["coarse"]), occupancy=cfg["occupancy"], scale=cfg["scale"])
    slam.H, slam.W, slam.fx, slam.fy, slam.cx, slam.cy = update_cam(cfg)
    dec = NICEDecoders(coarse=slam.coarse, reference_draws=True)
    slam.bound = load_bound(cfg)
    load_pretrain(cfg, dec)
    c = grid_init(cfg, slam.bound)
    slam.shared_c = {k: v.to(device) for k, v in c.items()}
    slam.shared_decoders = dec.to(device)
    slam.renderer = FusedRenderer(cfg, SimpleNamespace(nice=True), slam)
    return slam
