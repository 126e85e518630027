"""Frames of the sequence fixtures (tests/make_golden_slam_sequences.py): scene_util.make_frame images on a smooth ground-truth path."""
import numpy as np
import torch

import scene_util as su

FRAME_SEED0 = 100


def path_pose(scene, k):
    """Ground-truth c2w [4,4] float32 of frame k: a slow arc around the room0 bound centre (~2.3 cm and ~0.6 degrees per frame)."""
    b = su.scene_bound(scene)
    ctr = (b[:, 0] + b[:, 1]) / 2
    a = 0.01 * k
    ca, sa = np.cos(a), np.sin(a)
    c2w = torch.eye(4, dtype=torch.float64)
    c2w[:3, :3] = torch.tensor([[ca, 0.0, sa], [0.0, 1.0, 0.0], [-sa, 0.0, ca]], dtype=torch.float64)
    c2w[:3, 3] = ctr + torch.tensor([0.02 * k, 0.005 * k, -0.01 * k], dtype=torch.float64)
    return c2w.float()


def sequence(scene, n):
    """Frame-reader items (idx, gt_color [H,W,3] float64, gt_depth [H,W] float32, gt_c2w [4,4])."""
    out = []
    for k in range(n):
        depth, color = su.make_frame(scene, FRAME_SEED0 + k)
        out.append((k, color, depth, path_pose(scene, k)))
    return out


def pose_dev(a, b):
    """(translation in m, rotation angle in rad) between two c2w."""
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    t = float((a[:3, 3] - b[:3, 3]).norm())
    cos = float(((a[:3, :3].T @ b[:3, :3]).trace() - 1) / 2)
    return t, float(np.arccos(min(1.0, max(-1.0, cos))))


def per_frame(est_a, log_a, est_b, log_b, n):
    """Per frame k: pose deviation (t, r) of estimate_c2w_list[k] and the largest relative deviation of the per-iteration losses of the
    frame's tracking and mapping calls (logs in run_log's form, the same calls in the same order)."""
    out = {k: dict(zip(("t", "r"), pose_dev(est_a[k], est_b[k])), map_loss=0.0, track_loss=0.0) for k in range(n)}
    for a, b in zip(log_a, log_b):
        key = "track_loss" if b["kind"] == "track" else "map_loss"
        la, lb = torch.as_tensor(a["losses"]).double(), torch.as_tensor(b["losses"]).double()
        out[b["idx"]][key] = max(out[b["idx"]][key], float(((la - lb).abs() / lb.abs()).max()))
    return out


def rel_dev(a, b):
    """Largest |a - b| / (1 + |b|)."""
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return float(((a - b).abs() / (1 + b.abs())).max())
