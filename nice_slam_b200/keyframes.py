"""Device-resident keyframe store (SURVEY.md 8f-4).

The reference keeps every keyframe's colour / depth image on the HOST (`keyframe_dict.append({... 'color': gt_color.cpu(), 'depth':
gt_depth.cpu(), 'est_c2w': cur_c2w.clone()})`, src/Mapper.py:612-617), copies the full images of every window keyframe back to the device in
EVERY joint iteration (:439-440) and projects 1600 points into every keyframe with numpy on the host for the overlap selection (:196-218).
Here the images stay on the GPU (a 680 x 1200 RGB-D keyframe is 13 MB; a 2000-frame Replica run keeps ~40 of them), the overlap counts come
from one kernel launch (nsb_keyframe_overlap) and the per-frame pixel samples of a window from one gather (nsb_keyframe_gather).
The selection policy itself -- sort by percent_inside, numpy permutation, first k (:219-227) -- is the reference's, on the host.
"""
import ctypes as C

import numpy as np
import torch

from . import _lib
from .renderer import _VP, _stream


def pick_overlap(counts, n_points, k, rng=np.random):
    """The selection policy of Mapper.keyframe_selection_overlap (Mapper.py:218-227) on per-keyframe overlap counts of n_points points:
    keyframes with percent_inside > 0, sorted by it (stable, descending), permuted with numpy's RNG, first k."""
    lst = sorted([{"id": i, "percent_inside": c / n_points} for i, c in enumerate(counts)], key=lambda d: d["percent_inside"], reverse=True)
    sel = [d["id"] for d in lst if d["percent_inside"] > 0.00]
    return list(rng.permutation(np.array(sel))[:k])


class KeyframeStore:
    def __init__(self, H, W, fx, fy, cx, cy, device, capacity=16):
        self.H, self.W, self.fx, self.fy, self.cx, self.cy = int(H), int(W), float(fx), float(fy), float(cx), float(cy)
        self.dev = torch.device(device)
        self.idx = []                                   # frame index of every keyframe (keyframe_list, Mapper.py:611)
        self.est_c2w = []                               # [4,4] float32 host tensors (the reference's keyframe_dict[k]['est_c2w'])
        self.gt_c2w = []
        self._cap = 0
        self.depth = self.color = self.w2c = None
        self._grow(int(capacity))
        self._t = {}

    def __len__(self):
        return len(self.idx)

    def _grow(self, cap):
        depth = torch.empty(cap, self.H, self.W, dtype=torch.float32, device=self.dev)
        color = torch.empty(cap, self.H, self.W, 3, dtype=torch.float32, device=self.dev)
        w2c = torch.zeros(cap, 16, dtype=torch.float32, device=self.dev)
        if self._cap:
            depth[: self._cap].copy_(self.depth); color[: self._cap].copy_(self.color); w2c[: self._cap].copy_(self.w2c)
        self.depth, self.color, self.w2c, self._cap = depth, color, w2c, cap

    @staticmethod
    def _w2c(c2w):
        """numpy.linalg.inv of the float32 pose, exactly as Mapper.py:199-200 computes it."""
        m = torch.as_tensor(c2w).detach().float().cpu()
        if m.shape[0] == 3:
            m = torch.cat([m, torch.tensor([[0.0, 0.0, 0.0, 1.0]])], 0)
        return m, torch.from_numpy(np.linalg.inv(m.numpy())).float().reshape(16)

    def append(self, idx, gt_color, gt_depth, est_c2w, gt_c2w=None):
        """Mapper.py:611-617: register frame `idx` as a keyframe (images are copied into the device-resident store)."""
        k = len(self.idx)
        if k == self._cap:
            self._grow(2 * self._cap)
        self.depth[k].copy_(torch.as_tensor(gt_depth).to(self.dev, torch.float32))
        self.color[k].copy_(torch.as_tensor(gt_color).to(self.dev, torch.float32))
        m, inv = self._w2c(est_c2w)
        self.w2c[k].copy_(inv)
        self.idx.append(int(idx)); self.est_c2w.append(m); self.gt_c2w.append(None if gt_c2w is None else torch.as_tensor(gt_c2w).detach().cpu())
        return k

    def update_pose(self, k, est_c2w):
        """Pose write-back after bundle adjustment (Mapper.py:521-540)."""
        m, inv = self._w2c(est_c2w)
        self.est_c2w[k] = m
        self.w2c[k].copy_(inv)

    def overlap_counts(self, rays_o, rays_d, gt_depth, n_samples=16, edge=20, n_keyframes=None):
        """int32 [K] (device): points of the current frame's rays that project inside each of the first K keyframes (Mapper.py:186-216)."""
        K = len(self.idx) if n_keyframes is None else int(n_keyframes)
        counts = torch.zeros(max(K, 1), dtype=torch.int32, device=self.dev)
        t = self._t.get(n_samples)
        if t is None:
            t = self._t[n_samples] = torch.linspace(0.0, 1.0, steps=n_samples).to(self.dev)
        ro, rd, gd = (x.to(self.dev, torch.float32).contiguous() for x in (rays_o, rays_d, gt_depth))
        _lib.check(_lib.lib().nsb_keyframe_overlap(_VP(ro.data_ptr()), _VP(rd.data_ptr()), _VP(gd.data_ptr()), int(ro.shape[0]), _VP(t.data_ptr()), int(n_samples),
                                                   _VP(self.w2c.data_ptr()), K, self.H, self.W, self.fx, self.fy, self.cx, self.cy, int(edge),
                                                   _VP(counts.data_ptr()), _stream()), "nsb_keyframe_overlap")
        return counts[:K]

    def select_overlap(self, rays_o, rays_d, gt_depth, k, n_samples=16, n_keyframes=None, rng=np.random):
        """Mapper.keyframe_selection_overlap (src/Mapper.py:166-228) given the caller's pixel draw (get_samples, torch RNG): ids of up to k
        keyframes with overlap, sorted by percent_inside (stable, descending), permuted with numpy's RNG, as the reference does."""
        counts = self.overlap_counts(rays_o, rays_d, gt_depth, n_samples, n_keyframes=n_keyframes).cpu().numpy()
        return pick_overlap(counts, int(rays_o.shape[0]) * int(n_samples), k, rng)

    def stage(self, gt_color, gt_depth):
        """Copy a frame's images into the first free slot without registering it as a keyframe (the mapper's current frame, which it samples
        like a keyframe).  Returns the slot; the next append() overwrites it."""
        k = len(self.idx)
        if k == self._cap:
            self._grow(2 * self._cap)
        self.depth[k].copy_(torch.as_tensor(gt_depth).to(self.dev, torch.float32))
        self.color[k].copy_(torch.as_tensor(gt_color).to(self.dev, torch.float32))
        return k

    def sample(self, slots, pix_i, pix_j):
        """gt_depth [F,n] and gt_color [F,n,3] (float32, device) of pixels (pix_i, pix_j) ([F,n] integer tensors, the caller's get_sample_uv draws)
        of the keyframes `slots` ([F] ints) -- Mapper.py:437-462 without the host->device copy of the whole images."""
        F, n = pix_i.shape
        s = torch.as_tensor(slots, dtype=torch.int32).to(self.dev)
        pi = pix_i.to(self.dev, torch.int32).contiguous(); pj = pix_j.to(self.dev, torch.int32).contiguous()
        od = torch.empty(F, n, dtype=torch.float32, device=self.dev); oc = torch.empty(F, n, 3, dtype=torch.float32, device=self.dev)
        _lib.check(_lib.lib().nsb_keyframe_gather(_VP(self.depth.data_ptr()), _VP(self.color.data_ptr()), _VP(s.data_ptr()), _VP(pi.data_ptr()), _VP(pj.data_ptr()),
                                                  F, n, self.H, self.W, _VP(od.data_ptr()), _VP(oc.data_ptr()), _stream()), "nsb_keyframe_gather")
        return od, oc
