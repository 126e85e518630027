"""The per-frame camera optimisation of Tracker.run for NICE-SLAM (src/Tracker.py:188-253 around optimize_cam_in_batch, :71-128), assembled from
the library's pieces: the frame's RGB-D resident on the device -> per iteration ONE sampler launch (draws -> rays of the current camera tensor,
sensor samples, bbox pre-filter, compaction: nsb_track_samples) + the fused tracking iteration (steps.IterationContext, kind 'track', with d c2w)
+ ONE pose-step launch (best-pose bookkeeping, quad2rotation chain, Adam: nsb_track_pose_step).  Pixel draws come from torch's generator with
the very call select_uv makes (src/common.py:92-107), so the caller's CUDA random stream advances as under the reference.  Grids and decoders
are read only.  Host reads: the kept-ray count of every iteration (it sizes the render) and one small block at the end of the frame."""
import ctypes as C

import torch

from . import _lib
from .mapping import tensor_from_c2w
from .renderer import _VP, _stream, require_default_sampling
from .steps import IterationContext

BETAS, EPS = (0.9, 0.999), 1e-8                 # torch.optim.Adam defaults (Tracker.py:207-219)


class FusedTrackingLoop:
    def __init__(self, renderer, c, decoders, capacity, ignore_edge_W=20, ignore_edge_H=20, pixels=None, iters=10, lr=0.001,
                 seperate_LR=False, handle_dynamic=True, use_color_in_tracking=True, w_color_loss=0.5, const_speed_assumption=True,
                 generator=None):
        """c / decoders: the tracker's grids and decoders (read only); capacity: rays per iteration the buffers are sized for
        (cfg['tracking']['pixels']).  The other arguments are cfg['tracking'] settings under the reference's names; pixels defaults to
        capacity.  generator: the torch.Generator (on the grids' device) the pixel draws come from; None draws from torch's default one."""
        require_default_sampling(renderer, "FusedTrackingLoop")
        self.r, self.c, self.dec, self.capacity = renderer, c, decoders, int(capacity)
        self.pixels = self.capacity if pixels is None else int(pixels)
        if not 1 <= self.pixels <= self.capacity:
            raise RuntimeError("FusedTrackingLoop: pixels=%d does not fit capacity %d" % (self.pixels, self.capacity))
        self.ignore_edge_W, self.ignore_edge_H, self.iters, self.lr = int(ignore_edge_W), int(ignore_edge_H), int(iters), float(lr)
        self.seperate_LR, self.handle_dynamic, self.use_color = bool(seperate_LR), bool(handle_dynamic), bool(use_color_in_tracking)
        self.w_color_loss, self.const_speed_assumption = float(w_color_loss), bool(const_speed_assumption)
        self.generator = generator
        H, W = int(renderer.H), int(renderer.W)
        self.H0, self.H1, self.W0, self.W1 = self.ignore_edge_H, H - self.ignore_edge_H, self.ignore_edge_W, W - self.ignore_edge_W
        if self.iters < 1 or self.H0 < 0 or self.W0 < 0 or self.H1 <= self.H0 or self.W1 <= self.W0:
            raise RuntimeError("FusedTrackingLoop: empty pixel region or no iterations (H=%d, W=%d, ignore_edge_H=%d, ignore_edge_W=%d, iters=%d)"
                               % (H, W, self.ignore_edge_H, self.ignore_edge_W, self.iters))
        self.n_region = (self.H1 - self.H0) * (self.W1 - self.W0)
        self.dev = next(iter(c.values())).device
        dev, n, f32 = self.dev, self.capacity, torch.float32
        self.ctx = IterationContext(renderer, n, "color", dev, kind="track", host_staging=False)
        self.rays_o, self.rays_d, self.gt_depth, self.gt_color = self.ctx.device_views()      # the sampler writes the context's input block
        self.dirs = torch.empty(n, 3, dtype=f32, device=dev)
        self.kept_index = torch.empty(n, dtype=torch.int32, device=dev)
        self.count = torch.zeros(1, dtype=torch.int32, device=dev)
        self.depth = torch.empty(H, W, dtype=f32, device=dev)                     # the frame, resident for its iterations
        self.color = torch.empty(H, W, 3, dtype=torch.float64, device=dev)
        self.cam = torch.empty(7, dtype=f32, device=dev)                          # camera tensor being optimised
        self.adam_m = torch.empty(7, dtype=f32, device=dev)
        self.adam_v = torch.empty(7, dtype=f32, device=dev)
        self.candidate = torch.empty(7, dtype=f32, device=dev)
        self.c2w = torch.empty(4, 4, dtype=f32, device=dev)
        self.losses = torch.empty(self.iters, dtype=torch.float64, device=dev)   # per-iteration losses of the last frame
        self.best = torch.empty(2, dtype=torch.float64, device=dev)              # [running minimum, its iteration]
        self.best_iter = None
        self._bound = (C.c_double * 6)(*renderer._bounds()[0])

    def initial_pose(self, pre_c2w, prev_prev_c2w=None):
        """Start pose of a frame (Tracker.py:190-200): with const_speed_assumption and the pose before the previous one,
        (pre_c2w @ prev_prev_c2w^-1) @ pre_c2w in float32 on the device, else pre_c2w.  [4,4] float32 on the device."""
        pre = torch.as_tensor(pre_c2w).to(self.dev).float()
        if self.const_speed_assumption and prev_prev_c2w is not None:
            delta = pre @ torch.as_tensor(prev_prev_c2w).to(self.dev).float().inverse()
            return delta @ pre
        return pre

    def track_frame(self, gt_color, gt_depth, init_c2w, draws=None):
        """Optimise the camera of one frame for `iters` iterations and return the chosen pose, [4,4] float32 on the device (Tracker.py:248-253).
        gt_color [H,W,3], gt_depth [H,W]: the frame (copied to the device once).  init_c2w: the start pose ([4,4] or [3,4], converted by
        mapping.tensor_from_c2w on the host, as the reference's get_tensor_from_camera does) or a camera tensor [7] [qw,qx,qy,qz,tx,ty,tz].  draws: optional [iters, pixels] flat indices into the
        edge-cropped region; without it every iteration draws torch.randint(n_region, (pixels,)) on the frame's device (from self.generator),
        as select_uv does.
        Afterwards self.losses holds the per-iteration losses (device float64) and self.best_iter the chosen iteration."""
        L = _lib.lib()
        st = _stream()
        self.depth.copy_(torch.as_tensor(gt_depth).reshape(self.depth.shape), non_blocking=True)
        self.color.copy_(torch.as_tensor(gt_color).reshape(self.color.shape), non_blocking=True)
        init = torch.as_tensor(init_c2w)
        self.cam.copy_(init.reshape(7) if init.numel() == 7 else tensor_from_c2w(init))
        self.adam_m.zero_(); self.adam_v.zero_()
        self.best.copy_(torch.tensor([1e10, -1.0], dtype=torch.float64), non_blocking=True)     # current_min_loss, Tracker.py:224
        if draws is not None:
            draws = torch.as_tensor(draws).to(self.dev, torch.int64).contiguous()
            if tuple(draws.shape) != (self.iters, self.pixels):
                raise RuntimeError("FusedTrackingLoop: draws must be [iters, pixels] = [%d, %d], got %s" % (self.iters, self.pixels, tuple(draws.shape)))
            if int(draws.min()) < 0 or int(draws.max()) >= self.n_region:
                raise RuntimeError("FusedTrackingLoop: draws must lie in [0, %d)" % self.n_region)
        # seperate_LR = False: the candidate is the camera tensor AFTER the iteration's step -- optimizer.step() updates the very tensor that
        # Tracker.run clones afterwards.  seperate_LR = True: the tensor the loss was evaluated at -- run() rebuilds camera_tensor =
        # torch.cat([quad, T]) at the top of each iteration, and the step moves quad and T, not that copy (Tracker.py:222-247).
        post_step = 0 if self.seperate_LR else 1
        quat_lr = self.lr * 0.2 if self.seperate_LR else self.lr
        for it in range(self.iters):
            n = self.sample(draws[it] if draws is not None else torch.randint(self.n_region, (self.pixels,), device=self.dev,
                                                                                         generator=self.generator))
            if n == 0:
                raise RuntimeError("FusedTrackingLoop: the bbox pre-filter kept no ray in iteration %d (the reference fails in median())" % it)
            self.iterate(n)
            _lib.check(L.nsb_track_pose_step(_VP(self.cam.data_ptr()), _VP(self.ctx.loss.data_ptr()), _VP(self.ctx.d_c2w.data_ptr()),
                                             _VP(self.adam_m.data_ptr()), _VP(self.adam_v.data_ptr()), self.lr, quat_lr, BETAS[0], BETAS[1], EPS,
                                             it + 1, post_step, _VP(self.losses.data_ptr()), _VP(self.best.data_ptr()),
                                             _VP(self.candidate.data_ptr()), _VP(self.c2w.data_ptr()), st), "nsb_track_pose_step")
        best = self.best.cpu()
        self.best_iter = int(best[1])
        if self.best_iter < 0:
            raise RuntimeError("FusedTrackingLoop: no iteration of this frame had a finite loss below 1e10 (the reference has no candidate pose)")
        return self.c2w.clone()

    def sample(self, draws_row):
        """get_samples + the bbox pre-filter for one iteration under the current camera tensor self.cam (nsb_track_samples): the kept rays go
        to self.rays_o / rays_d / dirs / gt_depth / gt_color (and their draw slots to self.kept_index).  draws_row: int64 [pixels] on the
        device.  Returns the kept count (a 4-byte read)."""
        _lib.check(_lib.lib().nsb_track_samples(_VP(self.cam.data_ptr()), _VP(draws_row.data_ptr()), self.pixels, _VP(self.depth.data_ptr()),
                                                _VP(self.color.data_ptr()), self.depth.shape[0], self.depth.shape[1], self.H0, self.H1, self.W0, self.W1,
                                                float(self.r.fx), float(self.r.fy), float(self.r.cx), float(self.r.cy), self._bound,
                                                _VP(self.rays_o.data_ptr()), _VP(self.rays_d.data_ptr()), _VP(self.dirs.data_ptr()),
                                                _VP(self.gt_depth.data_ptr()), _VP(self.gt_color.data_ptr()), _VP(self.kept_index.data_ptr()),
                                                _VP(self.count.data_ptr()), _stream()), "nsb_track_samples")
        return int(self.count.item())

    def iterate(self, n):
        """The fused tracking iteration on the first n sampled rays: loss -> self.ctx.loss, d c2w -> self.ctx.d_c2w, ray gradients ->
        self.ctx.d_rays_o / d_rays_d."""
        self.ctx.run(self.c, self.dec, self.rays_o[:n], self.rays_d[:n], self.gt_depth[:n], self.gt_color[:n], w_color=self.w_color_loss,
                     handle_dynamic=self.handle_dynamic, use_color=self.use_color, dirs=self.dirs[:n])
