"""The joint-iteration loop of Mapper.optimize_map for NICE-SLAM (src/Mapper.py:296-379 set-up, :389-520 loop, :521-540 pose write-back),
assembled from the library's pieces: frustum mask on the device (or every voxel) -> voxel slot tables -> per iteration one fused mapping
iteration (compact voxel gradients + the optimised decoders' gradients, steps.IterationContext) + fused Adam on the selected voxels (in place
on the shared grids), on the optimised decoders and -- with bundle adjustment -- on the camera tensors of the window (optim.FusedMapperAdam).
Pixel draws stay with the caller (the reference's get_sample_uv, torch RNG); with BA the rays are regenerated from the current camera
tensors every iteration (nsb_window_rays), exactly as Mapper.py:437-462 does through get_camera_from_tensor + get_samples."""
import ctypes as C

import torch

from . import _lib
from .renderer import _VP, _stream, require_default_sampling

from ._lib import STAGE_DECODERS
from .masked import MaskedVoxels, frustum_voxel_mask
from .optim import FusedMapperAdam
from .steps import IterationContext

GRID_OF = {"middle": "grid_middle", "fine": "grid_fine", "color": "grid_color", "coarse": "grid_coarse"}


class FusedMappingLoop:
    def __init__(self, renderer, c, decoders, c2w, depth, keys=("grid_middle", "grid_fine", "grid_color"), w_color=0.2, capacity=1024,
                 fix_fine=True, fix_color=False, frustum_feature_selection=True):
        """c: the shared grids dict (updated in place); c2w / depth: pose and sensor depth of the current frame (frustum selection);
        capacity: rays per iteration the buffers are sized for (cfg['mapping']['pixels']).  fix_fine / fix_color /
        frustum_feature_selection: the mapper's settings of the same names (Mapper.py:296-345): a decoder that is not fixed is optimised
        in the stages that evaluate it; without frustum feature selection every voxel of each grid is a parameter (c2w / depth unused).
        The colour-refinement pass of the last frame (Mapper.py:578-586) is fix_color=True, frustum_feature_selection=False."""
        require_default_sampling(renderer, "FusedMappingLoop")
        self.r, self.c, self.dec, self.w_color, self.capacity = renderer, c, decoders, w_color, int(capacity)
        self.fix_fine, self.fix_color, self.frustum_feature_selection = bool(fix_fine), bool(fix_color), bool(frustum_feature_selection)
        if frustum_feature_selection:
            self.masked = {k: MaskedVoxels(c[k], frustum_voxel_mask(renderer, c2w, k, c[k], depth)) for k in keys}
        else:                                                     # Mapper.py:302-312: the whole grid, through the same slot tables
            self.masked = {k: MaskedVoxels(c[k], torch.ones(c[k].shape[2:], dtype=torch.bool, device=c[k].device)) for k in keys}
        self.adam = FusedMapperAdam()
        self._ctx = {}
        self.n_frames = 0
        self.ba = None

    # ------------------------------------------------------------------------------------------ bundle adjustment
    def enable_ba(self, window_c2w, fixed_row, cam_lr, camera_tensors=None):
        """window_c2w: [F,3,4] (or [F,4,4]) starting poses of the window rows (selected keyframes ..., current frame), Mapper.py:253-262;
        fixed_row: the row that is NOT optimised (the oldest frame, Mapper.py:350) or None; cam_lr = cfg['mapping']['BA_cam_lr'].
        camera_tensors: [F - 1, 7] float32 [quaternion | translation] of the optimised rows in row order (get_tensor_from_camera); derived
        from the poses if omitted."""
        dev = next(iter(self.c.values())).device
        w = torch.as_tensor(window_c2w).float()[:, :3, :4].contiguous()
        F = w.shape[0]
        rows = [r for r in range(F) if r != fixed_row]
        if camera_tensors is None:
            camera_tensors = torch.stack([tensor_from_c2w(w[r]) for r in rows])
        cam_row = torch.full((F,), -1, dtype=torch.int32)
        for k, r in enumerate(rows):
            cam_row[r] = k
        self.ba = dict(cams=camera_tensors.detach().float().contiguous().clone().to(dev), cam_row=cam_row.to(dev), fixed=w.reshape(F, 12).to(dev),
                       lr=float(cam_lr), c2w=torch.empty(F, 12, dtype=torch.float32, device=dev), d_cams=torch.zeros(len(rows), 7, dtype=torch.float32, device=dev),
                       m=torch.zeros(len(rows), 7, dtype=torch.float32, device=dev), v=torch.zeros(len(rows), 7, dtype=torch.float32, device=dev), step=0)
        self.n_frames = F
        self._ctx = {}

    def window_c2w(self):
        """Current poses of the window rows, [F,3,4] (what Mapper.py:521-540 writes back into keyframe_dict / cur_c2w)."""
        b = self.ba
        F = self.n_frames
        dummy = torch.empty(0, dtype=torch.float32, device=b["cams"].device)
        _lib.check(_lib.lib().nsb_window_rays(_VP(b["cams"].data_ptr()), _VP(b["cam_row"].data_ptr()), _VP(b["fixed"].data_ptr()), F,
                                              None, None, None, 0, 1.0, 1.0, 0.0, 0.0, _VP(b["c2w"].data_ptr()), None, None, None, _stream()), "nsb_window_rays")
        return b["c2w"].view(F, 3, 4).clone()

    def window_rays(self, pix_i, pix_j, frame_of_ray):
        """rays_o, rays_d, dirs [N,3] of pixels (pix_i, pix_j) (float32 [N]) of window rows frame_of_ray (int32 [N]) under the CURRENT poses."""
        b, r = self.ba, self.r
        n = pix_i.shape[0]
        dev = pix_i.device
        ro, rd, dirs = (torch.empty(n, 3, dtype=torch.float32, device=dev) for _ in range(3))
        _lib.check(_lib.lib().nsb_window_rays(_VP(b["cams"].data_ptr()), _VP(b["cam_row"].data_ptr()), _VP(b["fixed"].data_ptr()), self.n_frames,
                                              _VP(pix_i.data_ptr()), _VP(pix_j.data_ptr()), _VP(frame_of_ray.data_ptr()), n,
                                              float(r.fx), float(r.fy), float(r.cx), float(r.cy), _VP(b["c2w"].data_ptr()),
                                              _VP(ro.data_ptr()), _VP(rd.data_ptr()), _VP(dirs.data_ptr()), _stream()), "nsb_window_rays")
        return ro, rd, dirs

    def iteration_ba(self, stage, pix_i, pix_j, gt_depth, gt_color, lr):
        """One joint iteration with bundle adjustment.  pix_i, pix_j, gt_depth: [F, n] (one row of draws per window row, as the
        reference's per-frame get_samples calls produce them); gt_color: [F, n, 3].  Rays come from the current camera tensors, the bbox
        pre-filter (Mapper.py:469-481) is applied, then the fused iteration, the voxel / decoder Adam steps and the pose Adam step (its
        learning rate is BA_cam_lr in stage 'color' and 0 otherwise, Mapper.py:417-424; the Adam state advances in every stage)."""
        L = _lib.lib()
        F, n = pix_i.shape
        dev = pix_i.device
        fid = torch.arange(F, dtype=torch.int32, device=dev).repeat_interleave(n)
        ro, rd, dirs = self.window_rays(pix_i.reshape(-1).float().contiguous(), pix_j.reshape(-1).float().contiguous(), fid)
        gd = gt_depth.reshape(-1).float().contiguous()
        keep8 = torch.empty(F * n, dtype=torch.uint8, device=dev)
        b6 = (C.c_double * 6)(*self.r._bounds()[0])
        _lib.check(L.nsb_bbox_prefilter(_VP(ro.data_ptr()), _VP(rd.data_ptr()), _VP(gd.data_ptr()), F * n, b6, _VP(keep8.data_ptr()), _stream()), "nsb_bbox_prefilter")
        keep = keep8.bool()
        offs = torch.zeros(F + 1, dtype=torch.int32, device=dev)
        offs[1:] = keep.view(F, n).sum(1).cumsum(0).int()
        ro, rd, dirs, gd = ro[keep].contiguous(), rd[keep].contiguous(), dirs[keep].contiguous(), gd[keep].contiguous()
        gc = gt_color.reshape(-1, 3).float()[keep].contiguous()
        ctx = self._context(ro.shape[0], stage, dev)
        loss = ctx.run(self.c, self.dec, ro, rd, gd, gc, w_color=self.w_color)
        ctx.finish_packed(dirs, offs)
        self._optimiser_step(ctx, stage, lr)
        b = self.ba
        b["step"] += 1
        _lib.check(L.nsb_adam_poses(_VP(b["cams"].data_ptr()), _VP(b["cam_row"].data_ptr()), F, _VP(ctx.d_frames.data_ptr()), _VP(b["m"].data_ptr()),
                                    _VP(b["v"].data_ptr()), _VP(b["d_cams"].data_ptr()), b["lr"] if stage == "color" else 0.0,
                                    self.adam.betas[0], self.adam.betas[1], self.adam.eps, b["step"], _stream()), "nsb_adam_poses")
        return loss

    def grad_decoders(self, stage):
        """The decoders whose parameters get a gradient at `stage`: those of parameter group 0 (the fine decoder unless fix_fine, the colour
        decoder unless fix_color, Mapper.py:336-341) that the stage evaluates (decoder.py:317-342); torch's Adam skips the others."""
        return tuple(lvl for lvl, fixed in (("fine", self.fix_fine), ("color", self.fix_color)) if not fixed and lvl in STAGE_DECODERS[stage])

    def _context(self, n, stage, device):
        """ONE context per stage, sized for a capacity: the ray count after the bbox pre-filter changes almost every iteration
        (Mapper.py:471-481) and must not allocate a fresh set of buffers each time.  The capacity grows geometrically if ever exceeded."""
        ctx = self._ctx.get(stage)
        if ctx is None or ctx.n < n:
            cap = max(n, self.capacity, 2 * ctx.n if ctx is not None else 0)
            grids = tuple(GRID_OF[l] for l in STAGE_DECODERS[stage] if GRID_OF[l] in self.masked)
            ctx = IterationContext(self.r, cap, stage, device, kind="map", grad_grids=grids,
                                   grad_decoders=self.grad_decoders(stage), masked=self.masked, host_staging=False,
                                   n_frames=self.n_frames)
            self._ctx[stage] = ctx
        return ctx

    def iteration(self, stage, rays_o, rays_d, gt_depth, gt_color, lr):
        """One joint iteration at `stage`; lr = dict(decoders=, middle=, fine=, color=) as cfg['mapping']['stage'][stage] x lr_factor
        (Mapper.py:412-416).  Returns the loss tensor (device, float64)."""
        ctx = self._context(rays_o.shape[0], stage, rays_o.device)
        loss = ctx.run(self.c, self.dec, rays_o, rays_d, gt_depth, gt_color, w_color=self.w_color)
        self._optimiser_step(ctx, stage, lr)
        return loss

    def _optimiser_step(self, ctx, stage, lr):
        """optimizer.step() (Mapper.py:504) for the parameters that received a gradient (Adam skips the others): the selected voxels of the
        stage's grids and the stage's optimised decoders (grad_decoders), all at the decoders_lr of the stage -- one launch
        (optim.FusedMapperAdam.step_all)."""
        vox = [(key, self.c[key], self.masked[key], ctx.d_grid[key], lr[key[5:]]) for key in ctx.grad_grids]
        dec = [(lvl, self.dec, ctx.d_flat[lvl], lr["decoders"]) for lvl in ctx.grad_decoders]
        self.adam.step_all(vox, dec, renderer=self.r)


def tensor_from_c2w(c2w):
    """get_tensor_from_camera (src/common.py:179-200): c2w [3,4] or [4,4] -> float32 [qw,qx,qy,qz,tx,ty,tz] (CPU tensor).  Host-side set-up
    arithmetic (the reference uses mathutils' Matrix.to_quaternion on the host): Shepperd's method in float64."""
    m = torch.as_tensor(c2w).detach().double().cpu()
    R, t = m[:3, :3], m[:3, 3]
    tr = float(R[0, 0] + R[1, 1] + R[2, 2])
    if tr > 0:
        s = (tr + 1.0) ** 0.5 * 2
        q = [0.25 * s, float(R[2, 1] - R[1, 2]) / s, float(R[0, 2] - R[2, 0]) / s, float(R[1, 0] - R[0, 1]) / s]
    elif R[0, 0] > R[1, 1] and R[0, 0] > R[2, 2]:
        s = float(1.0 + R[0, 0] - R[1, 1] - R[2, 2]) ** 0.5 * 2
        q = [float(R[2, 1] - R[1, 2]) / s, 0.25 * s, float(R[0, 1] + R[1, 0]) / s, float(R[0, 2] + R[2, 0]) / s]
    elif R[1, 1] > R[2, 2]:
        s = float(1.0 + R[1, 1] - R[0, 0] - R[2, 2]) ** 0.5 * 2
        q = [float(R[0, 2] - R[2, 0]) / s, float(R[0, 1] + R[1, 0]) / s, 0.25 * s, float(R[1, 2] + R[2, 1]) / s]
    else:
        s = float(1.0 + R[2, 2] - R[0, 0] - R[1, 1]) ** 0.5 * 2
        q = [float(R[1, 0] - R[0, 1]) / s, float(R[0, 2] + R[2, 0]) / s, float(R[1, 2] + R[2, 1]) / s, 0.25 * s]
    return torch.tensor(q + t.tolist(), dtype=torch.float32)
