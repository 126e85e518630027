"""The joint-iteration loop of Mapper.optimize_map for NICE-SLAM (src/Mapper.py:296-379 set-up, :389-520 loop, :521-540 pose write-back),
assembled from the library's pieces: frustum mask on the device (or every voxel) -> voxel slot tables -> per iteration one fused mapping
iteration (compact voxel gradients + the optimised decoders' gradients, steps.IterationContext) + fused Adam on the selected voxels (in place
on the shared grids), on the optimised decoders and -- with bundle adjustment -- on the camera tensors of the window (optim.FusedMapperAdam).
Pixel draws stay with the caller (the reference's get_sample_uv, torch RNG); with BA the rays are regenerated from the current camera
tensors every iteration (nsb_window_rays), exactly as Mapper.py:437-462 does through get_camera_from_tensor + get_samples.

FusedMapper runs a whole optimize_map call on top of it: keyframe selection and the window over a keyframes.KeyframeStore, the stage
schedule and learning rates, per iteration the reference's pixel draws + ONE sampler launch (nsb_map_samples: rays of every window row,
sensor samples, bbox pre-filter, compaction, row offsets) + the fused iteration and Adam steps, and the pose write-back."""
import ctypes as C

import numpy as np
import torch

from . import _lib
from .renderer import _VP, _stream, require_default_sampling

from ._lib import STAGE_DECODERS
from .masked import MaskedVoxels, frustum_voxel_mask
from .optim import FusedMapperAdam
from .steps import IterationContext

GRID_OF = {"middle": "grid_middle", "fine": "grid_fine", "color": "grid_color", "coarse": "grid_coarse"}
NSB_MAP_MAX_ROWS = 64           # window rows nsb_map_samples takes (include/nice_slam_b200.h)


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
        return self.iteration_sampled(stage, ro, rd, dirs, gd, gc, offs, lr)

    def iteration_sampled(self, stage, rays_o, rays_d, dirs, gt_depth, gt_color, frame_offsets, lr):
        """One joint iteration on a batch that is already sampled, pre-filtered and compacted (iteration_ba's, or nsb_map_samples'):
        the fused iteration, the voxel / decoder Adam steps and, with bundle adjustment, the per-row pose gradients (dirs, frame_offsets
        [F+1]) and the pose Adam step."""
        ctx = self._context(rays_o.shape[0], stage, rays_o.device)
        loss = ctx.run(self.c, self.dec, rays_o, rays_d, gt_depth, gt_color, w_color=self.w_color)
        if self.ba is None:
            self._optimiser_step(ctx, stage, lr)
            return loss
        ctx.finish_packed(dirs, frame_offsets)
        self._optimiser_step(ctx, stage, lr)
        b = self.ba
        b["step"] += 1
        _lib.check(_lib.lib().nsb_adam_poses(_VP(b["cams"].data_ptr()), _VP(b["cam_row"].data_ptr()), self.n_frames, _VP(ctx.d_frames.data_ptr()),
                                             _VP(b["m"].data_ptr()), _VP(b["v"].data_ptr()), _VP(b["d_cams"].data_ptr()), b["lr"] if stage == "color" else 0.0,
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


def map_stage(it, num_joint_iters, middle_iter_ratio, fine_iter_ratio, coarse_mapper=False):
    """The stage of joint iteration `it` (Mapper.py:403-410)."""
    if coarse_mapper:
        return "coarse"
    if it <= int(num_joint_iters * middle_iter_ratio):
        return "middle"
    if it <= int(num_joint_iters * fine_iter_ratio):
        return "fine"
    return "color"


def stage_lrs(stage_cfg, stage, lr_factor):
    """Learning rates of a stage (Mapper.py:412-416): cfg['mapping']['stage'][stage][<group>_lr] x lr_factor."""
    st = stage_cfg[stage]
    return {g: st[g + "_lr"] * lr_factor for g in ("decoders", "coarse", "middle", "fine", "color")}


def window_rows(selected, n_keyframes):
    """Rows of the window (Mapper.py:267-272): the selected keyframe ids, the last keyframe, then the current frame (-1).  Returns (rows,
    the row of the oldest keyframe -- not optimised under bundle adjustment -- or None for an empty store)."""
    rows = [int(k) for k in selected]
    fixed = None
    if n_keyframes > 0:
        rows.append(n_keyframes - 1)
        fixed = rows.index(min(rows))
    return rows + [-1], fixed


def random_select(l, k, rng=np.random):
    """common.random_select (src/common.py:66-71): k of 0..l-1 in numpy's random order."""
    return list(rng.permutation(np.array(range(l)))[:min(l, k)])


class FusedMapper:
    def __init__(self, renderer, c, decoders, store, pixels=1000, mapping_window_size=5, middle_iter_ratio=0.4, fine_iter_ratio=0.6, stage=None,
                 BA_cam_lr=0.001, w_color_loss=0.2, keyframe_selection_method="overlap", fix_fine=True, fix_color=False,
                 frustum_feature_selection=True, coarse_mapper=False, generator=None, rng=None):
        """renderer / c / decoders: the mapper's renderer, shared grids (updated in place) and decoders; store: the keyframes
        (keyframes.KeyframeStore, device-resident images).  The other arguments are cfg['mapping'] settings under the reference's names
        (`stage` is the per-stage learning-rate dict); the coarse mapper always selects keyframes globally (Mapper.py:78-80) and optimises
        grid_coarse only.  generator / rng: the torch.Generator (on the grids' device) of the pixel draws and the numpy RandomState of the
        keyframe selection; None takes torch's default generator and numpy's global state."""
        require_default_sampling(renderer, "FusedMapper")
        if stage is None:
            raise RuntimeError("FusedMapper: the per-stage learning rates (cfg['mapping']['stage']) are required")
        self.r, self.c, self.dec, self.store = renderer, c, decoders, store
        self.pixels, self.window_size = int(pixels), int(mapping_window_size)
        self.middle_iter_ratio, self.fine_iter_ratio = float(middle_iter_ratio), float(fine_iter_ratio)
        self.stage_cfg, self.BA_cam_lr, self.w_color_loss = stage, float(BA_cam_lr), float(w_color_loss)
        self.coarse_mapper = bool(coarse_mapper)
        self.generator, self.rng = generator, (np.random if rng is None else rng)
        self.keyframe_selection_method = "global" if self.coarse_mapper else keyframe_selection_method
        self.fix_fine, self.fix_color, self.frustum_feature_selection = bool(fix_fine), bool(fix_color), bool(frustum_feature_selection)
        self.keys = ("grid_coarse",) if self.coarse_mapper else ("grid_middle", "grid_fine", "grid_color")
        self.dev = next(iter(c.values())).device
        dev, n, f32 = self.dev, max(self.pixels, 1), torch.float32
        self.rays_o, self.rays_d, self.dirs, self.gt_color = (torch.empty(n, 3, dtype=f32, device=dev) for _ in range(4))
        self.gt_depth = torch.empty(n, dtype=f32, device=dev)
        self.count = torch.zeros(1, dtype=torch.int32, device=dev)
        self.offsets = torch.zeros(NSB_MAP_MAX_ROWS + 1, dtype=torch.int32, device=dev)
        self.draws = torch.empty(n, dtype=torch.int64, device=dev)
        self.losses = None
        self.window = self.fixed_row = self.pixs_per_image = self.stages = None
        self._contexts = {}                                       # one IterationContext per stage, kept across calls
        self._bound = (C.c_double * 6)(*renderer._bounds()[0])

    def select_window(self, slot_cur, cur_c2w):
        """Keyframe ids the window draws from (Mapper.py:256-265), before the last keyframe and the current frame are added."""
        K = len(self.store)
        if K == 0:
            return []
        if self.keyframe_selection_method == "global":
            return random_select(K - 1, self.window_size - 2, self.rng)
        if self.keyframe_selection_method != "overlap":
            raise RuntimeError("FusedMapper: unknown keyframe_selection_method %r" % self.keyframe_selection_method)
        H, W = self.store.H, self.store.W
        k = torch.randint(H * W, (100,), device=self.dev, generator=self.generator)       # keyframe_selection_overlap's get_samples(0, H, 0, W, 100, ...)
        pi, pj = (k % W).float(), (k // W).float()
        fixed = cur_c2w.to(self.dev, torch.float32)[:3, :4].reshape(1, 12).contiguous()
        cam_row = torch.full((1,), -1, dtype=torch.int32, device=self.dev)
        c2w, ro, rd = (torch.empty(m, dtype=torch.float32, device=self.dev) for m in ((12,), (100, 3), (100, 3)))
        frame = torch.zeros(100, dtype=torch.int32, device=self.dev)
        _lib.check(_lib.lib().nsb_window_rays(None, _VP(cam_row.data_ptr()), _VP(fixed.data_ptr()), 1, _VP(pi.data_ptr()), _VP(pj.data_ptr()),
                                              _VP(frame.data_ptr()), 100, float(self.r.fx), float(self.r.fy), float(self.r.cx), float(self.r.cy),
                                              _VP(c2w.data_ptr()), _VP(ro.data_ptr()), _VP(rd.data_ptr()), None, _stream()), "nsb_window_rays")
        gd, _ = self.store.sample([slot_cur], pi.view(1, -1), pj.view(1, -1))
        return self.store.select_overlap(ro, rd, gd.view(-1), self.window_size - 2, n_keyframes=K - 1, rng=self.rng)

    def map_frame(self, num_joint_iters, lr_factor, cur_gt_color, cur_gt_depth, cur_c2w, ba, draws=None, selection=None):
        """One Mapper.optimize_map call (src/Mapper.py:230-540) for the current frame (cur_gt_color [H,W,3], cur_gt_depth [H,W], estimated pose
        cur_c2w [4,4]) against the keyframes of the store.  ba: bundle adjustment (the reference's self.BA).  draws: optional
        [num_joint_iters, F, pixs_per_image] flat pixel indices (k = j * W + i) of every window row; without it each iteration calls
        torch.randint(H*W, (pixs_per_image,)) once per row in row order (from self.generator), as the reference's get_samples does.  selection: optional keyframe
        ids replacing the keyframe selection (and its random draws).  Afterwards self.losses holds the per-iteration losses (device float64),
        self.window the window's keyframe ids (-1: the current frame), self.fixed_row its fixed row and self.stages the stage schedule.
        Returns the optimised current pose [4,4] (device float32) with bundle adjustment, else None; the optimised keyframe poses are
        written back into the store."""
        if ba and self.coarse_mapper:
            raise RuntimeError("FusedMapper: the coarse mapper has no bundle adjustment (Mapper.py:602-603)")
        iters = int(num_joint_iters)
        store, dev = self.store, self.dev
        cur_c2w = torch.as_tensor(cur_c2w).to(dev, torch.float32)
        slot_cur = store.stage(cur_gt_color, cur_gt_depth)
        selected = list(selection) if selection is not None else self.select_window(slot_cur, cur_c2w)
        rows, fixed_row = window_rows(selected, len(store))
        F = len(rows)
        ppi = self.pixels // F
        if ppi == 0:
            raise RuntimeError("FusedMapper: %d pixels over a window of %d rows leaves no pixel per row" % (self.pixels, F))
        if F > NSB_MAP_MAX_ROWS:
            raise RuntimeError("FusedMapper: a window of %d rows exceeds the sampler's %d" % (F, NSB_MAP_MAX_ROWS))
        H, W = store.H, store.W
        if draws is not None:
            draws = torch.as_tensor(draws).to(dev, torch.int64).contiguous()
            if tuple(draws.shape) != (iters, F, ppi):
                raise RuntimeError("FusedMapper: draws must be [iters, F, pixs_per_image] = [%d, %d, %d], got %s" % (iters, F, ppi, tuple(draws.shape)))
            if int(draws.min()) < 0 or int(draws.max()) >= H * W:
                raise RuntimeError("FusedMapper: draws must lie in [0, %d)" % (H * W))
        self.window, self.fixed_row, self.pixs_per_image = rows, fixed_row, ppi
        self.stages = [map_stage(it, iters, self.middle_iter_ratio, self.fine_iter_ratio, self.coarse_mapper) for it in range(iters)]
        # the window's poses: keyframe estimates and the current estimate, rows in window order
        poses = torch.stack([store.est_c2w[k][:3, :4].float() if k >= 0 else cur_c2w[:3, :4].cpu() for k in rows])
        slots = torch.tensor([k if k >= 0 else slot_cur for k in rows], dtype=torch.int32).to(dev)
        loop = FusedMappingLoop(self.r, self.c, self.dec, cur_c2w, store.depth[slot_cur], keys=self.keys, w_color=self.w_color_loss,
                                capacity=self.pixels, fix_fine=self.fix_fine, fix_color=self.fix_color,
                                frustum_feature_selection=self.frustum_feature_selection)
        if ba:
            loop.enable_ba(poses, fixed_row, self.BA_cam_lr)
            cams, cam_row, fixed = loop.ba["cams"], loop.ba["cam_row"], loop.ba["fixed"]
        else:                                                      # every row keeps its pose
            cams, cam_row, fixed = None, torch.full((F,), -1, dtype=torch.int32, device=dev), poses.reshape(F, 12).contiguous().to(dev)
        loop._ctx = {s: ctx.rebind(loop.masked, loop.n_frames) for s, ctx in self._contexts.items()}
        lrs = {s: stage_lrs(self.stage_cfg, s, lr_factor) for s in set(self.stages)}
        self.losses = torch.empty(iters, dtype=torch.float64, device=dev)
        L, st = _lib.lib(), _stream()
        n_draws = F * ppi
        draw_buf = self.draws[:n_draws].view(F, ppi)
        for it, stage in enumerate(self.stages):
            if draws is not None:
                d = draws[it]
            else:
                for f in range(F):                                 # the reference's per-row get_samples draws, in row order
                    torch.randint(H * W, (ppi,), out=draw_buf[f], generator=self.generator)
                d = draw_buf
            _lib.check(L.nsb_map_samples(_VP(d.data_ptr()), F, ppi, _VP(slots.data_ptr()), _VP(store.depth.data_ptr()), _VP(store.color.data_ptr()),
                                         H, W, _VP(cams.data_ptr()) if cams is not None else None, _VP(cam_row.data_ptr()), _VP(fixed.data_ptr()),
                                         float(self.r.fx), float(self.r.fy), float(self.r.cx), float(self.r.cy), self._bound,
                                         _VP(self.rays_o.data_ptr()), _VP(self.rays_d.data_ptr()), _VP(self.dirs.data_ptr()),
                                         _VP(self.gt_depth.data_ptr()), _VP(self.gt_color.data_ptr()), _VP(self.offsets.data_ptr()),
                                         _VP(self.count.data_ptr()), st), "nsb_map_samples")
            n = int(self.count.item())
            if n == 0:
                raise RuntimeError("FusedMapper: the bbox pre-filter kept no ray in iteration %d (the reference fails in the render's "
                                   "max of an empty batch)" % it)
            loss = loop.iteration_sampled(stage, self.rays_o[:n], self.rays_d[:n], self.dirs[:n], self.gt_depth[:n], self.gt_color[:n],
                                          self.offsets[:F + 1], lrs[stage])
            self.losses[it:it + 1].copy_(loss)
        self._contexts.update(loop._ctx)
        if not ba:
            return None
        c2w = loop.window_c2w().cpu()                              # Mapper.py:521-540: write the optimised poses back
        bottom = torch.tensor([[0.0, 0.0, 0.0, 1.0]])
        new_cur = None
        for r, k in enumerate(rows):
            if r == fixed_row:
                continue
            pose = torch.cat([c2w[r], bottom], 0)
            if k >= 0:
                store.update_pose(k, pose)
            else:
                new_cur = pose.to(dev)
        return new_cur


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
