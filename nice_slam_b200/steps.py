"""Fused optimisation iterations (no autograd graph, no per-call allocations).

`IterationContext` owns the device buffers of one (batch size, stage) configuration and enqueues a whole
Tracker.optimize_cam_in_batch-style or Mapper.optimize_map-style iteration -- batch depth maxima, render forward,
loss seeds, render backward -- with ONE C call (nsb_tracking_iteration / nsb_mapping_iteration).  The optimiser
step itself (Adam on the pose / masked voxels / colour decoder) stays in PyTorch, as in the reference.

`run_host()` is the end-to-end entry used by bench.py's `e2e` figure: inputs come from pinned host memory, the loss
and the ray gradients are read back to pinned host memory, both copies inside the call.
"""
import ctypes as C

import torch

from . import _lib
from ._lib import LEVELS, STAGE_DECODERS
from .renderer import _VP, _inputs, _linspaces, _stream, _Call, _require_cuda, acts_buffer, require_default_sampling

KERNEL_LAUNCHES_PER_ITERATION = 2       # render_fwd + render_bwd for batches <= 1024 rays: the forward reduces the batch depth maxima itself and
                                        # its last CTA computes the loss seeds, the backward's last CTA produces d c2w; larger batches add
                                        # batch_max + seeds launches, decoder gradients an unpack launch


def packed_layout(n_frames, grad_decoders, masked_counts):
    """Sections of the packed float32 gradient block of a mapping iteration: {name: (offset, numel)}, total floats.
    [loss,0,0,0 | 'frames': 12 per keyframe | 'dec_<level>': canonical flat decoder order | '<grid key>': [n_selected,32] compact]"""
    L = _lib.lib()
    up4 = lambda v: (v + 3) & ~3
    off, sect = 4, {}
    sect["frames"] = (off, 12 * n_frames); off += up4(12 * n_frames)
    for lvl in grad_decoders:
        nf = L.nsb_flat_decoder_floats(LEVELS.index(lvl))
        sect["dec_" + lvl] = (off, nf); off += up4(nf)
    for key, count in masked_counts:
        sect[key] = (off, 32 * count); off += 32 * count
    return sect, off


def capture_graph(body):
    """CUDA graph of one call of `body`, after two warm-up calls outside capture (lazy attribute setup, decoder packing)."""
    cur = torch.cuda.current_stream()
    side = torch.cuda.Stream()
    side.wait_stream(cur)
    with torch.cuda.stream(side):
        body(); body()
    cur.wait_stream(side)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        body()
    return g


def host_io_body(ctx, host_io, d_result, h_result, can_push, enqueue):
    """Graph body: enqueue(push) between the move of ctx's input block from pinned host memory and the move of d_result to the pinned block
    h_result (host_io: see IterationContext.build_graph).  push = "sm_push" and can_push: the launch that completes d_result stores it itself."""
    sm, push = host_io in ("sm", "sm_push"), host_io == "sm_push" and can_push

    def body():
        if sm:
            ctx.copy_in_sm()
        elif host_io:
            ctx.d_in.copy_(ctx.h_in, non_blocking=True)
        enqueue(push)
        if sm and not push:
            ctx.copy_out_sm(h_result, d_result)
        elif host_io and not sm:
            h_result.copy_(d_result, non_blocking=True)
    return body


class IterationContext:
    def __init__(self, renderer, n_rays, stage, device, kind="track", grad_grids=(), grad_decoders=(), coarse_mapper=False,
                 masked=None, n_frames=0, host_staging=True):
        """masked: {grid key: masked.MaskedVoxels} -- those grids get COMPACT [n_selected,32] gradients (Mapper.py:317-333) instead of
        dense ones; n_frames: keyframes of the bundle-adjustment window whose d c2w is wanted (pose_grad_frames)."""
        require_default_sampling(renderer, "IterationContext")
        L = _lib.lib()
        self.r, self.n, self.stage, self.kind = renderer, int(n_rays), stage, kind
        self.n_last = self.n                  # rays of the last run() (<= capacity n)
        self.dev = torch.device(device)
        self.levels = STAGE_DECODERS[stage]
        self.render_with_depth = not (kind == "map" and (stage == "coarse" or coarse_mapper))
        S = renderer.N_samples + (renderer.N_surface if (self.render_with_depth and stage != "coarse") else 0)
        self.S = S
        n, dev = self.n, self.dev
        f64, f32 = torch.float64, torch.float32
        self.depth = torch.empty(n, dtype=f64, device=dev)
        self.var = torch.empty(n, dtype=f64, device=dev)
        self.rgb = torch.empty(n, 3, dtype=f32, device=dev)
        self.z_vals = torch.empty(n, S, dtype=f64, device=dev)
        self.raw = torch.empty(n, S, 4, dtype=f32, device=dev)
        self.masks = torch.empty(n, S, 15, dtype=torch.int32, device=dev)
        self.g_depth = torch.empty(n, dtype=f64, device=dev)
        self.g_rgb = torch.empty(n, 3, dtype=f32, device=dev)
        # results that travel back to the host live in ONE block so that the end-to-end form needs a single D2H copy:
        #   [d_rays_o | d_rays_d] f32 (6n) | pad to 8 B | loss f64 | d c2w f64 [3,4]
        res_off = ((n * 6 * 4 + 7) // 8) * 8
        self.d_res = torch.zeros(res_off + 13 * 8, dtype=torch.uint8, device=dev)
        self.loss = self.d_res[res_off: res_off + 8].view(f64)
        self.depth_max = torch.zeros(2, dtype=f32, device=dev)
        self.ws = torch.zeros(L.nsb_iteration_workspace_bytes(n), dtype=torch.uint8, device=dev)     # zeroed once: holds the split counters
        # stand-alone scratch for the split-phase (sharded) forms, which call the pieces of an iteration one by one (dist.py)
        self.seeds_ws = torch.empty(max(L.nsb_tracking_seeds_workspace(n), 16), dtype=torch.uint8, device=dev)
        self.bwd_ws = torch.empty(L.nsb_backward_workspace_bytes(), dtype=torch.uint8, device=dev)
        self.split_ws = torch.zeros(max(L.nsb_split_workspace_bytes(n, S), 16), dtype=torch.uint8, device=dev)   # decoder-parallel CTAs (small batches)
        self.split_bytes = L.nsb_split_workspace_bytes(n, S)
        self.pose_counter = torch.zeros(1, dtype=torch.int32, device=dev)      # arrival counter of the fused pose gradient (self-resetting)
        self.d_out = self.d_res[: n * 24].view(f32)                      # [d_rays_o | d_rays_d]
        self.d_rays_o = self.d_out[: 3 * n].view(n, 3)
        self.d_rays_d = self.d_out[3 * n:].view(n, 3)
        self.d_c2w = self.d_res[res_off + 8:].view(f64).view(3, 4)
        # device-side inputs (run_host copies into these; run() can alias caller tensors instead)
        # ... and the per-iteration inputs in one block (a single H2D copy):  [rays_o | rays_d | gt_depth] f32 (7n) | pad | gt_color
        col_dt = f64 if kind == "track" else f32
        col_off = ((n * 7 * 4 + 7) // 8) * 8
        col_bytes = n * 3 * (8 if col_dt == f64 else 4)
        self.d_in = torch.zeros(col_off + col_bytes, dtype=torch.uint8, device=dev)
        self.d_in32 = self.d_in[: n * 28].view(f32)
        self.gt_color = self.d_in[col_off:].view(col_dt).view(n, 3)
        self.grad_grids = tuple(grad_grids)
        self.grad_decoders = tuple(grad_decoders)
        self.masked = dict(masked or {})
        self.n_frames = int(n_frames)
        # packed float32 gradient block = what a sharded mapping iteration all-reduces in ONE collective (SURVEY.md 8e):
        #   [loss, 0, 0, 0 | d c2w of the keyframes (12 each) | decoder grads (canonical flat order) | compact voxel grads]
        # every section starts on a 16-byte boundary (the voxel scatter uses 16-byte vector reductions)
        sect, off = packed_layout(self.n_frames, self.grad_decoders, [(k, self.masked[k].count) for k in self.grad_grids if k in self.masked])
        self.sections = sect
        self.packed = torch.zeros(off, dtype=f32, device=dev)
        self.d_frames = self.packed[4: 4 + 12 * self.n_frames].view(self.n_frames, 12)
        self.d_grid = {key: self.packed[sect[key][0]: sect[key][0] + sect[key][1]].view(-1, 32) for key in self.grad_grids if key in self.masked}
        self.d_flat = {lvl: self.packed[sect["dec_" + lvl][0]: sect["dec_" + lvl][0] + sect["dec_" + lvl][1]] for lvl in self.grad_decoders}
        # layer outputs of the fine / colour decoders, kept by the forward when their weight gradients are wanted: the backward then computes them
        # on the tensor cores (nsb_forward_outputs.acts / acts_levels); 640 B per sample point and decoder.  A set with the middle or coarse
        # decoder takes the FP32-FMA pass, which reads no acts, unless the library option wgrad_all is on (then every decoder's are kept).
        self.acts, self.acts_levels = acts_buffer(self.grad_decoders, self.levels, n, S, dev)
        self.buf = _lib.IterationBuffers(self.depth.data_ptr(), self.var.data_ptr(), self.rgb.data_ptr(), self.z_vals.data_ptr(),
                                         self.raw.data_ptr(), self.masks.data_ptr(), self.g_depth.data_ptr(), self.g_rgb.data_ptr(), self.loss.data_ptr(),
                                         self.depth_max.data_ptr(), self.ws.data_ptr(), self.ws.numel(), None, None,
                                         self.acts.data_ptr() if self.acts is not None else None, self.acts_levels)
        self.ev_bwd = None
        # pinned host staging for run_host(): [rays_o | rays_d | gt_depth] f32, gt_color, and the read-back block
        cuda = dev.type == "cuda" and host_staging      # (pin_memory is a synchronising cudaHostAlloc: skipped when run_host() is never used)
        self.h_in = torch.zeros(self.d_in.numel(), dtype=torch.uint8).pin_memory() if cuda else None
        self.h_in32 = self.h_in[: n * 28].view(f32) if cuda else None
        self.h_col = self.h_in[col_off:].view(col_dt).view(n, 3) if cuda else None
        self.h_res = torch.zeros(self.d_res.numel(), dtype=torch.uint8).pin_memory() if cuda else None
        self.h_out = self.h_res[: n * 24].view(f32) if cuda else None
        self.h_loss = self.h_res[res_off: res_off + 8].view(f64) if cuda else None
        self.h_pose = self.h_res[res_off + 8:].view(f64).view(3, 4) if cuda else None
        self.h_pose13 = torch.empty(13, dtype=f64).pin_memory() if cuda else None
        self.h2d_bytes = self.d_in.numel()
        self.d2h_bytes = self.d_res.numel()

    # ------------------------------------------------------------------------------------------
    def _grads(self, c):
        """nsb_backward_args with the output pointers of this context; (re)zeroes the accumulation buffers."""
        bw = _lib.BackwardArgs()
        bw.d_rays_o, bw.d_rays_d = self.d_rays_o.data_ptr(), self.d_rays_d.data_ptr()
        for lvl in self.levels:
            key, li = "grid_" + lvl, LEVELS.index(lvl)
            if key in self.grad_grids:
                if key in self.masked:                            # compact gradient of the frustum-selected voxels
                    if self.masked[key].count > 0:
                        bw.d_grid[li] = self.d_grid[key].data_ptr()
                        bw.slot_map[li] = self.masked[key].slot_map.data_ptr()
                else:                                             # dense gradient with the grid's own strides
                    g = c[key]
                    if key not in self.d_grid or self.d_grid[key].stride() != g.stride():
                        self.d_grid[key] = torch.empty_strided(g.size(), g.stride(), dtype=g.dtype, device=g.device)
                    bw.d_grid[li] = self.d_grid[key].data_ptr()
            if lvl in self.d_flat:
                bw.d_flat[li] = self.d_flat[lvl].data_ptr()
        self.zero_grads()
        return bw

    def render_structs(self, c, decoders):
        """(call, grids, RenderInputs, ForwardOutputs, BackwardArgs) of a render over the context's device inputs (device_views) and
        buffers, for the split-phase forms that call the render entry points one by one (dist.py).  Keep call and grids alive while the
        structs are used: they own the packed decoders the inputs point at.  (Re)zeroes the accumulation buffers."""
        ro, rd, gd, _ = self.device_views()
        call, grids, _ = self.r._call(c, decoders, self.stage, gd if self.render_with_depth else None, self.dev)
        t_u, t_s = _linspaces(self.r.N_samples, self.r.N_surface, self.dev)
        inp = _inputs(call, ro, rd, self.depth_max, t_u, t_s, [g.detach() for g in grids])
        acts = self.acts.data_ptr() if self.acts is not None else None
        split = self.split_ws.data_ptr() if self.split_bytes else None
        fo = _lib.ForwardOutputs(self.depth.data_ptr(), self.var.data_ptr(), self.rgb.data_ptr(), self.z_vals.data_ptr(), self.raw.data_ptr(), None,
                                 self.masks.data_ptr(), split, self.split_bytes, acts, self.acts_levels)
        bw = self._grads(c)
        bw.z_vals, bw.raw, bw.g_depth, bw.g_rgb, bw.masks = (self.z_vals.data_ptr(), self.raw.data_ptr(), self.g_depth.data_ptr(),
                                                              self.g_rgb.data_ptr(), self.masks.data_ptr())
        bw.split_workspace, bw.split_workspace_bytes, bw.acts, bw.acts_levels = split, self.split_bytes, acts, self.acts_levels
        return call, grids, inp, fo, bw

    def zero_grads(self):
        if self.packed.numel() > 4:
            self.packed.zero_()                                   # one memset: loss slot, keyframe poses, decoder and compact voxel grads
        for key, t in self.d_grid.items():
            if key not in self.masked:
                t.zero_()

    def finish_packed(self, dirs=None, frame_offsets=None):
        """After run(): loss -> packed[0] and, for a BA window, d c2w of every keyframe -> packed frames section."""
        self.packed[0:1].copy_(self.loss)
        if self.n_frames > 0:
            _lib.check(_lib.lib().nsb_pose_grad_frames(_VP(dirs.data_ptr()), _VP(self.d_rays_o.data_ptr()), _VP(self.d_rays_d.data_ptr()),
                                                       _VP(frame_offsets.data_ptr()), self.n_frames, _VP(self.d_frames.data_ptr()), _stream()),
                       "nsb_pose_grad_frames")
        return self.packed

    def run(self, c, decoders, rays_o, rays_d, gt_depth, gt_color, w_color=None, handle_dynamic=True, use_color=True, dirs=None, result_to_host=False):
        """Enqueue one iteration on the current stream (inputs already on the device).  Results stay on the device:
        self.loss, self.depth/var/rgb, self.d_rays_o/d, self.d_grid[key], self.d_flat[level]; with `dirs` (camera-frame ray directions
        [N,3]) also self.d_c2w, produced by the backward kernel itself.  result_to_host (needs dirs): the CTA that produces d c2w also stores
        the result block [d_rays_o | d_rays_d | loss | d c2w] into the pinned host block self.h_res (nsb_backward_args.result_dst)."""
        L = _lib.lib()
        n = self._check_inputs(rays_o, rays_d, gt_depth, gt_color)
        call, grids, _ = self.r._call(c, decoders, self.stage, gt_depth if self.render_with_depth else None, self.dev)
        t_u, t_s = _linspaces(self.r.N_samples, self.r.N_surface, self.dev)
        inp = _inputs(call, rays_o, rays_d, self.depth_max, t_u, t_s, [g.detach() for g in grids])
        bw = self._grads(c)
        if dirs is not None:
            _require_cuda(dirs, "dirs")
            bw.pose_dirs, bw.d_c2w, bw.pose_counter = dirs.data_ptr(), self.d_c2w.data_ptr(), self.pose_counter.data_ptr()
        if result_to_host:
            if dirs is None or self.h_res is None:
                raise RuntimeError("nice_slam_b200: result_to_host needs dirs and a context with host staging")
            bw.result_dst, bw.result_src, bw.result_bytes = self._mapped(self.h_res), self.d_res.data_ptr(), self.d_res.numel()
        if self.kind == "track":
            w = 0.5 if w_color is None else w_color
            _lib.check(L.nsb_tracking_iteration(C.byref(inp), C.byref(self.buf), _VP(gt_color.data_ptr()), w, int(handle_dynamic),
                                                int(use_color), C.byref(bw), _stream()), "nsb_tracking_iteration")
        else:
            w = 0.2 if w_color is None else w_color
            _lib.check(L.nsb_mapping_iteration(C.byref(inp), C.byref(self.buf), _VP(gt_depth.data_ptr()), _VP(gt_color.data_ptr()), w,
                                               C.byref(bw), _stream()), "nsb_mapping_iteration")
        return self.loss

    def _check_inputs(self, rays_o, rays_d, gt_depth, gt_color):
        """The kernels read these tensors through raw pointers: refuse anything that is not exactly what they expect (a stride-0 expand()
        view such as the reference's rays_o, a float64 depth, a batch larger than the context's buffers ...) instead of reading garbage.
        Batches SMALLER than the context's capacity are fine (every buffer is sized for self.n; the bbox pre-filter of the mapper makes the
        count vary per iteration, Mapper.py:471-481).  Returns the batch size."""
        n = int(rays_o.shape[0])
        if n < 1 or n > self.n:
            raise RuntimeError("nice_slam_b200: batch of %d rays does not fit this IterationContext (capacity %d)" % (n, self.n))
        col_dt = torch.float64 if self.kind == "track" else torch.float32
        for t, nm, shape, dt in ((rays_o, "rays_o", (n, 3), torch.float32), (rays_d, "rays_d", (n, 3), torch.float32),
                                 (gt_depth, "gt_depth", (n,), torch.float32), (gt_color, "gt_color", (n, 3), col_dt)):
            _require_cuda(t, nm)
            if tuple(t.shape) != shape or t.dtype != dt or not t.is_contiguous():
                raise RuntimeError("nice_slam_b200: %s must be a contiguous %s tensor of shape %s, got %s %s%s" %
                                   (nm, dt, shape, t.dtype, tuple(t.shape), "" if t.is_contiguous() else " (non-contiguous)"))
        self.n_last = n
        return n

    def time_backward(self, enable=True):
        """Profiling hook: have the library record CUDA events around the backward launch of every run()."""
        if enable:
            self.ev_bwd = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
            for e in self.ev_bwd:
                e.record()                                  # materialise the cudaEvent_t handle
            self.buf.event_bwd_begin, self.buf.event_bwd_end = self.ev_bwd[0].cuda_event, self.ev_bwd[1].cuda_event
        else:
            self.ev_bwd = None
            self.buf.event_bwd_begin = self.buf.event_bwd_end = None

    def pose_grad(self, dirs):
        """d c2w [3,4] (f64, device) of the last run() from the ray gradients (nsb_pose_grad)."""
        _lib.check(_lib.lib().nsb_pose_grad(_VP(dirs.data_ptr()), _VP(self.d_rays_o.data_ptr()), _VP(self.d_rays_d.data_ptr()), self.n_last,
                                            _VP(self.d_c2w.data_ptr()), _stream()), "nsb_pose_grad")
        return self.d_c2w

    # ------------------------------------------------------------------------------------------ CUDA graph
    def device_views(self):
        """(rays_o, rays_d, gt_depth, gt_color) views of the context-owned input block (fixed addresses for graphs)."""
        n = self.n
        return self.d_in32[: 3 * n].view(n, 3), self.d_in32[3 * n: 6 * n].view(n, 3), self.d_in32[6 * n:], self.gt_color

    def load_device_inputs(self, rays_o, rays_d, gt_depth, gt_color):
        ro, rd, gd, gc = self.device_views()
        for dst, src, nm in ((ro, rays_o, "rays_o"), (rd, rays_d, "rays_d"), (gd, gt_depth, "gt_depth"), (gc, gt_color, "gt_color")):
            if tuple(src.shape) != tuple(dst.shape):
                raise RuntimeError("nice_slam_b200: %s has shape %s, this IterationContext holds %s" % (nm, tuple(src.shape), tuple(dst.shape)))
            dst.copy_(src)                    # copy_ converts dtype / strides (a stride-0 expand() view is materialised here)

    def build_graph(self, c, decoders, dirs=None, host_io=False, **kw):
        """Capture one whole iteration into a CUDA graph (launch-bound small batches: one graph launch instead of
        4-6 kernel launches + Python glue).  Inputs are read from the context-owned block (load_device_inputs) or,
        with host_io, copied from the pinned staging block inside the graph; results stay in the context's buffers
        (and, with host_io, are copied to the pinned read-back block inside the graph).  host_io = True: copy-engine transfers
        (cudaMemcpyAsync nodes); host_io = "sm": both blocks moved by nsb_copy_block launches over the mapped host views; host_io = "sm_push": the
        input block as for "sm", the result block stored to pinned memory by the backward's last CTA (needs dirs; else as "sm").
        Re-capture after anything that changes pointers (grids re-created) or the decoders' packed image."""
        ro, rd, gd, gc = self.device_views()
        body = host_io_body(self, host_io, self.d_res, self.h_res, dirs is not None,
                            lambda push: self.run(c, decoders, ro, rd, gd, gc, dirs=dirs, result_to_host=push, **kw))
        return capture_graph(body)

    def _mapped(self, t):
        """Device view of a pinned host tensor (nsb_host_device_pointer); resolved once, outside any graph capture."""
        key = t.data_ptr()
        m = getattr(self, "_mapped_ptrs", None)
        if m is None:
            m = self._mapped_ptrs = {}
        if key not in m:
            p = _lib.lib().nsb_host_device_pointer(_VP(key))
            if not p:
                raise RuntimeError("nice_slam_b200: " + _lib.lib().nsb_last_error().decode())
            m[key] = p
        return m[key]

    def copy_in_sm(self):
        """h_in (pinned) -> d_in by nsb_copy_block on the current stream."""
        _lib.check(_lib.lib().nsb_copy_block(_VP(self.d_in.data_ptr()), _VP(self._mapped(self.h_in)), self.d_in.numel(), _stream()), "nsb_copy_block")

    def copy_out_sm(self, dst, src):
        """src (device) -> dst (pinned, of equal size) by nsb_copy_block on the current stream."""
        _lib.check(_lib.lib().nsb_copy_block(_VP(self._mapped(dst)), _VP(src.data_ptr()), src.numel() * src.element_size(), _stream()), "nsb_copy_block")

    def stage_host_inputs(self, rays_o, rays_d, gt_depth, gt_color):
        """Fill the pinned host block from CPU tensors (outside the timed region of a benchmark)."""
        n = self.n
        self.h_in32[: 3 * n].copy_(rays_o.reshape(-1))
        self.h_in32[3 * n: 6 * n].copy_(rays_d.reshape(-1))
        self.h_in32[6 * n:].copy_(gt_depth.reshape(-1))
        self.h_col.copy_(gt_color)

    def run_host(self, c, decoders, **kw):
        """End-to-end: pinned host inputs -> device -> iteration -> loss + ray gradients back to pinned host memory.
        Returns (loss float, d_rays [N,6] pinned host view).  Synchronises the current stream."""
        n = self.n
        self.d_in.copy_(self.h_in, non_blocking=True)
        ro, rd, gd = self.d_in32[: 3 * n].view(n, 3), self.d_in32[3 * n: 6 * n].view(n, 3), self.d_in32[6 * n:]
        self.run(c, decoders, ro, rd, gd, self.gt_color, **kw)
        self.h_res.copy_(self.d_res, non_blocking=True)
        torch.cuda.current_stream().synchronize()
        return float(self.h_loss[0]), self.h_out.view(2, n, 3)
