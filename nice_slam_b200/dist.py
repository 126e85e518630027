"""Ray-sharded data parallelism (one process per GPU, torch.distributed: NCCL on GPUs, gloo in the CPU tests).

Rays are independent given replicated (grids, decoders, pose); what is NOT per-ray in the reference and therefore
needs an exchange when a batch is sharded (SURVEY.md section 8e):
  * torch.max(gt_depth) / torch.max(gt_depth*1.2)        (src/utils/Renderer.py:109,144)  -> all-reduce MAX of 2 floats
  * tmp.median() of the tracking residuals               (src/Tracker.py:113)             -> all-gather of the residuals
  * the scalar loss and every gradient that is summed over rays (pose, voxel, decoder grads) -> all-reduce SUM
The exchange helpers below work on whatever device the tensors live on (so the gloo tests exercise the same code).
"""
import torch
import torch.distributed as dist


MAX_BATCH_DEPTHS = 8192          # NSB_MAX_BATCH_DEPTHS (include/nice_slam_b200.h)


def world():
    if dist.is_available() and dist.is_initialized():
        return dist.get_rank(), dist.get_world_size()
    return 0, 1


def shard_bounds(n, rank, world_size):
    """Contiguous [lo, hi) slice of an n-ray batch for `rank` (sizes differ by at most one)."""
    base, rem = divmod(n, world_size)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def exchange_depth_max(depth_max):
    """In place: element-wise MAX over ranks of [max(gt), max(gt*1.2)]."""
    if world()[1] > 1:
        dist.all_reduce(depth_max, op=dist.ReduceOp.MAX)
    return depth_max


def gather_residuals(res_local, counts=None):
    """All shards' tracking residuals, concatenated in rank order (equal shard sizes unless `counts` is given)."""
    rank, ws = world()
    if ws == 1:
        return res_local
    if counts is None:
        out = torch.empty(ws * res_local.numel(), dtype=res_local.dtype, device=res_local.device)
        dist.all_gather_into_tensor(out, res_local.contiguous())
        return out
    parts = [torch.empty(c, dtype=res_local.dtype, device=res_local.device) for c in counts]
    dist.all_gather(parts, res_local.contiguous())
    return torch.cat(parts)


def reduce_sum(packed):
    """In place SUM all-reduce of a packed gradient buffer ([loss | pose grads | decoder grads | voxel grads])."""
    if world()[1] > 1:
        dist.all_reduce(packed, op=dist.ReduceOp.SUM)
    return packed


class PeerExchange:
    """NVLink peer-memory exchange buffers for the *_peers kernels (include/nice_slam_b200.h): one symmetric buffer per rank, mapped on
    every rank through torch's symmetric-memory allocator (the plumbing); the exchanges themselves happen inside our kernels.
    `PeerExchange.create` returns None when symmetric memory is not available (single process, CPU, unsupported fabric) -- the callers
    then use the NCCL collectives."""

    def __init__(self, buf, handle, counters, max_rays):
        from . import _lib
        self.buf, self.handle, self.counters, self.max_rays = buf, handle, counters, max_rays
        rank, ws = world()
        self.struct = _lib.Peers()
        self.struct.rank, self.struct.world, self.struct.max_rays = rank, ws, max_rays
        ptrs = list(handle.buffer_ptrs)
        for r in range(ws):
            self.struct.buffer[r] = ptrs[r]
        self.struct.counters = counters.data_ptr()

    @staticmethod
    def create(max_rays, device):
        rank, ws = world()
        if ws < 2 or ws > 8 or torch.device(device).type != "cuda":
            return None
        ok = 1.0
        px = None
        try:
            import torch.distributed._symmetric_memory as symm
            from . import _lib
            nbytes = _lib.lib().nsb_peer_buffer_bytes(max_rays)
            buf = symm.empty(nbytes, dtype=torch.uint8, device=device)
            buf.zero_()
            handle = symm.rendezvous(buf, dist.group.WORLD)
            counters = torch.zeros(4, dtype=torch.int64, device=device)
            px = PeerExchange(buf, handle, counters, max_rays)
            torch.cuda.synchronize()
        except Exception:                                     # noqa: BLE001 -- any failure means "no peer memory here"
            ok = 0.0
        flag = torch.tensor([ok], device=device)
        dist.all_reduce(flag, op=dist.ReduceOp.MIN)           # all ranks take the same path (also a barrier after the zero fill)
        return px if flag.item() > 0.5 else None


class ShardedTrackingIteration:
    """One tracking iteration on this rank's shard of a global ray batch (split-phase: the exchanges sit between the
    kernels).  With world_size == 1 it degenerates to the same kernels without collectives.

    prepare() builds every ctypes structure once (pointers are fixed: the context's own input block); enqueue() then
    only issues the kernels and the three collectives, so it can be replayed from a CUDA graph (NCCL collectives are
    graph-capturable) -- build_graph() returns None if capture is not possible and the caller falls back to enqueue()."""

    def __init__(self, ctx, exchange="auto"):
        """exchange: 'auto' = in-kernel exchanges over NVLink peer memory when available, else NCCL; 'nccl' = NCCL collectives."""
        from .renderer import require_default_sampling
        require_default_sampling(ctx.r, "ShardedTrackingIteration")
        self.ctx = ctx                      # steps.IterationContext(kind='track')
        dev = ctx.dev
        self.res = torch.empty(ctx.n, dtype=torch.float64, device=dev)
        self.allres = torch.empty(ctx.n * world()[1], dtype=torch.float64, device=dev)
        self.packed = torch.zeros(13, dtype=torch.float64, device=dev)      # [loss | d_c2w(12)]
        self.peers = PeerExchange.create(ctx.n, dev) if exchange == "auto" else None
        self._p = None
        # every rank's shard must have the same number of rays: the pooled median indexes the gathered residuals as [world][n] and
        # all_gather_into_tensor needs equal sizes (pad the global batch to a multiple of the world size, or pass `counts` to gather_residuals)
        if world()[1] > 1:
            nn = torch.tensor([ctx.n, -ctx.n], dtype=torch.int64, device=dev)
            dist.all_reduce(nn, op=dist.ReduceOp.MAX)
            if int(nn[0]) != -int(nn[1]):
                raise RuntimeError("nice_slam_b200: ShardedTrackingIteration needs equal shard sizes on all ranks (got %d here, max %d, min %d)"
                                   % (ctx.n, int(nn[0]), -int(nn[1])))
        self.fused = self.peers is not None and ctx.n <= 512          # whole iteration in two launches (exchanges inside the render kernels)

    def prepare(self, c, decoders, dirs, w_color=0.5, handle_dynamic=True, use_color=True, global_gt_depth=None):
        """global_gt_depth: the sensor depths of the WHOLE batch (a ray-sharded tracker splits a pixel list every rank knows: same frame, same
        draws).  The batch depth maxima (Renderer.py:109,144) are then reduced locally over the full list (one tiny launch) and the iteration keeps
        only the two exchanges that sit at kernel tails (median pool, [loss | d c2w] sum); without it every forward CTA first waits for all ranks'
        shard maxima -- which exposes the launch skew between the ranks' independent graph replays."""
        from . import _lib
        from .renderer import _inputs, _linspaces
        x = self.ctx
        ro, rd, gd, gc = x.device_views()
        call, grids, _ = x.r._call(c, decoders, x.stage, gd, x.dev)
        t_u, t_s = _linspaces(x.r.N_samples, x.r.N_surface, x.dev)
        inp = _inputs(call, ro, rd, x.depth_max, t_u, t_s, [g.detach() for g in grids])
        fo = _lib.ForwardOutputs(x.depth.data_ptr(), x.var.data_ptr(), x.rgb.data_ptr(), x.z_vals.data_ptr(), x.raw.data_ptr(), None,
                                 x.masks.data_ptr(), x.split_ws.data_ptr() if x.split_bytes else None, x.split_bytes,
                                 x.acts.data_ptr() if x.acts is not None else None)
        bw = x._grads(c)
        bw.acts = x.acts.data_ptr() if x.acts is not None else None
        if x.split_bytes:
            bw.split_workspace, bw.split_workspace_bytes = x.split_ws.data_ptr(), x.split_bytes
        bw.z_vals, bw.raw, bw.g_depth, bw.g_rgb, bw.masks = (x.z_vals.data_ptr(), x.raw.data_ptr(), x.g_depth.data_ptr(),
                                                              x.g_rgb.data_ptr(), x.masks.data_ptr())
        self._p = dict(call=call, grids=grids, lin=(t_u, t_s), inp=inp, fo=fo, bw=bw, dirs=dirs, gd=gd, gc=gc,
                       w_color=w_color, hd=int(handle_dynamic), uc=int(use_color), ggd=global_gt_depth)

    def enqueue(self, out13_ptr=None):
        """out13_ptr (fused two-launch form only): device-visible address that receives [loss | d c2w] instead of self.packed -- e.g. the mapped
        view of a pinned host block, so that the summing CTA's 13 stores are the read-back."""
        import ctypes as C
        from . import _lib
        from .renderer import _VP, _stream
        L = _lib.lib()
        x, p = self.ctx, self._p
        n = x.n
        st = _stream()
        if self.peers is not None and self.fused:
            # TWO launches, no collective: depth maxima + median pool are exchanged inside the forward launch, [loss | d c2w] inside the backward's
            bw = p["bw"]
            bw.pose_dirs, bw.d_c2w, bw.pose_counter = p["dirs"].data_ptr(), x.d_c2w.data_ptr(), x.pose_counter.data_ptr()
            inp = p["inp"]
            inp.depth_max = None                                       # shard maxima reduced + exchanged inside the forward kernel ...
            if p["ggd"] is not None:                                   # ... or, the full batch's depths known locally: reduced there, no exchange
                if p["ggd"].numel() <= MAX_BATCH_DEPTHS:
                    inp.gt_depth_batch, inp.n_batch = p["ggd"].data_ptr(), p["ggd"].numel()
                else:
                    _lib.check(L.nsb_batch_max_depth(_VP(p["ggd"].data_ptr()), p["ggd"].numel(), _VP(x.depth_max.data_ptr()), st), "nsb_batch_max_depth")
                    inp.depth_max = x.depth_max.data_ptr()
            _lib.check(L.nsb_tracking_iteration_peers(C.byref(inp), C.byref(x.buf), _VP(p["gc"].data_ptr()), p["w_color"], p["hd"], p["uc"], C.byref(bw),
                                                      C.byref(self.peers.struct), _VP(out13_ptr or self.packed.data_ptr()), st), "nsb_tracking_iteration_peers")
            return self.packed
        if self.peers is not None:
            # five kernels, no collective launch: the three exchanges happen inside batch_max / seeds / pose_grad over peer memory
            px = C.byref(self.peers.struct)
            _lib.check(L.nsb_batch_max_depth_peers(_VP(p["gd"].data_ptr()), n, _VP(x.depth_max.data_ptr()), px, st), "nsb_batch_max_depth_peers")
            _lib.check(L.nsb_render_forward(C.byref(p["inp"]), C.byref(p["fo"]), st), "nsb_render_forward")
            _lib.check(L.nsb_tracking_seeds_peers(_VP(x.depth.data_ptr()), _VP(x.var.data_ptr()), _VP(x.rgb.data_ptr()), _VP(p["gd"].data_ptr()),
                                                  _VP(p["gc"].data_ptr()), n, p["w_color"], p["hd"], p["uc"], px,
                                                  _VP(x.g_depth.data_ptr()), _VP(x.g_rgb.data_ptr()), _VP(x.loss.data_ptr()),
                                                  _VP(x.seeds_ws.data_ptr()), L.nsb_tracking_seeds_workspace(n), st), "nsb_tracking_seeds_peers")
            _lib.check(L.nsb_render_backward(C.byref(p["inp"]), C.byref(p["bw"]), st), "nsb_render_backward")
            _lib.check(L.nsb_pose_grad_peers(_VP(p["dirs"].data_ptr()), _VP(x.d_rays_o.data_ptr()), _VP(x.d_rays_d.data_ptr()), n,
                                             _VP(x.loss.data_ptr()), _VP(self.packed.data_ptr()), px, st), "nsb_pose_grad_peers")
            return self.packed
        _lib.check(L.nsb_batch_max_depth(_VP(p["gd"].data_ptr()), n, _VP(x.depth_max.data_ptr()), st), "nsb_batch_max_depth")
        exchange_depth_max(x.depth_max)
        _lib.check(L.nsb_render_forward(C.byref(p["inp"]), C.byref(p["fo"]), st), "nsb_render_forward")
        pool, n_pool = None, 0
        if p["hd"] and world()[1] > 1:
            _lib.check(L.nsb_tracking_residuals(_VP(x.depth.data_ptr()), _VP(x.var.data_ptr()), _VP(p["gd"].data_ptr()), n,
                                                _VP(self.res.data_ptr()), st), "nsb_tracking_residuals")
            dist.all_gather_into_tensor(self.allres, self.res)
            pool, n_pool = _VP(self.allres.data_ptr()), self.allres.numel()
        _lib.check(L.nsb_tracking_seeds(_VP(x.depth.data_ptr()), _VP(x.var.data_ptr()), _VP(x.rgb.data_ptr()), _VP(p["gd"].data_ptr()),
                                        _VP(p["gc"].data_ptr()), n, p["w_color"], p["hd"], p["uc"], pool, n_pool,
                                        _VP(x.g_depth.data_ptr()), _VP(x.g_rgb.data_ptr()), _VP(self.packed.data_ptr()),
                                        _VP(x.seeds_ws.data_ptr()), L.nsb_tracking_seeds_workspace(n), st), "nsb_tracking_seeds")
        _lib.check(L.nsb_render_backward(C.byref(p["inp"]), C.byref(p["bw"]), st), "nsb_render_backward")
        _lib.check(L.nsb_pose_grad(_VP(p["dirs"].data_ptr()), _VP(x.d_rays_o.data_ptr()), _VP(x.d_rays_d.data_ptr()), n,
                                   _VP(self.packed.data_ptr() + 8), st), "nsb_pose_grad")
        reduce_sum(self.packed)             # [global loss | global d_c2w]  (the seeds kernel wrote the local loss into packed[0])
        return self.packed

    def build_graph(self, host_io=False):
        """CUDA graph of enqueue() (and, with host_io, of the pinned-host copies around it); None if capture fails."""
        x = self.ctx

        sm = host_io in ("sm", "sm_push")

        def body():
            if sm:                                                 # the blocks moved by nsb_copy_block launches over the mapped host views
                x.copy_in_sm()
            elif host_io:
                x.d_in.copy_(x.h_in, non_blocking=True)
            push = host_io == "sm_push" and self.peers is not None and self.fused       # the summing CTA stores [loss | d c2w] to pinned memory itself
            self.enqueue(out13_ptr=x._mapped(x.h_pose13) if push else None)
            if sm and not push:
                x.copy_out_sm(x.h_pose13, self.packed)
            elif host_io and not sm:
                x.h_pose13.copy_(self.packed, non_blocking=True)
        try:
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
        except Exception:
            torch.cuda.synchronize()
            return None

    def run(self, c, decoders, rays_o, rays_d, dirs, gt_depth, gt_color, w_color=0.5, handle_dynamic=True, use_color=True):
        """Convenience: copy the shard into the context's input block, prepare and enqueue once."""
        self.ctx.load_device_inputs(rays_o, rays_d, gt_depth, gt_color)
        self.prepare(c, decoders, dirs, w_color, handle_dynamic, use_color)
        return self.enqueue()


class ShardedMappingIteration:
    """One Mapper.optimize_map joint iteration (src/Mapper.py:482-503) on this rank's shard of the window's ray batch.
    Replicated: grids, decoders, poses.  Exchanges: MAX of the batch depth maxima before sampling (Renderer.py:109,144) and ONE
    SUM all-reduce of the context's packed float32 block [loss | keyframe pose grads | decoder grads | compact voxel grads]
    (steps.IterationContext.packed) -- after it every rank holds the full-batch gradients and takes the identical optimiser step.
    Split-phase like ShardedTrackingIteration; graph-capturable."""

    def __init__(self, ctx):
        assert ctx.kind == "map"
        from .renderer import require_default_sampling
        require_default_sampling(ctx.r, "ShardedMappingIteration")
        self.ctx = ctx
        self._p = None

    def prepare(self, c, decoders, dirs=None, frame_offsets=None, w_color=0.2, global_gt_depth=None):
        """global_gt_depth: the sensor depths of the WHOLE batch (every rank samples the same window pixels from replicated keyframes, so it
        has them): the batch depth maxima (Renderer.py:109,144) are then computed locally on the full batch before sharding and the iteration
        needs exactly ONE collective, the all-reduce of the packed gradient block (SURVEY.md 8e).  None: MAX all-reduce of the shard maxima."""
        from . import _lib
        from .renderer import _inputs, _linspaces
        x = self.ctx
        ro, rd, gd, gc = x.device_views()
        call, grids, _ = x.r._call(c, decoders, x.stage, gd if x.render_with_depth else None, x.dev)
        t_u, t_s = _linspaces(x.r.N_samples, x.r.N_surface, x.dev)
        inp = _inputs(call, ro, rd, x.depth_max, t_u, t_s, [g.detach() for g in grids])
        fo = _lib.ForwardOutputs(x.depth.data_ptr(), x.var.data_ptr(), x.rgb.data_ptr(), x.z_vals.data_ptr(), x.raw.data_ptr(), None,
                                 x.masks.data_ptr(), x.split_ws.data_ptr() if x.split_bytes else None, x.split_bytes,
                                 x.acts.data_ptr() if x.acts is not None else None)
        bw = x._grads(c)
        bw.acts = x.acts.data_ptr() if x.acts is not None else None
        if x.split_bytes:
            bw.split_workspace, bw.split_workspace_bytes = x.split_ws.data_ptr(), x.split_bytes
        bw.z_vals, bw.raw, bw.g_depth, bw.g_rgb, bw.masks = (x.z_vals.data_ptr(), x.raw.data_ptr(), x.g_depth.data_ptr(),
                                                              x.g_rgb.data_ptr(), x.masks.data_ptr())
        bw.workspace = x.bwd_ws.data_ptr()
        self._p = dict(call=call, grids=grids, lin=(t_u, t_s), inp=inp, fo=fo, bw=bw, dirs=dirs, offs=frame_offsets, gd=gd, gc=gc,
                       w_color=w_color, uc=int(x.stage == "color"), ggd=global_gt_depth)
        self.collectives_per_step = (1 if (global_gt_depth is not None or not x.render_with_depth) else 2) if world()[1] > 1 else 0

    def enqueue(self):
        import ctypes as C
        from . import _lib
        from .renderer import _VP, _stream
        L = _lib.lib()
        x, p = self.ctx, self._p
        n, st = x.n, _stream()
        x.zero_grads()
        if x.render_with_depth:
            if p["ggd"] is not None:                               # maxima of the full batch, no exchange
                _lib.check(L.nsb_batch_max_depth(_VP(p["ggd"].data_ptr()), p["ggd"].numel(), _VP(x.depth_max.data_ptr()), st), "nsb_batch_max_depth")
            else:
                _lib.check(L.nsb_batch_max_depth(_VP(p["gd"].data_ptr()), n, _VP(x.depth_max.data_ptr()), st), "nsb_batch_max_depth")
                exchange_depth_max(x.depth_max)
        _lib.check(L.nsb_render_forward(C.byref(p["inp"]), C.byref(p["fo"]), st), "nsb_render_forward")
        _lib.check(L.nsb_mapping_seeds(_VP(x.depth.data_ptr()), _VP(x.rgb.data_ptr()), _VP(p["gd"].data_ptr()), _VP(p["gc"].data_ptr()), n,
                                       p["w_color"], p["uc"], _VP(x.g_depth.data_ptr()), _VP(x.g_rgb.data_ptr()), _VP(x.loss.data_ptr()), st),
                   "nsb_mapping_seeds")
        _lib.check(L.nsb_render_backward(C.byref(p["inp"]), C.byref(p["bw"]), st), "nsb_render_backward")
        x.finish_packed(p["dirs"], p["offs"])
        return reduce_sum(x.packed)

    def build_graph(self):
        try:
            cur = torch.cuda.current_stream()
            side = torch.cuda.Stream()
            side.wait_stream(cur)
            with torch.cuda.stream(side):
                self.enqueue(); self.enqueue()
            cur.wait_stream(side)
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                self.enqueue()
            return g
        except Exception:
            torch.cuda.synchronize()
            return None
