"""Fused Adam for the mapper's parameters (SURVEY.md 8f-2): the frustum-selected voxels of the shared grids, updated in place from the
compact gradients of a mapping iteration (no `val_grad = val[mask]` copy in, no `val[mask] = val_grad` copy back), and the colour
decoder, from its flat gradient.  Same arithmetic as torch.optim.Adam with its defaults (src/Mapper.py:365-379, :412-419, :504): one
launch per optimiser step instead of the ~10 element-wise launches per tensor of the stock optimiser.  Pose parameters stay with
torch (their gradient needs the quaternion chain of get_camera_from_tensor)."""
import ctypes as C

import torch

from . import _lib
from ._lib import LEVELS
from .decoders import decoder_params_struct, named_params
from .renderer import _stream, grid_struct


class FusedMapperAdam:
    """State (exp_avg, exp_avg_sq, step) per parameter group; one C call per step."""

    def __init__(self, betas=(0.9, 0.999), eps=1e-8):
        self.betas, self.eps = betas, eps
        self.state = {}

    def _st(self, name, numel, device):
        st = self.state.get(name)
        if st is None or st["m"].numel() != numel:
            st = dict(m=torch.zeros(numel, dtype=torch.float32, device=device), v=torch.zeros(numel, dtype=torch.float32, device=device), step=0)
            self.state[name] = st
        return st

    def step_all(self, voxel_items, decoder_items=(), renderer=None):
        """The mapper's whole optimizer.step() (Mapper.py:504) in ONE launch.  voxel_items: [(key, grid, masked, grad, lr)] (at most four):
        grid is the shared [1,32,D,H,W] tensor (updated in place), masked its masked.MaskedVoxels, grad the compact [n_selected,32] gradient;
        decoder_items: [(level_name, decoders, grad_flat, lr)] (at most two), the decoders that received a gradient in this iteration, whose
        parameter tensors are updated in place: each keeps its own Adam state and step count, as torch.optim.Adam does for the parameters of
        one group whose .grad is set.  Pass the FusedRenderer so that its packed-weight cache of every stepped decoder is invalidated (raw
        pointer writes do not bump the tensors' version counters)."""
        items = [it for it in voxel_items if it[2].count > 0]
        if len(items) > 4:
            raise RuntimeError("nice_slam_b200: at most four voxel groups per fused optimiser step")
        if len(decoder_items) > 2:
            raise RuntimeError("nice_slam_b200: at most two decoders per fused optimiser step")
        groups = (_lib.AdamVoxelGroup * max(len(items), 1))()
        for q, (key, grid, masked, grad, lr) in enumerate(items):
            st = self._st(key, masked.count * 32, grid.device)
            st["step"] += 1
            g = groups[q]
            g.grid = grid_struct(grid.detach())
            g.slot_map, g.grad, g.exp_avg, g.exp_avg_sq = masked.slot_map.data_ptr(), grad.data_ptr(), st["m"].data_ptr(), st["v"].data_ptr()
            g.lr, g.step = float(lr), st["step"]
        decs = (_lib.AdamDecoderItem * max(len(decoder_items), 1))()
        for k, (level_name, decoders, grad_flat, lr) in enumerate(decoder_items):
            st = self._st("dec_" + level_name, grad_flat.numel(), grad_flat.device)
            st["step"] += 1
            d = decs[k]
            d.level, d.params = LEVELS.index(level_name), C.pointer(self._decoder_struct(decoders, level_name))
            d.grad_flat, d.exp_avg, d.exp_avg_sq, d.lr, d.step = grad_flat.data_ptr(), st["m"].data_ptr(), st["v"].data_ptr(), float(lr), st["step"]
        _lib.check(_lib.lib().nsb_adam_mapper_step_decoders(groups, len(items), decs, len(decoder_items), self.betas[0], self.betas[1], self.eps,
                                                            _stream()), "nsb_adam_mapper_step_decoders")
        if decoder_items and renderer is not None:
            renderer.invalidate_decoders(tuple(it[0] for it in decoder_items))

    def _decoder_struct(self, decoders, level_name):
        """nsb_decoder_params of a decoder, cached on the storage pointers of its parameters (building it walks ~20 tensors)."""
        p = named_params(decoders, level_name)
        key = tuple(t.data_ptr() for t in p.values())
        hit = self.state.get(("dp", level_name))
        if hit is None or hit[0] != key:
            hit = (key, decoder_params_struct(decoders, level_name))
            self.state[("dp", level_name)] = hit
        return hit[1]
