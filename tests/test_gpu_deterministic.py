"""GPU: option "deterministic" -- voxel and decoder-weight gradients summed in an order fixed by the data.

  * nsb_voxel_grad_ordered bit for bit against a numpy float32 sequential sum in (point, corner) order: dense channels-last and strided
    grids, the compact slot buffer with unselected voxels, one voxel hit by 10^4 contributions, points on cell faces, on the bound and
    outside it, an empty batch;
  * repeatability: five drop-in mapping calls (render_batch_ray + loss.backward(), every decoder trainable, dense and masked voxel
    gradients) give equal tensors, with split_model 0 and 1 alike; the coarse stage too;
  * the deterministic gradients stay within float32 summation-order noise of the default mode's;
  * a backward whose split workspace was sized with the option off is refused, not run (drop-in and fused iteration);
  * one fused IterationContext serves a smaller then a larger batch and matches a fresh context bit for bit;
  * exact invariants (torch.equal, on non-zero tensors, with the kernels that ran checked in a profiler trace): the mode leaves the forward
    and the ray gradients unchanged; channels-last and NCDHW grids give the same bits; compact (val[mask]) voxel gradients equal the dense
    ones at the mask, drop-in and fused; a split workspace left full of NaN by an earlier call gives the same bits as a zeroed one;
  * the mode's dispatch edges: S < 8 (ray-group kernels) refused by name, small_rays ignored, a tracking call on the default kernels;
  * two replays of the golden sequences (FusedSLAM, coarse mapper off and on) give equal poses, losses, grids, decoders and checkpoint
    contents, within test_gpu_slam's bars against the reference."""
import os

import numpy as np
import pytest
import torch

import scene_util as su
from gpu_util import make_renderer, rel
from oracle import f64_ref as fr
from oracle import torch_port as tp
from test_gpu_f64 import GRIDS
from test_gpu_wgrad_all import kernel_names

pytestmark = pytest.mark.gpu
DEV = "cuda"


class option:
    """A library option for the duration of a block, restored afterwards."""

    def __init__(self, **values):
        self.values = values

    def __enter__(self):
        from nice_slam_b200 import _lib
        self.prev = {k: _lib.get_option(k) for k in self.values}
        for k, v in self.values.items():
            _lib.set_option(k, v)

    def __exit__(self, *exc):
        from nice_slam_b200 import _lib
        for k in sorted(self.prev, key=lambda k: k != "deterministic"):      # (deterministic first: it refuses some values of the others)
            _lib.set_option(k, self.prev[k])


# ------------------------------------------------------------------------------------ the ordered reduction alone
def _f32(x):
    return np.float32(x)


def ref_voxel_grad(xn, dc, D, H, W, slot_map, d_grid):
    """numpy restatement: tri_axis / make_tri / tri_weight of nsb_geom.cuh in float32, one sequential float32 sum per voxel channel in
    ascending (point, corner) order onto d_grid's values.  d_grid: [D, H, W, 32] (dense) or [n_selected, 32] (compact)."""
    out = d_grid.astype(np.float32).copy()
    size = (W, H, D)
    for p in range(xn.shape[0]):
        i0, w0, w1 = [0] * 3, [0] * 3, [0] * 3
        for a in range(3):
            mx = _f32(size[a] - 1)
            u = _f32(_f32(_f32(xn[p, a]) + _f32(1.0)) * _f32(0.5)) * mx
            u = _f32(u)
            if u <= 0:
                u = _f32(0.0)
            elif u >= mx:
                u = mx
            i0[a] = int(np.floor(u))
            f0 = _f32(i0[a])
            w0[a] = _f32(_f32(f0 + _f32(1.0)) - u)
            w1[a] = _f32(u - f0)
        for k in range(8):
            x, y, z = i0[0] + (k & 1), i0[1] + ((k >> 1) & 1), i0[2] + ((k >> 2) & 1)
            if not (x < W and y < H and z < D):
                continue
            wx = w1[0] if k & 1 else w0[0]
            wy = w1[1] if k & 2 else w0[1]
            wz = w1[2] if k & 4 else w0[2]
            w = _f32(_f32(wx * wy) * wz)
            if slot_map is not None:
                s = int(slot_map[(z * H + y) * W + x])
                if s < 0:
                    continue
                row = out[s]
            else:
                row = out[z, y, x]
            row += (w * dc[p]).astype(np.float32)          # one float32 product and one float32 add per channel, in order
    return out


def run_ordered(xn, dc, D, H, W, layout, slot_map=None, init=None):
    """nsb_voxel_grad_ordered on the device; returns d_grid as [D, H, W, 32] (dense) or [n_selected, 32] (compact)."""
    import ctypes as C
    from nice_slam_b200 import _lib
    L = _lib.lib()
    n = xn.shape[0]
    if slot_map is not None:
        n_sel = int((slot_map >= 0).sum())
        g = torch.zeros(max(n_sel, 1), 32, dtype=torch.float32, device=DEV)
        strides = (1, 0, 0, 32)
    elif layout == "channels_last":
        g = torch.zeros(D, H, W, 32, dtype=torch.float32, device=DEV)
        strides = (1, H * W * 32, W * 32, 32)
    else:                                                         # the reference's contiguous [32, D, H, W]
        g = torch.zeros(32, D, H, W, dtype=torch.float32, device=DEV)
        strides = (D * H * W, H * W, W, 1)
    if init is not None:
        (g.copy_(torch.from_numpy(init)) if slot_map is not None or layout == "channels_last"
         else g.copy_(torch.from_numpy(init).permute(3, 0, 1, 2)))
    grid = _lib.Grid(None, D, H, W, *strides)
    xn_d = torch.from_numpy(np.ascontiguousarray(xn, dtype=np.float32)).to(DEV)
    dc_d = torch.from_numpy(np.ascontiguousarray(dc, dtype=np.float32)).to(DEV)
    sm = torch.from_numpy(slot_map.astype(np.int32)).to(DEV) if slot_map is not None else None
    ws = torch.empty(max(L.nsb_voxel_grad_ordered_workspace(n), 16), dtype=torch.uint8, device=DEV)
    _lib.check(L.nsb_voxel_grad_ordered(C.byref(grid), sm.data_ptr() if sm is not None else None, xn_d.data_ptr(), dc_d.data_ptr(), n,
                                        g.data_ptr(), ws.data_ptr(), ws.numel(), torch.cuda.current_stream().cuda_stream), "nsb_voxel_grad_ordered")
    torch.cuda.synchronize()
    if slot_map is None and layout != "channels_last":
        g = g.permute(1, 2, 3, 0)
    return g.cpu().numpy()


def _points(rng, n, D, H, W):
    """Random points with the special positions mixed in: cell faces (lattice coordinates), the bound (+-1) and outside it."""
    xn = rng.uniform(-1.0, 1.0, size=(n, 3)).astype(np.float32)
    size = np.array([W, H, D], dtype=np.float32)
    k = n // 5
    lat = rng.integers(0, size.astype(np.int64), size=(k, 3)).astype(np.float32)
    xn[:k] = (lat / (size - 1) * 2 - 1).astype(np.float32)          # on cell faces
    xn[k: 2 * k] = rng.choice(np.array([-1.0, 1.0], np.float32), size=(k, 3))
    xn[2 * k: 3 * k] = rng.uniform(-1.6, 1.6, size=(k, 3)).astype(np.float32)
    return xn


@pytest.mark.parametrize("layout", ["channels_last", "ncdhw", "compact"])
def test_ordered_voxel_gradient_bit_exact(layout):
    rng = np.random.default_rng({"channels_last": 1, "ncdhw": 2, "compact": 3}[layout])
    D, H, W = 5, 7, 6
    n = 700
    xn = _points(rng, n, D, H, W)
    dc = rng.standard_normal((n, 32)).astype(np.float32)
    slot_map = None
    if layout == "compact":
        sel = rng.random(D * H * W) < 0.6
        slot_map = np.where(sel, np.cumsum(sel) - 1, -1).astype(np.int32)
        init = rng.standard_normal((int(sel.sum()), 32)).astype(np.float32)
    else:
        init = rng.standard_normal((D, H, W, 32)).astype(np.float32)
    got = run_ordered(xn, dc, D, H, W, layout, slot_map, init)
    want = ref_voxel_grad(xn, dc, D, H, W, slot_map, init)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), np.abs(got - want).max()


def test_ordered_voxel_gradient_hot_voxel():
    """12 000 points in one cell (one voxel gets 12 000 contributions per corner) plus scattered ones."""
    rng = np.random.default_rng(4)
    D, H, W = 4, 4, 4
    hot = (np.array([1.2, 2.4, 0.7], np.float32) + rng.uniform(0, 0.6, size=(12000, 3)).astype(np.float32)) / 3 * 2 - 1
    xn = np.concatenate([hot.astype(np.float32), _points(rng, 300, D, H, W)])
    dc = rng.standard_normal((xn.shape[0], 32)).astype(np.float32)
    got = run_ordered(xn, dc, D, H, W, "channels_last")
    want = ref_voxel_grad(xn, dc, D, H, W, None, np.zeros((D, H, W, 32), np.float32))
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), np.abs(got - want).max()


def test_ordered_voxel_gradient_empty_batch():
    init = np.arange(3 * 3 * 3 * 32, dtype=np.float32).reshape(3, 3, 3, 32)
    got = run_ordered(np.zeros((0, 3), np.float32), np.zeros((0, 32), np.float32), 3, 3, 3, "channels_last", init=init)
    assert np.array_equal(got, init)


# ------------------------------------------------------------------------------------ the drop-in mapping call
def _scene():
    sc = su.load_scenes()["room0"]
    return sc, su.make_grids(sc, "soft"), su.load_decoders("soft")


def mapping_call(sc, grids, dec_state, stage, n_rays=996, masked=False, seed=2100):
    """One drop-in mapping call (every decoder trainable, the grids of the stage graded) -> dict of loss and gradients."""
    renderer, c, dec = make_renderer(sc, grids, dec_state, DEV)
    ro, rd, gd, gc = (t.to(DEV) for t in su.make_rays(sc, n_rays, seed=seed))
    for p in dec.parameters():
        p.requires_grad_(True)
    graded = {"coarse": ("grid_coarse",), "middle": ("grid_middle",), "fine": ("grid_fine",),
              "color": ("grid_fine", "grid_color", "grid_middle")}[stage]
    leaves = {}
    for k in list(c):
        c[k] = c[k].detach()
        if k in graded:
            if masked:                                            # the reference mapper's val[mask] parameterisation (Mapper.py:317-333)
                g = torch.Generator().manual_seed(7)
                mask = (torch.rand(c[k].shape[2:], generator=g) < 0.7).to(DEV)
                val = c[k][:, :, mask].clone().requires_grad_(True)
                full = c[k].clone()
                full[:, :, mask] = val
                leaves[k], c[k] = val, full
            else:
                c[k] = c[k].clone().requires_grad_(True)
                leaves[k] = c[k]
    ro = ro.clone().requires_grad_(True)
    depth, var, color = renderer.render_batch_ray(c, dec, rd, ro, DEV, stage, gt_depth=gd if stage != "coarse" else None)
    loss = tp.mapping_loss(depth, color, gd, gc.float(), stage)
    loss.backward()
    torch.cuda.synchronize()
    out = {"loss": loss.detach().clone(), "d_rays_o": ro.grad.clone()}
    out.update({"d_" + k: v.grad.clone() for k, v in leaves.items()})
    out.update({"d_" + n: p.grad.clone() for n, p in dec.named_parameters() if p.grad is not None})
    return out


def _equal(a, b):
    assert a.keys() == b.keys()
    return [k for k in a if not torch.equal(a[k], b[k])]


@pytest.mark.parametrize("stage,masked", [("color", False), ("color", True), ("fine", False), ("middle", True), ("coarse", False)])
def test_mapping_call_repeats_bit_for_bit(stage, masked):
    sc, grids, dec_state = _scene()
    runs = []
    for split_model in (1, 0):
        with option(deterministic=1, split_model=split_model):
            for _ in range(5 if split_model else 2):
                runs.append(mapping_call(sc, grids, dec_state, stage, masked=masked))
    for i, r in enumerate(runs[1:], 1):
        diff = _equal(runs[0], r)
        assert not diff, (i, diff)


@pytest.mark.parametrize("stage", ["color", "coarse"])
def test_deterministic_gradients_match_default_mode(stage):
    """The two modes add the same float32 products in different orders: a relative difference of float32 summation noise."""
    sc, grids, dec_state = _scene()
    with option(deterministic=1):
        det = mapping_call(sc, grids, dec_state, stage)
    dflt = mapping_call(sc, grids, dec_state, stage)
    for k in det:
        assert rel(det[k], dflt[k]) < 1e-4, (k, rel(det[k], dflt[k]))


def test_workspace_sized_for_the_other_mode_is_refused():
    """A forward run with the option off sizes its split workspace without the deterministic buffers; turning the option on before the
    backward makes the backward fail with an error naming the option (no launch)."""
    sc, grids, dec_state = _scene()
    renderer, c, dec = make_renderer(sc, grids, dec_state, DEV)
    ro, rd, gd, gc = (t.to(DEV) for t in su.make_rays(sc, 996, seed=2200))
    c["grid_fine"] = c["grid_fine"].detach().clone().requires_grad_(True)
    depth, var, color = renderer.render_batch_ray(c, dec, rd, ro, DEV, "fine", gt_depth=gd)
    loss = tp.mapping_loss(depth, color, gd, gc.float(), "fine")
    with option(deterministic=1):
        with pytest.raises(RuntimeError, match="deterministic"):
            loss.backward()
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------ the fused iteration with a varying batch
def _iteration(ctx, c, dec, ro, rd, gd, gc):
    ctx.run(c, dec, ro, rd, gd, gc)
    torch.cuda.synchronize()
    out = {"loss": ctx.loss.clone(), "d_rays_o": ctx.d_rays_o[: ro.shape[0]].clone()}
    out.update({"d_" + k: v.clone() for k, v in ctx.d_grid.items()})
    out.update({"d_" + k: v.clone() for k, v in ctx.d_flat.items()})
    return out


@pytest.mark.parametrize("stage", ["color", "coarse"])
def test_iteration_context_serves_a_smaller_then_a_larger_batch(stage):
    """One deterministic IterationContext (capacity 996 rays) runs 400 rays, then 996: the second call equals the same 996-ray call on a
    fresh context bit for bit (the mode's buffers never reach the ray counters a larger batch uses), and repeats exactly."""
    from nice_slam_b200.steps import IterationContext
    sc, grids, dec_state = _scene()
    with option(deterministic=1):
        renderer, c, dec = make_renderer(sc, grids, dec_state, DEV)
        for p in dec.parameters():
            p.requires_grad_(True)
        ro, rd, gd, gc = (t.to(DEV).contiguous() for t in su.make_rays(sc, 996, seed=2300))
        gc = gc.float().contiguous()
        graded = ("grid_coarse",) if stage == "coarse" else ("grid_middle", "grid_fine", "grid_color")
        decs = ("coarse",) if stage == "coarse" else ("middle", "fine", "color")
        kw = dict(kind="map", grad_grids=graded, grad_decoders=decs, coarse_mapper=stage == "coarse")
        ctx = IterationContext(renderer, 996, stage, DEV, **kw)
        _iteration(ctx, c, dec, ro[:400].contiguous(), rd[:400].contiguous(), gd[:400].contiguous(), gc[:400].contiguous())
        grown = _iteration(ctx, c, dec, ro, rd, gd, gc)
        again = _iteration(ctx, c, dec, ro, rd, gd, gc)
        fresh = _iteration(IterationContext(renderer, 996, stage, DEV, **kw), c, dec, ro, rd, gd, gc)
    assert not _equal(grown, fresh), _equal(grown, fresh)
    assert not _equal(grown, again), _equal(grown, again)
    with option(deterministic=0, wgrad_all=1):            # the same kernels (every decoder's weight gradients on the tensor cores), atomic sums
        dflt = _iteration(IterationContext(renderer, 996, stage, DEV, **kw), c, dec, ro, rd, gd, gc)
    for k in dflt:
        assert rel(grown[k], dflt[k]) < 1e-4, (k, rel(grown[k], dflt[k]))


def test_iteration_workspace_sized_with_the_option_off_names_it():
    from nice_slam_b200.steps import IterationContext
    sc, grids, dec_state = _scene()
    renderer, c, dec = make_renderer(sc, grids, dec_state, DEV)
    ro, rd, gd, gc = (t.to(DEV).contiguous() for t in su.make_rays(sc, 200, seed=2400))
    ctx = IterationContext(renderer, 200, "color", DEV, kind="map", grad_grids=("grid_fine",), grad_decoders=("color",))
    with option(deterministic=1):
        with pytest.raises(RuntimeError, match="deterministic"):
            ctx.run(c, dec, ro, rd, gd, gc.float().contiguous())
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------ exact invariants
FWD = ("depth", "var", "rgb", "raw", "z_vals", "masks", "d_rays_o", "d_rays_d")     # the same arithmetic in every mode and layout
FORMS = {"grids": lambda stage: (), "color_wg": lambda stage: ("color",), "all": lambda stage: fr.STAGE_DECODERS[stage]}


def render_call(stage, n_rays=97, form="grids", n_samples=17, n_surface=16, seed=3000, channels_last=True, voxel_masks=None, attempts=3):
    """One drop-in render_batch_ray (soft room0 scene, the grids of the stage graded, the decoders of `form` trainable) and the backward of
    seeded random cotangents of depth, var and rgb, traced.  voxel_masks {grid key: [D, H, W] bool}: that grid takes the reference mapper's
    val[mask] parameterisation (Mapper.py:317-333, the mask repeated over the channels), which the renderer serves with compact gradients.
    -> (dict of outputs and gradients, kernel names of the call).  A trace without a render forward and a render backward kernel has lost
    device records (see test_gpu_wgrad_all._profiled), and the call is run again."""
    from torch.profiler import ProfilerActivity, profile
    from nice_slam_b200.masked import MaskedVoxels
    sc, grids, dec_state = _scene()
    gdec = FORMS[form](stage)
    for _ in range(attempts):
        renderer, c, dec = make_renderer(sc, grids, dec_state, DEV, channels_last=channels_last, n_samples=n_samples, n_surface=n_surface)
        ro, rd, gd, _ = su.make_rays(sc, n_rays, seed=seed)
        g = torch.Generator().manual_seed(seed)
        cot = (torch.randn(n_rays, dtype=torch.float64, generator=g), torch.randn(n_rays, dtype=torch.float64, generator=g),
               torch.randn(n_rays, 3, generator=g))
        cot = tuple(x.to(DEV) for x in cot)
        r1, r2 = ro.to(DEV).requires_grad_(True), rd.to(DEV).requires_grad_(True)
        for n, p in dec.named_parameters():
            p.requires_grad_(n.split("_decoder.")[0] in gdec)
        leaves = {}
        for k in list(c):
            c[k] = c[k].detach()
            if k not in GRIDS[stage]:
                continue
            if voxel_masks is not None and k in voxel_masks:
                m5 = voxel_masks[k].to(DEV).unsqueeze(0).unsqueeze(0).expand_as(c[k])
                val = c[k][m5].clone().requires_grad_(True)
                full = c[k].clone()
                full[m5] = val
                leaves[k], c[k] = val, full
            else:
                c[k] = c[k].clone().requires_grad_(True)
                leaves[k] = c[k]
        aux = {}
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            d, u, col = renderer.render_batch_ray(c, dec, r2, r1, DEV, stage, gt_depth=gd.to(DEV), aux=aux)
            ((d * cot[0]).sum() + (u * cot[1]).sum() + (col * cot[2]).sum()).backward()
            torch.cuda.synchronize()
        names = kernel_names(prof)
        if any(x.startswith("render_fwd") for x in names) and any(x.startswith("render_bwd") for x in names):
            break
    if voxel_masks is not None:                                   # the compact path served the masked grids
        assert sum(isinstance(v, MaskedVoxels) for v in renderer._mask_cache.values()) == len(voxel_masks), renderer._mask_cache
    # (the saved ReLU words of the stage's decoders: word 5 * dec_pos + layer; the others are not written.  rgb: the colour stage's alone)
    out = dict(depth=d.detach(), var=u.detach(), raw=aux["raw"], z_vals=aux["z_vals"],
               masks=aux["masks"][..., : 5 * len(fr.STAGE_DECODERS[stage])], d_rays_o=r1.grad, d_rays_d=r2.grad)
    if stage == "color":
        out["rgb"] = col.detach()
    out.update({"d_" + k: v.grad for k, v in leaves.items()})
    out.update({"d_" + n: p.grad for n, p in dec.named_parameters() if p.grad is not None})
    assert set(k.split("_decoder.")[0][2:] for k in out if "_decoder." in k) == set(gdec), sorted(out)
    return out, names


def backward_kernel(stage, form, det):
    """The tile backward kernel that produces the call's voxel (and, with decoders graded, weight) gradients."""
    base = "render_bwd_tile" if form == "grids" else "render_bwd_wg_coarse_tile" if stage == "coarse" else "render_bwd_wg_tile"
    return base + ("_det" if det else "") + "_kernel"


def check_kernels(names, stage, form, det):
    """The intended backward ran, and every render backward of the call is of the mode's family (kDet or default)."""
    bwd = sorted(set(x for x in names if x.startswith("render_bwd")))
    assert backward_kernel(stage, form, det) in bwd, (stage, form, det, bwd)
    assert all(("_det_" in x) == bool(det) for x in bwd), (det, bwd)
    assert not any(x.startswith("render_fwd_tc") or x == "render_bwd_kernel" for x in names), names


def assert_bits(a, b, keys, what):
    """torch.equal on each of `keys` (every decoder gradient for keys = None), each non-zero; decoder gradients non-zero per decoder."""
    keys = sorted(a) if keys is None else [k for k in keys if k != "rgb" or "rgb" in a or "rgb" in b]
    assert set(keys) <= set(a) and set(keys) <= set(b), (what, sorted(a), sorted(b))
    differ = [k for k in keys if not torch.equal(a[k], b[k])]
    assert not differ, (what, [(k, float((a[k].double() - b[k].double()).abs().max())) for k in differ])
    for k in keys:
        if "_decoder." not in k:
            assert float(a[k].double().abs().max()) > 0, (what, k)
    for lvl in set(k.split("_decoder.")[0] for k in keys if "_decoder." in k):
        assert max(float(a[k].abs().max()) for k in keys if k.startswith(lvl + "_decoder.")) > 0, (what, lvl)


@pytest.mark.parametrize("stage,form", [(s, "grids") for s in ("coarse", "middle", "fine", "color")] + [("color", "color_wg")] +
                         [(s, "all") for s in ("coarse", "middle", "fine", "color")])
def test_mode_leaves_forward_and_ray_gradients_unchanged(stage, form):
    """The forward is the same kernel in both modes, and the kDet backward differs from the default one only in where dL/dc and the weight
    partials go: the ray parts are summed in (tile, decoder) order either way.  Form "all" is set beside option wgrad_all, which puts every
    decoder's weight gradients on the same kernel family as the mode does."""
    with option(deterministic=0, wgrad_all=int(form == "all")):
        dflt, nd = render_call(stage, form=form)
    with option(deterministic=1):
        det, nt = render_call(stage, form=form)
    check_kernels(nd, stage, form, 0)
    check_kernels(nt, stage, form, 1)
    assert_bits(det, dflt, FWD, "mode %s %s" % (stage, form))


@pytest.mark.parametrize("det", [1, 0])
@pytest.mark.parametrize("stage,form", [("coarse", "all"), ("middle", "grids"), ("fine", "all"), ("color", "color_wg"), ("color", "all")])
def test_channels_last_and_ncdhw_grids_give_identical_bits(stage, form, det):
    """gather_issue loads the same floats through either layout's addressing and gather_consume / gather_tile_kt run one fmaf chain on them,
    so the forward and the ray gradients are bit-identical; in deterministic mode the ordered voxel sum keys a voxel by its index, not its
    address, so every voxel and decoder gradient is too."""
    runs = {}
    for cl in (True, False):
        with option(deterministic=det, wgrad_all=1):
            runs[cl], names = render_call(stage, form=form, channels_last=cl, seed=3100)
        check_kernels(names, stage, form, det)
    assert_bits(runs[False], runs[True], None if det else FWD, "layout %s %s det=%d" % (stage, form, det))


def _voxel_masks(stage, kind):
    """{grid key: [D, H, W] bool} for the grids of the stage: 'random' selects about 70 % of the voxels; 'half' leaves out the voxels of
    x index < W / 2, so every corner of the samples in that half takes the slot -1 path."""
    sc, grids, _ = _scene()
    g = torch.Generator().manual_seed(31)
    out = {}
    for k in GRIDS[stage]:
        D, H, W = grids[k].shape[2:]
        if kind == "random":
            out[k] = torch.rand(D, H, W, generator=g) < 0.7
        else:
            out[k] = torch.ones(D, H, W, dtype=torch.bool)
            out[k][:, :, : W // 2] = False
    return out


@pytest.mark.parametrize("kind", ["random", "half"])
@pytest.mark.parametrize("stage", ["coarse", "middle", "fine", "color"])
def test_compact_voxel_gradients_equal_the_dense_ones(stage, kind):
    """The ordered voxel sum takes each voxel's (point, corner) list in the same order whether its key is a slot or a linear voxel index:
    the drop-in val[mask] gradient equals the dense call's gradient at the mask, bit for bit, with every decoder graded."""
    masks = _voxel_masks(stage, kind)
    with option(deterministic=1):
        dense, nd = render_call(stage, form="all", seed=3200)
        comp, nc = render_call(stage, form="all", seed=3200, voxel_masks=masks)
    check_kernels(nd, stage, "all", 1)
    check_kernels(nc, stage, "all", 1)
    assert_bits(comp, dense, FWD + tuple(k for k in dense if "_decoder." in k), "compact %s %s" % (stage, kind))
    for k, m in masks.items():
        g = dense["d_" + k]
        m5 = m.to(DEV).unsqueeze(0).unsqueeze(0).expand_as(g)
        want = g[m5]
        assert float(want.abs().max()) > 0, k
        assert float(g[~m5].abs().max()) > 0, k                   # samples did reach the voxels left out
        assert torch.equal(comp["d_" + k], want), (k, float((comp["d_" + k] - want).abs().max()))


@pytest.mark.parametrize("stage", ["color", "coarse"])
def test_masked_iteration_compact_gradients_equal_the_dense_ones(stage):
    """The fused mapping iteration (IterationContext) with MaskedVoxels: its compact gradients equal the dense context's at the mask bit for
    bit (test_gpu_parity.test_masked_mapping_iteration_packed_block holds the default mode to rel < 1e-5)."""
    from nice_slam_b200.masked import MaskedVoxels
    from nice_slam_b200.steps import IterationContext
    sc, grids, dec_state = _scene()
    masks = _voxel_masks(stage, "random")
    keys = tuple(masks)
    decs = ("coarse",) if stage == "coarse" else ("middle", "fine", "color")
    with option(deterministic=1):
        renderer, c, dec = make_renderer(sc, grids, dec_state, DEV)
        ro, rd, gd, gc = (t.to(DEV).contiguous() for t in su.make_rays(sc, 330, seed=3300))
        gc = gc.float().contiguous()
        kw = dict(kind="map", grad_grids=keys, grad_decoders=decs, coarse_mapper=stage == "coarse")
        dense = IterationContext(renderer, 330, stage, DEV, **kw)
        dense.run(c, dec, ro, rd, gd, gc)
        mv = {k: MaskedVoxels(c[k], masks[k]) for k in keys}
        ctx = IterationContext(renderer, 330, stage, DEV, masked=mv, **kw)
        ctx.run(c, dec, ro, rd, gd, gc)
        torch.cuda.synchronize()
    assert torch.equal(ctx.loss, dense.loss)
    for k in keys:
        m5 = masks[k].to(DEV).unsqueeze(0).unsqueeze(0).expand_as(dense.d_grid[k])
        want = dense.d_grid[k][m5]
        assert float(want.abs().max()) > 0, k
        assert torch.equal(mv[k].to_reference(ctx.d_grid[k]), want), (k, float((mv[k].to_reference(ctx.d_grid[k]) - want).abs().max()))
    for lvl in decs:
        assert float(dense.d_flat[lvl].abs().max()) > 0 and torch.equal(ctx.d_flat[lvl], dense.d_flat[lvl]), lvl


def _poison_split_workspace(monkeypatch):
    """Every drop-in forward's split workspace comes back from _forward_setup filled with 0xFF bytes (NaN as float32) -- as a workspace
    reused by an earlier call may be -- except the ray-completion counters at its end and the 16 bytes in front of them, which split_layout
    (nsb_render.cu) requires to start at zero.  Any NaN in a result is then a read of a region the call did not write first."""
    import nice_slam_b200.renderer as R
    setup = R._forward_setup

    def poisoned(call, ro):
        res = setup(call, ro)
        split = res[3][5]
        if split is not None:
            keep = 16 + (4 * ro.shape[0] + 15) // 16 * 16
            assert split.numel() > keep
            split[: split.numel() - keep].fill_(0xFF)
        return res

    monkeypatch.setattr(R, "_forward_setup", poisoned)


POISON_CASES = [("coarse", 97, 33, "all", False), ("coarse", 1408, 256, "grids", True), ("fine", 97, 256, "grids", False),
                ("fine", 1408, 33, "all", True), ("color", 97, 33, "color_wg", True), ("color", 1408, 33, "grids", False),
                ("color", 97, 256, "all", False), ("color", 1408, 256, "color_wg", False)]


@pytest.mark.parametrize("det", [1, 0])
@pytest.mark.parametrize("stage,n_rays,S,form,compact", POISON_CASES)
def test_dirty_split_workspace_gives_the_bits_of_a_clean_one(stage, n_rays, S, form, compact, det, monkeypatch):
    """The same call on a zeroed and on a NaN-filled split workspace (tile kernels: S >= 8, small_rays 0).  Deterministic mode: every output
    and gradient bit-identical.  Default mode: forward and ray gradients bit-identical, voxel and weight gradients (float atomics) finite and
    within float32 summation-order noise."""
    ns, nsurf = (S, 16) if stage == "coarse" else (S - 16, 16)
    masks = _voxel_masks(stage, "random") if compact else None
    kw = dict(stage=stage, n_rays=n_rays, form=form, n_samples=ns, n_surface=nsurf, seed=3400 + n_rays, voxel_masks=masks)
    with option(deterministic=det, wgrad_all=int(form == "all"), small_rays=0):
        clean, names = render_call(**kw)
        _poison_split_workspace(monkeypatch)
        dirty, names_dirty = render_call(**kw)
    check_kernels(names, stage, form, det)
    check_kernels(names_dirty, stage, form, det)
    what = "dirty %s N=%d S=%d %s compact=%d det=%d" % (stage, n_rays, S, form, compact, det)
    if det:
        assert_bits(dirty, clean, None, what)
        return
    assert_bits(dirty, clean, FWD, what)
    for k in clean:
        if k not in FWD:
            assert bool(torch.isfinite(dirty[k]).all()), (what, k)
            assert rel(dirty[k], clean[k]) < 1e-4, (what, k, rel(dirty[k], clean[k]))


# ------------------------------------------------------------------------------------ the mode's dispatch edges
def test_ray_group_family_backward_is_refused_by_name():
    """S = 7 < kMinSamples takes the round-1 ray-group kernels, whose backward adds voxel gradients with atomics: the mode refuses it with an
    error naming the option, before any backward kernel runs."""
    from torch.profiler import ProfilerActivity, profile
    sc, grids, dec_state = _scene()
    with option(deterministic=1):
        renderer, c, dec = make_renderer(sc, grids, dec_state, DEV, n_samples=5, n_surface=2)
        for p in dec.parameters():
            p.requires_grad_(False)
        ro, rd, gd, _ = (t.to(DEV) for t in su.make_rays(sc, 64, seed=3500))
        c["grid_fine"] = c["grid_fine"].detach().clone().requires_grad_(True)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            depth, var, color = renderer.render_batch_ray(c, dec, rd, ro, DEV, "fine", gt_depth=gd)
            with pytest.raises(RuntimeError, match="deterministic"):
                depth.sum().backward()
            torch.cuda.synchronize()
    names = kernel_names(prof)
    assert "render_fwd_tc_kernel" in names, names
    assert not any(x.startswith("render_bwd") for x in names), names
    assert c["grid_fine"].grad is None


def test_small_rays_leaves_a_mapping_call_on_the_tile_kernels():
    """small_rays = 64 would send a 16-ray call to the ray-group kernels; in deterministic mode a call with voxel and weight gradients stays on
    the kDet tile backward, and its bits are those of small_rays = 0."""
    runs = {}
    for small in (64, 0):
        with option(deterministic=1, small_rays=small):
            runs[small], names = render_call("color", n_rays=16, form="color_wg", seed=3600)
        check_kernels(names, "color", "color_wg", 1)
    assert_bits(runs[64], runs[0], None, "small_rays")


def test_tracking_call_runs_the_default_kernels():
    """A tracking-form call (ray gradients only) has no order-dependent sum: deterministic mode leaves it on the default kernels, with the
    bits of the mode off."""
    sc, grids, dec_state = _scene()
    runs = {}
    for det in (1, 0):
        with option(deterministic=det):
            runs[det], names = _tracking_call(sc, grids, dec_state)
        assert "render_bwd_tile_kernel" in names and not any("_det_" in x for x in names), (det, names)
    assert_bits(runs[1], runs[0], ("depth", "var", "rgb", "d_rays_o", "d_rays_d"), "tracking")


def _tracking_call(sc, grids, dec_state):
    from test_gpu_wgrad_all import _profiled
    renderer, c, dec = make_renderer(sc, grids, dec_state, DEV)
    for p in dec.parameters():
        p.requires_grad_(False)                                   # (the fused tracker's form: the pose alone is optimised)
    ro, rd, gd, gc = (t.to(DEV) for t in su.make_rays(sc, 200, seed=3700))
    out = {}

    def track():
        r1 = ro.clone().requires_grad_(True)
        r2 = rd.clone().requires_grad_(True)
        depth, var, color = renderer.render_batch_ray(c, dec, r2, r1, DEV, "color", gt_depth=gd)
        tp.tracking_loss(depth, var, color, gd, gc.double(), sc["tracking"]["w_color_loss"]).backward()
        out.update(depth=depth.detach(), var=var.detach(), rgb=color.detach(), d_rays_o=r1.grad, d_rays_d=r2.grad)

    names = _profiled(track)
    return out, names


# ------------------------------------------------------------------------------------ whole sequences
@pytest.mark.parametrize("name,coarse", [("blocks", False), ("blocks", True), ("every1", False)])
def test_sequence_replays_repeat_bit_for_bit(name, coarse, tmp_path):
    """Two deterministic replays of a golden sequence (FusedSLAM: tracking loop, mapping loop with its BA window and fused Adam, the coarse
    mapper when on): every pose, every run_log loss, every grid and decoder tensor equal, and every checkpoint's
    contents equal tensor by tensor.  The
    replay stays within test_gpu_slam's bars against the reference's run."""
    from test_gpu_slam import REF, cfg_of, load, slam_for
    from slam_sequences import per_frame, sequence
    case = load(name)
    sc = su.load_scenes()["room0"]
    runs = []
    with option(deterministic=1):
        for i in range(2):
            cfg = cfg_of(case)
            cfg["coarse"] = coarse
            d = tmp_path / str(i)
            d.mkdir()
            slam = slam_for(sc, cfg, ckpt_dir=str(d))
            est, gt = slam.run(sequence(sc, case["n"]), replay=case["replay"])
            runs.append((slam, est, d))
    (a, ea, da), (b, eb, db) = runs
    assert torch.equal(ea, eb)
    assert len(a.run_log) == len(b.run_log)
    for x, y in zip(a.run_log, b.run_log):
        assert (x["kind"], x["idx"]) == (y["kind"], y["idx"])
        assert torch.equal(torch.as_tensor(x["losses"]), torch.as_tensor(y["losses"])), (x["kind"], x["idx"])
    assert all(torch.equal(a.c[k], b.c[k]) for k in a.c)
    sa, sb = a.dec.state_dict(), b.dec.state_dict()
    assert all(torch.equal(sa[k], sb[k]) for k in sa)
    files = sorted(os.listdir(da))
    assert files and files == sorted(os.listdir(db))
    for f in files:                                           # (the legacy format's storage keys are storage addresses: compare contents)
        ca = torch.load(da / f, map_location="cpu", weights_only=False)
        cb = torch.load(db / f, map_location="cpu", weights_only=False)
        assert ca.keys() == cb.keys(), f
        for k in ca:
            x, y = ca[k], cb[k]
            if isinstance(x, dict) and x and all(torch.is_tensor(v) for v in x.values()):
                assert x.keys() == y.keys() and all(torch.equal(x[j], y[j]) for j in x), (f, k)
            elif isinstance(x, list) and x and torch.is_tensor(x[0]):
                assert len(x) == len(y) and all(torch.equal(u, v) for u, v in zip(x, y)), (f, k)
            elif torch.is_tensor(x):
                assert torch.equal(x, y), (f, k)
            else:
                assert x == y, (f, k)
    if not coarse:
        dev = per_frame(ea, a.run_log, case["estimate_c2w_list"], case["run_log"], case["n"])
        for k, dd in dev.items():
            for q, bar in zip(("t", "r", "map_loss", "track_loss"), REF[name][k]):
                assert dd[q] <= bar, (k, q, dd[q], bar)
