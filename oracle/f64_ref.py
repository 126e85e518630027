"""ORACLE (test infrastructure, NOT product code) -- float64 restatement of the render-and-backprop path of
oracle/torch_port.py, used as the truth that the CUDA kernels and the float32 port are both measured against.

It takes the same discrete decisions as the float32 path, so that the only difference left is precision:
  * sample positions: tp.sample_z_vals (float64 and bit-exact already); in-bound test: tp.in_bound_mask;
  * the two float32 rounding points of the reference are kept: the normalised grid coordinate (`vgrid.float()`, torch_port.sample_grid)
    and the point cast `p.float()` in front of the Fourier embedding.  Both are straight-through: the value is the float32 one, the
    derivative is that of the float64 expression (autograd passes a cast's gradient through unchanged, as in the reference);
  * voxel cell and border clip: from the float32 unnormalised coordinate, computed as ATen's grid sampler does
    (GridSampler.h: ((x + 1) / 2) * (size - 1), clip to [0, size - 1], clipped coordinates get no gradient); the trilinear weights and the
    gather are float64, from the float64 value of the same coordinate.  When the float32 and float64 coordinates straddle a cell boundary
    the weights extrapolate linearly from the float32 cell instead of jumping a cell;
  * ReLU decisions: a mask passed in (the CUDA kernels' saved words, or the port's signs), else the float64 pre-activation's own sign.
Everything else -- trilinear weights, gather, embedding argument and sin, every layer, sigmoid, cumprod with `1 - alpha + 1e-10`,
compositing -- is float64.  The fine decoder's middle-grid features are detached, as under torch.no_grad() in torch_port.mlp_xyz.

Masks are bool [P, n_dec, 5, 32]: point, decoder in STAGE_DECODERS order (NICE.forward's order, the kernels' `dec_pos`), layer, unit.
"""
import torch
import torch.nn.functional as F
from torch.overrides import TorchFunctionMode

from oracle import torch_port as tp

STAGE_DECODERS = {"coarse": ("coarse",), "middle": ("middle",), "fine": ("fine", "middle"), "color": ("fine", "color", "middle")}
STAGE_GRIDS = {"coarse": ("coarse",), "middle": ("middle",), "fine": ("fine", "middle"), "color": ("fine", "color", "middle")}


# ----------------------------------------------------------------------------- discrete decisions
def _cell(p, shape, bound):
    """ATen's border / align_corners decisions for points p [P,3] f64 on a [D,H,W] grid: float32 cell index i0 [P,3] (x, y, z) and the
    clip flags lo / hi [P,3] -- all taken from the float32 unnormalised coordinate."""
    x32 = tp.normalize_coords(p.detach(), bound).float()
    size = torch.tensor([shape[2], shape[1], shape[0]], dtype=torch.float32)
    u = ((x32 + 1) / 2) * (size - 1)
    lo, hi = u <= 0, u >= size - 1
    i0 = torch.floor(torch.minimum(torch.maximum(u, torch.zeros_like(u)), size - 1)).long()
    return dict(i0=i0, lo=lo, hi=hi)


def decide(rays_o, rays_d, stage, gt_depth, bound, grid_shapes, n_samples=32, n_surface=16, coarse_enlarge=2):
    """Everything discrete about one batch: z_vals, in-bound mask and the voxel cells of every stage grid."""
    z = tp.sample_z_vals(rays_o.float(), rays_d.float(), gt_depth, bound, n_samples, n_surface, stage)
    p = (rays_o.float()[:, None, :] + rays_d.float()[:, None, :] * z[..., None]).reshape(-1, 3)
    cells = {}
    for lvl in STAGE_GRIDS[stage]:
        b = bound * coarse_enlarge if lvl == "coarse" else bound
        cells[lvl] = _cell(p, grid_shapes[lvl], b)
    return dict(z_vals=z, inb=tp.in_bound_mask(p, bound), cells=cells, coarse_enlarge=coarse_enlarge)


# ----------------------------------------------------------------------------- differentiable float64 path
def _straight32(x, round32):
    """x rounded to float32 in value, d/dx = 1."""
    return x + (x.detach().float().double() - x.detach()) if round32 else x


def _trilinear(grid, p, bound, cell, round32):
    """grid [1,32,D,H,W] f64, p [P,3] f64 -> [P,32] f64."""
    D, H, W = grid.shape[2:]
    size = torch.tensor([W, H, D], dtype=torch.float64)
    x = _straight32(tp.normalize_coords(p, bound), round32)
    u = ((x + 1) / 2) * (size - 1)
    u = torch.where(cell["lo"], torch.zeros_like(u), torch.where(cell["hi"], (size - 1).expand_as(u), u))
    i0 = cell["i0"]
    f = u - i0.double()
    flat = grid.reshape(32, -1).t()
    out = 0
    for dz in (0, 1):
        for dy in (0, 1):
            for dx in (0, 1):
                ix = torch.clamp(i0[:, 0] + dx, max=W - 1)        # the +1 corner of a clipped-high axis has weight 0
                iy = torch.clamp(i0[:, 1] + dy, max=H - 1)
                iz = torch.clamp(i0[:, 2] + dz, max=D - 1)
                w = (f[:, 0] if dx else 1 - f[:, 0]) * (f[:, 1] if dy else 1 - f[:, 1]) * (f[:, 2] if dz else 1 - f[:, 2])
                out = out + w[:, None] * flat[(iz * H + iy) * W + ix]
    return out


def _mlp(W, c, emb, mask, pre):
    """MLP (emb given) / MLP_no_xyz (emb None) with the ReLU decisions of `mask` [P,5,32] (None: own signs); appends the five
    pre-activations to `pre` and returns (output, mask used)."""
    h = emb if emb is not None else c
    used = []
    for i in range(5):
        u = F.linear(h, W["pts_linears.%d.weight" % i], W["pts_linears.%d.bias" % i])
        m = (u.detach() > 0) if mask is None else mask[:, i]
        used.append(m)
        pre.append(u.detach())
        h = u * m.double()
        if emb is not None:
            h = h + F.linear(c, W["fc_c.%d.weight" % i], W["fc_c.%d.bias" % i])
        if i == 2:
            h = torch.cat([emb if emb is not None else c, h], -1)
    return F.linear(h, W["output_linear.weight"], W["output_linear.bias"]), torch.stack(used, 1)


def decode(p, grids, dec, stage, bound, fixed, masks=None, round32=True):
    """NICE.forward + eval_points' out-of-bound rule for points p [P,3] f64 with the decisions `fixed` (cells, inb, coarse_enlarge,
    optional fine_mid) -> raw [P,4] (occupancy logit in channel 3), pre-activations [P,n_dec,5,32], ReLU decisions used [P,n_dec,5,32]."""
    P = p.shape[0]
    levels = STAGE_DECODERS[stage]
    feat = {}
    for lvl in STAGE_GRIDS[stage]:
        b = bound * fixed["coarse_enlarge"] if lvl == "coarse" else bound
        feat[lvl] = _trilinear(grids["grid_" + lvl], p, b, fixed["cells"][lvl], round32)
    pf = _straight32(p, round32)
    pre, used, out = [], [], {}
    for j, lvl in enumerate(levels):
        mask = None if masks is None else masks[:, j]
        if lvl == "coarse":
            o, m = _mlp(dec[lvl], feat[lvl], None, mask, pre)
        else:
            emb = torch.sin(pf @ dec[lvl]["embedder._B"])
            c = torch.cat([feat["fine"], fixed.get("fine_mid", feat["middle"]).detach()], 1) if lvl == "fine" else feat[lvl]
            o, m = _mlp(dec[lvl], c, emb, mask, pre)
        out[lvl] = o
        used.append(m)
    if stage == "color":
        rgb_pt = out["color"][:, :3]
        occ = out["fine"][:, 0] + out["middle"][:, 0]
    else:
        rgb_pt = torch.zeros(P, 3, dtype=torch.float64)
        occ = out[stage][:, 0] + (out["middle"][:, 0] if stage == "fine" else 0)
    occ = torch.where(fixed["inb"], occ, torch.full_like(occ, 100.0))
    raw = torch.cat([rgb_pt, occ[:, None]], 1)
    return raw, torch.stack(pre, 1).reshape(P, len(levels), 5, 32), torch.stack(used, 1)


def eval_points(p, grids, dec, stage, bound, coarse_enlarge=2):
    """tp.eval_points in float64 (own ReLU signs): p [P,3] f64, grids / dec float32 -> raw [P,4] f64."""
    p = p.double()
    cells = {lvl: _cell(p, tuple(grids["grid_" + lvl].shape[2:]), bound * coarse_enlarge if lvl == "coarse" else bound)
             for lvl in STAGE_GRIDS[stage]}
    fixed = dict(cells=cells, inb=tp.in_bound_mask(p, bound), coarse_enlarge=coarse_enlarge)
    g = {k: v.double() for k, v in grids.items()}
    d = {lvl: {k: v.double() for k, v in W.items()} for lvl, W in dec.items()}
    return decode(p, g, d, stage, bound, fixed)[0]


def render_batch_ray(grids, dec, rays_d, rays_o, stage, gt_depth, bound, n_samples=32, n_surface=16, coarse_enlarge=2,
                     masks=None, fixed=None, round32=True):
    """float64 depth, var, rgb [N], [N], [N,3] and aux dict(z_vals, raw [N,S,4] (occupancy logit in channel 3), pre [P,n_dec,5,32],
    masks [P,n_dec,5,32] (the decisions used), fixed (the discrete decisions, see decide)).
    grids: {"grid_<level>": f64 [1,32,D,H,W]}; dec: {level: {name: f64 tensor}}; rays f64 or f32 (differentiable when f64 leaves).
    fixed: decisions to reuse (central differences; its optional "fine_mid" [P,32] freezes the middle features the fine decoder sees, which
    carry no gradient); round32=False drops the two float32 rounding points (smooth in every input)."""
    if fixed is None:
        shapes = {lvl: tuple(grids["grid_" + lvl].shape[2:]) for lvl in STAGE_GRIDS[stage]}
        fixed = decide(rays_o.detach(), rays_d.detach(), stage, gt_depth, bound, shapes, n_samples, n_surface, coarse_enlarge)
    z = fixed["z_vals"]
    n, S = z.shape
    p = (rays_o.double()[:, None, :] + rays_d.double()[:, None, :] * z[..., None]).reshape(-1, 3)
    raw, pre, used = decode(p, grids, dec, stage, bound, fixed, masks, round32)
    raw = raw.reshape(n, S, 4)
    alpha = torch.sigmoid(10 * raw[..., 3])
    ones = torch.ones(n, 1, dtype=torch.float64)
    weights = alpha * torch.cumprod(torch.cat([ones, 1. - alpha + 1e-10], -1), -1)[:, :-1]
    rgb = torch.sum(weights[..., None] * raw[..., :3], -2)
    depth = torch.sum(weights * z, -1)
    var = torch.sum(weights * (z - depth[:, None]) ** 2, -1)
    aux = dict(z_vals=z, points=p.detach(), raw=raw.detach(), pre=pre, masks=used, fixed=fixed)
    return depth, var, rgb, aux


def run(grids, dec, rays_o, rays_d, stage, gt_depth, bound, g_depth, g_var, g_rgb, grad_grids=(), grad_decoders=(),
        n_samples=32, n_surface=16, coarse_enlarge=2, masks=None):
    """Forward + float64 autograd backward with the fixed cotangents g_depth / g_var / g_rgb (inputs are the float32 ones, promoted).
    Returns dict(depth, var, rgb, raw, pre, masks, d_rays_o, d_rays_d, d_grid_<level> (dense), d_dec {level: {name: grad}})."""
    ro = rays_o.detach().double().requires_grad_(True)
    rd = rays_d.detach().double().requires_grad_(True)
    g = {k: v.detach().double().requires_grad_(k in grad_grids) for k, v in grids.items()}
    dw = {lvl: {k: v.detach().double().requires_grad_(lvl in grad_decoders) for k, v in W.items()} for lvl, W in dec.items()}
    shapes = {lvl: tuple(g["grid_" + lvl].shape[2:]) for lvl in STAGE_GRIDS[stage]}
    fixed = decide(rays_o, rays_d, stage, gt_depth, bound, shapes, n_samples, n_surface, coarse_enlarge)
    d, u, c, aux = render_batch_ray(g, dw, rd, ro, stage, gt_depth, bound, masks=masks, fixed=fixed)
    ((d * g_depth.double()).sum() + (u * g_var.double()).sum() + (c * g_rgb.double()).sum()).backward()
    out = dict(depth=d.detach(), var=u.detach(), rgb=c.detach(), raw=aux["raw"], pre=aux["pre"], masks=aux["masks"], z_vals=aux["z_vals"],
               fixed=fixed, d_rays_o=ro.grad, d_rays_d=rd.grad)
    for k in grad_grids:
        out["d_" + k] = g[k].grad if g[k].grad is not None else torch.zeros_like(g[k])
    out["d_dec"] = {lvl: {k: v.grad if v.grad is not None else torch.zeros_like(v) for k, v in dw[lvl].items()} for lvl in grad_decoders}
    return out


# ----------------------------------------------------------------------------- the float32 port with its ReLU decisions
class _ReluSigns(TorchFunctionMode):
    def __init__(self):
        super().__init__()
        self.signs = []

    def __torch_function__(self, func, types, args=(), kwargs=None):
        if func is F.relu:
            self.signs.append(args[0].detach() > 0)
        return func(*args, **(kwargs or {}))


def port_run(grids, dec, rays_o, rays_d, stage, gt_depth, bound, g_depth, g_var, g_rgb, grad_grids=(), grad_decoders=(),
             n_samples=32, n_surface=16):
    """tp.render_batch_ray (float32) forward + backward with the same cotangents; also returns the port's per-point raw and its ReLU
    decisions as a mask [P,n_dec,5,32] (recorded from the F.relu calls, which run in STAGE_DECODERS order)."""
    ro = rays_o.detach().clone().requires_grad_(True)
    rd = rays_d.detach().clone().requires_grad_(True)
    g = {k: v.detach().clone().requires_grad_(k in grad_grids) for k, v in grids.items()}
    dw = {lvl: {k: v.detach().clone().requires_grad_(lvl in grad_decoders) for k, v in W.items()} for lvl, W in dec.items()}
    with _ReluSigns() as rec:
        d, u, c, aux = tp.render_batch_ray(g, dw, rd, ro, stage, gt_depth, bound, n_samples, n_surface, return_aux=True)
    ((d * g_depth).sum() + (u * g_var).sum() + (c * g_rgb).sum()).backward()
    n_dec = len(STAGE_DECODERS[stage])
    P = aux["raw"].shape[0] * aux["raw"].shape[1]
    masks = torch.stack(rec.signs, 1).reshape(P, n_dec, 5, 32)
    out = dict(depth=d.detach(), var=u.detach(), rgb=c.detach(), raw=aux["raw"], masks=masks, z_vals=aux["z_vals"],
               d_rays_o=ro.grad, d_rays_d=rd.grad)
    for k in grad_grids:
        out["d_" + k] = g[k].grad if g[k].grad is not None else torch.zeros_like(g[k])
    out["d_dec"] = {lvl: {k: v.grad if v.grad is not None else torch.zeros_like(v) for k, v in dw[lvl].items()} for lvl in grad_decoders}
    return out


def unpack_masks(words, n_dec):
    """The kernels' saved ReLU words [N,S,15] int32 (word 5 * dec_pos + layer, bit j = unit j) -> bool [P,n_dec,5,32]."""
    w = words.reshape(-1, 15)[:, : 5 * n_dec].long() & 0xFFFFFFFF
    bits = (w[..., None] >> torch.arange(32, device=w.device)) & 1
    return bits.bool().reshape(-1, n_dec, 5, 32)


# ----------------------------------------------------------------------------- error metrics
def errors(x, t):
    """Errors of x against the truth t: max-norm relative, L2 relative, and the per-element |x - t| / (|t| + 1e-3 max|t|) summarised by
    its maximum and 99.9th percentile over the elements where either side is non-zero (voxels no sample touches do not dilute it).
    An all-zero truth gives the absolute error in every metric."""
    x = torch.as_tensor(x).detach().double().cpu().reshape(-1)
    t = torch.as_tensor(t).detach().double().cpu().reshape(-1)
    e = (x - t).abs()
    tmax = float(t.abs().max()) if t.numel() else 0.0
    if tmax == 0.0:
        v = float(e.max()) if e.numel() else 0.0
        return dict(max=v, l2=v, pe_max=v, pe_999=v)
    sel = (t != 0) | (x != 0)
    pe = e[sel] / (t[sel].abs() + 1e-3 * tmax)
    k = max(1, int(0.999 * pe.numel() + 0.5))
    return dict(max=float(e.max()) / tmax, l2=float(e.norm() / t.norm()), pe_max=float(pe.max()), pe_999=float(pe.kthvalue(k).values))
