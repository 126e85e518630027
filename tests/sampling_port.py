"""ORACLE (test infrastructure): the reference's other sampling settings on top of oracle/torch_port.py -- lindisp, perturb with
given uniforms, and hierarchical importance sampling (src/utils/Renderer.py:152-196, sample_pdf src/common.py:19-63) -- with the
same torch ops in the same order and dtypes.  tests/make_golden_sampling.py asserts bit-identity with the unmodified reference on
every fixture it writes (tests/golden/sampling/); tests/test_sampling_port.py re-checks it against them.

The random draws are inputs here: t_rand [N, n_samples] (torch.rand(z_vals.shape), Renderer.py:165) and, for importance sampling
with perturb > 0, u [N, n_importance] (common.py:37).
"""
import torch

from oracle import torch_port as tp


def sample_z_vals(rays_o, rays_d, gt_depth, bound, n_samples, n_surface, stage, lindisp=False, t_rand=None):
    """torch_port.sample_z_vals plus lindisp (Renderer.py:154-157) and the perturb jitter (:159-166) before the merge."""
    if stage == "coarse":
        gt_depth = None
    if gt_depth is None:
        n_surface = 0
        near = 0.01
    else:
        gt_depth = gt_depth.reshape(-1, 1)
        near = gt_depth.repeat(1, n_samples) * 0.01
    with torch.no_grad():
        o = rays_o.detach().unsqueeze(-1)
        d = rays_d.detach().unsqueeze(-1)
        t = (bound.unsqueeze(0) - o) / d
        far_bb, _ = torch.min(torch.max(t, dim=2)[0], dim=1)
        far_bb = far_bb.unsqueeze(-1)
        far_bb += 0.01
    far = torch.clamp(far_bb, 0, torch.max(gt_depth * 1.2)) if gt_depth is not None else far_bb
    if n_surface > 0:
        nz = gt_depth > 0
        g = gt_depth[nz].unsqueeze(-1).repeat(1, n_surface)
        ts = torch.linspace(0., 1., steps=n_surface).double()
        z_nz = 0.95 * g * (1. - ts) + 1.05 * g * ts
        z_surf = torch.zeros(gt_depth.shape[0], n_surface).double()
        nz = nz.squeeze(-1)
        z_surf[nz, :] = z_nz
        z_zero = 0.001 * (1. - ts) + torch.max(gt_depth) * ts
        z_surf[~nz, :] = z_zero
    tv = torch.linspace(0., 1., steps=n_samples)
    if lindisp:
        z_vals = 1. / (1. / near * (1. - tv) + 1. / far * tv)
    else:
        z_vals = near * (1. - tv) + far * tv
    if t_rand is not None:
        mids = .5 * (z_vals[..., 1:] + z_vals[..., :-1])
        upper = torch.cat([mids, z_vals[..., -1:]], -1)
        lower = torch.cat([z_vals[..., :1], mids], -1)
        z_vals = lower + (upper - lower) * t_rand
    if n_surface > 0:
        z_vals, _ = torch.sort(torch.cat([z_vals, z_surf.double()], -1), -1)
    return z_vals


def sample_pdf(bins, weights, n_importance, u=None):
    """Inverse-cdf sampling of common.py:19-63.  u None: torch.linspace(0, 1, n_importance) (det=True); else the given [N, n] uniforms.
    Works in the dtypes of its inputs (float32 weights in the reference; the tests also run it in float64)."""
    weights = weights + 1e-5
    pdf = weights / torch.sum(weights, -1, keepdim=True)
    cdf = torch.cumsum(pdf, -1)
    cdf = torch.cat([torch.zeros_like(cdf[..., :1]), cdf], -1)
    if u is None:
        u = torch.linspace(0., 1., steps=n_importance).expand(list(cdf.shape[:-1]) + [n_importance])
    u = u.to(cdf.dtype).contiguous()
    inds = torch.searchsorted(cdf, u, right=True)
    below = torch.max(torch.zeros_like(inds - 1), inds - 1)
    above = torch.min((cdf.shape[-1] - 1) * torch.ones_like(inds), inds)
    inds_g = torch.stack([below, above], -1)
    shape = [inds_g.shape[0], inds_g.shape[1], cdf.shape[-1]]
    cdf_g = torch.gather(cdf.unsqueeze(1).expand(shape), 2, inds_g)
    bins_g = torch.gather(bins.unsqueeze(1).expand(shape), 2, inds_g)
    denom = cdf_g[..., 1] - cdf_g[..., 0]
    denom = torch.where(denom < 1e-5, torch.ones_like(denom), denom)
    t = (u - cdf_g[..., 0]) / denom
    return bins_g[..., 0] + t * (bins_g[..., 1] - bins_g[..., 0])


def render_batch_ray(grids, dec, rays_d, rays_o, stage, gt_depth, bound, n_samples=32, n_surface=16, lindisp=False, t_rand=None,
                     n_importance=0, u=None, return_aux=False):
    """Renderer.render_batch_ray (Renderer.py:63-198) with the sampling settings.  With n_importance > 0 the outputs are those of the
    second pass; aux holds the final z_vals and, as z_vals0 / weights0, the first pass's samples and weights."""
    n_rays = rays_o.shape[0]
    z_vals = sample_z_vals(rays_o, rays_d, gt_depth, bound, n_samples, n_surface, stage, lindisp, t_rand)
    pts = rays_o[..., None, :] + rays_d[..., None, :] * z_vals[..., :, None]
    raw = tp.eval_points(pts.reshape(-1, 3), grids, dec, stage, bound).reshape(n_rays, z_vals.shape[1], -1)
    depth, var, rgb, weights = tp.composite(raw, z_vals)
    aux = dict(z_vals=z_vals, weights=weights)
    if n_importance > 0:
        z_mid = .5 * (z_vals[..., 1:] + z_vals[..., :-1])
        z_samples = sample_pdf(z_mid, weights[..., 1:-1], n_importance, u).detach()
        aux.update(z_vals0=z_vals, weights0=weights.detach())
        z_vals, _ = torch.sort(torch.cat([z_vals, z_samples], -1), -1)
        pts = rays_o[..., None, :] + rays_d[..., None, :] * z_vals[..., :, None]
        raw = tp.eval_points(pts.reshape(-1, 3), grids, dec, stage, bound).reshape(n_rays, z_vals.shape[1], -1)
        depth, var, rgb, weights = tp.composite(raw, z_vals)
        aux.update(z_vals=z_vals, weights=weights)
    if return_aux:
        return depth, var, rgb, aux
    return depth, var, rgb
