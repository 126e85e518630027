"""Generate tests/golden/sampling/*.pt: the UNMODIFIED reference Renderer.render_batch_ray (imported from the reference checkout through
tests/ref_harness.py) with the sampling settings of its `rendering:` block that the shipped NICE configs leave off -- perturb, lindisp
and N_importance (src/utils/Renderer.py:152-196) -- on room0 'soft', 96 rays, with autograd gradients for random output seeds.

    python tests/make_golden_sampling.py        # needs the reference checkout

The CPU generator is seeded before every call; the uniforms the reference draws (torch.rand, Renderer.py:165 and common.py:37) are
recorded, and so is the next draw after the call (the caller's random stream must advance the same way).  tests/sampling_port.py
reproduces every fixture bit for bit (asserted here).  The files live in a subdirectory: the render_*.pt cases of tests/golden/ are the
default sampler's.
"""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import make_golden as mg        # noqa: E402
import sampling_port as spt     # noqa: E402
import scene_util as su         # noqa: E402
from oracle import torch_port as tp   # noqa: E402

OUT = os.path.join(su.GOLDEN, "sampling")
LV = {"coarse": ["coarse"], "middle": ["middle"], "fine": ["fine", "middle"], "color": ["fine", "color", "middle"]}
PRIMARY = {"coarse": "grid_coarse", "middle": "grid_middle", "fine": "grid_fine", "color": "grid_fine"}
# name: (stage, perturb, lindisp, N_importance, rng seed)
CASES = {
    "render_color_perturb": ("color", 1.0, False, 0, 11),
    "render_coarse_perturb": ("coarse", 1.0, False, 0, 12),
    "render_color_lindisp": ("color", 0.0, True, 0, 13),
    "render_color_importance": ("color", 0.0, False, 12, 14),
    "render_color_importance_perturb": ("color", 1.0, False, 12, 15),
    "render_coarse_importance": ("coarse", 0.0, False, 12, 16),
}


def rays(sc, n, seed):
    """n rays with gt_depth > 0 (a lindisp ray without sensor depth has z = 0 / NaN; that case has its own block)."""
    ro, rd, gd, gc = su.make_rays(sc, 4 * n, seed=seed)
    keep = torch.nonzero(gd > 0).reshape(-1)[:n]
    assert keep.numel() == n
    ro, rd, gd = ro[keep].clone(), rd[keep].clone(), gd[keep].clone()
    ro[:8, 0] += 5.0               # some rays leave the bound early -> out-of-bound samples
    return ro, rd, gd


def reference_call(renderer, fn):
    """Run fn() with torch.rand recorded; returns (result, [drawn tensors])."""
    drawn = []
    _rand = torch.rand

    def rand_rec(*a, **k):
        r = _rand(*a, **k)
        drawn.append(r.clone())
        return r
    torch.rand = rand_rec
    try:
        out = fn()
    finally:
        torch.rand = _rand
    return out, drawn


def gen_case(name, stage, perturb, lindisp, n_imp, seed, sc, cfg, slam, renderer, n=96):
    renderer.perturb, renderer.lindisp, renderer.N_importance = perturb, lindisp, n_imp
    ns, nsf = cfg["rendering"]["N_samples"], cfg["rendering"]["N_surface"]
    ro, rd, gd = rays(sc, n, 3)
    gt = None if stage == "coarse" else gd
    ro1, rd1 = ro.clone().requires_grad_(True), rd.clone().requires_grad_(True)
    c = {k: v.clone().requires_grad_(k[5:] in LV[stage]) for k, v in slam.shared_c.items()}
    for p in slam.shared_decoders.parameters():
        p.grad = None
        p.requires_grad_(True)
    torch.manual_seed(seed)
    (d, u, col), drawn = reference_call(renderer, lambda: renderer.render_batch_ray(c, slam.shared_decoders, rd1, ro1, "cpu", stage, gt_depth=gt))
    next_draw = torch.rand(8)
    t_rand = drawn.pop(0) if perturb > 0 else None
    u_imp = drawn.pop(0) if (n_imp > 0 and perturb > 0) else None
    assert not drawn
    g = torch.Generator().manual_seed(55)
    gD = torch.randn(n, generator=g, dtype=torch.float64)
    gV = torch.randn(n, generator=g, dtype=torch.float64) * 3
    gC = torch.randn(n, 3, generator=g)
    ((d * gD).sum() + (u * gV).sum() + (col * gC).sum()).backward()
    # the port on the recorded uniforms: bit-identical outputs
    d2, u2, c2, aux = spt.render_batch_ray(slam.shared_c, tp.decoders_state(slam.shared_decoders), rd, ro, stage, gt, slam.bound, ns, nsf,
                                           lindisp=lindisp, t_rand=t_rand, n_importance=n_imp, u=u_imp, return_aux=True)
    assert torch.equal(d2, d.detach()) and torch.equal(u2, u.detach()) and torch.equal(c2, col.detach()), name
    z = aux["z_vals"]
    pts = (ro[:, None, :] + rd[:, None, :] * z[:, :, None]).reshape(-1, 3)
    bnd = slam.bound * 2 if stage == "coarse" else slam.bound
    cidx = mg.corner_indices(pts, bnd, sc["shapes"][PRIMARY[stage]]).reshape(n, -1, 3)
    case = dict(scene="room0", variant="soft", stage=stage, perturb=perturb, lindisp=lindisp, n_importance=n_imp, seed=seed,
                t_rand=t_rand, u_importance=u_imp, next_draw=next_draw,
                rays_o=ro, rays_d=rd, gt_depth=gt, g_depth=gD, g_var=gV, g_rgb=gC,
                depth=d.detach(), var=u.detach(), rgb=col.detach(), z_vals=z, corner_idx=cidx,
                z_vals0=aux.get("z_vals0"), d_rays_o=ro1.grad, d_rays_d=rd1.grad,
                d_grid={k: su.grid_summary(c[k].grad) for k in c if c[k].grad is not None},
                d_dec={l: {k: v.grad.clone() for k, v in getattr(slam.shared_decoders, l + "_decoder").named_parameters()
                           if v.grad is not None} for l in LV[stage]})
    if lindisp:
        # forward-only block with sensor depth 0 on half of the rays: 1/near = inf -> z = 0, and NaN at t = 1 (the reference's behaviour)
        ro0, rd0, gd0 = ro[:32].clone(), rd[:32].clone(), gd[:32].clone()
        gd0[::2] = 0.0
        with torch.no_grad():
            d0, u0, c0 = renderer.render_batch_ray(slam.shared_c, slam.shared_decoders, rd0, ro0, "cpu", stage, gt_depth=gd0)
            d3, u3, c3, aux0 = spt.render_batch_ray(slam.shared_c, tp.decoders_state(slam.shared_decoders), rd0, ro0, stage, gd0, slam.bound,
                                                    ns, nsf, lindisp=True, return_aux=True)
        assert torch.equal(d3.isnan(), d0.isnan()) and torch.equal(d3[~d3.isnan()], d0[~d0.isnan()])
        assert bool(d0.isnan().any())
        case["zero_depth"] = dict(rays_o=ro0, rays_d=rd0, gt_depth=gd0, depth=d0, var=u0, rgb=c0, z_vals=aux0["z_vals"])
    renderer.perturb, renderer.lindisp, renderer.N_importance = 0.0, False, 0
    return case


def main():
    import warnings
    warnings.filterwarnings("ignore")
    os.makedirs(OUT, exist_ok=True)
    sc, cfg, slam, renderer = mg.ref_scene("room0", "soft")
    for name, (stage, perturb, lindisp, n_imp, seed) in CASES.items():
        case = gen_case(name, stage, perturb, lindisp, n_imp, seed, sc, cfg, slam, renderer)
        path = os.path.join(OUT, name + ".pt")
        torch.save(case, path)
        print("wrote sampling/%-36s %8.1f KB" % (name + ".pt", os.path.getsize(path) / 1024))


if __name__ == "__main__":
    main()
