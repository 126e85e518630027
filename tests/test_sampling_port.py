"""CPU: the sampling port (tests/sampling_port.py: lindisp, perturb, importance sampling) against the fixtures the unmodified reference
produced (tests/golden/sampling/, tests/make_golden_sampling.py), bit for bit; and the ctypes mirror of nsb_sampling against the C struct."""
import ctypes as C
import glob
import os
import subprocess
import tempfile

import pytest
import torch

import sampling_port as spt
import scene_util as su

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = sorted(glob.glob(os.path.join(su.GOLDEN, "sampling", "*.pt")))
LV = {"coarse": ["coarse"], "middle": ["middle"], "fine": ["fine", "middle"], "color": ["fine", "color", "middle"]}


def load(path):
    case = torch.load(path, map_location="cpu", weights_only=False)
    sc = su.load_scenes()[case["scene"]]
    return case, sc, su.make_grids(sc, case["variant"]), su.load_decoders(case["variant"])


def test_all_sampling_fixtures_present():
    names = {os.path.basename(p)[:-3] for p in CASES}
    assert names == {"render_color_perturb", "render_coarse_perturb", "render_color_lindisp", "render_color_importance",
                     "render_color_importance_perturb", "render_coarse_importance"}


@pytest.mark.parametrize("path", CASES, ids=[os.path.basename(p)[:-3] for p in CASES])
def test_sampling_port_matches_reference_fixture(path):
    case, sc, grids, dec = load(path)
    bound = su.scene_bound(sc)
    stage = case["stage"]
    r = sc["rendering"]
    ro = case["rays_o"].clone().requires_grad_(True)
    rd = case["rays_d"].clone().requires_grad_(True)
    g = {k: v.clone().requires_grad_(k[5:] in LV[stage]) for k, v in grids.items()}
    dw = {n: {k: v.clone().requires_grad_(True) for k, v in W.items()} for n, W in dec.items()}
    d, u, c, aux = spt.render_batch_ray(g, dw, rd, ro, stage, case["gt_depth"], bound, r["N_samples"], r["N_surface"], lindisp=case["lindisp"],
                                        t_rand=case["t_rand"], n_importance=case["n_importance"], u=case["u_importance"], return_aux=True)
    assert torch.equal(aux["z_vals"], case["z_vals"])
    assert torch.equal(d.detach(), case["depth"]) and torch.equal(u.detach(), case["var"]) and torch.equal(c.detach(), case["rgb"])
    ((d * case["g_depth"]).sum() + (u * case["g_var"]).sum() + (c * case["g_rgb"]).sum()).backward()
    assert torch.equal(ro.grad, case["d_rays_o"]) and torch.equal(rd.grad, case["d_rays_d"])
    for k, summ in case["d_grid"].items():
        mine = su.grid_summary(g[k].grad)
        assert mine["nnz"] == summ["nnz"] and torch.equal(mine["val"], summ["val"])
    for lvl, gd in case["d_dec"].items():
        for k, v in gd.items():
            assert torch.equal(dw[lvl][k].grad, v), (lvl, k)
    if "zero_depth" in case:                       # lindisp rays with sensor depth 0: z = 0, NaN at t = 1 -> NaN depth, as the reference
        zd = case["zero_depth"]
        with torch.no_grad():
            d0, _, _, aux0 = spt.render_batch_ray(grids, dec, zd["rays_d"], zd["rays_o"], stage, zd["gt_depth"], bound, r["N_samples"],
                                                  r["N_surface"], lindisp=True, return_aux=True)
        assert torch.equal(aux0["z_vals"].isnan(), zd["z_vals"].isnan()) and torch.equal(d0.isnan(), zd["depth"].isnan())
        assert torch.equal(d0[~d0.isnan()], zd["depth"][~zd["depth"].isnan()])
        assert bool(zd["depth"].isnan().any()) and bool((zd["gt_depth"] > 0).any())


def test_sampling_struct_size_matches_the_header():
    """sizeof(_lib.Sampling) == sizeof(nsb_sampling), compiled with gcc."""
    from nice_slam_b200 import _lib
    prog = r'''
#include <stdio.h>
#include <stddef.h>
#include "nice_slam_b200.h"
int main(){ printf("%zu %zu %zu %zu\n", sizeof(nsb_sampling), offsetof(nsb_sampling, t_rand), offsetof(nsb_sampling, z_vals), offsetof(nsb_sampling, S)); return 0; }
'''
    with tempfile.TemporaryDirectory() as td:
        src = os.path.join(td, "s.c")
        open(src, "w").write(prog)
        exe = os.path.join(td, "s")
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), src, "-o", exe])
        got = [int(x) for x in subprocess.check_output([exe]).split()]
    S = _lib.Sampling
    assert got == [C.sizeof(S), S.t_rand.offset, S.z_vals.offset, S.S.offset]
