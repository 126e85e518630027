"""GPU: a whole Mapper.optimize_map call through mapping.FusedMapper -- its window sampler (nsb_map_samples) against the reference's per-row
get_samples + torch.cat + bbox pre-filter restated, whole calls against the real runs of tests/make_golden_mapper_frames.py, the random
draws it makes, and its errors."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import scene_util as su
from gpu_util import make_renderer, rel
from oracle import torch_port as tp

pytestmark = pytest.mark.gpu
DEV = "cuda"
VP = C.c_void_p
GOLD = os.path.join(su.GOLDEN, "mapper_frames")
CASES = ("ba_overlap", "no_ba", "first_frame", "coarse")
TOL = 1e-4                                  # test_gpu_parity's bar for one render on the same inputs


@pytest.fixture(scope="module")
def room0():
    return su.load_scenes()["room0"]


def fresh(sc):
    renderer, c, dec = make_renderer(sc, su.make_grids(sc, "soft"), su.load_decoders("soft"), DEV)
    return renderer, c, dec


def store_with(sc, seeds):
    from nice_slam_b200.keyframes import KeyframeStore
    cam = sc["cam"]
    store = KeyframeStore(cam["H"], cam["W"], cam["fx"], cam["fy"], cam["cx"], cam["cy"], DEV, capacity=2)
    for k, s in enumerate(seeds):
        depth, color = su.make_frame(sc, s)
        store.append(5 * k, color, depth, su.make_pose(sc, s))
    return store


def test_window_sampler_matches_per_row_get_samples_and_prefilter(room0):
    """nsb_map_samples on 5 rows x 333 draws (1665 > 1024: two compaction rounds, row boundaries inside warps) against per-row
    get_samples + cat + bbox pre-filter: kept mask, order, count and row offsets exact, depth / colour bit-exact, rays within the
    nsb_window_rays bars, dirs exact.  Rows mix camera tensors (one with a non-unit quaternion) and fixed poses and read four store slots;
    one slot has a band of far depths, another only far depths, so its row loses every ray."""
    from nice_slam_b200 import _lib
    from nice_slam_b200.mapping import tensor_from_c2w
    L = _lib.lib()
    sc = room0
    cam = sc["cam"]
    H, W = cam["H"], cam["W"]
    store = store_with(sc, [30, 31, 32])
    depth, color = su.make_frame(sc, 33)
    depth[200:260] = 40.0
    store.append(15, color, depth, su.make_pose(sc, 33))
    gone = store.stage(color, torch.full_like(depth, 1e6))               # slot 4: every ray exits the bound before its depth
    slots = torch.tensor([0, 3, gone, 1, 3], dtype=torch.int32)
    cam_row = torch.tensor([0, -1, 1, -1, 2], dtype=torch.int32)
    poses = torch.stack([su.make_pose(sc, s)[:3] for s in (40, 41, 42, 43, 44)])
    cams = torch.stack([tensor_from_c2w(poses[r]) for r in (0, 2, 4)])
    cams[1, :4] *= 1.04
    F, n = 5, 333
    draws = torch.randint(H * W, (F, n), generator=torch.Generator().manual_seed(12))
    out = {k: torch.full((F * n, 3), float("nan"), device=DEV) for k in ("ro", "rd", "dirs", "gc")}
    gd = torch.full((F * n,), float("nan"), device=DEV)
    offs = torch.full((F + 1,), -7, dtype=torch.int32, device=DEV)
    count = torch.zeros(1, dtype=torch.int32, device=DEV)
    d = {k: v.to(DEV).contiguous() for k, v in dict(draws=draws, slots=slots, cam_row=cam_row, cams=cams, fixed=poses.reshape(F, 12)).items()}
    b6 = (C.c_double * 6)(*su.scene_bound(sc).reshape(6).tolist())
    _lib.check(L.nsb_map_samples(VP(d["draws"].data_ptr()), F, n, VP(d["slots"].data_ptr()), VP(store.depth.data_ptr()), VP(store.color.data_ptr()),
                                 H, W, VP(d["cams"].data_ptr()), VP(d["cam_row"].data_ptr()), VP(d["fixed"].data_ptr()), cam["fx"], cam["fy"],
                                 cam["cx"], cam["cy"], b6, VP(out["ro"].data_ptr()), VP(out["rd"].data_ptr()), VP(out["dirs"].data_ptr()),
                                 VP(gd.data_ptr()), VP(out["gc"].data_ptr()), VP(offs.data_ptr()), VP(count.data_ptr()), None), "nsb_map_samples")
    # restatement: Mapper.py:437-481 -- per row get_samples(0, H, 0, W, ...) under its pose, cat, pre-filter
    sd, scol = store.depth.cpu(), store.color.cpu()
    ro, rd, dirs, wgd, wgc = [], [], [], [], []
    for f in range(F):
        k = draws[f]
        i, j = (k % W).float(), (k // W).float()
        pose = tp.camera_from_tensor(cams[cam_row[f]]) if cam_row[f] >= 0 else poses[f]
        o, dd = tp.rays_from_uv(i, j, pose, cam["fx"], cam["fy"], cam["cx"], cam["cy"])
        ro.append(o); rd.append(dd)
        dirs.append(torch.stack([(i - cam["cx"]) / cam["fx"], -(j - cam["cy"]) / cam["fy"], -torch.ones_like(i)], -1))
        wgd.append(sd[int(slots[f])].reshape(-1)[k]); wgc.append(scol[int(slots[f])].reshape(-1, 3)[k])
    ro, rd, dirs, wgd, wgc = (torch.cat(x) for x in (ro, rd, dirs, wgd, wgc))
    keep = tp.bbox_prefilter(ro, rd, wgd, su.scene_bound(sc))
    kept = int(count.item())
    per_row = keep.view(F, n).sum(1)
    assert kept == int(keep.sum()) and 0 < kept < F * n
    assert int(per_row[2]) == 0 and bool((per_row[[0, 1, 3, 4]] > 0).all()), per_row
    want_offs = torch.cat([torch.zeros(1, dtype=torch.long), per_row.cumsum(0)]).int()
    assert torch.equal(offs.cpu(), want_offs), (offs.cpu(), want_offs)
    assert torch.equal(gd[:kept].cpu(), wgd[keep]) and torch.equal(out["gc"][:kept].cpu(), wgc[keep])
    assert float((out["ro"][:kept].cpu() - ro[keep]).abs().max()) <= 1e-6 and float((out["rd"][:kept].cpu() - rd[keep]).abs().max()) <= 2e-6
    assert torch.equal(out["dirs"][:kept].cpu(), dirs[keep])
    # the rays are nsb_window_rays' to the bit (same device code), on the kept rays' pixels
    pi = (draws.reshape(-1) % W).float()[keep].to(DEV).contiguous(); pj = (draws.reshape(-1) // W).float()[keep].to(DEV).contiguous()
    fid = torch.arange(F, dtype=torch.int32).repeat_interleave(n)[keep].to(DEV).contiguous()
    c2w, wro, wrd = torch.empty(F, 12, device=DEV), torch.empty(kept, 3, device=DEV), torch.empty(kept, 3, device=DEV)
    _lib.check(L.nsb_window_rays(VP(d["cams"].data_ptr()), VP(d["cam_row"].data_ptr()), VP(d["fixed"].data_ptr()), F, VP(pi.data_ptr()), VP(pj.data_ptr()),
                                 VP(fid.data_ptr()), kept, cam["fx"], cam["fy"], cam["cx"], cam["cy"], VP(c2w.data_ptr()), VP(wro.data_ptr()),
                                 VP(wrd.data_ptr()), None, None), "nsb_window_rays")
    assert torch.equal(out["ro"][:kept], wro) and torch.equal(out["rd"][:kept], wrd)


def test_track_sampler_still_gives_window_rays_bits(room0):
    """After nsb_track_samples moved onto the shared sampler loop: on the inputs of test_gpu_tracking's sampler test, its rays are
    nsb_window_rays' to the bit, and its kept set, order, samples and dirs are the restatement's exactly."""
    from nice_slam_b200 import _lib
    from nice_slam_b200.mapping import tensor_from_c2w
    L = _lib.lib()
    sc = room0
    cam = sc["cam"]
    H, W = cam["H"], cam["W"]
    H0, H1, W0, W1 = 30, H - 45, 70, W - 10
    depth, color = su.make_frame(sc, 3)
    depth[200:260] = 40.0
    camera = tensor_from_c2w(su.make_pose(sc, 3))
    camera[:4] *= 1.03
    n, Wr = 3000, W1 - W0
    draws = torch.randint((H1 - H0) * Wr, (n,), generator=torch.Generator().manual_seed(8))
    d = dict(cam=camera.to(DEV), draws=draws.to(DEV), depth=depth.to(DEV), color=color.to(DEV))
    ro, rd, dirs = (torch.full((n, 3), float("nan"), device=DEV) for _ in range(3))
    gd = torch.full((n,), float("nan"), device=DEV)
    gc = torch.full((n, 3), float("nan"), dtype=torch.float64, device=DEV)
    kept = torch.full((n,), -1, dtype=torch.int32, device=DEV)
    count = torch.zeros(1, dtype=torch.int32, device=DEV)
    b6 = (C.c_double * 6)(*su.scene_bound(sc).reshape(6).tolist())
    _lib.check(L.nsb_track_samples(VP(d["cam"].data_ptr()), VP(d["draws"].data_ptr()), n, VP(d["depth"].data_ptr()), VP(d["color"].data_ptr()), H, W,
                                   H0, H1, W0, W1, cam["fx"], cam["fy"], cam["cx"], cam["cy"], b6, VP(ro.data_ptr()), VP(rd.data_ptr()),
                                   VP(dirs.data_ptr()), VP(gd.data_ptr()), VP(gc.data_ptr()), VP(kept.data_ptr()), VP(count.data_ptr()), None),
               "nsb_track_samples")
    k = int(count.item())
    i, j = (W0 + draws % Wr).float(), (H0 + draws // Wr).float()
    wro, wrd = tp.rays_from_uv(i, j, tp.camera_from_tensor(camera), cam["fx"], cam["fy"], cam["cx"], cam["cy"])
    keep = tp.bbox_prefilter(wro, wrd, depth[H0:H1, W0:W1].reshape(-1)[draws], su.scene_bound(sc))
    assert k == int(keep.sum()) and torch.equal(kept[:k].cpu().long(), torch.nonzero(keep).reshape(-1))
    assert torch.equal(gd[:k].cpu(), depth[H0:H1, W0:W1].reshape(-1)[draws][keep])
    assert torch.equal(gc[:k].cpu(), color[H0:H1, W0:W1].reshape(-1, 3)[draws][keep])
    want_dirs = torch.stack([(i - cam["cx"]) / cam["fx"], -(j - cam["cy"]) / cam["fy"], -torch.ones_like(i)], -1)
    assert torch.equal(dirs[:k].cpu(), want_dirs[keep])
    cam_row = torch.zeros(1, dtype=torch.int32, device=DEV)
    pi, pj = i[keep].to(DEV).contiguous(), j[keep].to(DEV).contiguous()
    fid = torch.zeros(k, dtype=torch.int32, device=DEV)
    c2w, wro_d, wrd_d = torch.empty(12, device=DEV), torch.empty(k, 3, device=DEV), torch.empty(k, 3, device=DEV)
    _lib.check(L.nsb_window_rays(VP(d["cam"].data_ptr()), VP(cam_row.data_ptr()), None, 1, VP(pi.data_ptr()), VP(pj.data_ptr()), VP(fid.data_ptr()), k,
                                 cam["fx"], cam["fy"], cam["cx"], cam["cy"], VP(c2w.data_ptr()), VP(wro_d.data_ptr()), VP(wrd_d.data_ptr()), None, None),
               "nsb_window_rays")
    assert torch.equal(ro[:k], wro_d) and torch.equal(rd[:k], wrd_d)


def load(name):
    return torch.load(os.path.join(GOLD, name + ".pt"), map_location="cpu", weights_only=False)


def mapper_for(case, sc, renderer, c, dec, store):
    from nice_slam_b200 import FusedMapper
    return FusedMapper(renderer, c, dec, store, coarse_mapper=case["coarse_mapper"], **case["settings"])


@pytest.mark.parametrize("name", CASES)
def test_whole_call_against_real_optimize_map(room0, name):
    """One optimize_map call with the reference's recorded draws and window: the first iteration's loss within TOL (its inputs are the
    reference's), the window and stage schedule the reference used, every loss within 5 %; afterwards poses within 0.1 x the reference's
    update with the fixed row unchanged, the store's w2c the inverse of the written-back poses, > 99 % of the sampled voxels and decoder
    parameters within 2e-3 (1 + |v|), and every voxel outside the selection untouched.  The first frame runs at lr_first_factor = 5 times
    the rates: its voxels are held to 1e-2 (1 + |v|) for > 97 %, its decoders only through the losses."""
    from nice_slam_b200.masked import MaskedVoxels, frustum_voxel_mask
    case = load(name)
    sc = room0
    renderer, c, dec = fresh(sc)
    start = {k: v.clone() for k, v in c.items()}
    store = store_with(sc, case["keyframe_seeds"])
    mapper = mapper_for(case, sc, renderer, c, dec, store)
    depth, color = su.make_frame(sc, case["frame_seed"])
    c2w = su.make_pose(sc, case["frame_seed"])
    F = case["draws"].shape[1]
    got = mapper.map_frame(case["iters"], case["lr_factor"], color, depth, c2w, case["ba"], draws=case["draws"], selection=case["selection"])
    K = len(case["keyframe_seeds"])
    assert mapper.window == [*case["selection"], *([K - 1] if K else []), -1] and len(mapper.window) == F
    assert mapper.stages == case["stages"] and mapper.pixs_per_image == case["settings"]["pixels"] // F
    losses = mapper.losses.cpu()
    want = case["losses"]
    assert abs(float(losses[0]) - float(want[0])) <= TOL * abs(float(want[0])), (losses[0], want[0])
    assert bool(torch.isfinite(losses).all()) and float(((losses - want).abs() / want.abs()).max()) < 0.05, (losses, want)
    if case["ba"]:
        fixed = mapper.fixed_row
        rows = mapper.window
        start_pose = torch.stack([su.make_pose(sc, case["keyframe_seeds"][k]) if k >= 0 else c2w for k in rows])
        want_pose = torch.stack([case["keyframe_est_c2w"][k] if k >= 0 else case["cur_c2w"] for k in rows])
        got_pose = torch.stack([store.est_c2w[k] if k >= 0 else got.cpu() for k in rows])
        assert torch.equal(got_pose[fixed], start_pose[fixed])
        for r in range(F):
            if r == fixed:
                continue
            upd = float((want_pose[r] - start_pose[r]).norm())
            assert float((got_pose[r] - want_pose[r]).norm()) < 0.1 * upd, (r, float((got_pose[r] - want_pose[r]).norm()), upd)
        for k in range(K):
            assert float((store.w2c[k].cpu().view(4, 4) @ store.est_c2w[k] - torch.eye(4)).abs().max()) < 1e-5
        assert got.shape == (4, 4) and torch.equal(got[3].cpu(), torch.tensor([0.0, 0.0, 0.0, 1.0]))
    else:
        assert got is None
    # Adam's first steps are sign-like and the losses are L1: a voxel whose gradient sits within rounding of zero can step the other way,
    # by up to its learning rate, which the first frame's lr_first_factor (5) multiplies -- there ~2 % of the middle grid's sampled voxels
    # land outside 1e-2 (1 + |v|) of the reference, against < 1 % at 2e-3 (1 + |v|) in the calls at lr_factor 1
    bar, share = (2e-3, 0.99) if case["lr_factor"] <= 1 else (2e-3 * case["lr_factor"], 0.97)
    for key, fin in case["final"].items():
        sel = frustum_voxel_mask(renderer, c2w, key, c[key], depth.to(DEV))
        mv = MaskedVoxels(c[key], sel)
        after = mv.to_reference(mv.gather(c[key])).cpu()
        close = (after[fin["idx"].long()] - fin["val"]).abs() <= bar * (1 + fin["val"].abs())
        assert float(close.float().mean()) > share, (key, float(close.float().mean()))
        outside = (~sel).view(1, 1, *sel.shape).expand_as(c[key])
        assert torch.equal(c[key][outside], start[key][outside]), key
    if case["lr_factor"] > 1:
        return                                  # sign-like steps at 5x the rate leave ~half the colour decoder's weights a rate apart
    for lvl, want_dec in case["decoders"].items():
        mine = {k: v.detach().cpu() for k, v in getattr(dec, lvl + "_decoder").state_dict().items()}
        for k, v in want_dec.items():
            close = (mine[k].reshape(v.shape) - v).abs() <= 2e-3 * (1 + v.abs())
            assert float(close.float().mean()) > 0.99, (lvl, k, float(close.float().mean()))


def test_default_draws_follow_the_reference_randint_sequence(room0):
    """Without draws and selection, map_frame makes the reference's random calls in its order: the overlap selection's
    torch.randint(H*W, (100,)) and numpy permutation, then per iteration one torch.randint(H*W, (pixs_per_image,)) per window row.  After
    the same seed the CUDA generator is where that sequence of direct calls leaves it; replaying the sequence as draws and selection
    consumes nothing and gives the same call: the same window and first loss to the bit; the later losses to 1e-6 and the grids to the
    whole-call bar, since the backward's gradient sums are not bit-reproducible run to run."""
    from nice_slam_b200 import FusedMapper
    sc = room0
    s = dict(load("no_ba")["settings"], pixels=300)
    H, W = sc["cam"]["H"], sc["cam"]["W"]
    depth, color = su.make_frame(sc, 50)
    c2w = su.make_pose(sc, 50)

    def run(**kw):
        renderer, c, dec = fresh(sc)
        mapper = FusedMapper(renderer, c, dec, store_with(sc, [10, 11, 12]), **s)
        mapper.map_frame(4, 1.0, color, depth, c2w, False, **kw)
        return mapper, {k: v.clone() for k, v in c.items()}
    torch.cuda.manual_seed(99); np.random.seed(99)
    m0, g0 = run()
    state = torch.cuda.get_rng_state()
    F, ppi = len(m0.window), m0.pixs_per_image
    torch.cuda.manual_seed(99)
    torch.randint(H * W, (100,), device=DEV)
    draws = torch.stack([torch.stack([torch.randint(H * W, (ppi,), device=DEV) for _ in range(F)]) for _ in range(4)])
    assert torch.equal(torch.cuda.get_rng_state(), state)
    m1, g1 = run(draws=draws, selection=m0.window[:-2])
    assert torch.equal(torch.cuda.get_rng_state(), state)
    assert m1.window == m0.window and float(m1.losses[0]) == float(m0.losses[0])
    assert rel(m1.losses, m0.losses) < 1e-6, (m0.losses, m1.losses)
    for k in g0:                              # the whole-call bar: sign-like Adam steps amplify the rounding of a few voxels
        close = (g1[k] - g0[k]).abs() <= 2e-3 * (1 + g0[k].abs())
        assert float(close.float().mean()) > 0.99, (k, float(close.float().mean()))


def test_errors(room0):
    """Bundle adjustment in the coarse mapper, a window wider than the pixel budget, and an iteration whose pre-filter keeps no ray raise."""
    from nice_slam_b200 import FusedMapper
    sc = room0
    case = load("no_ba")
    renderer, c, dec = fresh(sc)
    depth, color = su.make_frame(sc, 2)
    c2w = su.make_pose(sc, 2)
    coarse = FusedMapper(renderer, c, dec, store_with(sc, []), coarse_mapper=True, **case["settings"])
    with pytest.raises(RuntimeError, match="coarse mapper"):
        coarse.map_frame(2, 1.0, color, depth, c2w, True)
    narrow = FusedMapper(renderer, c, dec, store_with(sc, [10, 11, 12]), **dict(case["settings"], pixels=3))
    with pytest.raises(RuntimeError, match="no pixel per row"):
        narrow.map_frame(2, 1.0, color, depth, c2w, False, selection=[0, 1])
    empty = FusedMapper(renderer, c, dec, store_with(sc, []), **case["settings"])
    with pytest.raises(RuntimeError, match="kept no ray"):
        empty.map_frame(2, 1.0, color, torch.full_like(depth, 1e6), c2w, False)
