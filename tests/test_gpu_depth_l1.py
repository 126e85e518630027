"""GPU: the 2D reconstruction metric (recon.eval_depth_l1, nice_slam_b200.depth, nsb_depth.cu) against the float64 oracle
(oracle/depth_l1.py): the rasterizer pixel by pixel on room0 meshes, watertightness on a box room, the metric per view, the view sampler's
accept / reject decisions against check_proj, bit-identical repeats, the CLI and input checks."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

import scene_util as su
from cull_scene import box_room, room_poses
from gpu_util import make_renderer
from oracle import depth_l1 as od
from test_gpu_recon import mesh_cfg, moved

pytestmark = pytest.mark.gpu
DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD_LOG = os.path.join(ROOT, "nice_slam_b200", "csrc", "build.log")


@pytest.fixture(scope="module")
def room():
    """room0's 'soft' grids meshed at resolutions 64 and 128 (as test_gpu_recon.py's fixture): {R: (vertices f64, faces int64)}."""
    from nice_slam_b200.mesh import FusedMesher
    sc = su.load_scenes()["room0"]
    renderer, c, dec = make_renderer(sc, su.make_grids(sc, "soft"), su.load_decoders("soft"), DEV)
    out = {}
    with torch.no_grad():
        for R in (64, 128):
            m = FusedMesher(renderer, mesh_cfg(R))
            v, f, _ = m.marching_cubes(m.lattice(c, dec, None))
            out[R] = (v.cpu().numpy(), f.cpu().numpy().astype(np.int64))
    return out


def f32_ulp(x):
    return np.spacing(np.abs(np.asarray(x, np.float32))).astype(np.float64)


def compare(gpu, v, f, c2w, H, W, fx, fy, cx, cy, zn, zf=20.0):
    """The GPU depth [H,W] against the oracle: non-ambiguous pixels both background or within 1 float32 ulp; ambiguous ones 0 or within
    1 ulp of a face that may cover them.  -> (the oracle's image with each ambiguous pixel replaced by the GPU's value, ambiguous count)."""
    want, amb, cand = od.raycast(v, f, c2w, H, W, fx, fy, cx, cy, zn, zf)
    g = gpu.astype(np.float64)
    ok = ~amb
    assert np.array_equal(g[ok] == 0, want[ok] == 0), np.argwhere(ok & ((g == 0) != (want == 0)))[:5]
    hit = ok & (want > 0)
    assert np.all(np.abs(g[hit] - want[hit]) <= f32_ulp(want[hit]))
    for p, zs in cand.items():
        i, j = divmod(p, W)
        assert g[i, j] == 0 or np.abs(np.array(zs) - g[i, j]).min() <= f32_ulp(g[i, j]), (i, j, g[i, j], zs)
    out = np.where(amb, g, np.asarray(want, np.float32).astype(np.float64))
    return out, int(amb.sum())


def room_views(v, n, seed, near_wall):
    """c2w [n,4,4] inside room0's mesh: candidates of the metric's sampling box, and with near_wall, cameras 2-4 cm from a vertex looking
    along a random direction (walls cross the near plane, faces lie behind the camera)."""
    from nice_slam_b200 import depth as dp
    rng = np.random.default_rng(seed)
    ext, T = dp.sampling_box(v)
    c2w = dp.candidates(rng.random((n, 6)), ext, T)
    if near_wall:
        k = rng.integers(0, len(v), n)
        pos = v[k] + rng.normal(size=(n, 3)) * 0.02
        c2w = dp.view_matrix(rng.normal(size=(n, 3)), dp.UP, pos)
    return c2w


# ------------------------------------------------------------------------------------------------ the rasterizer
@pytest.mark.parametrize("res", [64, 128])
def test_rasterizer_matches_oracle_on_room0(room, res):
    from nice_slam_b200 import depth as dp
    v, f = room[res]
    H, W = 48, 64
    fx = fy = 300.0 * W / 500
    cx, cy = W / 2 - 0.5, H / 2 - 0.5
    zn = dp.default_z_near(v)
    c2w = np.concatenate([room_views(v, 4, res, False), room_views(v, 4, res + 1, True)])
    got = dp.render_depth(v, f, c2w, H, W, fx, fy, cx, cy).cpu().numpy()
    n_amb, n_hit = 0, 0
    for k in range(len(c2w)):
        _, a = compare(got[k], v, f, c2w[k], H, W, fx, fy, cx, cy, zn)
        n_amb += a
        n_hit += int((got[k] > 0).sum())
    print("room0@%d: %d ambiguous pixels of %d, %d hits" % (res, n_amb, len(c2w) * H * W, n_hit))
    assert n_hit > len(c2w) * H * W // 4
    assert n_amb < 50


def analytic_box_depth(c2w, size, H, W, fx, fy, cx, cy):
    """z of every pixel's ray from inside the box [0, size]: the least exit distance over the axes, in float64."""
    j, i = np.meshgrid(np.arange(W, dtype=np.float64), np.arange(H, dtype=np.float64))
    d = np.stack([(j - cx) / fx, (i - cy) / fy, np.ones_like(j)], -1)
    dw = d @ c2w[:3, :3].T
    o = c2w[:3, 3]
    with np.errstate(divide="ignore"):
        t = np.where(dw > 0, (np.asarray(size) - o) / dw, np.where(dw < 0, -o / dw, np.inf))
    return t.min(-1)


def test_box_room_is_watertight_at_500x500():
    from nice_slam_b200 import depth as dp
    size = (4.0, 3.0, 2.5)
    v, f = box_room(0.25, size)
    views = [((1.0, 0.0, 0.0), (2.0, 1.5, 1.25)),                     # the centre, axis-aligned: pixel centres fall on edges and vertices
             ((0.0, 1.0, 0.0), (2.0, 1.5, 1.25)),
             ((-1.0, 0.0, 0.0), (0.05, 1.5, 1.25)),                   # 5 cm from a wall, facing it
             ((0.0, 1.0, 0.0), (0.05, 0.75, 1.0)),                    # 5 cm from a wall, looking along it
             ((1.0, 1.0, 0.7), (0.3, 0.3, 0.3)),                      # across the room from a corner
             ((-1.0, -1.0, -0.8), (0.4, 0.5, 0.3)),                   # into a corner
             ((1.0, 0.75, 0.625), (2.0, 1.5, 1.25)),                  # at the far corner from the centre, through a vertex
             ((0.3, -0.2, 1.0), (1.0, 2.0, 0.5))]                     # up at the ceiling
    c2w = dp.view_matrix(np.array([d for d, _ in views]), dp.UP, np.array([p for _, p in views]))
    got = dp.render_depth(v, f, c2w).cpu().numpy()
    zn = dp.default_z_near(v)
    for k in range(len(views)):
        want = analytic_box_depth(c2w[k], size, 500, 500, 300.0, 300.0, 249.5, 249.5)
        assert want.min() > zn * 1.01
        assert (got[k] == 0).sum() == 0, (k, np.argwhere(got[k] == 0)[:5])
        err = np.abs(got[k].astype(np.float64) - want)
        assert np.all(err <= 2 * f32_ulp(want)), (k, err.max())


# ------------------------------------------------------------------------------------------------ the metric
def test_depth_l1_of_a_moved_copy_is_zero(room):
    from nice_slam_b200.recon import eval_depth_l1
    v, f = room[128]
    mv, M = moved(v, 0.0, (0.0, 0.0, 1.0), (0.03, 0.01, -0.02))        # a translation: both meshes keep one z_near
    r = eval_depth_l1((mv, f), (v, f), np.zeros((0, 3)), align=True, n_views=200)
    assert np.abs(r["transform"] - np.linalg.inv(M)).max() < 1e-6
    assert r["depth_l1"] < 1e-3 and r["rejected"] == 0 and r["candidates"] == 200


def test_depth_l1_of_a_box_room_without_a_wall_matches_oracle():
    from nice_slam_b200 import depth as dp
    from nice_slam_b200.recon import eval_depth_l1
    size = (4.0, 3.0, 2.5)
    v, f = box_room(0.25, size)
    wall = np.all(np.isclose(v[f][..., 0], size[0]), axis=1)          # the faces of the wall at x = 4
    H, W, focal = 60, 60, 36.0
    r = eval_depth_l1((v, f[~wall]), (v, f), np.zeros((0, 3)), align=False, n_views=12, seed=5, H=H, W=W, focal=focal)
    zn = dp.default_z_near(v)
    assert r["depth_l1"] > 0
    for k, c in enumerate(r["c2w"]):
        g = dp.render_depth(v, f, c[None], H, W, focal, focal).cpu().numpy()[0]
        rr = dp.render_depth(v, f[~wall], c[None], H, W, focal, focal).cpu().numpy()[0]
        gw, _ = compare(g, v, f, c, H, W, focal, focal, W / 2 - .5, H / 2 - .5, zn)
        rw, _ = compare(rr, v, f[~wall], c, H, W, focal, focal, W / 2 - .5, H / 2 - .5, zn)
        want = od.view_error(gw, rw)
        assert abs(r["view_errors"][k] - want) <= 1e-9 * want, (k, r["view_errors"][k], want)


def test_depth_l1_of_room0_64_against_128_matches_oracle(room):
    from nice_slam_b200 import depth as dp
    from nice_slam_b200.recon import eval_depth_l1
    gv, gf = room[128]
    rv, rf = room[64]
    H, W, focal = 40, 40, 24.0
    r = eval_depth_l1((rv, rf), (gv, gf), np.zeros((0, 3)), align=True, n_views=4, seed=2, H=H, W=W, focal=focal)
    assert np.isfinite(r["depth_l1"]) and r["depth_l1"] > 0
    T = r["transform"]
    av = rv @ T[:3, :3].T + T[:3, 3]
    for k, c in enumerate(r["c2w"]):
        g = dp.render_depth(gv, gf, c[None], H, W, focal, focal).cpu().numpy()[0]
        rr = dp.render_depth(av, rf, c[None], H, W, focal, focal).cpu().numpy()[0]
        gw, _ = compare(g, gv, gf, c, H, W, focal, focal, W / 2 - .5, H / 2 - .5, dp.default_z_near(gv))
        rw, _ = compare(rr, av, rf, c, H, W, focal, focal, W / 2 - .5, H / 2 - .5, dp.default_z_near(av))
        want = od.view_error(gw, rw)
        assert abs(r["view_errors"][k] - want) <= 1e-9 * want
    print("room0@64 vs @128: Depth L1 %.4f cm" % r["depth_l1"])


def test_repeats_are_bit_identical(room):
    from nice_slam_b200.recon import eval_depth_l1
    v, f = room[128]
    mv, _ = moved(v, 0.3, (0.0, 0.0, 1.0), (0.02, 0.0, 0.0))
    a = eval_depth_l1((mv, f), room[64], np.zeros((0, 3)), n_views=50)
    b = eval_depth_l1((mv, f), room[64], np.zeros((0, 3)), n_views=50)
    assert a["view_errors"].tobytes() == b["view_errors"].tobytes() and a["depth_l1"] == b["depth_l1"]
    assert np.array_equal(a["c2w"], b["c2w"]) and np.array_equal(a["transform"], b["transform"])


# ------------------------------------------------------------------------------------------------ view sampling
@pytest.fixture(scope="module")
def unseen_box():
    """box_room(0.1) and the vertices that 24 poses inside it do not see (cull.cull_mesh): an unseen-region cloud."""
    from nice_slam_b200.cull import cull_mesh
    v, f = box_room(0.1)
    seen, _ = cull_mesh(v, f, room_poses(24, 3, max_pitch_deg=50.0))
    return v, v[seen.cpu().numpy() == 0]


def test_view_sampling_rejects_as_check_proj_and_is_batch_independent(unseen_box):
    from nice_slam_b200 import depth as dp
    v, unseen = unseen_box
    assert 0 < len(unseen) < len(v)
    n = 24
    runs = [dp.sample_views(v, unseen, n, seed=11, batch=b) for b in (1, 7, 256)]
    c2w, drawn, rejected = runs[0]
    for c, d, r in runs[1:]:
        assert np.array_equal(c, c2w) and d == drawn and r == rejected
    print("views: %d accepted of %d candidates (%d rejected), %d unseen points" % (n, drawn, rejected, len(unseen)))
    ext, T = dp.sampling_box(v)
    cand = dp.candidates(np.random.default_rng(11).random((drawn, 6)), ext, T)
    gpu = dp.views_see_any(torch.from_numpy(unseen).to(DEV), torch.from_numpy(dp.check_proj_w2c(cand)).to(DEV)).cpu().numpy().astype(bool)
    assert np.array_equal(cand[~gpu], c2w) and (~gpu).sum() == n
    flips = 0
    for k in range(drawn):
        want = od.check_proj(unseen, 500, 500, 300., 300., 249.5, 249.5, cand[k])
        if want != gpu[k]:
            u, vv, z = od.check_proj_uvz(unseen, 500, 500, 300., 300., 249.5, 249.5, cand[k])
            with np.errstate(invalid="ignore"):
                border = np.minimum(np.minimum(np.abs(u), np.abs(u - 500)), np.minimum(np.abs(vv), np.abs(vv - 500))) < 1e-3
            assert (border | (np.abs(z) < 1e-5)).any(), k
            flips += 1
            print("candidate %d: check_proj %s, GPU %s (a point within rounding of the border)" % (k, want, gpu[k]))
    assert flips <= 2
    for c in c2w:                                                       # no accepted view sees an unseen point
        u, vv, z = od.check_proj_uvz(unseen, 500, 500, 300., 300., 249.5, 249.5, c)
        with np.errstate(invalid="ignore"):
            inside = (z <= 0) & (u > 1e-3) & (u < 500 - 1e-3) & (vv > 1e-3) & (vv < 500 - 1e-3)
        assert not inside.any()


def test_view_sampling_without_unseen_points_and_the_cap(unseen_box):
    from nice_slam_b200 import depth as dp
    v, unseen = unseen_box
    c2w, drawn, rejected = dp.sample_views(v, np.zeros((0, 3)), 10, seed=1)
    assert drawn == 10 and rejected == 0
    assert np.array_equal(c2w, dp.candidates(np.random.default_rng(1).random((10, 6)), *dp.sampling_box(v)))
    with pytest.raises(ValueError, match="cap of 3 candidates"):
        dp.sample_views(v, v, 2, seed=1, max_candidates=3)           # every vertex unseen: every view is rejected


# ------------------------------------------------------------------------------------------------ CLI and input checks
def test_cli_prints_depth_l1(room, tmp_path):
    from nice_slam_b200.mesh import write_ply
    gt, rec = str(tmp_path / "gt.ply"), str(tmp_path / "rec.ply")
    write_ply(gt, *room[128])
    write_ply(rec, *room[64])
    np.save(str(tmp_path / "gt_pc_unseen.npy"), np.array([[100.0, 100.0, 100.0]]))
    env = dict(os.environ, PYTHONPATH=ROOT)
    cmd = [sys.executable, "-m", "nice_slam_b200.recon", "--rec_mesh", rec, "--gt_mesh", gt]
    out = subprocess.run(cmd + ["-2d"], cwd=ROOT, env=env, capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    lines = out.stdout.strip().splitlines()
    assert len(lines) == 1 and lines[0].startswith("Depth L1: ") and np.isfinite(float(lines[0].split()[-1]))
    out = subprocess.run(cmd + ["-3d", "-2d"], cwd=ROOT, env=env, capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    lines = out.stdout.strip().splitlines()
    assert [l.split(":")[0] for l in lines] == ["accuracy", "completion", "completion ratio", "Depth L1"]


def test_bad_input_raises():
    from nice_slam_b200 import depth as dp
    v, f = box_room(1.0)
    c = np.eye(4)[None]
    bad = v.copy()
    bad[3, 1] = np.nan
    with pytest.raises(ValueError, match="not all finite"):
        dp.render_depth(bad, f, c)
    with pytest.raises(ValueError, match="face indices outside"):
        dp.render_depth(v, np.concatenate([f, [[0, 1, len(v)]]]), c)
    with pytest.raises(ValueError, match="face indices outside"):
        dp.render_depth(v, np.concatenate([f, [[0, -1, 2]]]), c)
    with pytest.raises(ValueError, match="empty"):
        dp.render_depth(v, np.zeros((0, 3), np.int64), c)
    with pytest.raises(ValueError, match="c2w must be"):
        dp.render_depth(v, f, np.eye(4)[:3])
    with pytest.raises(ValueError, match="c2w must be"):
        dp.render_depth(v, f, np.eye(3)[None])
    nan_pose = np.eye(4)[None].copy()
    nan_pose[0, 0, 3] = np.inf
    with pytest.raises(ValueError, match="c2w entries are not all finite"):
        dp.render_depth(v, f, nan_pose)
    with pytest.raises(ValueError, match="z_near"):
        dp.render_depth(v, f, c, z_near=0.0)


def test_new_kernels_have_no_spills():
    if not os.path.exists(BUILD_LOG):
        pytest.skip("build log not available")
    found, cur = {}, None
    for line in open(BUILD_LOG):
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            cur = m.group(1)
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur and "nsb_depth_cu" in cur:
            found[cur] = tuple(int(x) for x in m.groups())
    for k in ("raster_faces_kernel", "raster_large_kernel", "views_see_any_kernel", "depth_l1_kernel", "depth_fill_kernel", "depth_finish_kernel"):
        ent = {n: s for n, s in found.items() if re.search(r"\d%s" % k, n)}
        assert ent, k
        for n, (stack, st, ld) in ent.items():
            assert st == 0 and ld == 0, (n, stack, st, ld)
