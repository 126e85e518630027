"""GPU: reconstruction metrics (nice_slam_b200.recon, nsb_recon.cu) against the float64 oracle (oracle/recon.py) and scipy's cKDTree:
surface sampling, exact nearest neighbours, the ICP pass and loop, bit-identical repeats, and the metric of a FusedSLAM run's
final_mesh_eval_rec.ply."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
from scipy.spatial import cKDTree

import scene_util as su
from gpu_util import make_renderer
from oracle import recon as orc

pytestmark = pytest.mark.gpu
DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MC_BOUND = [[-2.9, 8.9], [-3.2, 5.5], [-3.5, 3.3]]                   # configs/Replica/room0.yaml: mapping.marching_cubes_bound


def mesh_cfg(resolution, **meshing):
    m = dict(resolution=resolution, level_set=0, clean_mesh_bound_scale=1.02, remove_small_geometry_threshold=0.2, get_largest_components=False,
             color_mesh_extraction_method="direct_point_query", depth_test=False, mesh_coarse_level=False, eval_rec=False, clean_mesh=True)
    m.update(meshing)
    return dict(meshing=m, mapping=dict(marching_cubes_bound=MC_BOUND), scale=1)


@pytest.fixture(scope="module")
def room():
    """room0's 'soft' grids meshed (lattice without a hull + marching cubes) at resolutions 64 and 128: {R: (vertices f64, faces int64)}."""
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


def moved(v, angle, axis, t):
    """(v moved by a rigid motion about the centroid, its 4x4)."""
    ctr = np.eye(4)
    ctr[:3, 3] = v.mean(0)
    M = ctr @ orc.rigid(angle, axis, t) @ np.linalg.inv(ctr)
    return orc.transform_points(v, M), M


# ------------------------------------------------------------------------------------------------ sampling
def check_sampling(v, f, count, seed):
    from nice_slam_b200.recon import sample_surface
    g = torch.Generator(device=DEV)
    g.manual_seed(seed)
    pts, face = sample_surface(v, f, count, g)
    g.manual_seed(seed)
    u = torch.rand(count, 3, dtype=torch.float64, device=DEV, generator=g).cpu().numpy()
    want_pts, want_face = orc.sample_surface(v, f, u)
    pts, face = pts.cpu().numpy(), face.cpu().numpy()
    cum = np.cumsum(orc.face_areas(v, f))
    pick = u[:, 0] * cum[-1]
    diff = np.nonzero(face != want_face)[0]
    for s in diff:                                   # only picks within 1e-12 relative of every cumulative boundary between the two faces
        lo, hi = sorted((face[s], want_face[s]))
        assert np.abs(cum[lo:hi] - pick[s]).max() <= 1e-12 * cum[-1], (s, face[s], want_face[s])
    same = face == want_face
    assert np.abs(pts[same] - want_pts[same]).max() <= 1e-12 * max(1.0, np.abs(v).max())
    return len(diff)


def test_sampling_matches_oracle_with_zero_area_faces(room):
    v, f = room[64]
    deg = np.array([[0, 0, 0], [1, 1, 2], [3, 4, 3]] * 50, dtype=np.int64)           # zero-area faces spread through the list
    ff = np.insert(f, np.linspace(0, len(f), len(deg)).astype(np.int64), deg, axis=0)
    assert (orc.face_areas(v, ff) == 0).sum() >= len(deg)
    assert check_sampling(v, ff, 300001, 3) < 5
    _, face = orc.sample_surface(v, ff, np.random.default_rng(0).random((10000, 3)))
    assert not np.isin(face, np.nonzero(orc.face_areas(v, ff) == 0)[0]).any()


def test_sampling_a_single_face():
    v = np.array([[0.1, 0.2, 0.3], [1.5, 0.2, -0.3], [0.4, 2.0, 0.9]])
    assert check_sampling(v, np.array([[0, 1, 2]]), 1000, 5) == 0
    assert check_sampling(v, np.array([[0, 1, 2]]), 1, 6) == 0


# ------------------------------------------------------------------------------------------------ nearest neighbours
def check_nn(t, q, radius=None):
    """GPU against cKDTree: the GPU's pick is optimal under numpy's d2 (the kernel's formula, bit for bit), no worse than cKDTree's,
    the smaller index on an exact tie; squared distances equal cKDTree's to 1e-12 relative; -1 exactly where cKDTree finds nothing."""
    from nice_slam_b200.recon import NearestNeighbours
    t, q = np.ascontiguousarray(t, dtype=np.float64), np.ascontiguousarray(q, dtype=np.float64)
    d2, idx = NearestNeighbours(t).query(q, radius=radius, squared=True)
    d2, idx = d2.cpu().numpy(), idx.cpu().numpy().astype(np.int64)
    dk, jk = cKDTree(t).query(q, distance_upper_bound=np.inf if radius is None else radius)
    none = ~np.isfinite(dk)
    assert np.array_equal(idx < 0, none)
    assert np.all(np.isinf(d2[none]))
    ok = ~none
    mine = ((q[ok] - t[idx[ok]]) ** 2).sum(1)
    theirs = ((q[ok] - t[jk[ok]]) ** 2).sum(1)
    assert np.array_equal(d2[ok], mine)
    assert np.all(mine <= theirs)
    tie = mine == theirs
    assert np.all(idx[ok][tie] <= jk[ok][tie])
    assert np.all(np.abs(d2[ok] - dk[ok] ** 2) <= 1e-12 * dk[ok] ** 2)
    return idx, d2


def _rng(seed):
    return np.random.default_rng(seed)


def test_nn_uniform_clouds():
    check_nn(_rng(0).random((100000, 3)) * 10, _rng(1).random((50000, 3)) * 12 - 1)
    check_nn(_rng(2).random((3000, 3)) * [10, 0.5, 3], _rng(3).random((3000, 3)) * 10)          # a flat box


def test_nn_surface_clouds(room):
    v, f = room[128]
    t, _ = orc.sample_surface(v, f, _rng(4).random((200000, 3)))
    q, _ = orc.sample_surface(v, f, _rng(5).random((100000, 3)))
    check_nn(t, q)
    check_nn(t, q + _rng(6).normal(scale=0.05, size=q.shape))


def test_nn_duplicates_and_one_cell():
    base = _rng(7).random((1000, 3))
    t = np.repeat(base, 5, axis=0)[_rng(8).permutation(5000)]
    idx, d2 = check_nn(t, np.concatenate([base, base + 1e-3]))
    assert np.all(d2[:1000] == 0)
    same = np.tile([[0.5, -1.25, 3.0]], (500, 1))                   # every target in one cell (zero extent)
    idx, d2 = check_nn(same, _rng(9).random((300, 3)))
    assert np.all(idx == 0)
    check_nn(0.5 + 1e-9 * _rng(10).random((400, 3)), _rng(11).random((200, 3)))


def test_nn_far_target_and_far_queries():
    t = np.concatenate([_rng(12).random((2000, 3)) * 5, [[1e4, 2.0, 2.0]]])
    check_nn(t, np.concatenate([_rng(13).random((2000, 3)) * 6, [[9999.0, 2.0, 2.0], [5e3, 0, 0]]]))
    t = _rng(14).random((5000, 3)) * 4
    far = np.concatenate([_rng(15).normal(size=(500, 3)) * 1e3, [[-1e3, 2, 2], [2, 1e3, 2], [2, 2, -5e2], [1e6, -1e6, 1e6]]])
    check_nn(t, far)


@pytest.mark.parametrize("n,m", [(1, 1), (1, 1000), (257, 1), (1000, 257), (333, 777), (4097, 2049)])
def test_nn_sizes(n, m):
    check_nn(_rng(n).random((n, 3)) * 3, _rng(m + 1).random((m, 3)) * 4 - 0.5)


@pytest.mark.parametrize("radius", [0.0, 0.05, 0.3, 1.0, 100.0])
def test_nn_radius(radius, room):
    idx, _ = check_nn(_rng(16).random((2000, 3)) * 10, _rng(17).random((5000, 3)) * 12 - 1, radius)
    if radius == 0.0:
        assert np.all(idx == -1)
    v, _ = room[64]
    check_nn(v, v[::7] + _rng(18).normal(scale=0.05, size=v[::7].shape), radius)


# ------------------------------------------------------------------------------------------------ repeats and ICP
def test_bit_identical_repeats(room):
    from nice_slam_b200.recon import NearestNeighbours, icp_sums
    v, _ = room[128]
    q = torch.from_numpy(v[::3] + _rng(19).normal(scale=0.02, size=v[::3].shape)).to(DEV)
    a = NearestNeighbours(v).query(q, squared=True)
    b = NearestNeighbours(v).query(q, squared=True)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    nn = NearestNeighbours(v)
    src = torch.from_numpy(moved(v[v[:, 0] < np.median(v[:, 0])], 2.0, (0, 0, 1), (0.03, 0, 0))[0]).to(DEV)
    s1, s2 = icp_sums(nn, src, np.eye(4), 0.1), icp_sums(nn, src, np.eye(4), 0.1)
    assert s1.tobytes() == s2.tobytes() and s1[0] > 0


def test_icp_matches_oracle_and_recovers_the_motion(room):
    from nice_slam_b200.recon import icp_align
    v, _ = room[128]
    crop = v[(v[:, 0] < np.quantile(v[:, 0], 0.7)) & (v[:, 2] > np.quantile(v[:, 2], 0.1))]
    src, M = moved(crop, 0.8, (0.2, 0.3, 1.0), (0.02, -0.015, 0.01))
    T, fit, rmse, it = icp_align(src, v, 0.1)                                                  # an exact copy: both end at rounding level
    Tw, fitw, rmsew, itw = orc.icp_align(src, v, 0.1)
    assert it == itw and it < 30
    assert np.abs(T - Tw).max() < 1e-9
    assert fit == fitw == 1.0 and rmse < 1e-9 and rmsew < 1e-9
    assert np.abs(T - np.linalg.inv(M)).max() < 1e-6
    noisy = src + _rng(20).normal(scale=1e-3, size=src.shape)                                  # 1 mm noise: a real rmse to compare
    T, fit, rmse, it = icp_align(noisy, v, 0.1)
    Tw, fitw, rmsew, itw = orc.icp_align(noisy, v, 0.1)
    assert it == itw and it < 30
    assert np.abs(T - Tw).max() < 1e-9
    assert abs(fit - fitw) < 1e-12 and abs(rmse - rmsew) < 1e-12 and 1e-3 < rmse < 1e-2
    T0, fit0, rmse0, it0 = icp_align(src, v, 0.1, max_iteration=0)
    assert it0 == 0 and np.array_equal(T0, np.eye(4)) and 0 < fit0 < fit
    T1, fit1, rmse1, it1 = icp_align(src + 10.0, v, 0.1)                                       # no pairs: identity, 0, 0
    assert np.array_equal(T1, np.eye(4)) and fit1 == 0.0 and rmse1 == 0.0 and it1 == 1


# ------------------------------------------------------------------------------------------------ end to end
@pytest.fixture(scope="module")
def fused_run(tmp_path_factory):
    """The every1 replay with mesh_dir and meshing.eval_rec: its final_mesh_eval_rec.ply."""
    from test_gpu_slam import cfg_of, load, slam_for
    from slam_sequences import sequence
    sc = su.load_scenes()["room0"]
    case = load("every1")
    cfg = cfg_of(case, mesh_freq=100, no_mesh_on_first_frame=True, marching_cubes_bound=MC_BOUND)
    cfg["meshing"], cfg["scale"] = mesh_cfg(64, eval_rec=True)["meshing"], 1
    mesh_dir = str(tmp_path_factory.mktemp("recon") / "mesh")
    slam = slam_for(sc, cfg, mesh_dir=mesh_dir)
    slam.run(sequence(sc, case["n"]), replay=case["replay"])
    return os.path.join(mesh_dir, "final_mesh_eval_rec.ply")


def test_eval_recon_of_a_fused_run_matches_oracle(fused_run, room):
    from nice_slam_b200.recon import NearestNeighbours, eval_recon, read_ply, sample_surface
    assert os.path.exists(fused_run)
    gv, gf = room[128]
    r = eval_recon(fused_run, (gv, gf), align=True, seed=3)
    rv, rf, _ = read_ply(fused_run)
    rv = rv @ r["transform"][:3, :3].T + r["transform"][:3, 3]
    g = torch.Generator(device=DEV)
    g.manual_seed(3)
    rec_pts = sample_surface(rv, rf, 200000, g)[0]
    gt_pts = sample_surface(gv, gf, 200000, g)[0]
    acc, comp, ratio, _, d_comp = orc.metrics(rec_pts.cpu().numpy(), gt_pts.cpu().numpy())
    assert abs(r["accuracy"] - 100 * acc) < 1e-9 and abs(r["completion"] - 100 * comp) < 1e-9
    mine = NearestNeighbours(rec_pts).query(gt_pts)[0].cpu().numpy()
    flip = (mine < 0.05) != (d_comp < 0.05)
    assert np.all(np.abs(d_comp[flip] - 0.05) < 1e-12)
    assert abs(r["completion_ratio"] - 100 * ratio) <= 100 * flip.sum() / len(d_comp) + 1e-12
    assert np.isfinite(r["accuracy"]) and np.isfinite(r["completion"]) and 0 < r["completion_ratio"] < 100      # a partial scan


def test_eval_recon_aligns_a_moved_copy(room):
    from nice_slam_b200.recon import eval_recon
    v, f = room[128]
    mv, M = moved(v, 1.0, (0.1, -0.2, 1.0), (0.03, 0.01, -0.02))
    # two independent samplings of one surface are 1 / (2 sqrt(density)) apart on average: 0.65 cm at 6000 samples per m^2
    n = max(200000, int(6000 * orc.face_areas(v, f).sum()))
    r = eval_recon((mv, f), (v, f), align=True, n_samples=n)
    assert np.abs(r["transform"] - np.linalg.inv(M)).max() < 1e-6
    assert r["fitness"] == 1.0
    assert r["accuracy"] < 1.0 and r["completion"] < 1.0 and r["completion_ratio"] > 99.0


def test_cli_prints_the_three_lines(fused_run, room, tmp_path):
    from nice_slam_b200.mesh import write_ply
    gt = str(tmp_path / "gt.ply")
    write_ply(gt, *room[64])
    env = dict(os.environ, PYTHONPATH=ROOT)
    out = subprocess.run([sys.executable, "-m", "nice_slam_b200.recon", "--rec_mesh", fused_run, "--gt_mesh", gt, "-3d"], cwd=ROOT, env=env,
                         capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    lines = out.stdout.strip().splitlines()
    assert [l.split(":")[0] for l in lines] == ["accuracy", "completion", "completion ratio"]
    assert all(np.isfinite(float(l.split()[-1])) for l in lines)
    out = subprocess.run([sys.executable, "-m", "nice_slam_b200.recon", "--rec_mesh", fused_run, "--gt_mesh", gt, "-2d"], cwd=ROOT, env=env,
                         capture_output=True, text=True)
    assert out.returncode != 0 and "not supported" in out.stderr
