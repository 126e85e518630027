"""GPU: ground-truth culling (nice_slam_b200.cull, nsb_cull_*) against the float64 oracle of cull_mesh.py (oracle/cull.py) on a FusedMesher
mesh and on a 2.4 M-vertex room with 2000 poses, the CLI's PLY pass-through, the 3D metric against culled and unculled ground truth,
and the errors."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import scene_util as su
from cull_scene import box_room, room_poses, write_ply_with_extras, write_traj
from gpu_util import make_renderer
from oracle import cull as oc

pytestmark = pytest.mark.gpu
DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MC_BOUND = [[-2.9, 8.9], [-3.2, 5.5], [-3.5, 3.3]]                   # configs/Replica/room0.yaml: mapping.marching_cubes_bound
T40 = 2.0 ** 40


def _np(x):
    return x.cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)


def check_against_oracle(v, f, c2w):
    """The kernel's seen mask against the oracle's (at most max(3, 1e-5 V) differ, each within rounding of a decision under some pose),
    the kept faces against the kernel's own mask, and a second call's bits."""
    from nice_slam_b200.cull import cull_mesh
    seen, kept = cull_mesh(v, f, c2w)
    seen, kept = _np(seen).astype(bool), _np(kept)
    w2c = oc.w2c_list(c2w)
    want = oc.seen_mask(v, w2c)
    diff = np.nonzero(seen != want)[0]
    assert len(diff) <= max(3, 1e-5 * len(v)), len(diff)
    assert oc.near_border(v[diff], w2c).all(), diff[~oc.near_border(v[diff], w2c)][:10]
    assert kept.dtype == np.int32 and np.array_equal(kept, oc.kept_faces(f, seen))
    s2, k2 = cull_mesh(v, f, c2w)
    assert np.array_equal(_np(s2), seen.astype(np.uint8)) and np.array_equal(_np(k2), kept)
    return seen, want


def test_fused_mesher_mesh_against_oracle():
    """The marching-cubes mesh of room0's 'soft' grids (resolution 64, as tests/test_gpu_mesh.py) and its five synthetic keyframe poses."""
    from nice_slam_b200.keyframes import KeyframeStore
    from nice_slam_b200.mesh import FusedMesher
    sc = su.load_scenes()["room0"]
    renderer, c, dec = make_renderer(sc, su.make_grids(sc, "soft"), su.load_decoders("soft"), DEV)
    cam = sc["cam"]
    store = KeyframeStore(cam["H"], cam["W"], cam["fx"], cam["fy"], cam["cx"], cam["cy"], DEV)
    for k in range(5):
        depth, color = su.make_frame(sc, 300 + k)
        store.append(10 * k, color, depth, su.make_pose(sc, 300 + k))
    cfg = dict(meshing=dict(resolution=64, level_set=0, clean_mesh_bound_scale=1.02, remove_small_geometry_threshold=0.2,
                            get_largest_components=False, color_mesh_extraction_method="direct_point_query", depth_test=False),
               mapping=dict(marching_cubes_bound=MC_BOUND), scale=1)
    m = FusedMesher(renderer, cfg)
    v, f, _ = m.marching_cubes(m.lattice(c, dec, m.hull(store)))
    v, f = _np(v).astype(np.float64), _np(f).astype(np.int64)
    seen, want = check_against_oracle(v, f, torch.stack(store.est_c2w))
    assert len(f) > 1000 and 0 < want.sum() < len(want), (len(f), want.sum(), len(want))


def test_large_room_many_pose_tiles_against_oracle():
    v, f = box_room(0.005)
    c2w = room_poses(2000, 1, 25.0)
    assert len(v) >= 2_000_000 and len(v) % 256 and len(c2w) % 256
    seen, want = check_against_oracle(v, f, c2w)
    assert 0.002 < 1 - want.mean() < 0.05                                    # unseen vertices run every pose tile


def test_frame_border_nonfinite_poses_and_no_poses():
    """Analytic cases on the device (oracle cases of tests/test_cull_oracle.py): at depth 2^40 the pixel coordinates are exact."""
    from nice_slam_b200.cull import cull_faces, cull_mesh, cull_seen
    unit = dict(H=680, W=1200, fx=1.0, fy=1.0, cx=0.0, cy=0.0)
    uv = [(0, 340), (1200, 340), (600, 0), (600, 680), (0, 0), (1200, 680), (600, 340), (0.5, 340), (1199.5, 340), (600, 0.5), (600, 679.5)]
    v = torch.tensor([[u * T40, -w * T40, 0.0] for u, w in uv], dtype=torch.float64, device=DEV)
    w0 = torch.eye(4)
    w0[2, 3] = -T40
    behind, nan = w0.clone(), w0.clone()
    behind[2, 3] = T40
    nan[0, 1] = float("nan")
    expect = [0] * 6 + [1] * 5
    for poses, want in (([w0], expect), ([behind], [0] * 11), ([nan], [0] * 11), ([nan, behind, w0], expect)):
        w = torch.stack(poses).to(DEV)
        assert cull_seen(v, w, **unit).tolist() == want
        assert oc.seen_mask(v.cpu().numpy(), w.cpu().numpy(), **unit).astype(int).tolist() == want
    faces = torch.tensor([[0, 1, 2], [0, 6, 1], [3, 4, 5], [10, 2, 3]], dtype=torch.int32, device=DEV)
    assert cull_faces(faces, cull_seen(v, w0[None].to(DEV), **unit)).tolist() == [1, 3]
    vv, ff = box_room(0.5)
    seen, kept = cull_mesh(vv, ff, np.zeros((0, 4, 4)))
    assert seen.shape == (len(vv),) and int(seen.sum()) == 0 and kept.numel() == 0
    c2w = room_poses(30, 4)
    c2w[3] = np.nan
    c2w[5, 0, 0] = np.inf
    assert np.array_equal(_np(cull_mesh(vv, ff, c2w)[0]).astype(bool), oc.seen_mask(vv, oc.w2c_list(c2w)))


@pytest.fixture(scope="module")
def culled_room(tmp_path_factory):
    """A 150 k-vertex room with extra PLY properties, culled by the CLI with 40 level cameras (about a quarter of the room unseen)."""
    d = tmp_path_factory.mktemp("cull")
    v, f = box_room(0.02)
    c2w = room_poses(40, 2, 10.0)
    gt, traj, out = str(d / "room_mesh.ply"), str(d / "traj.txt"), str(d / "culled.ply")
    vbytes = write_ply_with_extras(gt, v, f)
    write_traj(traj, c2w)
    r = subprocess.run([sys.executable, "-m", "nice_slam_b200.cull", "--input_mesh", gt, "--traj", traj, "--output_mesh", out],
                       cwd=ROOT, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return dict(v=v, f=f, c2w=c2w, gt=gt, traj=traj, out=out, vbytes=vbytes, stdout=r.stdout)


def test_cli_culls_and_passes_records_through(culled_room):
    from nice_slam_b200.cull import cull_mesh, load_poses
    from nice_slam_b200.recon import read_ply, read_ply_records
    s = culled_room
    v32 = s["v"].astype(np.float32).astype(np.float64)
    _, kept = cull_mesh(v32, s["f"], load_poses(s["traj"]))
    kept = _np(kept)
    assert 0 < len(kept) < 0.9 * len(s["f"])
    assert s["stdout"].strip() == "kept %d of %d faces (%d vertices)" % (len(kept), len(s["f"]), len(s["v"]))
    rv, rf, rc = read_ply(s["out"])
    assert np.array_equal(rv, v32) and np.array_equal(rf, s["f"][kept])
    _, els = read_ply_records(s["out"])
    _, els_in = read_ply_records(s["gt"])
    assert els[0][2].tobytes() == s["vbytes"]
    assert els[1][2].tobytes() == els_in[1][2][kept].tobytes() and np.array_equal(els[1][2]["label"], kept)
    assert els[2][2].tobytes() == els_in[2][2].tobytes()


def test_metric_against_culled_and_unculled_ground_truth(culled_room):
    """A reconstruction of exactly the seen part completes the culled ground truth (sampling distance only) but not the whole room."""
    from nice_slam_b200.recon import eval_recon, read_ply
    s = culled_room
    rv, rf, _ = read_ply(s["out"])
    culled = eval_recon((rv, rf), s["out"], n_samples=500000)
    whole = eval_recon((rv, rf), s["gt"], n_samples=500000)
    assert culled["completion"] < 1.0 and culled["accuracy"] < 1.0, culled
    assert whole["completion"] > 3 * culled["completion"] and whole["completion"] > 2.0, whole
    assert whole["completion_ratio"] < culled["completion_ratio"] - 10, (culled, whole)


def test_errors_name_the_entry_point():
    from nice_slam_b200 import _lib
    from nice_slam_b200.cull import cull_faces, cull_mesh, cull_seen
    from nice_slam_b200.renderer import _VP, _stream
    v = torch.zeros(4, 3, dtype=torch.float64)
    w = torch.eye(4)[None]
    with pytest.raises(ValueError, match="nsb_cull_seen: vertices must be a CUDA tensor"):
        cull_seen(v, w.to(DEV))
    with pytest.raises(ValueError, match="nsb_cull_seen: w2c must be"):
        cull_seen(v.to(DEV), torch.eye(4, dtype=torch.float64, device=DEV)[None])
    faces = torch.tensor([[0, 1, 2]], dtype=torch.int32)
    with pytest.raises(ValueError, match="nsb_cull_faces: faces must be a CUDA tensor"):
        cull_faces(faces, torch.zeros(4, dtype=torch.uint8, device=DEV))
    with pytest.raises(ValueError, match="cull_mesh: face indices outside"):
        cull_mesh(v, np.array([[0, 1, 4]]), w)
    with pytest.raises(RuntimeError, match="nsb_cull_seen.*H and W"):
        cull_seen(v.to(DEV), w.to(DEV), H=0)
    L, vd, seen = _lib.lib(), v.to(DEV), torch.empty(4, dtype=torch.uint8, device=DEV)
    with pytest.raises(RuntimeError, match="nsb_cull_seen.*negative"):
        _lib.check(L.nsb_cull_seen(_VP(vd.data_ptr()), -1, None, 0, 600.0, 600.0, 599.5, 339.5, 680, 1200, _VP(seen.data_ptr()), _stream()),
                   "nsb_cull_seen")
    fd = faces.to(DEV)
    ws = torch.empty(8, dtype=torch.uint8, device=DEV)
    total = torch.empty(1, dtype=torch.int64, device=DEV)
    with pytest.raises(RuntimeError, match="nsb_cull_faces: workspace"):
        _lib.check(L.nsb_cull_faces(_VP(fd.data_ptr()), 1, _VP(seen.data_ptr()), _VP(ws.data_ptr()), 8, _VP(total.data_ptr()), _stream()),
                   "nsb_cull_faces")
    torch.cuda.synchronize()
