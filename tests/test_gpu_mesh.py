"""GPU: mesh extraction (nice_slam_b200.mesh.FusedMesher, nsb_mesh.cu) against the float64 oracle (oracle/mesh.py), the PLY files, the
errors, and meshing inside a FusedSLAM run."""
import copy
import os

import numpy as np
import pytest
import torch

import scene_util as su
from gpu_util import make_renderer, rel
from oracle import mesh as om
from oracle import torch_port as tp

pytestmark = pytest.mark.gpu
DEV = "cuda"
MC_BOUND = [[-2.9, 8.9], [-3.2, 5.5], [-3.5, 3.3]]                   # configs/Replica/room0.yaml: mapping.marching_cubes_bound


def mesh_cfg(resolution=64, **meshing):
    m = dict(resolution=resolution, level_set=0, clean_mesh_bound_scale=1.02, remove_small_geometry_threshold=0.2, get_largest_components=False,
             color_mesh_extraction_method="direct_point_query", depth_test=False, mesh_coarse_level=False, eval_rec=False, clean_mesh=True)
    m.update(meshing)
    return dict(meshing=m, mapping=dict(marching_cubes_bound=MC_BOUND), scale=1)


@pytest.fixture(scope="module")
def setup():
    from nice_slam_b200.keyframes import KeyframeStore
    from nice_slam_b200.mesh import FusedMesher
    sc = su.load_scenes()["room0"]
    grids, dec_state = su.make_grids(sc, "soft"), su.load_decoders("soft")
    renderer, c, dec = make_renderer(sc, grids, dec_state, DEV)
    cam = sc["cam"]
    store = KeyframeStore(cam["H"], cam["W"], cam["fx"], cam["fy"], cam["cx"], cam["cy"], DEV)
    frames = []
    for k in range(5):
        depth, color = su.make_frame(sc, 300 + k)
        c2w = su.make_pose(sc, 300 + k)
        store.append(10 * k, color, depth, c2w)
        frames.append((depth, c2w))
    mesher = FusedMesher(renderer, mesh_cfg())
    return dict(sc=sc, grids=grids, dec_state=dec_state, renderer=renderer, c=c, dec=dec, store=store, frames=frames, mesher=mesher,
                bound=su.scene_bound(sc))


@pytest.fixture(scope="module")
def volume(setup):
    """GPU hull and lattice at resolution 64, and the oracle's hull."""
    s = setup
    cam = s["sc"]["cam"]
    planes = s["mesher"].hull(s["store"])
    pts = [np.stack([f[1][:3, 3].double().numpy() for f in s["frames"]])]
    pts += [om.backproject(f[0].numpy(), f[1].double().numpy(), cam["fx"], cam["fy"], cam["cx"], cam["cy"]) for f in s["frames"]]
    want_planes = om.hull_equations(np.concatenate(pts), 1.02)
    z = s["mesher"].lattice(s["c"], s["dec"], planes)
    return dict(planes=planes, want_planes=want_planes, z=z)


def test_lattice_points_and_decode_match_oracle(setup, volume):
    s = setup
    axes = om.lattice_axes(MC_BOUND, 1, 64)
    for a, x in enumerate(axes):
        assert np.array_equal(s["mesher"].axes[a], x)
    p32 = om.lattice_points(axes)
    p = torch.from_numpy(p32)
    want = torch.cat([tp.eval_points(p[i:i + 65536], s["grids"], s["dec_state"], "fine", s["bound"])[:, 3] for i in range(0, len(p), 65536)])
    inb = om.in_bound_f32(p32, s["bound"].numpy())
    assert np.array_equal(want.numpy() == 100, ~inb)                        # float32 points: the port's mask is the float32 rule too
    hull_want = om.inside_hull(p32.astype(np.float64), volume["want_planes"])
    hull_got = om.inside_hull(p32.astype(np.float64), volume["planes"])
    assert (hull_want != hull_got).sum() <= 1e-3 * len(p32), (hull_want != hull_got).sum()
    z = volume["z"].reshape(-1).cpu()
    assert torch.equal(z == 100, torch.from_numpy(~(inb & hull_got)))
    keep = torch.from_numpy(inb & hull_got)
    assert keep.sum() > 1000
    assert rel(z[keep], want[keep]) < 1e-4


def test_lattice_without_hull_matches_eval_points_rule(setup):
    """No hull: 100 exactly where the float32 point is not strictly inside the float32 bound; the decode equals FusedRenderer.eval_points
    of the same float32 points where the float64 and float32 rules agree."""
    s = setup
    z = s["mesher"].lattice(s["c"], s["dec"], None).reshape(-1)
    p32 = om.lattice_points(s["mesher"].axes)
    inb = om.in_bound_f32(p32, s["bound"].numpy())
    assert torch.equal((z == 100).cpu(), torch.from_numpy(~inb))
    raw = s["renderer"].eval_points(torch.from_numpy(p32).double().to(DEV), s["dec"], s["c"], "fine", DEV)
    both = torch.from_numpy(inb) & (raw[:, 3] != 100).cpu()
    assert torch.equal(z.cpu()[both], raw[:, 3].cpu()[both])


def test_marching_cubes_matches_oracle(setup, volume):
    s = setup
    verts, faces, eid = s["mesher"].marching_cubes(volume["z"], with_edge_ids=True)
    ax = s["mesher"].axes
    wv, wf, weid = om.marching_cubes(volume["z"].cpu().numpy(), 0.0, [ax[a][2] - ax[a][1] for a in range(3)], [ax[a][0] for a in range(3)])
    assert len(wf) > 1000
    assert np.array_equal(eid.cpu().numpy(), weid)
    assert np.array_equal(verts.cpu().numpy(), wv)
    assert np.array_equal(eid.cpu().numpy()[faces.cpu().numpy()], weid[wf])


def test_seen_masks_clean_and_colors_match_oracle(setup, volume):
    s = setup
    m, store = s["mesher"], s["store"]
    cam = s["sc"]["cam"]
    verts, faces, _ = m.marching_cubes(volume["z"])
    v = verts.cpu().numpy()
    K = np.array([[cam["fx"], 0, cam["cx"]], [0, cam["fy"], cam["cy"]], [0, 0, 1.0]])
    w2c = store.w2c[: len(store)].cpu().numpy().reshape(-1, 4, 4)
    dmax = [float(store.depth[k].max()) for k in range(len(store))]
    est = torch.stack(store.est_c2w)
    for all_frames in (False, True):
        got = m.seen(verts, store, est, len(store) - 1, get_mask_use_all_frames=all_frames).cpu().numpy().astype(bool)
        ws = [np.linalg.inv(e.double().numpy()).astype(np.float32) for e in est] if all_frames else w2c
        want = om.seen_mask(v, ws, K, cam["H"], cam["W"], None if all_frames else dmax)
        assert 0 < want.sum() < len(want)
        assert (got != want).sum() <= max(3, 1e-4 * len(v)), (all_frames, (got != want).sum())
    seen = m.seen(verts, store, est, len(store) - 1)
    for largest, thr in ((False, 0.2), (True, 0.2), (False, 0.0)):
        m2 = copy.copy(m)
        m2.get_largest_components, m2.remove_small_geometry_threshold = largest, thr
        cv, cf = m2.clean(verts, faces, seen)
        wv, wf, _ = om.clean(v, faces.cpu().numpy().astype(np.int64), seen.cpu().numpy().astype(bool), thr, largest)
        assert np.array_equal(cv.cpu().numpy(), wv) and np.array_equal(cf.cpu().numpy(), wf), (largest, thr)
    cv, cf = m.clean(verts, faces, seen)
    col = m.colors(cv, s["c"], s["dec"]).cpu().numpy()
    p = torch.from_numpy(cv.cpu().numpy().astype(np.float32))
    want = om.colors_u8(tp.eval_points(p, s["grids"], s["dec_state"], "color", s["bound"])[:, :3].numpy())
    d = np.abs(col.astype(int) - want.astype(int))
    assert d.max() <= 1 and (d > 0).mean() < 0.01


def read_ply(path):
    with open(path, "rb") as f:
        data = f.read()
    end = data.index(b"end_header\n") + len(b"end_header\n")
    head = data[:end].decode("ascii").split("\n")
    assert head[1] == "format binary_little_endian 1.0"
    nv = int(next(h for h in head if h.startswith("element vertex")).split()[-1])
    nf = int(next(h for h in head if h.startswith("element face")).split()[-1])
    color = "property uchar red" in head
    vt = [("x", "<f8"), ("y", "<f8"), ("z", "<f8")] + ([("r", "u1"), ("g", "u1"), ("b", "u1"), ("a", "u1")] if color else [])
    v = np.frombuffer(data, dtype=vt, count=nv, offset=end)
    f = np.frombuffer(data, dtype=[("n", "u1"), ("i", "<i4", (3,))], count=nf, offset=end + v.nbytes)
    assert np.all(f["n"] == 3) and end + v.nbytes + f.nbytes == len(data)
    verts = np.stack([v["x"], v["y"], v["z"]], 1)
    cols = np.stack([v["r"], v["g"], v["b"], v["a"]], 1) if color else None
    return verts, f["i"].astype(np.int64), cols


def test_get_mesh_writes_ply(setup, tmp_path):
    s = setup
    est = torch.stack(s["store"].est_c2w)
    path = str(tmp_path / "m.ply")
    v, f, col = s["mesher"].get_mesh(path, s["c"], s["dec"], s["store"], est, 4)
    assert len(f) > 0 and v.dtype == np.float64 and f.dtype == np.int64 and col.dtype == np.uint8
    rv, rf, rc = read_ply(path)
    assert np.array_equal(rv, v) and np.array_equal(rf, f) and np.array_equal(rc[:, :3], col) and np.all(rc[:, 3] == 255)
    v2, f2, c2 = s["mesher"].get_mesh(None, s["c"], s["dec"], s["store"], est, 4, color=False, clean_mesh=False)
    assert c2 is None and len(f2) >= len(f)


def test_errors_and_empty_surface(setup, tmp_path):
    from nice_slam_b200.mesh import FusedMesher
    s = setup
    for key, val in (("mesh_coarse_level", True), ("depth_test", True), ("color_mesh_extraction_method", "render_ray_along_normal")):
        with pytest.raises(RuntimeError, match=key):
            FusedMesher(s["renderer"], mesh_cfg(**{key: val}))
    with pytest.raises(RuntimeError, match="show_forecast"):
        s["mesher"].get_mesh(None, s["c"], s["dec"], s["store"], None, 0, show_forecast=True)
    empty = FusedMesher(s["renderer"], mesh_cfg(32, level_set=1000.0))        # no lattice value above the level: no surface
    path = str(tmp_path / "none.ply")
    assert empty.get_mesh(path, s["c"], s["dec"], s["store"], torch.stack(s["store"].est_c2w), 4) is None
    assert not os.path.exists(path)


def test_fused_slam_writes_meshes(tmp_path):
    """The every1 replay with mesh_dir: the reference's files at its frames; meshing draws nothing from any generator; the run log
    equals a run without meshing within the fused-vs-fused bars; final_mesh.ply equals a separate get_mesh call on the final state."""
    from test_gpu_slam import FUSED, cfg_of, load, per_frame, slam_for, within
    from slam_sequences import sequence
    sc = su.load_scenes()["room0"]
    case = load("every1")
    cfg = cfg_of(case, mesh_freq=3, no_mesh_on_first_frame=True, marching_cubes_bound=MC_BOUND)
    cfg["meshing"], cfg["scale"] = mesh_cfg(48, eval_rec=True)["meshing"], 1
    mesh_dir = str(tmp_path / "mesh")
    slam = slam_for(sc, cfg, mesh_dir=mesh_dir)
    states = []
    orig = slam.mesher.get_mesh

    def watched(*a, **k):
        before = ([g.get_state() for g in slam.generators.values()], torch.get_rng_state(), torch.cuda.get_rng_state(),
                  np.random.get_state()[1].copy(), [r.get_state()[1].copy() for r in slam.rngs.values()])
        out = orig(*a, **k)
        after = ([g.get_state() for g in slam.generators.values()], torch.get_rng_state(), torch.cuda.get_rng_state(),
                 np.random.get_state()[1].copy(), [r.get_state()[1].copy() for r in slam.rngs.values()])
        states.append((before, after))
        return out
    slam.mesher.get_mesh = watched
    est, _ = slam.run(sequence(sc, case["n"]), replay=case["replay"])
    n = case["n"]
    mapped = [e["idx"] for e in slam.run_log if e["kind"] == "map"]
    want = {"%05d_mesh.ply" % i for i in mapped if i % 3 == 0 and i != 0} | {"final_mesh.ply", "%05d_mesh.ply" % (n - 1), "final_mesh_eval_rec.ply"}
    assert set(os.listdir(mesh_dir)) == want
    for before, after in states:
        assert all(torch.equal(a, b) for a, b in zip(before[0], after[0]))
        assert torch.equal(before[1], after[1]) and torch.equal(before[2], after[2]) and np.array_equal(before[3], after[3])
        assert all(np.array_equal(a, b) for a, b in zip(before[4], after[4]))
    assert slam.times["meshing"] > 0
    plain = slam_for(sc, cfg_of(case))
    est_b, _ = plain.run(sequence(sc, n), replay=case["replay"])
    assert "meshing" not in plain.times
    assert [(e["kind"], e["idx"]) for e in slam.run_log] == [(e["kind"], e["idx"]) for e in plain.run_log]
    within(per_frame(est, slam.run_log, est_b, plain.run_log, n), FUSED["every1"], "meshing")
    slam.mesher.get_mesh = orig
    v, f, col = slam.mesher.get_mesh(None, slam.c, slam.dec, slam.store, slam.estimate_c2w_list, n - 1)
    rv, rf, rc = read_ply(os.path.join(mesh_dir, "final_mesh.ply"))
    assert np.array_equal(rv, v) and np.array_equal(rf, f) and np.array_equal(rc[:, :3], col)
    with open(os.path.join(mesh_dir, "final_mesh.ply"), "rb") as a, open(os.path.join(mesh_dir, "%05d_mesh.ply" % (n - 1)), "rb") as b:
        assert a.read() == b.read()


def test_against_reference_mesher(setup):
    """tests/golden/mesh/room0.pt (the reference Mesher on CPU): the lattice pass at resolution 24 (no hull) against Mesher.eval_points to
    the eval_points bar with the same out-of-bound points; the float32 in-bound rule on points between float32(bound) and bound; the seen
    masks of both modes."""
    import ctypes as C
    from nice_slam_b200 import _lib
    from nice_slam_b200.keyframes import KeyframeStore
    from nice_slam_b200.mesh import FusedMesher
    from nice_slam_b200.renderer import _VP, _stream
    s = setup
    g = torch.load(os.path.join(su.GOLDEN, "mesh", "room0.pt"), map_location="cpu", weights_only=False)
    R = g["resolution"]
    m = FusedMesher(s["renderer"], mesh_cfg(R))
    z = m.lattice(s["c"], s["dec"], None).cpu()
    want = g["z"].reshape(R, R, R).permute(1, 0, 2)                          # meshgrid('xy') order -> [ix, iy, iz]
    assert torch.equal(z == 100, want == 100)
    assert rel(z[want != 100], want[want != 100]) < 1e-4
    ep = g["edge_points"].double().to(DEV).contiguous()
    inp, keep = m._render_inputs(s["c"], s["dec"], "color", DEV)
    raw = torch.empty(len(ep), 4, dtype=torch.float32, device=DEV)
    col = torch.empty(len(ep), 3, dtype=torch.uint8, device=DEV)
    _lib.check(_lib.lib().nsb_mesh_colors(C.byref(inp), _VP(ep.data_ptr()), len(ep), _VP(raw.data_ptr()), _VP(col.data_ptr()), _stream()), "colors")
    assert torch.equal(raw[:, 3].cpu() == 100, g["edge_z"] == 100)
    cam = s["sc"]["cam"]
    store = KeyframeStore(cam["H"], cam["W"], cam["fx"], cam["fy"], cam["cx"], cam["cy"], DEV)
    for k, sd in enumerate(g["keyframe_seeds"]):
        depth, color = su.make_frame(s["sc"], sd)
        store.append(k, color, depth, su.make_pose(s["sc"], sd))
    probe = g["probe"].double().to(DEV).contiguous()
    est = torch.stack(store.est_c2w)
    for key, all_frames in (("seen_kf", False), ("seen_all", True)):
        got = m.seen(probe, store, est, len(store) - 1, get_mask_use_all_frames=all_frames).cpu().bool()
        assert (got != g[key]).sum() <= 5, (key, int((got != g[key]).sum()))
