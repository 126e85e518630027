"""CPU checks of the mesh extraction's float64 oracle (oracle/mesh.py) and of the generated marching-cubes table."""
import itertools
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import mesh as om  # noqa: E402

SPACING = (0.1, 0.12, 0.09)
ORIGIN = (-1.3, -1.5, -1.1)


def _coords(shape):
    return [ORIGIN[a] + SPACING[a] * np.arange(shape[a]) for a in range(3)]


def _sphere(n=28, r=0.9):
    x, y, z = np.meshgrid(*_coords((n, n, n)), indexing="ij")
    return (r - np.sqrt(x * x + y * y + z * z)).astype(np.float32)        # occupied (> 0) inside the ball


def _torus(n=30, R=0.75, r=0.3):
    x, y, z = np.meshgrid(*_coords((n, n, n)), indexing="ij")
    return (r - np.sqrt((np.sqrt(x * x + y * y) - R) ** 2 + z * z)).astype(np.float32)


def _blobs(n=30):
    x, y, z = np.meshgrid(*_coords((n, n, n)), indexing="ij")
    f = np.exp(-((x - 0.45) ** 2 + y * y + z * z) / 0.12) + np.exp(-((x + 0.45) ** 2 + y * y + z * z) / 0.12)
    return (f - np.exp(-0.45 ** 2 / 0.12) * 1.8).astype(np.float32)            # the two blobs meet at a saddle at the origin


def _edges_count(faces):
    e = np.sort(np.concatenate([faces[:, [0, 1]], faces[:, [1, 2]], faces[:, [2, 0]]]), 1)
    _, cnt = np.unique(e, axis=0, return_counts=True)
    return cnt


def _euler(verts, faces):
    return len(np.unique(faces)) - len(_edges_count(faces)) + len(faces)


def _check_on_edges(vol, verts, eid, level=0.0):
    N = vol.size
    R = np.array(vol.shape)
    a, p = eid // N, eid % N
    ijk = np.stack([p // (R[1] * R[2]), (p // R[2]) % R[1], p % R[2]], 1)
    v0 = vol.ravel()[p].astype(np.float64)
    q = ijk.copy(); q[np.arange(len(a)), a] += 1
    v1 = vol[q[:, 0], q[:, 1], q[:, 2]].astype(np.float64)
    assert np.all((v0 > level) != (v1 > level))                              # every vertex on a crossed edge
    t = (level - v0) / (v1 - v0)
    want = ijk.astype(np.float64)
    want[np.arange(len(a)), a] += t
    assert np.array_equal(verts, want * np.array(SPACING) + np.array(ORIGIN))


def _check_winding(vol, verts, faces):
    """Face normals point from occupied (value > level) to free space: against the volume's gradient."""
    tri = verts[faces]
    n = np.cross(tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0])
    c = tri.mean(1)
    g = np.stack(np.gradient(vol.astype(np.float64), *SPACING), -1)
    ijk = np.clip(np.rint((c - np.array(ORIGIN)) / np.array(SPACING)).astype(int), 0, np.array(vol.shape) - 1)
    gc = g[ijk[:, 0], ijk[:, 1], ijk[:, 2]]
    big = np.linalg.norm(n, axis=1) > 1e-9
    assert np.mean((n * gc).sum(1)[big] < 0) > 0.99


@pytest.mark.parametrize("name,vol,euler", [("sphere", _sphere(), 2), ("torus", _torus(), 0), ("blobs", _blobs(), 2)])
def test_marching_cubes_closed_manifold(name, vol, euler):
    verts, faces, eid = om.marching_cubes(vol, 0.0, SPACING, ORIGIN)
    assert len(faces) > 100
    _check_on_edges(vol, verts, eid)
    assert np.all(_edges_count(faces) == 2), name                            # closed 2-manifold
    assert _euler(verts, faces) == euler, name
    _check_winding(vol, verts, faces)


def test_marching_cubes_corners_at_level():
    vol = np.round(_sphere() * 4).astype(np.float32) / 4                  # many corners exactly at the level (0): they count as free
    verts, faces, eid = om.marching_cubes(vol, 0.0, SPACING, ORIGIN)
    _check_on_edges(vol, verts, eid)
    assert np.all(_edges_count(faces) == 2)


@pytest.mark.parametrize("case", range(256))
def test_every_case_closes_across_neighbours(case):
    """Each sign pattern, embedded in a 4x4x4 lattice with random neighbours and free borders (every ambiguous face configuration
    appears between the centre cell and its neighbours): the surface is closed and sits on crossed edges."""
    rng = np.random.RandomState(case)
    vol = np.full((4, 4, 4), -1.0, np.float32)
    vol[1:3, 1:3, 1:3] = np.where(rng.rand(2, 2, 2) < 0.5, -0.5, 0.5) + rng.uniform(-0.2, 0.2, (2, 2, 2))
    for c in range(8):
        vol[1 + (c & 1), 1 + ((c >> 1) & 1), 1 + ((c >> 2) & 1)] = (0.3 + 0.1 * c) * (1 if (case >> c) & 1 else -1)
    verts, faces, eid = om.marching_cubes(vol, 0.0, SPACING, ORIGIN)
    _check_on_edges(vol, verts, eid)
    if len(faces):
        assert np.all(_edges_count(faces) == 2)


def test_table_is_regenerated_exactly():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "gen_mc_table.py"), "--check"])
    assert r.returncode == 0, "nsb_mc_table.h differs from tools/gen_mc_table.py's output"


def test_table_cases_are_complements():
    """Complementary sign patterns give the same triangles with opposite winding (the face rule is symmetric in inside / outside only
    for unambiguous cases, so compare the unambiguous ones)."""
    edges, cnt, tri = om.load_table()
    for k in range(256):
        if cnt[k] and cnt[255 - k] == cnt[k] and cnt[k] <= 2:
            a = {tuple(sorted(tri[k][3 * j: 3 * j + 3])) for j in range(cnt[k])}
            b = {tuple(sorted(tri[255 - k][3 * j: 3 * j + 3])) for j in range(cnt[k])}
            assert a == b


def test_hull_reduction_keeps_every_vertex():
    """Support points over K directions, then the points outside their hull: the hull of the survivors is the full hull."""
    from scipy.spatial import ConvexHull
    from nice_slam_b200.mesh import hull_directions
    rng = np.random.RandomState(3)
    for trial in range(5):
        pts = rng.randn(4000, 3) * np.array([2.0, 1.0, 0.5]) + rng.randn(3)
        d = hull_directions(128)
        sup = pts[np.unique(np.argmax(pts @ d.T, axis=0))]
        inner = ConvexHull(sup)
        out = np.any(pts @ inner.equations[:, :3].T + inner.equations[:, 3] > 0, axis=1)
        survivors = np.concatenate([sup, pts[out]])
        full = ConvexHull(pts)
        red = ConvexHull(survivors)
        assert {tuple(v) for v in pts[full.vertices]} == {tuple(v) for v in survivors[red.vertices]}
        assert out.sum() < len(pts) // 4


def test_clean_drops_unseen_faces_and_small_components():
    verts, faces, _ = om.marching_cubes(_blobs(), 0.0, SPACING, ORIGIN)
    seen = np.ones(len(verts), bool)
    v2, f2, ids = om.clean(verts, faces, seen, 0.0, False)
    assert len(f2) == len(faces) and np.array_equal(v2, verts)
    seen = verts[:, 0] > 0.3                                                # one blob seen in part
    v3, f3, ids = om.clean(verts, faces, seen, 0.0, False)
    assert 0 < len(f3) < len(faces) and np.array_equal(v3, verts[ids])
    v4, f4, _ = om.clean(verts, faces, np.ones(len(verts), bool), 1e9, False)
    assert len(f4) == 0


# ------------------------------------------------------------------------------------ against the reference Mesher (tests/make_golden_mesh.py)
def _golden():
    import torch
    return torch.load(os.path.join(ROOT, "tests", "golden", "mesh", "room0.pt"), map_location="cpu", weights_only=False)


def test_lattice_points_equal_reference_bit_for_bit():
    g = _golden()
    axes = om.lattice_axes(g["marching_cubes_bound"], g["scale"], g["resolution"])
    for a in range(3):
        assert np.array_equal(axes[a], g["axes"][a].numpy())
    R = g["resolution"]
    ref = g["grid_points"].numpy().reshape(R, R, R, 3).transpose(1, 0, 2, 3).reshape(-1, 3)      # meshgrid('xy') -> [ix, iy, iz]
    assert np.array_equal(om.lattice_points(axes).view(np.uint32), ref.view(np.uint32))


def test_in_bound_rule_is_the_float32_one():
    import scene_util as su
    g = _golden()
    bound = su.scene_bound(su.load_scenes()["room0"]).numpy()
    assert np.array_equal(om.in_bound_f32(g["edge_points"].numpy(), bound), g["edge_z"].numpy() != 100)
    R = g["resolution"]
    p = g["grid_points"].numpy()
    assert np.array_equal(om.in_bound_f32(p, bound), g["z"].numpy() != 100)
    assert 0 < (g["edge_z"].numpy() == 100).sum() < len(g["edge_z"])


def _near_threshold(p, w2c_list, K, H, W, lim):
    """Largest closeness (relative) of a deciding quantity to its threshold over the poses, float64."""
    q = np.concatenate([p, np.ones((len(p), 1))], 1)
    best = np.full(len(p), np.inf)
    for m, w2c in enumerate(w2c_list):
        cam = q @ np.asarray(w2c, np.float64).T
        cam[:, 0] *= -1
        uv = cam[:, :3] @ K.T
        z = uv[:, 2] + 1e-8
        u, v = uv[:, 0] / z, uv[:, 1] / z
        r = [np.abs(u) / max(W, 1), np.abs(u - W) / W, np.abs(v) / H, np.abs(v - H) / H]
        if lim is not None:
            r.append(np.abs(-cam[:, 2] - lim[m]) / lim[m])
        best = np.minimum(best, np.min(r, axis=0))
    return best


def test_seen_masks_equal_reference():
    import scene_util as su
    import torch
    g = _golden()
    sc = su.load_scenes()["room0"]
    cam = sc["cam"]
    K = np.array([[cam["fx"], 0, cam["cx"]], [0, cam["fy"], cam["cy"]], [0, 0, 1.0]])
    c2w = [su.make_pose(sc, s) for s in g["keyframe_seeds"]]
    w2c = [np.linalg.inv(c.numpy()).astype(np.float32) for c in c2w]
    lim = [float(su.make_frame(sc, s)[0].max()) for s in g["keyframe_seeds"]]
    p = g["probe"].numpy().astype(np.float64)
    for key, dmax in (("seen_kf", lim), ("seen_all", None)):
        want = g[key].numpy()
        got = om.seen_mask(p, w2c, K, cam["H"], cam["W"], dmax)
        assert 0 < want.sum() < len(want), key
        bad = got != want
        if bad.any():
            lims = None if dmax is None else np.float32(dmax) * np.float32(1.1)
            close = _near_threshold(p[bad], w2c, K, cam["H"], cam["W"], lims)
            assert np.all(close < 1e-6), (key, close)
        assert bad.sum() <= 5, (key, bad.sum())
