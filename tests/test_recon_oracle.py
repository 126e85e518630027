"""CPU: the PLY reader of nice_slam_b200.recon, the grid plan of nsb_nn_plan (a host function), and the float64 oracle of the
reconstruction metrics (oracle/recon.py) on analytic meshes."""
import ctypes as C
import os
import struct
import subprocess
import tempfile

import numpy as np
import pytest

from oracle import recon as orc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def box_room(size=(4.0, 3.0, 2.5), step=0.1):
    """Closed box [0, size] as a triangle mesh: every face a grid of squares at `step`, two triangles each; shared vertices per face."""
    verts, faces = [], []
    n = [int(round(s / step)) for s in size]
    for a in range(3):
        b, c = (a + 1) % 3, (a + 2) % 3
        for side in (0.0, size[a]):
            u = np.linspace(0, size[b], n[b] + 1)
            w = np.linspace(0, size[c], n[c] + 1)
            U, W = np.meshgrid(u, w, indexing="ij")
            P = np.zeros(U.shape + (3,))
            P[..., a], P[..., b], P[..., c] = side, U, W
            base = sum(len(v) for v in verts)
            verts.append(P.reshape(-1, 3))
            idx = base + np.arange(U.size).reshape(U.shape)
            q = np.stack([idx[:-1, :-1], idx[1:, :-1], idx[1:, 1:], idx[:-1, 1:]], -1).reshape(-1, 4)
            faces.append(np.concatenate([q[:, [0, 1, 2]], q[:, [0, 2, 3]]]))
    return np.concatenate(verts), np.concatenate(faces).astype(np.int64)


# ------------------------------------------------------------------------------------------------ read_ply
def test_read_ply_round_trips_write_ply(tmp_path):
    from nice_slam_b200.mesh import write_ply
    from nice_slam_b200.recon import read_ply
    rng = np.random.default_rng(0)
    v = rng.normal(size=(50, 3))
    f = rng.integers(0, 50, size=(70, 3)).astype(np.int64)
    col = rng.integers(0, 256, size=(50, 3)).astype(np.uint8)
    for colors in (None, col):
        p = str(tmp_path / ("c.ply" if colors is not None else "n.ply"))
        write_ply(p, v, f, colors)
        rv, rf, rc = read_ply(p)
        assert rv.dtype == np.float64 and rf.dtype == np.int64
        assert np.array_equal(rv, v) and np.array_equal(rf, f)
        assert (rc is None) if colors is None else np.array_equal(rc, col)


def _write(path, header, body):
    with open(path, "wb") as fh:
        fh.write(("\n".join(header) + "\nend_header\n").encode("ascii"))
        fh.write(body)


def test_read_ply_float_vertices_extra_properties_int_counts(tmp_path):
    from nice_slam_b200.recon import read_ply
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]], dtype=np.float32) + np.float32(0.25)
    f = np.array([[0, 1, 2], [0, 3, 1], [3, 2, 1]])
    head = ["ply", "format binary_little_endian 1.0", "comment made by hand", "element vertex 4", "property float nx", "property float x",
            "property float y", "property float z", "property uchar red", "property uchar green", "property uchar blue", "property double quality",
            "element face 3", "property int vertex_count_first_is_a_scalar", "property list int uint vertex_indices", "element edge 1",
            "property int vertex1", "property int vertex2"]
    body = b""
    for i, p in enumerate(v):
        body += struct.pack("<ffff", -1.0, *p) + bytes([10 * i, 20 * i, 30 * i]) + struct.pack("<d", 0.5 * i)
    for t in f:
        body += struct.pack("<i", 7) + struct.pack("<i", 3) + struct.pack("<III", *t)
    body += struct.pack("<ii", 0, 1)
    p = str(tmp_path / "hand.ply")
    _write(p, head, body)
    rv, rf, rc = read_ply(p)
    assert np.array_equal(rv, v.astype(np.float64)) and np.array_equal(rf, f)
    assert np.array_equal(rc, np.array([[10 * i, 20 * i, 30 * i] for i in range(4)], dtype=np.uint8))


@pytest.mark.parametrize("case,match", [("ascii", "ascii"), ("big", "big_endian"), ("quad", "face 1 has 4 vertices"), ("noz", "'z'"),
                                         ("truncated", "truncated"), ("range", "outside"), ("vlist", "list property")])
def test_read_ply_rejects(tmp_path, case, match):
    from nice_slam_b200.recon import read_ply
    fmt = {"ascii": "ascii", "big": "binary_big_endian"}.get(case, "binary_little_endian")
    axes = "xy" if case == "noz" else "xyz"
    head = ["ply", "format %s 1.0" % fmt, "element vertex 4"] + ["property double %s" % a for a in axes]
    if case == "vlist":
        head.append("property list uchar int neighbours")
    head += ["element face 2", "property list uchar int vertex_indices"]
    body = b"".join(struct.pack("<" + "d" * len(axes), *([float(i)] * len(axes))) for i in range(4))
    faces = [[0, 1, 2], [0, 2, 3, 1]] if case == "quad" else [[0, 1, 2], [0, 2, 9 if case == "range" else 3]]
    for t in faces:
        body += bytes([len(t)]) + struct.pack("<" + "i" * len(t), *t)
    if case == "truncated":
        body = body[:-5]
    p = str(tmp_path / ("%s.ply" % case))
    _write(p, head, body)
    with pytest.raises(ValueError, match=match):
        read_ply(p)


# ------------------------------------------------------------------------------------------------ the grid rule (host)
def _plan(box, n):
    from nice_slam_b200 import _lib
    g = _lib.NNGrid()
    _lib.check(_lib.lib().nsb_nn_plan((C.c_double * 6)(*box), n, C.byref(g)), "nsb_nn_plan")
    return g


@pytest.mark.parametrize("box,n", [((0, 0, 0, 10, 8, 3), 200000), ((-5, -5, -5, 5, 5, 5), 1), ((0, 0, 0, 1e4, 1, 1), 1000),
                                   ((1, 2, 3, 1, 2, 3), 50), ((0, 0, 0, 10, 10, 0), 1000), ((0, 0, 0, 1, 1, 1), 7)])
def test_grid_plan_bounds_cells_and_covers_the_box(box, n):
    g = _plan(box, n)
    dims = [g.dims[a] for a in range(3)]
    assert g.n_cells == dims[0] * dims[1] * dims[2] <= max(2 * n, 1)
    assert g.cell > 0 and g.slack > 0 and g.n_points == n
    for a in range(3):
        assert g.origin[a] == box[a]
        assert dims[a] >= 1 and (box[3 + a] - box[a]) / g.cell < dims[a]          # the box's far corner falls inside the last cell


def test_struct_size_matches_the_header():
    from nice_slam_b200 import _lib
    prog = '#include <stdio.h>\n#include "nice_slam_b200.h"\nint main(void) { printf("%zu", sizeof(nsb_nn_grid)); return 0; }\n'
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "s.c"), os.path.join(d, "s")
        open(src, "w").write(prog)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), src, "-o", exe])
        assert int(subprocess.check_output([exe])) == C.sizeof(_lib.NNGrid)


# ------------------------------------------------------------------------------------------------ the oracle
def test_oracle_sampling_lands_on_the_picked_face():
    v, f = box_room(step=0.5)
    u = np.random.default_rng(1).random((100000, 3))
    pts, face = orc.sample_surface(v, f, u)
    tri = v[f[face]]
    n = np.cross(tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0])
    assert np.abs(np.einsum("ij,ij->i", pts - tri[:, 0], n)).max() < 1e-12              # on the face's plane
    area = orc.face_areas(v, f)
    assert np.isclose(area.sum(), 2 * (4 * 3 + 3 * 2.5 + 4 * 2.5))
    counts = np.bincount(face, minlength=len(f))                                            # equal areas: about 212 each
    assert np.abs(counts / counts.mean() - 1).max() < 0.4


def test_oracle_metrics_of_a_mesh_against_itself():
    v, f = box_room(step=0.5)
    pts, _ = orc.sample_surface(v, f, np.random.default_rng(2).random((3000, 3)))
    acc, comp, ratio, _, _ = orc.metrics(pts, pts)
    assert (acc, comp, ratio) == (0.0, 0.0, 1.0)


def test_oracle_icp_recovers_a_rigid_motion():
    v, _ = box_room()
    ctr = v.mean(0)
    motion = orc.rigid(0.5, (0.3, -0.5, 0.8), (0.012, -0.008, 0.006))
    centred = np.eye(4)
    centred[:3, 3] = ctr
    M = centred @ motion @ np.linalg.inv(centred)                                            # about the room's centre
    src = orc.transform_points(v, M)
    T, fit, rmse, it = orc.icp_align(src, v, 0.1)
    assert np.abs(T - np.linalg.inv(M)).max() < 1e-9
    assert fit == 1.0 and rmse < 1e-9 and 1 <= it < 30
