"""float64 numpy restatement of the mesh extraction of nice_slam_b200.mesh.FusedMesher (Mesher.get_mesh, src/utils/Mesher.py:349-574).

Every step the CUDA path takes, with the same decisions and output order, in plain numpy / scipy:
  lattice        get_grid_uniform (:321-347): np.linspace axes, float32 points, the float32 in-bound rule of Mesher.eval_points (:301-304)
  hull           convex hull of camera centres + back-projected depth pixels (scipy over ALL candidates), scaled about its vertex mean
  marching_cubes the table of tools/gen_mc_table.py (parsed from nice_slam_b200/csrc/nsb_mc_table.h): one vertex per crossed lattice
                 edge, vertices in (lattice point, axis) order, faces in (cell, table) order
  seen_mask      point_masks' seen output (:53-212)
  clean          face culling, shared-edge components (scipy.sparse.csgraph), area filter, compaction (:469-511)
  colors         direct_point_query (:513-524, 555-556) through oracle.torch_port.eval_points
"""
import os
import re

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TABLE_H = os.path.join(ROOT, "nice_slam_b200", "csrc", "nsb_mc_table.h")


def load_table():
    """(edges [12,2], tri_count [256], tri [256, 3*max]) parsed from the generated header."""
    text = open(TABLE_H).read()
    nums = lambda name: [int(v) for v in re.findall(r"-?\d+", re.search(name + r"\[\d[^=]*=\s*\{(.*?)\};", text, re.S).group(1))]
    mt = int(re.search(r"#define NSB_MC_MAX_TRI (\d+)", text).group(1))
    return (np.array(nums("kMcEdge"), np.int64).reshape(12, 2), np.array(nums("kMcTriCount"), np.int64),
            np.array(nums("kMcTri"), np.int64).reshape(256, 3 * mt))


def lattice_axes(marching_cubes_bound, scale, resolution):
    """x, y, z of get_grid_uniform: np.linspace(lo - 0.05, hi + 0.05, R) of the float64 bound * scale."""
    b = np.array(marching_cubes_bound, dtype=np.float64) * scale
    return [np.linspace(b[a][0] - 0.05, b[a][1] + 0.05, resolution) for a in range(3)]


def lattice_points(axes):
    """float32 [Rx*Ry*Rz, 3] in [ix, iy, iz] order (the reference's meshgrid('xy') points, transposed)."""
    xx, yy, zz = np.meshgrid(axes[0].astype(np.float32), axes[1].astype(np.float32), axes[2].astype(np.float32), indexing="ij")
    return np.stack([xx.ravel(), yy.ravel(), zz.ravel()], 1)


def in_bound_f32(p32, bound):
    """Mesher.eval_points' mask: float32 points against the bound rounded to float32, strict."""
    b = np.asarray(bound, dtype=np.float64).astype(np.float32)
    return np.all((p32 < b[:, 1]) & (p32 > b[:, 0]), axis=1)


def backproject(depth, c2w, fx, fy, cx, cy):
    """World points of every pixel with depth > 0 (NICE camera: x = (u-cx)/fx d, y = -(v-cy)/fy d, z = -d), float64."""
    H, W = depth.shape
    v, u = np.nonzero(depth > 0)
    d = depth[v, u].astype(np.float64)
    cam = np.stack([(u - cx) / fx * d, -(v - cy) / fy * d, -d], 1)
    c2w = np.asarray(c2w, dtype=np.float64)
    return cam @ c2w[:3, :3].T + c2w[:3, 3]


def hull_equations(points, bound_scale):
    """scipy ConvexHull of `points`, scaled by bound_scale about the mean of its vertices -> equations [F,4] (n . x + d <= 0 inside)."""
    from scipy.spatial import ConvexHull
    h = ConvexHull(points)
    v = points[h.vertices]
    c = v.mean(0)
    return ConvexHull(c + bound_scale * (v - c)).equations


def inside_hull(p64, eq):
    """All half-spaces: ((n0 x + n1 y) + n2 z) + d <= 0, evaluated in that order."""
    s = ((eq[None, :, 0] * p64[:, 0:1] + eq[None, :, 1] * p64[:, 1:2]) + eq[None, :, 2] * p64[:, 2:3]) + eq[None, :, 3]
    return np.all(s <= 0, axis=1)


def marching_cubes(vol, level, spacing, origin):
    """vol float32 [Rx,Ry,Rz] -> (verts f64 [V,3], faces int64 [F,3], edge_id int64 [V]).  Corner inside iff value > level; vertex of edge
    (p, a) at ((p + t e_a) * spacing + origin), t = (level - v0) / (v1 - v0) in float64; edge id = a * N + linear(p)."""
    edges, tri_count, tri = load_table()
    R = np.array(vol.shape)
    N = int(R.prod())
    v = vol.astype(np.float64)
    inside = v > level
    idx = np.arange(N).reshape(vol.shape)
    strides = np.array([R[1] * R[2], R[2], 1])
    # crossed lattice edges, ordered by (point, axis)
    eids, ts = [], []
    for a in range(3):
        sl0 = [slice(None)] * 3; sl1 = [slice(None)] * 3
        sl0[a] = slice(0, R[a] - 1); sl1[a] = slice(1, R[a])
        cr = inside[tuple(sl0)] != inside[tuple(sl1)]
        p = idx[tuple(sl0)][cr]
        v0, v1 = v[tuple(sl0)][cr], v[tuple(sl1)][cr]
        eids.append(a * N + p); ts.append((level - v0) / (v1 - v0))
    eid = np.concatenate(eids); t = np.concatenate(ts)
    order = np.lexsort((eid // N, eid % N))
    eid, t = eid[order], t[order]
    a = eid // N; p = eid % N
    ijk = np.stack([p // strides[0], (p // strides[1]) % R[1], p % R[2]], 1).astype(np.float64)
    ijk[np.arange(len(a)), a] = ijk[np.arange(len(a)), a] + t
    verts = ijk * np.asarray(spacing, np.float64) + np.asarray(origin, np.float64)
    # cells, in linear order of their lower corner
    cidx = idx[:-1, :-1, :-1].ravel()
    case = np.zeros(cidx.shape, np.int64)
    for c in range(8):
        off = (c & 1) * strides[0] + ((c >> 1) & 1) * strides[1] + ((c >> 2) & 1) * strides[2]
        case |= inside.ravel()[cidx + off].astype(np.int64) << c
    faces_e = []
    cell_edge = np.zeros((12,), np.int64)
    for e in range(12):
        c0 = edges[e][0]; ax = e // 4
        cell_edge[e] = ax * N + (c0 & 1) * strides[0] + ((c0 >> 1) & 1) * strides[1] + ((c0 >> 2) & 1) * strides[2]
    has = tri_count[case] > 0
    for ci, k in zip(cidx[has], case[has]):
        for j in range(tri_count[k]):
            faces_e.append([cell_edge[tri[k][3 * j + m]] + ci for m in range(3)])
    faces_e = np.array(faces_e, np.int64).reshape(-1, 3)
    okey = (eid % N) * 3 + eid // N                                     # ascending: (point, axis) order
    faces = np.searchsorted(okey, (faces_e % N) * 3 + faces_e // N)
    return verts, faces, eid


def seen_mask(verts, w2c_list, K, H, W, depth_max=None):
    """point_masks' seen output in float64: cam = w2c [p, 1]; cam.x *= -1; uv = K cam; z = uv.z + 1e-8; 0 < u/z < W, 0 < v/z < H, z < 0;
    keyframe mode (depth_max given, one per pose) adds -cam.z < depth_max * 1.1."""
    p = np.concatenate([verts.astype(np.float32).astype(np.float64), np.ones((len(verts), 1))], 1)
    seen = np.zeros(len(verts), bool)
    for m, w2c in enumerate(w2c_list):
        cam = p @ np.asarray(w2c, np.float64).T
        cam[:, 0] *= -1
        uv = cam[:, :3] @ np.asarray(K, np.float64).T
        z = uv[:, 2] + 1e-8
        u, v = uv[:, 0] / z, uv[:, 1] / z
        s = (u < W) & (u > 0) & (v < H) & (v > 0) & (z < 0)
        if depth_max is not None:
            s &= -cam[:, 2] < np.float64(np.float32(depth_max[m]) * np.float32(1.1))
        seen |= s
    return seen


def face_areas(verts, faces):
    a, b, c = verts[faces[:, 0]], verts[faces[:, 1]], verts[faces[:, 2]]
    return np.sqrt((np.cross(b - a, c - a) ** 2).sum(1)) / 2


def clean(verts, faces, seen, threshold, largest):
    """Drop faces whose three vertices are unseen; components over shared edges; keep area > threshold (or the largest); compact.
    -> (verts, faces, kept vertex ids)."""
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components
    faces = faces[~(~seen[faces]).all(1)]
    F = len(faces)
    if F == 0:
        return verts[:0], faces, np.zeros(0, np.int64)
    e = np.concatenate([faces[:, [0, 1]], faces[:, [1, 2]], faces[:, [2, 0]]])
    key = np.sort(e, 1)
    key = key[:, 0] * (len(verts) + 1) + key[:, 1]
    fid = np.tile(np.arange(F), 3)
    o = np.argsort(key, kind="stable")
    same = key[o][1:] == key[o][:-1]
    g = coo_matrix((np.ones(int(same.sum())), (fid[o][1:][same], fid[o][:-1][same])), shape=(F, F))
    _, lab = connected_components(g, directed=False)
    area = np.bincount(lab, weights=face_areas(verts, faces))
    keepc = np.zeros(len(area), bool)
    if largest:
        keepc[area.argmax()] = True
    else:
        keepc = area > threshold
    faces = faces[keepc[lab]]
    used = np.zeros(len(verts), bool); used[faces.ravel()] = True
    ids = np.nonzero(used)[0]
    remap = np.cumsum(used) - 1
    return verts[ids], remap[faces], ids


def colors_u8(rgb):
    """uint8(clip(rgb, 0, 1) * 255), truncating as astype(np.uint8) does."""
    return (np.clip(np.asarray(rgb, np.float32), 0, 1) * 255).astype(np.uint8)
