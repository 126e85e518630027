"""Synthetic scenes for the culling tests and tools/bench_cull.py: a closed box room as a triangle mesh, camera poses inside it, and the
files cull_mesh.py reads (a PLY with extra vertex and face properties, a traj.txt)."""
import numpy as np

ROOM = (4.0, 3.0, 2.5)


def box_room(step, size=ROOM):
    """Closed box [0, size] (z up): every side a grid of squares at about `step`, two triangles each; vertices shared within a side."""
    verts, faces = [], []
    n = [max(1, int(round(s / step))) for s in size]
    for a in range(3):
        b, c = (a + 1) % 3, (a + 2) % 3
        for side in (0.0, size[a]):
            U, W = np.meshgrid(np.linspace(0, size[b], n[b] + 1), np.linspace(0, size[c], n[c] + 1), indexing="ij")
            P = np.zeros(U.shape + (3,))
            P[..., a], P[..., b], P[..., c] = side, U, W
            base = sum(len(v) for v in verts)
            verts.append(P.reshape(-1, 3))
            idx = base + np.arange(U.size).reshape(U.shape)
            q = np.stack([idx[:-1, :-1], idx[1:, :-1], idx[1:, 1:], idx[:-1, 1:]], -1).reshape(-1, 4)
            faces.append(np.concatenate([q[:, [0, 1, 2]], q[:, [0, 2, 3]]]))
    return np.concatenate(verts), np.concatenate(faces).astype(np.int64)


def room_poses(n, seed, max_pitch_deg=30.0, size=ROOM):
    """n c2w float32 [n,4,4] in the NICE convention (x right, y up, looking along -z): centres in the middle third of the room at
    1.1-1.4 m, any yaw, pitch within +-max_pitch_deg."""
    rs = np.random.RandomState(seed)
    out = np.zeros((n, 4, 4), np.float64)
    for k in range(n):
        c = np.array([rs.uniform(size[0] / 3, 2 * size[0] / 3), rs.uniform(size[1] / 3, 2 * size[1] / 3), rs.uniform(1.1, 1.4)])
        yaw, pitch = rs.uniform(0, 2 * np.pi), np.radians(rs.uniform(-max_pitch_deg, max_pitch_deg))
        f = np.array([np.cos(yaw) * np.cos(pitch), np.sin(yaw) * np.cos(pitch), np.sin(pitch)])
        r = np.cross(f, [0.0, 0.0, 1.0])
        r /= np.linalg.norm(r)
        u = np.cross(r, f)
        out[k, :3, 0], out[k, :3, 1], out[k, :3, 2], out[k, :3, 3], out[k, 3, 3] = r, u, -f, c, 1.0
    return out.astype(np.float32)


def write_traj(path, c2w):
    """traj.txt of NICE-convention poses: the flips of columns 1 and 2 undone (they are their own inverse), 16 numbers per line."""
    raw = np.array(c2w, np.float64).reshape(-1, 4, 4).copy()
    raw[:, :3, 1] *= -1
    raw[:, :3, 2] *= -1
    with open(path, "w") as fh:
        for m in raw:
            fh.write(" ".join(repr(float(x)) for x in m.reshape(16)) + "\n")


def write_ply_with_extras(path, verts, faces, seed=0):
    """Binary little-endian PLY: float x y z, float nx ny nz, uchar red green blue alpha per vertex; per face a uchar flag before and an
    int label after the vertex list; a trailing one-record 'extra' element.  -> the vertex element's bytes."""
    rs = np.random.RandomState(seed)
    V, F = len(verts), len(faces)
    vt = np.dtype([("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("nx", "<f4"), ("ny", "<f4"), ("nz", "<f4"),
                   ("red", "u1"), ("green", "u1"), ("blue", "u1"), ("alpha", "u1")])
    v = np.zeros(V, vt)
    v["x"], v["y"], v["z"] = verts[:, 0], verts[:, 1], verts[:, 2]
    v["nx"], v["ny"], v["nz"] = rs.normal(size=(3, V)).astype(np.float32)
    for c in ("red", "green", "blue", "alpha"):
        v[c] = rs.randint(0, 256, V)
    ft = np.dtype([("flag", "u1"), ("n", "u1"), ("i", "<i4", (3,)), ("label", "<i4")])
    f = np.zeros(F, ft)
    f["flag"], f["n"], f["i"], f["label"] = rs.randint(0, 256, F), 3, faces, np.arange(F)
    head = ["ply", "format binary_little_endian 1.0", "comment synthetic room", "element vertex %d" % V]
    head += ["property float %s" % a for a in ("x", "y", "z", "nx", "ny", "nz")] + ["property uchar %s" % a for a in ("red", "green", "blue", "alpha")]
    head += ["element face %d" % F, "property uchar flag", "property list uchar int vertex_indices", "property int label",
             "element extra 1", "property double value", "end_header"]
    with open(path, "wb") as fh:
        fh.write(("\n".join(head) + "\n").encode("ascii"))
        fh.write(v.tobytes())
        fh.write(f.tobytes())
        fh.write(np.array([3.25]).astype("<f8").tobytes())
    return v.tobytes()
