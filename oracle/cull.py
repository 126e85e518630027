"""float64 numpy restatement of the reference's src/tools/cull_mesh.py (the culling of nice_slam_b200.cull / nsb_cull_*).

  load_poses   the parser: 16 floats per line as float64, columns 1 and 2 of rows 0-2 negated, cast to float32
  w2c_list     np.linalg.inv of the float32 c2w (numpy inverts in float64 and rounds to float32), as cull_mesh.py:51
  project      u, v, z of every vertex under every pose, in float64 from the float32 vertex and w2c
  seen_mask    0 <= -z and 0 < u < W and 0 < v < H for some pose (strict, no edge, no depth limit)
  kept_faces   indices of the faces with a seen vertex, ascending (update_faces(~all three unseen))
"""
import numpy as np

H, W, FX, FY, CX, CY = 680, 1200, 600.0, 600.0, 599.5, 339.5


def load_poses(path):
    out = []
    for line in open(path):
        c2w = np.array(list(map(float, line.split())), dtype=np.float64).reshape(4, 4)
        c2w[:3, 1] *= -1
        c2w[:3, 2] *= -1
        out.append(c2w.astype(np.float32))
    return np.array(out, dtype=np.float32).reshape(-1, 4, 4)


def w2c_list(c2w):
    return [np.linalg.inv(np.asarray(c, np.float32)) for c in c2w]


def project(verts, w2c, H=H, W=W, fx=FX, fy=FY, cx=CX, cy=CY):
    """-> (u, v, z) float64 [V] of one pose: p = float32(vertex); cam = w2c [p, 1]; cam.x = -cam.x; uv = K cam (K float32);
    z = uv.z + 1e-5; u = uv.x / z; v = uv.y / z."""
    p = np.concatenate([np.asarray(verts, np.float64).astype(np.float32).astype(np.float64), np.ones((len(verts), 1))], 1)
    K = np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]], dtype=np.float32).astype(np.float64)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):           # non-finite poses give NaN
        cam = p @ np.asarray(w2c, np.float32).astype(np.float64).T
        cam[:, 0] *= -1
        uv = cam[:, :3] @ K.T
        z = uv[:, 2] + 1e-5
        return uv[:, 0] / z, uv[:, 1] / z, z


def seen_mask(verts, w2c_all, H=H, W=W, fx=FX, fy=FY, cx=CX, cy=CY):
    """Every pose is tested on the vertices no earlier pose has seen (the same result as testing all, in less time)."""
    verts = np.asarray(verts, np.float64)
    seen = np.zeros(len(verts), bool)
    todo = np.arange(len(verts))
    for w2c in w2c_all:
        if not len(todo):
            break
        u, v, z = project(verts[todo], w2c, H, W, fx, fy, cx, cy)
        with np.errstate(invalid="ignore"):
            s = (0 <= -z) & (u < W) & (u > 0) & (v < H) & (v > 0)
        seen[todo[s]] = True
        todo = todo[~s]
    return seen


def near_border(verts, w2c_all, H=H, W=W, fx=FX, fy=FY, cx=CX, cy=CY, px=0.01, dz=1e-4):
    """For each vertex: is there a pose under which the float64 decision is within rounding -- z within dz of 0, or (u, v) within px
    pixels of the frame's border while the other tests pass?"""
    verts = np.asarray(verts, np.float64)
    near = np.zeros(len(verts), bool)
    for w2c in w2c_all:
        u, v, z = project(verts, w2c, H, W, fx, fy, cx, cy)
        with np.errstate(invalid="ignore"):
            inside = (z <= dz) & (u > -px) & (u < W + px) & (v > -px) & (v < H + px)
            edge = np.minimum(np.minimum(np.abs(u), np.abs(u - W)), np.minimum(np.abs(v), np.abs(v - H))) < px
            near |= (np.abs(z) < dz) | (inside & edge)
    return near


def kept_faces(faces, seen):
    return np.nonzero(np.asarray(seen, bool)[np.asarray(faces)].any(axis=1))[0]
