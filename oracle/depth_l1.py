"""float64 numpy restatement of the reference's calc_2d_metric (src/tools/eval_recon.py:120-209), the checker of nice_slam_b200.depth and
recon.eval_depth_l1.  Written from the metric's semantics; shares no code with the kernels.

  raycast        brute-force depth of a mesh under one c2w: every pixel's ray against every face in front of the frustum's side planes,
                 with a per-pixel ambiguity flag and, for ambiguous pixels, the depths of every face that may cover them
  view_error     mean |gt - rec| over the pixels of two depth images (0 = background)
  check_proj     eval_recon.py's check_proj in float32 numpy, and check_proj_uvz, its (u, v, z) per point in float64
  viewmatrix     eval_recon.py's viewmatrix, one view at a time
  candidate      one candidate view from six uniforms: volume_rectangular's origin, the rounded target, viewmatrix
"""
import numpy as np

TOL = 1e-9


def _pixel_rays(H, W, fx, fy, cx, cy):
    j, i = np.meshgrid(np.arange(W, dtype=np.float64), np.arange(H, dtype=np.float64))
    d = np.stack([(j - cx) / fx, (i - cy) / fy, np.ones_like(j)], -1).reshape(-1, 3)
    return d


def raycast(vertices, faces, c2w, H, W, fx, fy, cx, cy, z_near, z_far, tol=TOL, chunk=256):
    """-> (depth f64 [H,W], ambiguous bool [H,W], candidates {pixel index i*W+j: sorted depths}).

    Camera space p_cam = R^T (p - t) of the OpenCV c2w.  The ray of pixel (i, j) is d = ((j - cx)/fx, (i - cy)/fy, 1).  For a face with
    camera-space vertices v0 v1 v2 and D = det(v0, v1, v2), the ray hits the face in front of the camera iff sgn(D) d.(v_k x v_k+1) > 0
    for the three edges; the depth is z = D / (N.d), N = (v1 - v0) x (v2 - v0); a hit counts iff z_near <= z <= z_far.  depth = the least
    counted z, 0 without one.
    A pixel is ambiguous if some face has every edge margin sgn(D) d.(v_k x v_k+1) / (|v_k x v_k+1| |d|) >= -tol and z within tol
    (relative) of [z_near, z_far], but not every margin > tol or z not inside the range by more than tol: its centre lies within rounding
    of an edge plane, or its depth within rounding of z_near or z_far.  candidates lists, for each ambiguous pixel, the depths of those
    faces (float64)."""
    v = np.asarray(vertices, dtype=np.float64)
    f = np.asarray(faces, dtype=np.int64)
    c2w = np.asarray(c2w, dtype=np.float64)
    R, t = c2w[:3, :3], c2w[:3, 3]
    vc = (v - t) @ R                                                  # R^T (p - t) for every vertex
    tri = vc[f]                                                       # [F,3,3]
    # faces that can hit a pixel: not wholly behind z_near or beyond z_far, not wholly outside a side plane of the frustum (a margin of
    # two pixels)
    z = tri[..., 2]
    keep = (z.max(1) >= z_near * (1 - tol)) & (z.min(1) <= z_far * (1 + tol))
    sx0, sx1 = (-2.0 - cx) / fx, (W + 1.0 - cx) / fx
    sy0, sy1 = (-2.0 - cy) / fy, (H + 1.0 - cy) / fy
    for s, a, sgn in ((sx1, 0, 1), (sx0, 0, -1), (sy1, 1, 1), (sy0, 1, -1)):
        keep &= ~(sgn * (tri[..., a] - s * z) > 0).all(1)
    tri = tri[keep]
    d = _pixel_rays(H, W, fx, fy, cx, cy)                             # [n,3]
    dn = np.linalg.norm(d, axis=1)
    n = len(d)
    best = np.full(n, np.inf)
    amb = np.zeros(n, bool)
    cand = {}
    for s0 in range(0, len(tri), chunk):
        T = tri[s0:s0 + chunk]
        a, b, c = T[:, 0], T[:, 1], T[:, 2]
        N = np.cross(b - a, c - a)
        D = np.einsum("fk,fk->f", N, a)
        sg = np.sign(D)
        marg = []
        for u, w in ((a, b), (b, c), (c, a)):
            e = np.cross(u, w)
            en = np.linalg.norm(e, axis=1)
            with np.errstate(divide="ignore", invalid="ignore"):
                marg.append((d @ e.T) * sg / (dn[:, None] * en[None, :]))
        marg = np.stack(marg)                                         # [3, n, f]
        with np.errstate(divide="ignore", invalid="ignore"):
            zz = D[None, :] / (d @ N.T)                               # [n, f]
        lo = marg.min(0)
        clear = (lo > tol) & (zz - z_near > tol * z_near) & (z_far - zz > tol * z_far)
        maybe = (lo >= -tol) & (zz >= z_near * (1 - tol)) & (zz <= z_far * (1 + tol))
        best = np.minimum(best, np.where(clear, zz, np.inf).min(1))
        unclear = maybe & ~clear
        amb |= unclear.any(1)
        for p, k in zip(*np.nonzero(maybe)):
            cand.setdefault(int(p), []).append(float(zz[p, k]))
    depth = np.where(np.isfinite(best), best, 0.0)
    cand = {p: sorted(cand.get(p, [])) for p in np.nonzero(amb)[0].tolist()}
    return depth.reshape(H, W), amb.reshape(H, W), cand


def view_error(gt_depth, rec_depth):
    """np.abs(gt_depth - rec_depth).mean() in float64 (eval_recon.py:203)."""
    return float(np.abs(np.asarray(gt_depth, np.float64) - np.asarray(rec_depth, np.float64)).mean())


def check_proj_uvz(points, W, H, fx, fy, cx, cy, c2w):
    """check_proj's projection in float64 from its float32 inputs -> (u, v, z) per point."""
    c = np.array(c2w, dtype=np.float64)
    c[:3, 1] *= -1.0
    c[:3, 2] *= -1.0
    w2c = np.linalg.inv(c).astype(np.float32).astype(np.float64)
    p = np.concatenate([np.asarray(points, np.float64), np.ones((len(points), 1))], 1).astype(np.float32).astype(np.float64)
    cam = p @ w2c.T
    cam[:, 0] *= -1
    K = np.array([[fx, 0.0, cx], [0.0, fy, cy], [0.0, 0.0, 1.0]], dtype=np.float32).astype(np.float64)
    uv = cam[:, :3] @ K.T
    z = uv[:, 2] + 1e-5
    with np.errstate(divide="ignore", invalid="ignore"):
        return uv[:, 0] / z, uv[:, 1] / z, z


def check_proj(points, W, H, fx, fy, cx, cy, c2w):
    """eval_recon.py:60-87 in float32 numpy: True iff some point projects strictly inside the image with 0 <= -z."""
    c = np.array(c2w, dtype=np.float64)
    c[:3, 1] *= -1.0
    c[:3, 2] *= -1.0
    w2c = np.linalg.inv(c).astype(np.float32)
    p = np.concatenate([np.asarray(points, np.float64), np.ones((len(points), 1))], 1).astype(np.float32)
    cam = (p @ w2c.T)[:, :3]
    cam[:, 0] *= -1
    K = np.array([[fx, 0.0, cx], [0.0, fy, cy], [0.0, 0.0, 1.0]], dtype=np.float64).astype(np.float32)
    uv = cam @ K.T
    z = uv[:, 2] + np.float32(1e-5)
    with np.errstate(divide="ignore", invalid="ignore"):
        u, v = uv[:, 0] / z, uv[:, 1] / z
        mask = (0 <= -z) & (u < W) & (u > 0) & (v < H) & (v > 0)
    return bool(mask.sum() > 0)


def viewmatrix(z, up, pos):
    z = np.asarray(z, np.float64)
    vec2 = z / np.linalg.norm(z)
    vec0 = np.cross(up, vec2)
    vec0 = vec0 / np.linalg.norm(vec0)
    vec1 = np.cross(vec2, vec0)
    vec1 = vec1 / np.linalg.norm(vec1)
    m = np.eye(4)
    m[:3, :] = np.stack([vec0, vec1, vec2, np.asarray(pos, np.float64)], 1)
    return m


def candidate(u6, extents, transform):
    """One candidate view of calc_2d_metric's loop from six uniforms: origin = transform applied to (u[:3] - 0.5) * extents
    (volume_rectangular); target = round(-10000 + 20000 u[3:], 2); c2w = viewmatrix(target - origin, [0, 0, -1], origin)."""
    u6 = np.asarray(u6, np.float64)
    p = np.append((u6[:3] - 0.5) * np.asarray(extents, np.float64), 1.0)
    origin = (np.asarray(transform, np.float64) @ p)[:3]
    target = np.array([round(-10000.0 + 20000.0 * x, 2) for x in u6[3:]])
    return viewmatrix(target - origin, np.array([0.0, 0.0, -1.0]), origin)
