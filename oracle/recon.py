"""float64 numpy / scipy restatement of the reconstruction metrics of nice_slam_b200.recon (calc_3d_metric and get_align_transformation,
src/tools/eval_recon.py:45-59, 91-117).

  sample_surface   trimesh.sample.sample_surface (trimesh 3.10.7) with the uniforms given: numpy's area order, np.cumsum,
                   np.searchsorted (left), the a + b > 1 fold, (a e1 + b e2) + v0
  metrics          accuracy / completion / completion ratio through scipy.spatial.cKDTree, as eval_recon.py computes them
  icp_align        open3d 0.13's registration_icp with TransformationEstimationPointToPoint, read as nice_slam_b200.recon.icp_align
                   states it: correspondences by cKDTree within the threshold (d < threshold, cKDTree's distance_upper_bound rule),
                   Umeyama without scaling (Eigen::umeyama: SVD of the cross-covariance, the reflection fix), T = update @ T

Neither trimesh nor open3d is available where this project is tested, so this restatement is not pinned against them: the sampling
follows trimesh 3.10.7's source as published, and the ICP loop follows open3d 0.13's RegistrationICP as published, with two differences
of rounding only -- the source points are transformed from the originals by T each iteration (open3d transforms its copy in place by
each update), and the cross-covariance is formed from the centred points here.
"""
import numpy as np
from scipy.spatial import cKDTree


def face_areas(vertices, faces):
    v = np.asarray(vertices, dtype=np.float64)
    f = np.asarray(faces, dtype=np.int64)
    c = np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]])
    return np.sqrt((c ** 2).sum(axis=1)) / 2.0


def sample_surface(vertices, faces, uniforms):
    """-> (points f64 [count,3], face index int64 [count]) for uniforms f64 [count,3] = (u0, u1, u2)."""
    v = np.asarray(vertices, dtype=np.float64)
    f = np.asarray(faces, dtype=np.int64)
    u = np.asarray(uniforms, dtype=np.float64)
    cum = np.cumsum(face_areas(v, f))
    face = np.minimum(np.searchsorted(cum, u[:, 0] * cum[-1]), len(f) - 1)
    origins = v[f[face, 0]]
    vectors = v[f[face, 1:]] - origins[:, None, :]
    lengths = u[:, 1:3, None].copy()
    test = lengths.sum(axis=1).reshape(-1) > 1.0
    lengths[test] -= 1.0
    lengths = np.abs(lengths)
    return (vectors * lengths).sum(axis=1) + origins, face.astype(np.int64)


def metrics(rec_points, gt_points, threshold=0.05):
    """(accuracy, completion, completion ratio) in the reference's units (m, m, fraction) and the two distance arrays."""
    d_acc, _ = cKDTree(gt_points).query(rec_points)
    d_comp, _ = cKDTree(rec_points).query(gt_points)
    return float(np.mean(d_acc)), float(np.mean(d_comp)), float(np.mean((d_comp < threshold).astype(np.float64))), d_acc, d_comp


def transform_points(points, T):
    return np.asarray(points, dtype=np.float64) @ T[:3, :3].T + T[:3, 3]


def correspondences(tree, target, source, T, threshold):
    """-> (fitness, inlier rmse, transformed source points of the pairs, their targets)."""
    p = transform_points(source, T)
    d, j = tree.query(p, distance_upper_bound=threshold)
    ok = np.isfinite(d)
    n = int(ok.sum())
    rmse = float(np.sqrt(np.sum(d[ok] ** 2) / n)) if n else 0.0
    return n / len(source), rmse, p[ok], target[j[ok]]


def umeyama(p, q):
    """Rigid T f64 [4,4] with T p ~ q (least squares), identity without pairs."""
    T = np.eye(4)
    if len(p) == 0:
        return T
    mp, mq = p.mean(0), q.mean(0)
    sigma = (q - mq).T @ (p - mp) / len(p)
    U, _, Vh = np.linalg.svd(sigma)
    S = np.ones(3)
    if np.linalg.det(U) * np.linalg.det(Vh) < 0:
        S[2] = -1.0
    R = U @ np.diag(S) @ Vh
    T[:3, :3], T[:3, 3] = R, mq - R @ mp
    return T


def icp_align(source, target, threshold=0.1, init=None, max_iteration=30, relative_fitness=1e-6, relative_rmse=1e-6):
    """-> (T f64 [4,4], fitness, inlier rmse, iterations)."""
    source = np.asarray(source, dtype=np.float64)
    target = np.asarray(target, dtype=np.float64)
    tree = cKDTree(target)
    T = np.eye(4) if init is None else np.array(init, dtype=np.float64)
    fit, rmse, p, q = correspondences(tree, target, source, T, threshold)
    it = 0
    while it < max_iteration:
        T = umeyama(p, q) @ T
        it += 1
        fit0, rmse0 = fit, rmse
        fit, rmse, p, q = correspondences(tree, target, source, T, threshold)
        if abs(fit0 - fit) < relative_fitness and abs(rmse0 - rmse) < relative_rmse:
            break
    return T, fit, rmse, it


def rigid(angle_deg, axis, t):
    """4x4 rotation by angle_deg about the unit of axis, then translation t."""
    a = np.asarray(axis, dtype=np.float64)
    a = a / np.linalg.norm(a)
    th = np.deg2rad(angle_deg)
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    T = np.eye(4)
    T[:3, :3] = np.eye(3) + np.sin(th) * K + (1 - np.cos(th)) * K @ K
    T[:3, 3] = t
    return T
