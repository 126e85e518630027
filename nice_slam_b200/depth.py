"""The views and the depth renders of the 2D reconstruction metric (calc_2d_metric, src/tools/eval_recon.py:120-209), which needs
trimesh and open3d's OpenGL visualiser on the host.  recon.eval_depth_l1 puts them together.

  oriented_bounds  trimesh.bounds.oriented_bounds restated: the minimum-volume box over the convex hull's face normals (scipy)
  view_matrix      viewmatrix(z, up, pos) of eval_recon.py: OpenCV camera axes x = up x z, y = z x x, z = dir
  check_proj_w2c   the w2c check_proj projects with: float32(inv(float64 c2w with columns 1 and 2 negated))
  views_see_any    check_proj over a batch of poses (nsb_views_see_any)
  sample_views     get_cam_position + the rejection loop of calc_2d_metric, from a seeded numpy stream
  render_depth     the z-depth of a mesh under c2w poses (nsb_depth_render): open3d's depth buffer restated as an exact ray-plane depth
"""
import numpy as np
import torch
from scipy.spatial import ConvexHull

from . import _lib
from .cull import _device_tensor
from .renderer import _VP, _stream

# calc_2d_metric's camera
H, W, FOCAL = 500, 500, 300.0
UP = np.array([0.0, 0.0, -1.0])
Z_FAR = 20.0
WORKSPACE_BYTES = 256 << 20          # bound on the rasterizer's queue per launch


# ---------------------------------------------------------------------------------------------- the sampling box
def _min_rectangle(q):
    """Minimum-area rectangle of 2D points q [n,2] over the directions of their hull's edges -> (area, unit direction u, (lo_u, hi_u),
    (lo_w, hi_w)) with w = u rotated by +90 degrees."""
    try:
        h = q[ConvexHull(q).vertices]
    except Exception:                                               # collinear: a zero-area box along the points' spread
        h = q
    e = np.roll(h, -1, axis=0) - h
    n = np.linalg.norm(e, axis=1)
    ok = n > 0
    if not ok.any():
        return 0.0, np.array([1.0, 0.0]), (h[0, 0], h[0, 0]), (h[0, 1], h[0, 1])
    u = e[ok] / n[ok, None]
    w = np.stack([-u[:, 1], u[:, 0]], 1)
    pu, pw = h @ u.T, h @ w.T                                       # [hull points, directions]
    area = (pu.max(0) - pu.min(0)) * (pw.max(0) - pw.min(0))
    k = int(np.argmin(area))
    return float(area[k]), u[k], (pu[:, k].min(), pu[:, k].max()), (pw[:, k].min(), pw[:, k].max())


def oriented_bounds(vertices):
    """trimesh.bounds.oriented_bounds(mesh, ordered=True) restated -> (to_origin f64 [4,4], extents f64 [3] ascending).

    For every face normal n of the vertices' convex hull (scipy's ConvexHull), the hull is projected onto the plane normal to n and the
    minimum-area rectangle over the projected hull's edge directions is taken; the box of least volume wins.  to_origin is the rigid
    transform that moves the box's centre to the origin with its edges along x, y, z in the order of the ascending extents (a rotation,
    det +1).  trimesh's choice among equal boxes, and the signs of its axes, are not reproduced: calc_2d_metric uses the box only through
    its centre, its axes up to sign and its extents, and samples it symmetrically about the centre."""
    v = np.asarray(vertices, dtype=np.float64).reshape(-1, 3)
    if len(v) == 0 or not np.isfinite(v).all():
        raise ValueError("oriented_bounds: need finite vertices [n,3] with n >= 1")
    try:
        hull = ConvexHull(v)
        pts, normals = v[hull.vertices], hull.equations[:, :3]
    except Exception:                                               # flat or degenerate: the principal axes give the normals to try
        pts = v
        c = v - v.mean(0)
        normals = np.linalg.svd(c, full_matrices=False)[2] if len(v) > 1 else np.eye(3)
    normals = np.unique(np.round(normals / np.linalg.norm(normals, axis=1, keepdims=True), 12), axis=0)
    best = None
    for n in normals:
        a = np.eye(3)[int(np.argmin(np.abs(n)))]
        b1 = np.cross(n, a)
        b1 /= np.linalg.norm(b1)
        b2 = np.cross(n, b1)
        area, u, (ul, uh), (wl, wh) = _min_rectangle(np.stack([pts @ b1, pts @ b2], 1))
        pn = pts @ n
        vol = area * (pn.max() - pn.min())
        if best is None or vol < best[0]:
            ax_u = u[0] * b1 + u[1] * b2
            ax_w = -u[1] * b1 + u[0] * b2
            centre = 0.5 * (ul + uh) * ax_u + 0.5 * (wl + wh) * ax_w + 0.5 * (pn.min() + pn.max()) * n
            best = (vol, np.stack([ax_u, ax_w, n]), np.array([uh - ul, wh - wl, pn.max() - pn.min()]), centre)
    _, axes, ext, centre = best
    order = np.argsort(ext, kind="stable")
    R = axes[order]
    if np.linalg.det(R) < 0:
        R[2] = -R[2]
    to_origin = np.eye(4)
    to_origin[:3, :3], to_origin[:3, 3] = R, -R @ centre
    return to_origin, ext[order]


def sampling_box(gt_vertices):
    """get_cam_position (eval_recon.py:62-70) -> (extents [3], transform [4,4]): the box's extents scaled by (0.3, 0.7, 0.7), transform =
    inv(to_origin) moved 0.4 along world z."""
    to_origin, extents = oriented_bounds(gt_vertices)
    extents = extents * np.array([0.3, 0.7, 0.7])
    transform = np.linalg.inv(to_origin)
    transform[2, 3] += 0.4
    return extents, transform


# ---------------------------------------------------------------------------------------------- views
def _normalize(x):
    return x / np.linalg.norm(x, axis=-1, keepdims=True)


def view_matrix(z, up, pos):
    """viewmatrix (eval_recon.py:15-21) of rows of z [n,3] and pos [n,3] -> c2w f64 [n,4,4]: columns x = normalize(up x z'), y =
    normalize(z' x x), z' = normalize(z), t = pos."""
    z = _normalize(np.asarray(z, dtype=np.float64).reshape(-1, 3))
    up = np.broadcast_to(np.asarray(up, dtype=np.float64), z.shape)
    x = _normalize(np.cross(up, z))
    y = _normalize(np.cross(z, x))
    c2w = np.zeros((len(z), 4, 4))
    c2w[:, :3, 0], c2w[:, :3, 1], c2w[:, :3, 2], c2w[:, :3, 3], c2w[:, 3, 3] = x, y, z, np.asarray(pos, dtype=np.float64).reshape(-1, 3), 1.0
    return c2w


def candidates(uniforms, extents, transform):
    """Candidate views from uniforms [n,6] (three for the origin, three for the target) -> c2w f64 [n,4,4].  origin = transform applied to
    (u - 0.5) * extents (trimesh.sample.volume_rectangular); target = round(-10^4 + 2 10^4 u, 2) (random.uniform, then round); c2w =
    view_matrix(target - origin, (0, 0, -1), origin)."""
    u = np.asarray(uniforms, dtype=np.float64).reshape(-1, 6)
    p = (u[:, :3] - 0.5) * extents
    origin = (transform @ np.concatenate([p, np.ones((len(p), 1))], 1).T).T[:, :3]
    target = np.round(-10000.0 + 20000.0 * u[:, 3:], 2)
    return view_matrix(target - origin, UP, origin)


def check_proj_w2c(c2w):
    """c2w f64 [n,4,4] -> the float32 w2c check_proj projects with: inv of the float64 pose with columns 1 and 2 of rows 0-2 negated
    (eval_recon.py:65-70; cull.w2c_of inverts the float32 pose instead)."""
    c = np.array(c2w, dtype=np.float64).reshape(-1, 4, 4)
    c[:, :3, 1] *= -1.0
    c[:, :3, 2] *= -1.0
    return np.linalg.inv(c).astype(np.float32)


def views_see_any(points, w2c, H=H, W=W, fx=FOCAL, fy=FOCAL, cx=None, cy=None):
    """nsb_views_see_any: points CUDA f64 [N,3], w2c CUDA f32 [P,4,4] -> u8 [P], 1 iff some point is inside pose p's frustum."""
    cx = W / 2.0 - 0.5 if cx is None else cx
    cy = H / 2.0 - 0.5 if cy is None else cy
    pts = _device_tensor(points, torch.float64, (None, 3), "points", "nsb_views_see_any")
    w = _device_tensor(w2c, torch.float32, (None, 4, 4), "w2c", "nsb_views_see_any")
    if pts.shape[0] >= 2 ** 31 or w.shape[0] >= 2 ** 31:
        raise ValueError("nsb_views_see_any: more than 2^31 - 1 points or poses")
    out = torch.empty(w.shape[0], dtype=torch.uint8, device=w.device)
    _lib.check(_lib.lib().nsb_views_see_any(_VP(pts.data_ptr()), pts.shape[0], _VP(w.data_ptr()), w.shape[0], float(fx), float(fy), float(cx),
                                            float(cy), int(H), int(W), _VP(out.data_ptr()), _stream()), "nsb_views_see_any")
    return out


def sample_views(gt_vertices, unseen_points, n, seed=0, H=H, W=W, fx=FOCAL, fy=FOCAL, cx=None, cy=None, batch=256, device="cuda",
                 max_candidates=None):
    """calc_2d_metric's views (eval_recon.py:152-172) -> (c2w f64 [n,4,4], candidates drawn, rejected).

    Candidates come from np.random.default_rng(seed): candidate k is candidates() of the stream's doubles [6k, 6k + 6), drawn `batch`
    candidates at a time (the stream is sequential, so blocks concatenate).  Each block is tested with one nsb_views_see_any launch; a
    candidate that sees an unseen point (check_proj) is rejected, and the first n accepted in candidate order are returned, so the result
    does not depend on `batch`.  `candidates drawn` counts up to the n-th accepted one.  An empty unseen cloud rejects nothing.  More than
    max_candidates (default 1000 n) candidates raise ValueError."""
    cx = W / 2.0 - 0.5 if cx is None else cx
    cy = H / 2.0 - 0.5 if cy is None else cy
    n, batch = int(n), int(batch)
    if n < 0 or batch < 1:
        raise ValueError("sample_views: need n >= 0 and batch >= 1")
    cap = 1000 * n if max_candidates is None else int(max_candidates)
    extents, transform = sampling_box(gt_vertices)
    dev = torch.device(device)
    unseen = np.asarray(unseen_points, dtype=np.float64).reshape(-1, 3)
    pts = torch.from_numpy(unseen).to(dev) if len(unseen) else None
    rng = np.random.default_rng(seed)
    out, drawn = [], 0
    while len(out) < n:
        if drawn >= cap:
            raise ValueError("sample_views: %d views accepted after the cap of %d candidates (max_candidates); the unseen points are "
                             "in view from almost everywhere in the sampling box" % (len(out), cap))
        m = min(batch, cap - drawn)
        c2w = candidates(rng.random((m, 6)), extents, transform)
        if pts is None:
            seen = np.zeros(m, dtype=bool)
        else:
            seen = views_see_any(pts, torch.from_numpy(check_proj_w2c(c2w)).to(dev), H, W, fx, fy, cx, cy).cpu().numpy().astype(bool)
        for k in np.nonzero(~seen)[0]:
            out.append(c2w[k])
            if len(out) == n:
                drawn += int(k) + 1
                break
        else:
            drawn += m
    c2w = np.array(out, dtype=np.float64).reshape(-1, 4, 4)
    return c2w, drawn, drawn - n


# ---------------------------------------------------------------------------------------------- depth
def default_z_near(vertices):
    """0.01 x the largest extent of the vertices' axis-aligned box: a restatement of the near plane open3d's ViewControl derives from the
    bounding box of the geometry in the window (max(0.01 E, distance - 3 E) as we read it, whose second term is negative for a camera
    inside the room; not verified against open3d)."""
    v = np.asarray(vertices.cpu() if isinstance(vertices, torch.Tensor) else vertices, dtype=np.float64).reshape(-1, 3)
    return 0.01 * float((v.max(0) - v.min(0)).max())


def _mesh_tensors(vertices, faces, dev, what):
    v = torch.as_tensor(vertices).to(device=dev, dtype=torch.float64).contiguous()
    f = torch.as_tensor(faces).to(device=dev)
    if v.dim() != 2 or v.shape[1] != 3 or f.dim() != 2 or f.shape[1] != 3:
        raise ValueError("%s: expected vertices [V,3] and faces [F,3], got %s and %s" % (what, tuple(v.shape), tuple(f.shape)))
    if v.shape[0] >= 2 ** 31 or f.shape[0] >= 2 ** 31:
        raise ValueError("%s: more than 2^31 - 1 vertices or faces" % what)
    if v.shape[0] == 0 or f.shape[0] == 0:
        raise ValueError("%s: the mesh is empty (%d vertices, %d faces)" % (what, v.shape[0], f.shape[0]))
    if f.dtype.is_floating_point or f.dtype == torch.bool:
        raise ValueError("%s: faces must be integers, got %s" % (what, f.dtype))
    if not bool(torch.isfinite(v).all()):
        raise ValueError("%s: vertex coordinates are not all finite" % what)
    if int(f.min()) < 0 or int(f.max()) >= v.shape[0]:
        raise ValueError("%s: face indices outside [0, %d)" % (what, v.shape[0]))
    return v, f.to(torch.int32).contiguous()


def render_depth(vertices, faces, c2w, H=H, W=W, fx=FOCAL, fy=FOCAL, cx=None, cy=None, z_near=None, z_far=Z_FAR, device="cuda"):
    """z-depth of the mesh (vertices [V,3], faces [F,3]) under the poses c2w [P,4,4] (OpenCV convention, as view_matrix) -> CUDA f32
    [P,H,W], 0 where no face is hit (nsb_depth_render; the rule is in include/nice_slam_b200.h).  What open3d's visualiser renders for
    calc_2d_metric, with the exact ray-plane depth in place of a 24-bit depth buffer (a difference of order 1e-5 m at room distances) and
    no face culling (mesh_show_back_face).  z_near defaults to default_z_near(vertices); z_far = 20 (set_constant_z_far(20))."""
    cx = W / 2.0 - 0.5 if cx is None else cx
    cy = H / 2.0 - 0.5 if cy is None else cy
    dev = torch.device(device)
    v, f = _mesh_tensors(vertices, faces, dev, "render_depth")
    c = torch.as_tensor(c2w).to(device=dev, dtype=torch.float64)
    if c.dim() == 2:
        c = c.unsqueeze(0)
    if c.dim() != 3 or tuple(c.shape[1:]) != (4, 4):
        raise ValueError("render_depth: c2w must be [P,4,4] (or [4,4]), got %s" % (tuple(c.shape),))
    if c.shape[0] >= 2 ** 31:
        raise ValueError("render_depth: more than 2^31 - 1 poses")
    if not bool(torch.isfinite(c).all()):
        raise ValueError("render_depth: c2w entries are not all finite")
    c = c.contiguous()
    zn = default_z_near(vertices) if z_near is None else float(z_near)
    if not (0.0 < zn <= float(z_far) < np.inf):
        raise ValueError("render_depth: need 0 < z_near <= z_far < inf, got %r, %r" % (zn, z_far))
    if int(H) < 1 or int(W) < 1:
        raise ValueError("render_depth: H and W must be >= 1")
    L, F, P = _lib.lib(), f.shape[0], c.shape[0]
    out = torch.empty(P, int(H), int(W), dtype=torch.float32, device=dev)
    step = max(1, min(P, (WORKSPACE_BYTES - 16) // (8 * F)))        # cameras per launch: the queue holds F x step entries
    ws = torch.empty(L.nsb_depth_render_workspace(F, step), dtype=torch.uint8, device=dev)
    for p0 in range(0, P, step):
        p1 = min(P, p0 + step)
        _lib.check(L.nsb_depth_render(_VP(v.data_ptr()), v.shape[0], _VP(f.data_ptr()), F, _VP(c[p0].data_ptr()), p1 - p0, float(fx), float(fy),
                                      float(cx), float(cy), int(H), int(W), zn, float(z_far), _VP(ws.data_ptr()), ws.numel(),
                                      _VP(out[p0].data_ptr()), _stream()), "nsb_depth_render")
    return out


def depth_l1(a, b):
    """nsb_depth_l1: CUDA f32 [P,H,W] pair -> f64 [P], mean |a - b| per view (float64, a fixed summation order)."""
    if a.shape != b.shape or a.dim() != 3 or a.dtype != torch.float32 or b.dtype != torch.float32 or not a.is_cuda or not b.is_cuda:
        raise ValueError("depth_l1: need two CUDA float32 [P,H,W] tensors of one shape")
    a, b = a.contiguous(), b.contiguous()
    out = torch.empty(a.shape[0], dtype=torch.float64, device=a.device)
    _lib.check(_lib.lib().nsb_depth_l1(_VP(a.data_ptr()), _VP(b.data_ptr()), a.shape[0], a.shape[1] * a.shape[2], _VP(out.data_ptr()), _stream()),
               "nsb_depth_l1")
    return out
