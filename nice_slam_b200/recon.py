"""Reconstruction metrics of a mesh against a ground-truth mesh on the GPU: the 3D and 2D metrics of the reference's
src/tools/eval_recon.py (calc_3d_metric, :91-117, with get_align_transformation, :45-59; calc_2d_metric, :120-209), which need trimesh
and open3d on the host.

  read_ply           binary little-endian triangle meshes (mesh.write_ply's, trimesh's and open3d's), validated
  read_ply_records   the same files as their header lines and raw records per element; write_ply_records writes them back
  sample_surface     trimesh.sample.sample_surface on the device (nsb_sample_surface), uniforms from a torch.Generator
  NearestNeighbours  exact nearest neighbours on a uniform grid (nsb_nn_*), the role of scipy's cKDTree in eval_recon.py
  icp_align          open3d 0.13's registration_icp, point to point (nsb_icp_sums per iteration, the 3x3 SVD on the host)
  eval_recon         accuracy (cm), completion (cm), completion ratio (% under 5 cm)
  eval_depth_l1      depth L1 (cm) over 1000 seeded interior views that do not see the unseen region (nice_slam_b200.depth: the
                     sampling box, the views, the depth rasterizer nsb_depth_render)

python -m nice_slam_b200.recon --rec_mesh A.ply --gt_mesh B.ply -3d -2d   prints eval_recon.py's three lines, then its "Depth L1: " line.
-2d reads the unseen-region point cloud beside the ground truth (B_pc_unseen.npy, as eval_recon.py:146); without it -2d exits non-zero
before any GPU work.
"""
import argparse
import ctypes as C
import os
import sys

import numpy as np
import torch

from . import _lib
from .renderer import _VP, _stream

# ---------------------------------------------------------------------------------------------- PLY input
_PLY_TYPES = {"char": "i1", "int8": "i1", "uchar": "u1", "uint8": "u1", "short": "i2", "int16": "i2", "ushort": "u2", "uint16": "u2",
              "int": "i4", "int32": "i4", "uint": "u4", "uint32": "u4", "float": "f4", "float32": "f4", "double": "f8", "float64": "f8"}


def _ply_type(name, what):
    if name not in _PLY_TYPES:
        raise ValueError("read_ply: %s has unknown type %r" % (what, name))
    return "<" + _PLY_TYPES[name]


def _parse_header(fh, path):
    """-> (header lines as read, line ends included, up to and including end_header; [(name, count, [property words])])."""
    if fh.readline().strip() != b"ply":
        raise ValueError("read_ply: %s is not a PLY file" % path)
    fh.seek(0)
    lines = [fh.readline()]
    elements, fmt = [], None
    while True:
        line = fh.readline()
        if not line:
            raise ValueError("read_ply: %s ends before end_header" % path)
        lines.append(line)
        w = line.decode("ascii", "replace").split()
        if not w or w[0] in ("comment", "obj_info"):
            continue
        if w[0] == "end_header":
            break
        if w[0] == "format":
            fmt = w[1] if len(w) > 1 else ""
        elif w[0] == "element" and len(w) == 3:
            elements.append((w[1], int(w[2]), []))
        elif w[0] == "property" and elements:
            elements[-1][2].append(tuple(w[1:]))
        else:
            raise ValueError("read_ply: %s: malformed header line %r" % (path, line.strip()))
    if fmt != "binary_little_endian":
        raise ValueError("read_ply: %s has format %r; only binary_little_endian is supported (not ascii or binary_big_endian)" % (path, fmt))
    return lines, elements


def _scalar_dtype(name, count, props, path):
    fields = []
    for p in props:
        if p[0] == "list":
            raise ValueError("read_ply: %s: element %r has a list property %r; only the face element may" % (path, name, p[-1]))
        fields.append((p[1], _ply_type(p[0], "property %s.%s" % (name, p[1]))))
    return np.dtype(fields)


def _open_records(path):
    """Parse the header -> (header lines, an iterator over (name, property words, records) in file order).  Each element is checked as
    the iterator reaches it, so a reader that consumes it element by element raises in file order."""
    with open(path, "rb") as fh:
        header, elements = _parse_header(fh, path)
        data = fh.read()

    def records():
        off = 0
        for name, n, props in elements:
            if n < 0:
                raise ValueError("read_ply: %s: element %r has a negative count" % (path, name))
            if name == "face":
                lists = [p for p in props if p[0] == "list"]
                if len(lists) != 1 or lists[0][-1] not in ("vertex_indices", "vertex_index"):
                    raise ValueError("read_ply: %s: element 'face' needs one list property vertex_indices" % path)
                fields = []
                for p in props:
                    if p[0] == "list":
                        ct, it = p[1], p[2]
                        if ct not in ("uchar", "uint8", "int", "int32", "uint", "uint32"):
                            raise ValueError("read_ply: %s: face list count type %r (uchar or int expected)" % (path, ct))
                        if it not in ("int", "int32", "uint", "uint32"):
                            raise ValueError("read_ply: %s: face list index type %r (int or uint expected)" % (path, it))
                        fields += [("__n", _ply_type(ct, "face count")), ("__i", _ply_type(it, "face index"), (3,))]
                    else:
                        fields.append((p[1], _ply_type(p[0], "property face.%s" % p[1])))
                dt = np.dtype(fields)
            else:
                dt = _scalar_dtype(name, n, props, path)
            need = dt.itemsize * n
            if off + need > len(data):
                raise ValueError("read_ply: %s: element %r is truncated (%d bytes, %d left)" % (path, name, need, len(data) - off))
            rec = np.frombuffer(data, dtype=dt, count=n, offset=off)
            off += need
            if name == "face":
                bad = np.nonzero(rec["__n"] != 3)[0]
                if len(bad):
                    raise ValueError("read_ply: %s: face %d has %d vertices; only triangles are supported" % (path, bad[0], rec["__n"][bad[0]]))
            yield name, props, rec

    return header, records()


def read_ply_records(path):
    """-> (header, elements): header = the header's lines as read (bytes, line ends included, "ply" to "end_header"); elements = [(name,
    property words, records)] in file order, records a read-only numpy structured array over the file's bytes (the face element's list
    property is the fields __n (count) and __i (three indices)).  The formats and checks of read_ply's file layer: binary little-endian,
    scalar properties, one triangle list property on 'face'; anything else raises ValueError as read_ply does.  write_ply_records writes
    such a pair back."""
    header, it = _open_records(path)
    return header, list(it)


def _mesh_of(path, elements):
    """read_ply's arrays of the (name, props, records) of a file, checked in file order."""
    verts, faces, colors = None, None, None
    for name, props, rec in elements:
        if name == "face":
            faces = rec["__i"].astype(np.int64)
        elif name == "vertex":
            dt = rec.dtype
            for a in "xyz":
                if a not in dt.names:
                    raise ValueError("read_ply: %s: element 'vertex' has no property %r" % (path, a))
                if dt[a] not in (np.dtype("<f4"), np.dtype("<f8")):
                    raise ValueError("read_ply: %s: vertex property %r must be float or double" % (path, a))
            verts = np.stack([rec[a].astype(np.float64) for a in "xyz"], 1)
            if all(c in dt.names for c in ("red", "green", "blue")):
                colors = np.stack([rec[c] for c in ("red", "green", "blue")], 1).astype(np.uint8)
    if verts is None:
        raise ValueError("read_ply: %s has no element 'vertex'" % path)
    if faces is None:
        faces = np.zeros((0, 3), dtype=np.int64)
    if not np.isfinite(verts).all():
        raise ValueError("read_ply: %s: vertex coordinates are not all finite" % path)
    if len(faces) and (faces.min() < 0 or faces.max() >= len(verts)):
        raise ValueError("read_ply: %s: face indices outside [0, %d)" % (path, len(verts)))
    return verts, faces, colors


def read_ply(path):
    """-> (vertices f64 [V,3], faces int64 [F,3], colours uint8 [V,3] or None).  Binary little-endian only; vertex x / y / z as float
    or double (other vertex properties are skipped by their sizes); faces as one list property with a uchar or int count and int or uint
    indices, every face a triangle.  Anything else raises ValueError naming the element or property."""
    return _mesh_of(path, _open_records(path)[1])


def write_ply_records(path, header, elements):
    """Write read_ply_records' (header, elements), with any element's records replaced (e.g. a subset of the faces): the header's lines
    unchanged except each 'element <name> <count>' line, whose count becomes the number of records given; then each element's records
    as their bytes, in order.  Records taken from the file (or indexed subsets of them) come out byte for byte."""
    counts = iter([len(rec) for _, _, rec in elements])
    out = []
    for line in header:
        w = line.split()
        if len(w) == 3 and w[0] == b"element":
            end = line[len(line.rstrip(b"\r\n")):]
            line = b"element %s %d" % (w[1], next(counts)) + end
        out.append(line)
    d = os.path.dirname(path)
    if d:
        os.makedirs(d, exist_ok=True)
    with open(path, "wb") as fh:
        fh.write(b"".join(out))
        for _, _, rec in elements:
            fh.write(np.ascontiguousarray(rec).tobytes())


# ---------------------------------------------------------------------------------------------- device steps
def _points(x, dev, what):
    t = torch.as_tensor(x).to(device=dev, dtype=torch.float64).contiguous()
    if t.dim() != 2 or t.shape[1] != 3:
        raise ValueError("%s: expected [n,3] points, got %s" % (what, tuple(t.shape)))
    if t.shape[0] >= 2 ** 31:
        raise ValueError("%s: more than 2^31 - 1 points" % what)
    return t


def sample_surface(vertices, faces, count, generator):
    """trimesh.sample.sample_surface of (vertices [V,3], faces [F,3]) on the generator's device -> (points f64 [count,3], face index
    int64 [count]).  The uniforms are one torch.rand(count, 3, float64) draw: column 0 picks the face, columns 1-2 the point."""
    dev = generator.device
    v = _points(vertices, dev, "sample_surface")
    f = torch.as_tensor(faces).to(device=dev, dtype=torch.int32).contiguous()
    if f.dim() != 2 or f.shape[1] != 3 or f.shape[0] < 1:
        raise ValueError("sample_surface: faces must be [F,3] with F >= 1, got %s" % (tuple(f.shape),))
    if int(f.min()) < 0 or int(f.max()) >= v.shape[0]:
        raise ValueError("sample_surface: face indices outside [0, %d)" % v.shape[0])
    u = torch.rand(int(count), 3, dtype=torch.float64, device=dev, generator=generator)
    return sample_surface_uniforms(v, f, u)


def sample_surface_uniforms(vertices, faces, uniforms):
    """sample_surface with the uniforms f64 [count,3] given (device tensors; faces int32)."""
    L, dev, F = _lib.lib(), vertices.device, faces.shape[0]
    u = uniforms.to(device=dev, dtype=torch.float64).contiguous()
    n = u.shape[0]
    ws = torch.empty(L.nsb_sample_surface_workspace(F), dtype=torch.uint8, device=dev)
    pts = torch.empty(n, 3, dtype=torch.float64, device=dev)
    idx = torch.empty(n, dtype=torch.int64, device=dev)
    _lib.check(L.nsb_sample_surface(_VP(vertices.data_ptr()), _VP(faces.data_ptr()), F, _VP(u.data_ptr()), n, _VP(ws.data_ptr()), ws.numel(),
                                    _VP(pts.data_ptr()), _VP(idx.data_ptr()), _stream()), "nsb_sample_surface")
    return pts, idx


class NearestNeighbours:
    """Exact nearest neighbours among targets [N,3] (N >= 1): a uniform grid built once on the device (include/nice_slam_b200.h gives
    the cell rule).  Equal distances go to the smaller target index."""

    def __init__(self, targets, device="cuda"):
        dev = targets.device if isinstance(targets, torch.Tensor) and targets.is_cuda else torch.device(device)
        t = _points(targets, dev, "NearestNeighbours")
        if t.shape[0] < 1:
            raise ValueError("NearestNeighbours: no targets")
        if not bool(torch.isfinite(t).all()):
            raise ValueError("NearestNeighbours: targets are not all finite")
        L, N = _lib.lib(), t.shape[0]
        ws = torch.empty(L.nsb_nn_bounds_workspace(N), dtype=torch.uint8, device=dev)
        box = torch.empty(6, dtype=torch.float64, device=dev)
        _lib.check(L.nsb_nn_bounds(_VP(t.data_ptr()), N, _VP(ws.data_ptr()), ws.numel(), _VP(box.data_ptr()), _stream()), "nsb_nn_bounds")
        g = _lib.NNGrid()
        _lib.check(L.nsb_nn_plan((C.c_double * 6)(*box.cpu().tolist()), N, C.byref(g)), "nsb_nn_plan")
        self.cell_start = torch.empty(g.n_cells + 1, dtype=torch.int64, device=dev)
        self.points = torch.empty(N, 3, dtype=torch.float64, device=dev)
        self.index = torch.empty(N, dtype=torch.int32, device=dev)
        g.cell_start, g.points, g.index = self.cell_start.data_ptr(), self.points.data_ptr(), self.index.data_ptr()
        ws = torch.empty(L.nsb_nn_build_workspace(g.n_cells), dtype=torch.uint8, device=dev)
        _lib.check(L.nsb_nn_build(_VP(t.data_ptr()), C.byref(g), _VP(ws.data_ptr()), ws.numel(), _stream()), "nsb_nn_build")
        self.grid, self.device, self.n = g, dev, N

    def query(self, points, radius=None, squared=False):
        """-> (distance f64 [M] -- squared with squared=True --, index int32 [M]) of each point's nearest target, on the device.  With a
        radius only targets at distance < radius count; a point with none gets index -1 and distance inf."""
        q = _points(points, self.device, "NearestNeighbours.query")
        if not bool(torch.isfinite(q).all()):
            raise ValueError("NearestNeighbours.query: points are not all finite")
        M = q.shape[0]
        d2 = torch.empty(M, dtype=torch.float64, device=self.device)
        idx = torch.empty(M, dtype=torch.int32, device=self.device)
        r = -1.0 if radius is None else float(radius)
        if radius is not None and not r >= 0.0:
            raise ValueError("NearestNeighbours.query: radius must be >= 0")
        _lib.check(_lib.lib().nsb_nn_query(C.byref(self.grid), _VP(q.data_ptr()), M, r, _VP(d2.data_ptr()), _VP(idx.data_ptr()), _stream()),
                   "nsb_nn_query")
        return (d2 if squared else torch.sqrt(d2)), idx


def icp_sums(nn, source, T, threshold):
    """One correspondence pass (nsb_icp_sums) -> float64 numpy [17]: pairs, sum d^2, sum p, sum q, sum p_i q_j (row i)."""
    L = _lib.lib()
    M = source.shape[0]
    ws = torch.empty(L.nsb_icp_workspace(M), dtype=torch.uint8, device=nn.device)
    sums = torch.empty(17, dtype=torch.float64, device=nn.device)
    Tc = (C.c_double * 16)(*np.asarray(T, dtype=np.float64).reshape(16).tolist())
    _lib.check(L.nsb_icp_sums(C.byref(nn.grid), _VP(source.data_ptr()), M, Tc, float(threshold), _VP(ws.data_ptr()), ws.numel(),
                              _VP(sums.data_ptr()), _stream()), "nsb_icp_sums")
    return sums.cpu().numpy()


def _umeyama_from_sums(s):
    """Eigen::umeyama(src, dst, false) from the pass's sums: sigma = sum (q - mq)(p - mp)^T / n = S^T / n - mq mp^T; U S V^T = svd(sigma);
    R = U diag(1, 1, det(U) det(V) < 0 ? -1 : 1) V^T; t = mq - R mp.  Identity without pairs."""
    T = np.eye(4)
    n = s[0]
    if n == 0:
        return T
    mp, mq = s[2:5] / n, s[5:8] / n
    sigma = s[8:17].reshape(3, 3).T / n - np.outer(mq, mp)
    U, _, Vh = np.linalg.svd(sigma)
    D = np.ones(3)
    if np.linalg.det(U) * np.linalg.det(Vh) < 0:
        D[2] = -1.0
    R = U @ np.diag(D) @ Vh
    T[:3, :3], T[:3, 3] = R, mq - R @ mp
    return T


def _fit(s, M):
    n = s[0]
    return n / M, (float(np.sqrt(s[1] / n)) if n else 0.0)


def icp_align(source, target, threshold=0.1, init=None, max_iteration=30, relative_fitness=1e-6, relative_rmse=1e-6, device="cuda"):
    """open3d 0.13's registration_icp(source, target, threshold, init, TransformationEstimationPointToPoint(), ICPConvergenceCriteria(
    relative_fitness, relative_rmse, max_iteration)), as get_align_transformation calls it -> (T f64 [4,4], fitness, inlier_rmse,
    iterations).

    Restated from open3d 0.13's RegistrationICP (open3d itself is not used):
      - correspondences: each source point, moved by T, is paired with its nearest target if that is at distance < threshold (strict,
        as FLANN's radius search and scipy's distance_upper_bound); fitness = pairs / M, inlier_rmse = sqrt(sum d^2 / pairs), 0 without
        pairs;
      - evaluate at init (identity if None); then up to max_iteration times: update = Umeyama without scaling on the pairs (identity
        without pairs), T = update @ T, re-evaluate, stop when |d fitness| < relative_fitness and |d rmse| < relative_rmse;
      - iterations = the number of updates applied.
    The source is transformed from the original points by T in every pass (open3d moves its copy by each update in turn): the two
    differ by rounding only.  Every source point counts, referenced by a face or not, as open3d's point cloud of mesh vertices."""
    dev = target.device if isinstance(target, torch.Tensor) and target.is_cuda else torch.device(device)
    src = _points(source, dev, "icp_align")
    nn = target if isinstance(target, NearestNeighbours) else NearestNeighbours(target, dev)
    M = src.shape[0]
    if M < 1:
        raise ValueError("icp_align: no source points")
    T = np.eye(4) if init is None else np.array(init, dtype=np.float64).reshape(4, 4)
    s = icp_sums(nn, src, T, threshold)
    fit, rmse = _fit(s, M)
    it = 0
    while it < max_iteration:
        T = _umeyama_from_sums(s) @ T
        it += 1
        fit0, rmse0 = fit, rmse
        s = icp_sums(nn, src, T, threshold)
        fit, rmse = _fit(s, M)
        if abs(fit0 - fit) < relative_fitness and abs(rmse0 - rmse) < relative_rmse:
            break
    return T, fit, rmse, it


# ---------------------------------------------------------------------------------------------- the metric
def _mesh(m, what):
    if isinstance(m, (str, bytes)) or hasattr(m, "__fspath__"):
        v, f, _ = read_ply(m)
    else:
        v, f = m
        v = np.asarray(v.cpu() if isinstance(v, torch.Tensor) else v, dtype=np.float64)
        f = np.asarray(f.cpu() if isinstance(f, torch.Tensor) else f, dtype=np.int64)
    if len(f) == 0:
        raise ValueError("eval_recon: the %s mesh has no faces" % what)
    return v, f


def eval_recon(rec, gt, align=True, n_samples=200000, seed=0, device="cuda"):
    """calc_3d_metric (eval_recon.py:91-117) of rec against gt (paths or (vertices, faces) pairs) -> dict(accuracy [cm], completion [cm],
    completion_ratio [%], transform, fitness, inlier_rmse, icp_iterations).

    With align, icp_align from every rec vertex to every gt vertex (threshold 0.1) and the rec vertices moved by it (v R^T + t, host
    float64, as trimesh's apply_transform).  Then n_samples surface samples of rec, then of gt, from one device generator seeded with
    seed; accuracy = mean distance from the rec samples to their nearest gt sample, completion = the other way, completion_ratio = the
    share of gt samples whose distance is < 0.05."""
    dev = torch.device(device)
    rv, rf = _mesh(rec, "rec")
    gv, gf = _mesh(gt, "gt")
    T, fit, rmse, it = np.eye(4), None, None, 0
    if align:
        T, fit, rmse, it = icp_align(rv, gv, 0.1, device=dev)
        rv = rv @ T[:3, :3].T + T[:3, 3]
    g = torch.Generator(device=dev)
    g.manual_seed(int(seed))
    rec_pts, _ = sample_surface(rv, rf, n_samples, g)
    gt_pts, _ = sample_surface(gv, gf, n_samples, g)
    d_acc, _ = NearestNeighbours(gt_pts).query(rec_pts)
    d_comp, _ = NearestNeighbours(rec_pts).query(gt_pts)
    return dict(accuracy=float(d_acc.mean()) * 100, completion=float(d_comp.mean()) * 100,
                completion_ratio=float((d_comp < 0.05).double().mean()) * 100, transform=T, fitness=fit, inlier_rmse=rmse, icp_iterations=it)


def unseen_path(gt_meshfile):
    """The unseen-region point cloud shipped beside a culled ground truth: gt_meshfile.replace('.ply', '_pc_unseen.npy') (eval_recon.py:146)."""
    return gt_meshfile.replace(".ply", "_pc_unseen.npy")


def eval_depth_l1(rec, gt, unseen_points, align=True, n_views=1000, seed=0, H=500, W=500, focal=300.0, device="cuda", view_batch=32):
    """calc_2d_metric (eval_recon.py:120-209) of rec against gt (paths or (vertices, faces) pairs); unseen_points: [N,3] (or a .npy path),
    the region no view may see -> dict(depth_l1 [cm], view_errors f64 [n_views] in m, c2w f64 [n_views,4,4], transform, candidates,
    rejected).

    With align, the rec vertices are moved by icp_align to the gt vertices (threshold 0.1), as eval_recon.  The views are
    depth.sample_views(gt vertices, unseen_points, n_views, seed); each view renders the gt and the aligned rec with depth.render_depth
    (z_far 20, each mesh's own z_near = depth.default_z_near, the rec's taken after alignment), and its error is the float64 mean of
    |gt depth - rec depth| over every pixel, a pixel one mesh misses counting the other's full depth.  depth_l1 = 100 x the mean of the
    view errors.  Views are rendered view_batch at a time; a repeat gives the same bits."""
    from . import depth as dp
    dev = torch.device(device)
    rv, rf = _mesh(rec, "rec")
    gv, gf = _mesh(gt, "gt")
    if isinstance(unseen_points, (str, bytes)) or hasattr(unseen_points, "__fspath__"):
        unseen_points = np.load(unseen_points)
    unseen = np.asarray(unseen_points, dtype=np.float64)
    if unseen.size and (unseen.ndim != 2 or unseen.shape[1] != 3 or not np.isfinite(unseen).all()):
        raise ValueError("eval_depth_l1: unseen_points must be finite [N,3], got shape %s" % (unseen.shape,))
    T = np.eye(4)
    if align:
        T = icp_align(rv, gv, 0.1, device=dev)[0]
        rv = rv @ T[:3, :3].T + T[:3, 3]
    cx, cy = W / 2.0 - 0.5, H / 2.0 - 0.5
    c2w, drawn, rejected = dp.sample_views(gv, unseen.reshape(-1, 3), n_views, seed, H, W, focal, focal, cx, cy, device=dev)
    zn_g, zn_r = dp.default_z_near(gv), dp.default_z_near(rv)
    errs = []
    for p0 in range(0, len(c2w), int(view_batch)):
        views = c2w[p0:p0 + int(view_batch)]
        dg = dp.render_depth(gv, gf, views, H, W, focal, focal, cx, cy, zn_g, dp.Z_FAR, dev)
        dr = dp.render_depth(rv, rf, views, H, W, focal, focal, cx, cy, zn_r, dp.Z_FAR, dev)
        errs.append(dp.depth_l1(dg, dr).cpu().numpy())
    errors = np.concatenate(errs) if errs else np.zeros(0)
    return dict(depth_l1=float(errors.mean()) * 100 if len(errors) else float("nan"), view_errors=errors, c2w=c2w, transform=T,
                candidates=drawn, rejected=rejected)


def main(argv=None):
    ap = argparse.ArgumentParser(description="Arguments to evaluate the reconstruction.")
    ap.add_argument("--rec_mesh", type=str, help="reconstructed mesh file path")
    ap.add_argument("--gt_mesh", type=str, help="ground truth mesh file path")
    ap.add_argument("-2d", "--metric_2d", action="store_true",
                    help="enable 2D metric (depth L1 over 1000 views; needs the gt's unseen-region cloud, <gt_mesh>_pc_unseen.npy)")
    ap.add_argument("-3d", "--metric_3d", action="store_true", help="enable 3D metric")
    a = ap.parse_args(argv)
    if (a.metric_3d or a.metric_2d) and (not a.rec_mesh or not a.gt_mesh):
        ap.error("-3d and -2d need --rec_mesh and --gt_mesh")
    unseen = None
    if a.metric_2d:                                    # checked before any GPU work, so a missing file costs no 3D run
        path = unseen_path(a.gt_mesh)
        if path == a.gt_mesh or not os.path.isfile(path):
            sys.exit("nice_slam_b200.recon: %s not found; the 2D metric (depth L1) without the ground truth's unseen-region point cloud "
                     "is not supported" % path)
        unseen = np.load(path)
    if a.metric_3d:
        r = eval_recon(a.rec_mesh, a.gt_mesh)
        print("accuracy: ", r["accuracy"])
        print("completion: ", r["completion"])
        print("completion ratio: ", r["completion_ratio"])
    if a.metric_2d:
        print("Depth L1: ", eval_depth_l1(a.rec_mesh, a.gt_mesh, unseen)["depth_l1"])


if __name__ == "__main__":
    main()
