"""Mesh extraction of a fused run's own state (Mesher.get_mesh, src/utils/Mesher.py:349-574) on the GPU.

FusedMesher reads the grids, the decoders, the mapper's KeyframeStore and estimate_c2w_list, and runs every step on the device:

  1. scene hull (get_bound_from_frames, :214-279): the convex hull of the keyframes' camera centres and back-projected depth pixels, scaled
     by clean_mesh_bound_scale about the mean of its vertices.  The support points of 128 fixed directions bound an inner polytope; only the
     pixels outside it (a few thousand) go to scipy.spatial.ConvexHull on the host.  This is the one deliberate deviation: the reference
     hulls the vertices of open3d's TSDF surface (voxel 4 scale/512, truncation 0.04 scale), which lie within about a voxel of these points;
  2. occupancy lattice (get_grid_uniform + eval_points at stage 'fine', :321-347, 281-319, 421-433): nsb_mesh_lattice_eval, the points
     generated inside the forward kernel, 100 outside the float32 bound or the hull;
  3. marching cubes (skimage's, :437-467): nsb_mc_count / nsb_mc_emit with the table of tools/gen_mc_table.py -- the same vertex set, but
     triangles may differ from skimage's in cells with an ambiguous face;
  4. seen masks (point_masks, :53-212): keyframes with their depth limit, or (get_mask_use_all_frames) estimate_c2w_list[0..idx];
  5. culling, shared-edge components, the area filter and compaction (:469-511);
  6. vertex colours (direct_point_query, :513-524, 555-556), then the vertices are divided by scale (:570).

The meshing reads the grids only and draws no random numbers.  Without a surface get_mesh returns None and writes nothing, as the
reference prints and returns (:459-463)."""
import ctypes as C
import os

import numpy as np
import torch

from . import _lib
from .renderer import _VP, _inputs, _linspaces, _stream

HULL_DIRECTIONS = 128


def hull_directions(k=HULL_DIRECTIONS):
    """k unit vectors spread over the sphere (Fibonacci lattice), float64 [k,3]."""
    i = np.arange(k, dtype=np.float64) + 0.5
    z = 1.0 - 2.0 * i / k
    r = np.sqrt(1.0 - z * z)
    phi = np.pi * (3.0 - np.sqrt(5.0)) * i
    return np.stack([r * np.cos(phi), r * np.sin(phi), z], 1)


def lattice_axes(marching_cubes_bound, scale, resolution):
    """x, y, z of get_grid_uniform (Mesher.py:331-339): np.linspace(lo - 0.05, hi + 0.05, R) of marching_cubes_bound * scale (float64)."""
    b = np.array(marching_cubes_bound, dtype=np.float64) * scale
    return [np.linspace(b[a][0] - 0.05, b[a][1] + 0.05, int(resolution)) for a in range(3)]


def write_ply(path, vertices, faces, colors=None):
    """Binary little-endian PLY: x y z double; red green blue alpha uchar (alpha 255) when colours are given; faces as list uchar int."""
    V, F = len(vertices), len(faces)
    vt = [("x", "<f8"), ("y", "<f8"), ("z", "<f8")]
    if colors is not None:
        vt += [("red", "u1"), ("green", "u1"), ("blue", "u1"), ("alpha", "u1")]
    v = np.empty(V, dtype=vt)
    v["x"], v["y"], v["z"] = vertices[:, 0], vertices[:, 1], vertices[:, 2]
    if colors is not None:
        v["red"], v["green"], v["blue"], v["alpha"] = colors[:, 0], colors[:, 1], colors[:, 2], 255
    f = np.empty(F, dtype=[("n", "u1"), ("i", "<i4", (3,))])
    f["n"], f["i"] = 3, faces
    head = ["ply", "format binary_little_endian 1.0", "element vertex %d" % V] + ["property double %s" % a for a in "xyz"]
    if colors is not None:
        head += ["property uchar %s" % a for a in ("red", "green", "blue", "alpha")]
    head += ["element face %d" % F, "property list uchar int vertex_indices", "end_header"]
    d = os.path.dirname(path)
    if d:
        os.makedirs(d, exist_ok=True)
    with open(path, "wb") as fh:
        fh.write(("\n".join(head) + "\n").encode("ascii"))
        fh.write(v.tobytes())
        fh.write(f.tobytes())


def _i32x3(v):
    return (C.c_int32 * 3)(*[int(x) for x in v])


def _f64x3(v):
    return (C.c_double * 3)(*[float(x) for x in v])


class FusedMesher:
    def __init__(self, renderer, cfg):
        """renderer: the run's FusedRenderer (its bound and decoder cache); cfg: the reference's config (meshing.*, mapping.marching_cubes_bound,
        scale).  Settings the fused path does not implement raise here, naming the setting."""
        m = cfg["meshing"]
        for key in ("mesh_coarse_level", "show_forecast", "depth_test"):
            if m.get(key):
                raise RuntimeError("FusedMesher: meshing.%s is not supported" % key)
        method = m.get("color_mesh_extraction_method", "direct_point_query")
        if method != "direct_point_query":
            raise RuntimeError("FusedMesher: meshing.color_mesh_extraction_method %r (iMAP*) is not supported; only 'direct_point_query'" % method)
        self.r = renderer
        self.resolution = int(m["resolution"])
        self.level_set = float(m["level_set"])
        self.clean_mesh_bound_scale = float(m["clean_mesh_bound_scale"])
        self.remove_small_geometry_threshold = float(m["remove_small_geometry_threshold"])
        self.get_largest_components = bool(m["get_largest_components"])
        self.scale = float(cfg["scale"])
        self.marching_cubes_bound = cfg["mapping"]["marching_cubes_bound"]
        self.axes = lattice_axes(self.marching_cubes_bound, self.scale, self.resolution)

    # ------------------------------------------------------------------------------------------ steps
    def _render_inputs(self, c, decoders, stage, dev):
        call, grids, _ = self.r._call(c, decoders, stage, None, dev)
        dummy = torch.zeros(1, 3, dtype=torch.float32, device=dev)
        t_u, t_s = _linspaces(self.r.N_samples, self.r.N_surface, dev)
        keep = [g.detach() for g in grids]
        return _inputs(call, dummy, dummy, None, t_u, t_s, keep), (call, keep, dummy)

    def hull(self, store):
        """Half-spaces f64 [P,4] (n . p + d <= 0 inside) of the scaled scene hull of the keyframes in `store`."""
        from scipy.spatial import ConvexHull                      # host step of the hull only
        M = len(store)
        if M == 0:
            raise RuntimeError("FusedMesher: the scene hull needs at least one keyframe")
        L, dev, H, W = _lib.lib(), store.dev, store.H, store.W
        depth = store.depth[:M].contiguous()
        c2w_h = torch.stack([m[:3, :4] for m in store.est_c2w[:M]]).double()
        c2w = c2w_h.to(dev).contiguous()
        cams = c2w_h[:, :, 3].numpy()
        cam_args = (store.fx, store.fy, store.cx, store.cy)
        dirs = torch.from_numpy(hull_directions()).to(dev).contiguous()
        best = torch.zeros(HULL_DIRECTIONS, dtype=torch.int64, device=dev)
        _lib.check(L.nsb_mesh_hull_support(_VP(depth.data_ptr()), M, H, W, _VP(c2w.data_ptr()), *cam_args, _VP(dirs.data_ptr()), HULL_DIRECTIONS,
                                           _VP(best.data_ptr()), _stream()), "nsb_mesh_hull_support")
        b = best.cpu().numpy().view(np.uint64)
        sup_ids = np.unique((b[b != 0] & np.uint64(0xffffffff)).astype(np.int64))
        sup = self._pixel_points(depth, H, W, c2w, cam_args, sup_ids)
        inner_pts = np.concatenate([cams, sup])
        flag = torch.empty(M * H * W, dtype=torch.uint8, device=dev)
        try:
            planes = torch.from_numpy(np.ascontiguousarray(ConvexHull(inner_pts).equations)).to(dev)
            n_planes = planes.shape[0]
        except Exception:                                          # (flat or too few points: every pixel is a candidate)
            planes, n_planes = None, 0
        _lib.check(L.nsb_mesh_hull_outside(_VP(depth.data_ptr()), M, H, W, _VP(c2w.data_ptr()), *cam_args,
                                           _VP(planes.data_ptr() if planes is not None else None), n_planes, 1e-9,
                                           _VP(flag.data_ptr()), _stream()), "nsb_mesh_hull_outside")
        out_ids = torch.nonzero(flag).reshape(-1).cpu().numpy()
        pts = np.concatenate([inner_pts, self._pixel_points(depth, H, W, c2w, cam_args, out_ids)])
        h = ConvexHull(pts)
        v = pts[h.vertices]
        ctr = v.mean(0)                                            # open3d's get_center of a triangle mesh: the vertex mean
        return ConvexHull(ctr + self.clean_mesh_bound_scale * (v - ctr)).equations

    def _pixel_points(self, depth, H, W, c2w, cam_args, ids):
        if len(ids) == 0:
            return np.zeros((0, 3))
        idt = torch.from_numpy(np.ascontiguousarray(ids, dtype=np.int64)).to(depth.device)
        out = torch.empty(len(ids), 3, dtype=torch.float64, device=depth.device)
        _lib.check(_lib.lib().nsb_mesh_hull_points(_VP(depth.data_ptr()), H, W, _VP(c2w.data_ptr()), *cam_args, _VP(idt.data_ptr()), len(ids),
                                                   _VP(out.data_ptr()), _stream()), "nsb_mesh_hull_points")
        return out.cpu().numpy()

    def lattice(self, c, decoders, planes=None):
        """z f32 [Rx,Ry,Rz] (device): stage-'fine' occupancy of the lattice, 100 outside the float32 bound or the hull `planes`."""
        dev = next(iter(c.values())).device
        inp, keep = self._render_inputs(c, decoders, "fine", dev)
        lat = _lib.MeshLattice()
        pl = None
        for a, x in enumerate(self.axes):
            lat.n[a] = len(x)
            lat.start[a], lat.stop[a] = float(x[0]), float(x[-1])
            lat.step[a] = float((x[-1] - x[0]) / (len(x) - 1)) if len(x) > 1 else 0.0
        if planes is not None:
            pl = torch.as_tensor(np.ascontiguousarray(planes, dtype=np.float64)).to(dev).contiguous()
            lat.planes, lat.n_planes = pl.data_ptr(), pl.shape[0]
        z = torch.empty(*[len(x) for x in self.axes], dtype=torch.float32, device=dev)
        _lib.check(_lib.lib().nsb_mesh_lattice_eval(C.byref(inp), C.byref(lat), _VP(z.data_ptr()), _stream()), "nsb_mesh_lattice_eval")
        return z

    def marching_cubes(self, z, with_edge_ids=False):
        """-> (vertices f64 [V,3], faces int32 [F,3], edge ids int64 [V] or None) on the device, in lattice coordinates of self.axes."""
        L, dev = _lib.lib(), z.device
        n = _i32x3(z.shape)
        ws = torch.empty(L.nsb_mc_workspace(z.numel()), dtype=torch.uint8, device=dev)
        totals = torch.zeros(2, dtype=torch.int64, device=dev)
        _lib.check(L.nsb_mc_count(_VP(z.data_ptr()), n, self.level_set, _VP(ws.data_ptr()), ws.numel(), _VP(totals.data_ptr()), _stream()), "nsb_mc_count")
        V, F = (int(v) for v in totals.cpu())
        x, y, w = self.axes
        origin = _f64x3((x[0], y[0], w[0]))
        spacing = _f64x3((x[2] - x[1], y[2] - y[1], w[2] - w[1]))                 # as the reference passes it (Mesher.py:446-448)
        verts = torch.empty(V, 3, dtype=torch.float64, device=dev)
        faces = torch.empty(F, 3, dtype=torch.int32, device=dev)
        eid = torch.empty(V, dtype=torch.int64, device=dev) if with_edge_ids else None
        if V:
            _lib.check(L.nsb_mc_emit(_VP(z.data_ptr()), n, self.level_set, origin, spacing, _VP(ws.data_ptr()), _VP(verts.data_ptr()),
                                     _VP(faces.data_ptr()), _VP(eid.data_ptr() if eid is not None else None), _stream()), "nsb_mc_emit")
        return verts, faces, eid

    def seen(self, verts, store, estimate_c2w_list, idx, get_mask_use_all_frames=False):
        """point_masks' seen output, uint8 [V] (device)."""
        L, dev = _lib.lib(), verts.device
        lim = None
        if get_mask_use_all_frames:
            c2w = torch.as_tensor(estimate_c2w_list)[: idx + 1].detach().cpu().numpy()
            w2c = torch.from_numpy(np.linalg.inv(c2w.astype(np.float64)).astype(np.float32).reshape(-1, 16)).to(dev)
        else:
            M = len(store)
            w2c = store.w2c[:M]
            lim = torch.empty(max(M, 1), dtype=torch.float32, device=dev)
            _lib.check(L.nsb_mesh_depth_limits(_VP(store.depth.data_ptr()), M, store.H * store.W, _VP(lim.data_ptr()), _stream()),
                       "nsb_mesh_depth_limits")
        w2c = w2c.contiguous()
        out = torch.empty(verts.shape[0], dtype=torch.uint8, device=dev)
        r = self.r
        _lib.check(L.nsb_mesh_seen(_VP(verts.data_ptr()), verts.shape[0], _VP(w2c.data_ptr()), w2c.shape[0],
                                   _VP(lim.data_ptr() if lim is not None else None), r.fx, r.fy, r.cx, r.cy, int(r.H), int(r.W),
                                   _VP(out.data_ptr()), _stream()), "nsb_mesh_seen")
        return out

    def clean(self, verts, faces, seen):
        """Culling, components, area filter (remove_small_geometry_threshold * scale^2, or the largest), compaction -> (verts, faces)."""
        L, dev = _lib.lib(), verts.device
        V, F = verts.shape[0], faces.shape[0]
        ws = torch.empty(L.nsb_mesh_clean_workspace(V, F), dtype=torch.uint8, device=dev)
        totals = torch.zeros(2, dtype=torch.int64, device=dev)
        thr = self.remove_small_geometry_threshold * self.scale * self.scale
        _lib.check(L.nsb_mesh_clean(_VP(verts.data_ptr()), V, _VP(faces.data_ptr()), F, _VP(seen.data_ptr()), thr, int(self.get_largest_components),
                                    _VP(ws.data_ptr()), ws.numel(), _VP(totals.data_ptr()), _stream()), "nsb_mesh_clean")
        nv, nf = (int(v) for v in totals.cpu())
        ov = torch.empty(nv, 3, dtype=torch.float64, device=dev)
        of = torch.empty(nf, 3, dtype=torch.int32, device=dev)
        _lib.check(L.nsb_mesh_compact(_VP(verts.data_ptr()), V, _VP(faces.data_ptr()), F, _VP(ws.data_ptr()), _VP(ov.data_ptr()),
                                      _VP(of.data_ptr()), _stream()), "nsb_mesh_compact")
        return ov, of

    def colors(self, verts, c, decoders):
        """uint8 [V,3] (device): direct_point_query of the float32-rounded vertices at stage 'color'."""
        dev = verts.device
        inp, keep = self._render_inputs(c, decoders, "color", dev)
        n = verts.shape[0]
        raw = torch.empty(max(n, 1), 4, dtype=torch.float32, device=dev)
        out = torch.empty(n, 3, dtype=torch.uint8, device=dev)
        _lib.check(_lib.lib().nsb_mesh_colors(C.byref(inp), _VP(verts.data_ptr()), n, _VP(raw.data_ptr()), _VP(out.data_ptr()), _stream()),
                   "nsb_mesh_colors")
        return out

    # ------------------------------------------------------------------------------------------ the whole extraction
    def get_mesh(self, path, c, decoders, store, estimate_c2w_list, idx, clean_mesh=True, get_mask_use_all_frames=False, color=True,
                 show_forecast=False):
        """Mesher.get_mesh (Mesher.py:349-574) for the NICE path -> (vertices f64 [V,3] / scale, faces int64 [F,3], colours uint8 [V,3] or
        None), host numpy; written to `path` (binary PLY) when given.  None, and no file, when the lattice has no surface."""
        if show_forecast:
            raise RuntimeError("FusedMesher: meshing.mesh_coarse_level / show_forecast is not supported")
        with torch.no_grad():
            planes = self.hull(store)
            z = self.lattice(c, decoders, planes)
            verts, faces, _ = self.marching_cubes(z)
            if faces.shape[0] == 0:
                return None
            if clean_mesh:
                seen = self.seen(verts, store, estimate_c2w_list, idx, get_mask_use_all_frames)
                verts, faces = self.clean(verts, faces, seen)
            cols = self.colors(verts, c, decoders).cpu().numpy() if color else None
            v = verts.cpu().numpy() / self.scale
            f = faces.cpu().numpy().astype(np.int64)
        if path is not None:
            write_ply(path, v, f, cols)
        return v, f, cols
