"""Cull a mesh to the camera frustums of a trajectory on the GPU: the reference's src/tools/cull_mesh.py, which makes the culled
ground-truth meshes the 3D reconstruction metric (nice_slam_b200.recon) is scored against.

  load_poses      traj.txt -> c2w float32 [N,4,4] in the NICE convention (cull_mesh.py's parser)
  c2w_from_traj   the parser's column flips and float32 cast of raw trajectory matrices
  cull_mesh       (vertices, faces, c2w) -> (seen mask u8 [V], kept face indices int32 [F']): nsb_cull_seen + nsb_cull_faces

python -m nice_slam_b200.cull --input_mesh A.ply --traj traj.txt --output_mesh B.ply [--H 680 --W 1200 --fx 600 --fy 600 --cx 599.5
--cy 339.5]   writes A without the faces whose three vertices no pose sees.  Every vertex stays, as in the reference (trimesh's
update_faces keeps them, and get_align_transformation aligns to all of them).  The output keeps the input's header and vertex records
byte for byte, and the kept face records with all their properties; trimesh re-encodes the vertex element on export, which is not
reproduced.  The formats are read_ply's: binary little-endian triangle meshes.
"""
import argparse

import numpy as np
import torch

from . import _lib
from .renderer import _VP, _stream

# cull_mesh.py:31-37: Replica's camera
H, W, FX, FY, CX, CY = 680, 1200, 600.0, 600.0, 599.5, 339.5


def c2w_from_traj(poses):
    """Raw trajectory matrices [N,4,4] (float64) -> c2w float32 [N,4,4] in the NICE convention: columns 1 and 2 of rows 0-2 negated in
    float64, then cast (cull_mesh.py:13-16)."""
    c2w = np.array(poses, dtype=np.float64).reshape(-1, 4, 4)
    c2w[:, :3, 1] *= -1
    c2w[:, :3, 2] *= -1
    return c2w.astype(np.float32)


def load_poses(path):
    """traj.txt (one pose per line: 16 numbers, a row-major c2w) -> c2w float32 [N,4,4] after c2w_from_traj.  A line without 16 numbers
    raises ValueError naming the line."""
    rows = []
    with open(path, "r") as fh:
        for k, line in enumerate(fh, 1):
            try:
                vals = [float(x) for x in line.split()]
            except ValueError:
                vals = None
            if vals is None or len(vals) != 16:
                raise ValueError("load_poses: %s line %d does not hold 16 numbers: %r" % (path, k, line.strip()[:80]))
            rows.append(vals)
    return c2w_from_traj(np.array(rows, dtype=np.float64).reshape(-1, 4, 4))


def w2c_of(c2w):
    """c2w [N,4,4] (array or tensor, NICE convention) -> w2c float32 [N,4,4] = np.linalg.inv(float32 c2w): numpy inverts in float64 and
    rounds to float32, as cull_mesh.py:51 does.  A pose with a non-finite entry gets an all-NaN w2c, which sees nothing."""
    c2w = c2w.detach().cpu().numpy() if isinstance(c2w, torch.Tensor) else np.asarray(c2w)
    c2w = c2w.astype(np.float32).reshape(-1, 4, 4)
    bad = ~np.isfinite(c2w).all(axis=(1, 2))
    ok = np.where(bad[:, None, None], np.eye(4, dtype=np.float32), c2w)
    try:
        w2c = np.linalg.inv(ok)
    except np.linalg.LinAlgError:
        k = next(i for i in range(len(ok)) if np.linalg.matrix_rank(ok[i].astype(np.float64)) < 4)
        raise ValueError("cull_mesh: pose %d is singular" % k) from None
    w2c[bad] = np.nan
    return w2c.astype(np.float32)


def _device_tensor(t, dtype, shape, what, entry):
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise ValueError("%s: %s must be a CUDA tensor" % (entry, what))
    if t.dtype != dtype or t.dim() != len(shape) or any(s is not None and t.shape[i] != s for i, s in enumerate(shape)):
        raise ValueError("%s: %s must be %s %s, got %s %s" % (entry, what, dtype, shape, t.dtype, tuple(t.shape)))
    return t.contiguous()


def cull_seen(vertices, w2c, H=H, W=W, fx=FX, fy=FY, cx=CX, cy=CY):
    """nsb_cull_seen: vertices CUDA f64 [V,3], w2c CUDA f32 [P,4,4] -> seen u8 [V] (1 = some pose sees the vertex)."""
    v = _device_tensor(vertices, torch.float64, (None, 3), "vertices", "nsb_cull_seen")
    w = _device_tensor(w2c, torch.float32, (None, 4, 4), "w2c", "nsb_cull_seen")
    if v.shape[0] >= 2 ** 31 or w.shape[0] >= 2 ** 31:
        raise ValueError("nsb_cull_seen: more than 2^31 - 1 vertices or poses")
    seen = torch.empty(v.shape[0], dtype=torch.uint8, device=v.device)
    _lib.check(_lib.lib().nsb_cull_seen(_VP(v.data_ptr()), v.shape[0], _VP(w.data_ptr()), w.shape[0], float(fx), float(fy), float(cx), float(cy),
                                        int(H), int(W), _VP(seen.data_ptr()), _stream()), "nsb_cull_seen")
    return seen


def cull_faces(faces, seen):
    """nsb_cull_faces + nsb_cull_faces_emit: faces CUDA int32 [F,3] (indices in [0, V), checked by the caller), seen CUDA u8 [V] ->
    int32 indices of the faces with a seen vertex, ascending."""
    f = _device_tensor(faces, torch.int32, (None, 3), "faces", "nsb_cull_faces")
    s = _device_tensor(seen, torch.uint8, (None,), "seen", "nsb_cull_faces")
    L, F, dev = _lib.lib(), f.shape[0], f.device
    ws = torch.empty(L.nsb_cull_faces_workspace(F), dtype=torch.uint8, device=dev)
    total = torch.empty(1, dtype=torch.int64, device=dev)
    _lib.check(L.nsb_cull_faces(_VP(f.data_ptr()), F, _VP(s.data_ptr()), _VP(ws.data_ptr()), ws.numel(), _VP(total.data_ptr()), _stream()),
               "nsb_cull_faces")
    kept = torch.empty(int(total), dtype=torch.int32, device=dev)
    if kept.numel():
        _lib.check(L.nsb_cull_faces_emit(F, _VP(ws.data_ptr()), _VP(kept.data_ptr()), _stream()), "nsb_cull_faces_emit")
    return kept


def cull_mesh(vertices, faces, c2w, H=H, W=W, fx=FX, fy=FY, cx=CX, cy=CY, device="cuda"):
    """cull_mesh.py's culling of (vertices [V,3], faces [F,3]) by the poses c2w [N,4,4] (arrays or tensors, in the NICE convention
    after the column flips: load_poses' output, or a FusedSLAM checkpoint's estimate_c2w_list / gt_c2w_list) -> (seen u8 [V], kept
    face indices int32 [F'] ascending), on the device.  A vertex is seen if some pose projects it strictly inside the H x W image in
    front of the camera (include/nice_slam_b200.h, nsb_cull_seen); a face is kept iff one of its vertices is seen."""
    dev = torch.device(device)
    v = torch.as_tensor(vertices).to(device=dev, dtype=torch.float64).contiguous()
    f = torch.as_tensor(faces).to(device=dev)
    if v.dim() != 2 or v.shape[1] != 3 or f.dim() != 2 or f.shape[1] != 3:
        raise ValueError("cull_mesh: expected vertices [V,3] and faces [F,3], got %s and %s" % (tuple(v.shape), tuple(f.shape)))
    if f.numel() and (int(f.min()) < 0 or int(f.max()) >= v.shape[0]):
        raise ValueError("cull_mesh: face indices outside [0, %d)" % v.shape[0])
    if f.shape[0] >= 2 ** 31:
        raise ValueError("cull_mesh: more than 2^31 - 1 faces")
    w2c = torch.from_numpy(w2c_of(c2w)).to(dev)
    seen = cull_seen(v, w2c, H, W, fx, fy, cx, cy)
    return seen, cull_faces(f.to(torch.int32).contiguous(), seen)


def main(argv=None):
    from .recon import _mesh_of, read_ply_records, write_ply_records
    ap = argparse.ArgumentParser(description="Arguments to cull the mesh.")
    ap.add_argument("--input_mesh", type=str, help="path to the mesh to be culled")
    ap.add_argument("--traj", type=str, help="path to the trajectory")
    ap.add_argument("--output_mesh", type=str, help="path to the output mesh")
    ap.add_argument("--H", type=int, default=H, help="image height (Replica: 680)")
    ap.add_argument("--W", type=int, default=W, help="image width (Replica: 1200)")
    ap.add_argument("--fx", type=float, default=FX)
    ap.add_argument("--fy", type=float, default=FY)
    ap.add_argument("--cx", type=float, default=CX)
    ap.add_argument("--cy", type=float, default=CY)
    a = ap.parse_args(argv)
    if not (a.input_mesh and a.traj and a.output_mesh):
        ap.error("--input_mesh, --traj and --output_mesh are required")
    header, elements = read_ply_records(a.input_mesh)
    verts, faces, _ = _mesh_of(a.input_mesh, elements)
    _, kept = cull_mesh(verts, faces, load_poses(a.traj), a.H, a.W, a.fx, a.fy, a.cx, a.cy)
    kept = kept.cpu().numpy()
    write_ply_records(a.output_mesh, header, [(n, p, rec[kept] if n == "face" else rec) for n, p, rec in elements])
    print("kept %d of %d faces (%d vertices)" % (len(kept), len(faces), len(verts)))


if __name__ == "__main__":
    main()
