"""Dumps what the decoder packing and the fused mapper's optimiser produce from fixed inputs, so that two builds can be compared byte
for byte:
  * the images nsb_pack_decoders writes for all four decoders (room0, soft decoders): raw, 3xTF32 tiles and units, FP16 units;
  * three FusedMapperAdam.step_all steps over three voxel groups (40 % of grid_middle / grid_fine / grid_color selected) and the fine and
    colour decoders, from seeded gradients: the grids, decoders and Adam state after each step;
  * d c2w of seeded ray gradients: nsb_pose_grad over the batch, nsb_pose_grad_frames over a ragged six-frame window, and nsb_adam_poses
    chaining the window's d c2w into five camera tensors.
The mapping loop itself is not a byte-level yardstick: its voxel gradients are summed with float atomics, so its state differs from run to
run of the same build.

    python tools/bit_identity_dump.py OUT.pt                 (needs a GPU)
    python tools/bit_identity_dump.py --compare A.pt B.pt    (exit status 1 unless every tensor is byte-identical)
"""
import ctypes as C
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch

VP = C.c_void_p


def dump(path):
    import scene_util as su
    from gpu_util import make_renderer
    from nice_slam_b200 import _lib
    from nice_slam_b200._lib import LEVELS
    from nice_slam_b200.masked import MaskedVoxels
    from nice_slam_b200.optim import FusedMapperAdam
    from nice_slam_b200.renderer import _PackCache
    L = _lib.lib()
    dev = torch.device("cuda")
    g = torch.Generator(device=dev).manual_seed(11)
    out = {}
    sc = su.load_scenes()["room0"]
    renderer, c, dec = make_renderer(sc, su.make_grids(sc, "soft"), su.load_decoders("soft"), dev)
    images, _ = _PackCache().get(dec, LEVELS, dev)
    for lvl, img in images.items():
        out["packed." + lvl] = img.clone()

    keys, levels = ("grid_middle", "grid_fine", "grid_color"), ("fine", "color")
    masked = {k: MaskedVoxels(c[k], torch.rand(c[k].shape[2:], device=dev, generator=g) < 0.4) for k in keys}
    fused = FusedMapperAdam()
    for step in range(3):
        voxel_items = [(k, c[k], masked[k], torch.randn(masked[k].count, 32, device=dev, generator=g) * 10.0 ** (-step), 0.005 if step else 0.1)
                       for k in keys]
        decoder_items = [(lvl, dec, torch.randn(L.nsb_flat_decoder_floats(LEVELS.index(lvl)), device=dev, generator=g) * 0.1, 0.005)
                         for lvl in levels]
        fused.step_all(voxel_items, decoder_items, renderer=renderer)
        for k in keys:
            out["%d.grid.%s" % (step, k)] = c[k].detach().clone()
        for k, v in dec.state_dict().items():
            out["%d.dec.%s" % (step, k)] = v.detach().clone()
        for name, st in fused.state.items():
            if isinstance(st, dict):
                out["%d.adam.%s.m" % (step, name)], out["%d.adam.%s.v" % (step, name)] = st["m"].clone(), st["v"].clone()

    n, offs = 996, torch.tensor([0, 100, 101, 350, 600, 996, 996], dtype=torch.int32, device=dev)
    F = offs.numel() - 1
    dirs, dro, drd = (torch.randn(n, 3, device=dev, generator=g) for _ in range(3))
    out["pose_grad"] = torch.zeros(12, dtype=torch.float64, device=dev)
    out["pose_grad_frames"] = torch.zeros(F, 12, device=dev)
    _lib.check(L.nsb_pose_grad(VP(dirs.data_ptr()), VP(dro.data_ptr()), VP(drd.data_ptr()), n, VP(out["pose_grad"].data_ptr()), None), "pose_grad")
    _lib.check(L.nsb_pose_grad_frames(VP(dirs.data_ptr()), VP(dro.data_ptr()), VP(drd.data_ptr()), VP(offs.data_ptr()), F,
                                      VP(out["pose_grad_frames"].data_ptr()), None), "pose_grad_frames")
    cams = torch.nn.functional.normalize(torch.randn(F - 1, 7, device=dev, generator=g), dim=1).contiguous()
    cam_row = torch.tensor([-1] + list(range(F - 1)), dtype=torch.int32, device=dev)
    m, v, d_cams = torch.zeros_like(cams), torch.zeros_like(cams), torch.zeros_like(cams)
    _lib.check(L.nsb_adam_poses(VP(cams.data_ptr()), VP(cam_row.data_ptr()), F, VP(out["pose_grad_frames"].data_ptr()), VP(m.data_ptr()),
                                VP(v.data_ptr()), VP(d_cams.data_ptr()), 0.001, 0.9, 0.999, 1e-8, 1, None), "adam_poses")
    out["camera_tensors"], out["d_camera_tensors"] = cams, d_cams
    torch.cuda.synchronize()
    torch.save({k: t.cpu() for k, t in out.items()}, path)
    print("wrote %d tensors to %s" % (len(out), path))


def as_bytes(t):
    return t.detach().contiguous().reshape(-1).view(torch.uint8)


def compare(a_path, b_path):
    a, b = torch.load(a_path, weights_only=True), torch.load(b_path, weights_only=True)
    bad = sorted(set(a) ^ set(b))
    for k in sorted(set(a) & set(b)):
        if a[k].dtype != b[k].dtype or a[k].shape != b[k].shape or not torch.equal(as_bytes(a[k]), as_bytes(b[k])):
            bad.append(k)
    print("%d tensors compared, %d differ%s" % (len(set(a) | set(b)), len(bad), (": " + ", ".join(bad)) if bad else ""))
    return 1 if bad else 0


def main():
    if len(sys.argv) == 4 and sys.argv[1] == "--compare":
        sys.exit(compare(sys.argv[2], sys.argv[3]))
    if len(sys.argv) != 2:
        sys.exit(__doc__)
    dump(sys.argv[1])


if __name__ == "__main__":
    main()
