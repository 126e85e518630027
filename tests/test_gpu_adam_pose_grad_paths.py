"""GPU: every C entry point of the fused Adam (nsb_adam_masked_voxels, nsb_adam_decoder, nsb_adam_mapper_step,
nsb_adam_mapper_step_decoders) and of the d c2w sums (nsb_pose_grad, nsb_pose_grad_frames) runs the same kernel, so their results must
agree bit for bit."""
import ctypes as C

import pytest
import torch

import scene_util as su
from gpu_util import make_renderer

pytestmark = pytest.mark.gpu
DEV = "cuda"
VP = C.c_void_p
NSB_ERR_ARG = -1
BETAS, EPS = (0.9, 0.999), 1e-8


def test_adam_entry_points_agree_bit_for_bit():
    """One voxel group (grid_middle, 40 % selected) and the colour decoder, three steps with changing gradients and learning rates, through
    (a) nsb_adam_masked_voxels + nsb_adam_decoder, (b) nsb_adam_mapper_step, (c) nsb_adam_mapper_step_decoders: parameters, exp_avg and
    exp_avg_sq equal.  step < 1 and a decoder given twice are refused."""
    from nice_slam_b200 import _lib
    from nice_slam_b200._lib import LEVELS
    from nice_slam_b200.decoders import decoder_params_struct
    from nice_slam_b200.masked import MaskedVoxels
    from nice_slam_b200.renderer import grid_struct
    L = _lib.lib()
    sc = su.load_scenes()["room0"]
    grids, dec_state = su.make_grids(sc, "soft"), su.load_decoders("soft")
    key, level = "grid_middle", LEVELS.index("color")
    g = torch.Generator(device=DEV).manual_seed(7)
    runs = []
    for _ in range(3):
        _, c, dec = make_renderer(sc, grids, dec_state, DEV)
        runs.append(dict(c=c, dec=dec))
    vm = torch.rand(runs[0]["c"][key].shape[2:], device=DEV, generator=g) < 0.4
    n_flat = L.nsb_flat_decoder_floats(level)
    for r in runs:
        r["mv"] = MaskedVoxels(r["c"][key], vm)
        r["grid"] = grid_struct(r["c"][key].detach())
        r["dp"] = decoder_params_struct(r["dec"], "color")
        r["state"] = [torch.zeros(r["mv"].count * 32, device=DEV), torch.zeros(r["mv"].count * 32, device=DEV),
                      torch.zeros(n_flat, device=DEV), torch.zeros(n_flat, device=DEV)]
    count = runs[0]["mv"].count
    assert count > 0

    def group(r, gv, lr, step):
        grp = _lib.AdamVoxelGroup()
        grp.grid = r["grid"]
        grp.slot_map, grp.grad, grp.exp_avg, grp.exp_avg_sq = r["mv"].slot_map.data_ptr(), gv.data_ptr(), r["state"][0].data_ptr(), r["state"][1].data_ptr()
        grp.lr, grp.step = lr, step
        return grp

    def item(r, gflat, lr, step):
        it = _lib.AdamDecoderItem()
        it.level, it.params = level, C.pointer(r["dp"])
        it.grad_flat, it.exp_avg, it.exp_avg_sq, it.lr, it.step = gflat.data_ptr(), r["state"][2].data_ptr(), r["state"][3].data_ptr(), lr, step
        return it

    def separate(r, gv, gflat, lr_v, lr_d, step):
        m, v, dm, dv = r["state"]
        rc = L.nsb_adam_masked_voxels(C.byref(r["grid"]), VP(r["mv"].slot_map.data_ptr()), VP(gv.data_ptr()), VP(m.data_ptr()), VP(v.data_ptr()),
                                      lr_v, BETAS[0], BETAS[1], EPS, step, None)
        return rc or L.nsb_adam_decoder(level, C.byref(r["dp"]), VP(gflat.data_ptr()), VP(dm.data_ptr()), VP(dv.data_ptr()),
                                        lr_d, BETAS[0], BETAS[1], EPS, step, None)

    def mapper_step(r, gv, gflat, lr_v, lr_d, step):
        _, _, dm, dv = r["state"]
        return L.nsb_adam_mapper_step(C.byref(group(r, gv, lr_v, step)), 1, level, C.byref(r["dp"]), VP(gflat.data_ptr()), VP(dm.data_ptr()),
                                      VP(dv.data_ptr()), lr_d, step, BETAS[0], BETAS[1], EPS, None)

    def mapper_step_decoders(r, gv, gflat, lr_v, lr_d, step):
        return L.nsb_adam_mapper_step_decoders(C.byref(group(r, gv, lr_v, step)), 1, C.byref(item(r, gflat, lr_d, step)), 1,
                                               BETAS[0], BETAS[1], EPS, None)

    paths = (separate, mapper_step, mapper_step_decoders)
    for step, (lr_v, lr_d) in enumerate([(0.1, 0.005), (0.005, 0.005), (0.005, 0.0)], start=1):
        gv = torch.randn(count, 32, device=DEV, generator=g) * (10.0 ** (1 - step))
        gflat = torch.randn(n_flat, device=DEV, generator=g) * 0.1
        for r, path in zip(runs, paths):
            assert path(r, gv, gflat, lr_v, lr_d, step) == 0, (path.__name__, L.nsb_last_error())
    torch.cuda.synchronize()
    a = runs[0]
    for r, path in zip(runs[1:], paths[1:]):
        assert torch.equal(r["c"][key], a["c"][key]), path.__name__
        for name, p in r["dec"].color_decoder.named_parameters():
            assert torch.equal(p, dict(a["dec"].color_decoder.named_parameters())[name]), (path.__name__, name)
        for s_r, s_a in zip(r["state"], a["state"]):
            assert torch.equal(s_r, s_a), path.__name__
    assert not torch.equal(a["c"][key], grids[key].to(DEV))                    # the steps did move the selected voxels

    # refused arguments: nothing is launched
    before = [t.clone() for t in a["state"]]
    gv, gflat = torch.zeros(count, 32, device=DEV), torch.zeros(n_flat, device=DEV)
    for path in paths:
        assert path(a, gv, gflat, 0.1, 0.1, 0) == NSB_ERR_ARG, path.__name__
    assert L.nsb_adam_decoder(level, C.byref(a["dp"]), VP(gflat.data_ptr()), VP(a["state"][2].data_ptr()), VP(a["state"][3].data_ptr()),
                              0.1, BETAS[0], BETAS[1], EPS, 0, None) == NSB_ERR_ARG
    twice = (_lib.AdamDecoderItem * 2)(item(a, gflat, 0.1, 1), item(a, gflat, 0.1, 1))
    assert L.nsb_adam_mapper_step_decoders(None, 0, twice, 2, BETAS[0], BETAS[1], EPS, None) == NSB_ERR_ARG
    torch.cuda.synchronize()
    assert all(torch.equal(t, b) for t, b in zip(a["state"], before))


@pytest.mark.parametrize("n", [1, 37, 1000, 3000])
def test_pose_grad_over_one_frame_equals_frames_form(n):
    """nsb_pose_grad over n rays, cast to float32 == nsb_pose_grad_frames with the single frame [0, n)."""
    from nice_slam_b200 import _lib
    L = _lib.lib()
    g = torch.Generator(device=DEV).manual_seed(n)
    dirs, dro, drd = (torch.randn(n, 3, device=DEV, generator=g) for _ in range(3))
    pose = torch.zeros(12, dtype=torch.float64, device=DEV)
    frames = torch.zeros(1, 12, device=DEV)
    offs = torch.tensor([0, n], dtype=torch.int32, device=DEV)
    _lib.check(L.nsb_pose_grad(VP(dirs.data_ptr()), VP(dro.data_ptr()), VP(drd.data_ptr()), n, VP(pose.data_ptr()), None), "pose_grad")
    _lib.check(L.nsb_pose_grad_frames(VP(dirs.data_ptr()), VP(dro.data_ptr()), VP(drd.data_ptr()), VP(offs.data_ptr()), 1, VP(frames.data_ptr()), None),
               "pose_grad_frames")
    torch.cuda.synchronize()
    assert torch.equal(pose.float(), frames[0])
    want = torch.cat([drd.double().T @ dirs.double(), dro.double().sum(0)[:, None]], dim=1).reshape(12)
    assert torch.allclose(pose, want, rtol=1e-9, atol=1e-9)
