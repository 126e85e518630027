"""Generate tests/golden/mapper_settings/*.pt: the UNMODIFIED reference Mapper.optimize_map (imported from the reference checkout through
tests/ref_harness.py) with the `mapping:` settings the shipped default leaves off -- fix_fine = False, and the colour-refinement pass of the
last frame (fix_color = True, frustum_feature_selection = False, middle / fine ratios 0, Mapper.py:578-586) -- on room0 'soft'.

    python tests/make_golden_mapper_settings.py        # needs the reference checkout

    joint_fix_fine_false.pt   five real joint iterations (3 x middle, fine, color) with the real torch.optim.Adam and fix_fine = False: the
                              fine decoder's parameters join the colour decoder's in parameter group 0 (Mapper.py:336-341).  Per-iteration
                              ray batches at the renderer boundary, the selected voxels after the loop, both decoders' final parameters.
    color_refine_ba.pt        real colour-refinement iterations with bundle adjustment on the window of make_golden._ba_setup: every voxel of
                              every grid is a parameter, no decoder is optimised.  The pixel draws of every window row and iteration, the
                              grids after the loop (samples over the whole grid) and the window poses.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import make_golden as mg        # noqa: E402
import ref_harness as rh        # noqa: E402
import scene_util as su         # noqa: E402
from oracle import torch_port as tp   # noqa: E402

OUT = os.path.join(su.GOLDEN, "mapper_settings")
KEYS = ("grid_middle", "grid_fine", "grid_color")


def save(name, obj):
    os.makedirs(OUT, exist_ok=True)
    path = os.path.join(OUT, name)
    torch.save(obj, path)
    print("wrote %-28s %8.1f KB" % (name, os.path.getsize(path) / 1024))


def stage_lrs(cfg, stage):
    st = cfg["mapping"]["stage"][stage]
    return dict(decoders=st["decoders_lr"], middle=st["middle_lr"], fine=st["fine_lr"], color=st["color_lr"])


def grid_samples(after, before, n=8192, seed=99):
    """A fixed random sample of a flat parameter vector after the loop, and norms of the whole."""
    g = torch.Generator().manual_seed(seed)
    pick = torch.randperm(after.numel(), generator=g)[:n].clone()
    return dict(idx=pick, val=after[pick].clone(), delta_norm=float((after - before).double().norm()), norm=float(after.double().norm()))


def gen_joint_fix_fine_false():
    rh.import_reference()
    import src.Mapper as mapper_mod
    sc, cfg, slam, renderer = mg.ref_scene("room0", "soft")
    mapper = rh.make_mapper(cfg, slam, renderer, coarse_mapper=False)
    mapper.fix_fine = False
    calls = mg.record_renderer(renderer)
    depth, color = su.make_frame(sc, 1)
    c2w = su.make_pose(sc, 1)
    samples = []
    _gs = mapper_mod.get_samples

    def get_samples_rec(*a, **k):
        r = _gs(*a, **k)
        samples.append([t.detach().clone() for t in r])
        return r
    mapper_mod.get_samples = get_samples_rec
    start = {k: v.detach().clone() for k, v in slam.shared_c.items()}
    dec_start = {lvl: {k: v.detach().clone() for k, v in getattr(slam.shared_decoders, lvl + "_decoder").state_dict().items()} for lvl in ("fine", "color")}
    try:
        torch.manual_seed(321)
        mapper.optimize_map(5, 1.0, 0, color, depth, c2w, [], [], c2w)
    finally:
        mapper_mod.get_samples = _gs
    its = []
    for it, call in enumerate(calls):
        s_o, s_d, s_gd, s_gc = samples[it]
        keep = tp.bbox_prefilter(s_o.float(), s_d.float(), s_gd.float(), slam.bound)
        assert torch.equal(s_o.float()[keep], call["rays_o"])
        its.append(dict(stage=call["stage"], rays_o=call["rays_o"], rays_d=call["rays_d"], gt_depth=call["gt_depth"],
                        gt_depth_loss=s_gd.float()[keep], gt_color=s_gc.float()[keep], lr=stage_lrs(cfg, call["stage"])))
    assert [it["stage"] for it in its] == ["middle"] * 3 + ["fine", "color"]
    final = {}
    for key in KEYS:
        m = mapper.get_mask_from_c2w(c2w, key, slam.shared_c[key].shape[2:], depth.numpy())
        vm = torch.from_numpy(np.ascontiguousarray(m)).permute(2, 1, 0).contiguous()
        m5 = vm.unsqueeze(0).unsqueeze(0).expand_as(slam.shared_c[key])
        final[key] = grid_samples(slam.shared_c[key][m5].detach().clone(), start[key][m5])
    decs = {lvl: {k: v.detach().clone() for k, v in getattr(slam.shared_decoders, lvl + "_decoder").state_dict().items()} for lvl in ("fine", "color")}
    for lvl in ("fine", "color"):                               # both decoders moved (the fine one in stage color only: decoders_lr is 0 in stage fine)
        assert any(not torch.equal(decs[lvl][k], dec_start[lvl][k]) for k in decs[lvl]), lvl
    save("joint_fix_fine_false.pt", dict(scene="room0", variant="soft", frame_seed=1, pose_seed=1, iterations=its, final=final,
                                         fine_decoder=decs["fine"], color_decoder=decs["color"], w_color_loss=cfg["mapping"]["w_color_loss"]))


def gen_color_refine_ba(n_it=5):
    rh.import_reference()
    import src.Mapper as mapper_mod
    sc, cfg, slam, renderer, mapper, kf_dict, kf_list, depth, color, c2w = mg._ba_setup()
    mapper.fix_color = True                                     # Mapper.py:578-586 (the window size of _ba_setup is kept)
    mapper.frustum_feature_selection = False
    mapper.middle_iter_ratio = 0.0
    mapper.fine_iter_ratio = 0.0
    samples, uv = [], []
    restore = mg._record_ba(mapper_mod, samples, uv)
    start = {k: v.detach().clone() for k, v in slam.shared_c.items()}
    dec_start = {k: v.detach().clone() for k, v in slam.shared_decoders.state_dict().items()}
    cam_hist = []
    _adam = torch.optim.Adam

    class SpyAdam(_adam):                                       # the real Adam; records the parameter groups before every step
        def step(self, *a, **k):
            cams = self.param_groups[5]["params"]
            cam_hist.append(dict(cam=torch.stack([c.detach().clone() for c in cams]), grad=torch.stack([c.grad.detach().clone() for c in cams]),
                                 n_decoder_params=len(self.param_groups[0]["params"])))
            return super().step(*a, **k)
    torch.optim.Adam = SpyAdam
    try:
        torch.manual_seed(778); np.random.seed(778)
        new_c2w = mapper.optimize_map(n_it, 1.0, 30, color, depth, c2w, kf_dict, kf_list, c2w)
    finally:
        torch.optim.Adam = _adam
        restore()
    assert all(h["n_decoder_params"] == 0 for h in cam_hist)   # fix_fine and fix_color: parameter group 0 is empty
    per_it = [samples[1 + 6 * it: 1 + 6 * (it + 1)] for it in range(n_it)]
    window0 = torch.stack([s["c2w"][:3] for s in per_it[0]])
    draws = [dict(i=torch.stack([f["i"] for f in fr]), j=torch.stack([f["j"] for f in fr]),
                  depth=torch.stack([f["depth"].float() for f in fr]), color=torch.stack([f["color"].float() for f in fr])) for fr in per_it]
    ident = []
    for r in range(6):
        hit = [k for k in range(5) if torch.allclose(su.make_pose(sc, 10 + k)[:3], window0[r][:3], atol=1e-5)]
        ident.append(hit[0] if hit else -1)
    final_c2w = torch.stack([(kf_dict[k]["est_c2w"] if k >= 0 else new_c2w)[:3].detach().clone() for k in ident])
    # the stage schedule of Mapper.py:403-409 with both ratios 0: the first iteration is a 'middle' one, every later one 'color'
    stages = ["middle" if it <= int(n_it * mapper.middle_iter_ratio) else ("fine" if it <= int(n_it * mapper.fine_iter_ratio) else "color") for it in range(n_it)]
    final, outside = {}, {}
    for key in KEYS:
        after = mapper.c[key].detach().reshape(-1).clone()
        before = start[key].reshape(-1)
        final[key] = grid_samples(after, before)
        m = mapper.get_mask_from_c2w(c2w, key, start[key].shape[2:], depth.numpy())
        vm = torch.from_numpy(np.ascontiguousarray(m)).permute(2, 1, 0).contiguous()
        out5 = (~vm).unsqueeze(0).unsqueeze(0).expand_as(start[key])
        outside[key] = int((mapper.c[key].detach()[out5] != start[key][out5]).sum())
        assert outside[key] > 0, key                            # voxels outside the current frustum move too
    assert all(torch.equal(v, dec_start[k]) for k, v in slam.shared_decoders.state_dict().items())
    save("color_refine_ba.pt", dict(scene="room0", variant="soft", frame_seed=1, pose_seed=1, keyframe_seeds=list(range(10, 15)), window_keyframes=ident,
                                    window_c2w=window0.clone(), final_c2w=final_c2w, camera_tensors=cam_hist[0]["cam"],
                                    camera_history=[dict(cam=h["cam"], grad=h["grad"]) for h in cam_hist], stages=stages,
                                    lrs=[stage_lrs(cfg, s) for s in stages], BA_cam_lr=cfg["mapping"]["BA_cam_lr"], draws=draws, final=final,
                                    moved_outside_frustum=outside, w_color_loss=cfg["mapping"]["w_color_loss"]))


if __name__ == "__main__":
    import warnings
    warnings.filterwarnings("ignore")
    gen_joint_fix_fine_false()
    gen_color_refine_ba()
