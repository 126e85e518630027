"""Generate tests/golden/mapper_frames/*.pt: whole calls of the UNMODIFIED reference Mapper.optimize_map (imported from the reference checkout
through tests/ref_harness.py) on CPU, room0 geometry, 'soft' grids.

    python tests/make_golden_mapper_frames.py        # needs the reference checkout

Each fixture stores seeds, not images (keyframes and the current frame: scene_util.make_frame / make_pose), the mapping settings, and what
the call did: the overlap selection's pixel draw, the keyframes the window drew from, every row's pixel draws of every iteration (flat
k = j * W + i, int32 [iteration][row][pixel]), the stage and loss of every iteration, the returned pose and every keyframe's est_c2w after
the call, a sample of the optimised voxels, and the decoders the call trains (fine unless fix_fine, colour unless fix_color) after it.

    ba_overlap.pt     five keyframes, bundle adjustment, overlap selection, the shipped 0.4 / 0.6 ratios (middle, fine and colour stages)
    no_ba.pt          three keyframes, no bundle adjustment
    first_frame.pt    an empty store: the window is the current frame alone, lr_first_factor
    coarse.pt         the coarse mapper: global selection, stage 'coarse', no depth guidance in the render
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

OUT = os.path.join(su.GOLDEN, "mapper_frames")
ITERS = 10
KEYFRAME_SEEDS = [10, 11, 12, 13, 14]
FRAME_SEED = 1
CASES = {
    "ba_overlap": dict(n_keyframes=5, ba=True, coarse_mapper=False, window=6, first=False, seed=901),
    "no_ba": dict(n_keyframes=3, ba=False, coarse_mapper=False, window=5, first=False, seed=902),
    "first_frame": dict(n_keyframes=0, ba=False, coarse_mapper=False, window=5, first=True, seed=903),
    "coarse": dict(n_keyframes=5, ba=False, coarse_mapper=True, window=5, first=False, seed=904),
}
SETTING_KEYS = ("pixels", "mapping_window_size", "middle_iter_ratio", "fine_iter_ratio", "stage", "BA_cam_lr", "w_color_loss",
                "keyframe_selection_method", "fix_fine", "fix_color", "frustum_feature_selection")
GRIDS = {False: ("grid_middle", "grid_fine", "grid_color"), True: ("grid_coarse",)}


def gen_case(name, spec):
    rh.import_reference()
    import src.Mapper as mapper_mod
    import src.common as common_mod
    sc, cfg, slam, renderer = mg.ref_scene("room0", "soft")
    mapper = rh.make_mapper(cfg, slam, renderer, coarse_mapper=spec["coarse_mapper"], BA=spec["ba"])
    mapper.mapping_window_size = spec["window"]
    W = cfg["cam"]["W"]
    kf_dict, kf_list = [], []
    for k in range(spec["n_keyframes"]):
        depth, color = su.make_frame(sc, KEYFRAME_SEEDS[k])
        c2w = su.make_pose(sc, KEYFRAME_SEEDS[k])
        kf_dict.append(dict(gt_c2w=c2w.clone(), idx=5 * k, color=color, depth=depth, est_c2w=c2w.clone()))
        kf_list.append(5 * k)
    mapper.keyframe_dict, mapper.keyframe_list = kf_dict, kf_list
    depth, color = su.make_frame(sc, FRAME_SEED)
    c2w = su.make_pose(sc, FRAME_SEED)
    lr_factor = cfg["mapping"]["lr_first_factor"] if spec["first"] else cfg["mapping"]["lr_factor"]
    uv, selection, losses = [], [], []
    _guv, _sel, _rs, _bw = common_mod.get_sample_uv, mapper.keyframe_selection_overlap, mapper_mod.random_select, torch.Tensor.backward

    def get_sample_uv_rec(*a, **k):
        r = _guv(*a, **k)
        uv.append((r[1].long() * W + r[0].long()).int())
        return r

    def selection_rec(*a, **k):
        r = _sel(*a, **k)
        selection.append([int(x) for x in r])
        return r

    def random_select_rec(*a, **k):
        r = _rs(*a, **k)
        selection.append([int(x) for x in r])
        return r

    def backward_rec(self, *a, **k):
        losses.append(float(self.detach()))
        return _bw(self, *a, **k)
    common_mod.get_sample_uv, mapper.keyframe_selection_overlap, mapper_mod.random_select, torch.Tensor.backward = \
        get_sample_uv_rec, selection_rec, random_select_rec, backward_rec
    start = {k: v.detach().clone() for k, v in slam.shared_c.items()}
    try:
        torch.manual_seed(spec["seed"]); np.random.seed(spec["seed"])
        new_c2w = mapper.optimize_map(ITERS, lr_factor, 30, color, depth, c2w, kf_dict, kf_list, c2w)
    finally:
        common_mod.get_sample_uv, mapper_mod.random_select, torch.Tensor.backward = _guv, _rs, _bw
    sel = selection[0] if selection else []
    overlap = mapper.keyframe_selection_method == "overlap" and spec["n_keyframes"] > 0
    overlap_draw = uv.pop(0) if overlap else None
    F = len(sel) + (1 if spec["n_keyframes"] else 0) + 1
    assert len(uv) == ITERS * F and len(losses) == ITERS, (len(uv), F, len(losses))
    draws = torch.stack([torch.stack(uv[it * F:(it + 1) * F]) for it in range(ITERS)])
    stages = ["coarse" if spec["coarse_mapper"] else
              ("middle" if it <= int(ITERS * mapper.middle_iter_ratio) else ("fine" if it <= int(ITERS * mapper.fine_iter_ratio) else "color"))
              for it in range(ITERS)]
    final = {}
    for key in GRIDS[spec["coarse_mapper"]]:
        m = mapper.get_mask_from_c2w(c2w, key, slam.shared_c[key].shape[2:], depth.numpy())
        vm = torch.from_numpy(np.ascontiguousarray(m)).permute(2, 1, 0).contiguous()
        m5 = vm.unsqueeze(0).unsqueeze(0).expand_as(slam.shared_c[key])
        final[key] = mg_samples(slam.shared_c[key][m5].detach().clone(), start[key][m5])
    settings = {k: cfg["mapping"][k] for k in SETTING_KEYS}
    settings.update(mapping_window_size=spec["window"], keyframe_selection_method=mapper.keyframe_selection_method)
    trained = [lvl for lvl, fixed in (("fine", mapper.fix_fine), ("color", mapper.fix_color)) if not fixed]       # Mapper.py:336-341
    decs = {lvl: {k: v.detach().clone() for k, v in getattr(slam.shared_decoders, lvl + "_decoder").state_dict().items()} for lvl in trained}
    obj = dict(scene="room0", variant="soft", frame_seed=FRAME_SEED, keyframe_seeds=KEYFRAME_SEEDS[:spec["n_keyframes"]], seed=spec["seed"],
               iters=ITERS, lr_factor=lr_factor, ba=spec["ba"], coarse_mapper=spec["coarse_mapper"], settings=settings,
               overlap_draw=overlap_draw, selection=sel, draws=draws, stages=stages, losses=torch.tensor(losses, dtype=torch.float64),
               cur_c2w=None if new_c2w is None else new_c2w.detach().clone(),
               keyframe_est_c2w=torch.stack([d["est_c2w"].detach().clone() for d in kf_dict]) if kf_dict else torch.zeros(0, 4, 4),
               final=final, decoders=decs)
    os.makedirs(OUT, exist_ok=True)
    path = os.path.join(OUT, name + ".pt")
    torch.save(obj, path)
    print("wrote %-16s %8.1f KB  selection %s  losses %s" % (name + ".pt", os.path.getsize(path) / 1024, sel, [round(x, 3) for x in losses]))


def mg_samples(after, before, n=2048, seed=99):
    """A fixed random sample of a flat parameter vector after the call, and norms of the whole."""
    g = torch.Generator().manual_seed(seed)
    pick = torch.randperm(after.numel(), generator=g)[:n].int()
    return dict(idx=pick, val=after[pick].clone(), delta_norm=float((after - before).double().norm()), norm=float(after.double().norm()))


if __name__ == "__main__":
    import warnings
    warnings.filterwarnings("ignore")
    for nm in (sys.argv[1:] or CASES):
        gen_case(nm, CASES[nm])
