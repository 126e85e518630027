"""GPU: the tile kernels element by element against the float64 reference (oracle/f64_ref.py), with the float32 port's own error as
the yardstick.

For every output tensor, the kernel's error against the float64 truth is set beside the float32 CPU port's error against the same truth,
each taken on its own ReLU decisions (the kernel's saved mask words / the port's signs; the float64 reference re-runs on each).  Four
metrics: max-norm relative, L2 relative, and the per-element error |x - t| / (|t| + 1e-3 max|t|) by its maximum and its 99.9th
percentile.  The kernel passes when every metric is within K x the port's + FLOOR.  Unlike a max-norm bar against the float32 port, this
sees small elements (voxels few samples hit, samples behind the surface, the rows of a ragged last tile) and says which side is wrong.

The kernels' saved ReLU bits are checked against the sign of the float64 pre-activation: a disagreement may only sit at a knife edge
(|u| <= TAU x that layer's largest |u|), and there must be few.

Run with `-s` to print the measured pairs ("f64 <case> <tensor> kernel <4 metrics> port <4 metrics>").  Bars from an H100 run (see DESIGN.md §2)."""
import pytest
import torch

import scene_util as su
from gpu_util import make_renderer
from oracle import f64_ref as fr
from oracle import torch_port as tp

pytestmark = pytest.mark.gpu
DEV = "cuda"
METRICS = ("max", "l2", "pe_max", "pe_999")
# Worst kernel / port ratio measured on an H100 80GB HBM3 (700 W), bars about 1.5x above it:
#  * stages with the Fourier embedding (middle, fine, colour; rays and points): max 9.1 (S = 127, var), L2 6.1 (same), per-element 3.5
#    (wgrad_tc = 0, colour fc_c.4 bias gradient);
#  * the coarse stage (MLP_no_xyz: the GEMMs alone set the error, and the float32 port's own error is smallest there): max 14.7 (var 6.6e-6
#    vs 4.5e-7), L2 18.8, per-element 25 (d_rays_o 1.7e-3 vs 6.8e-5).  3xTF32 drops lo*lo and the tensor core reads 10 mantissa bits of
#    each part, so the kernel sits above float32 rounding while staying near 1e-5 in max norm;
#  * fwd_f16 (colour stage; its backward is the 3xTF32 one): max 2.7 (soft grids x 30, var), L2 2.0, per-element 1.4.
# Deterministic mode (option deterministic) is held to the same bars; its worst ratios over the det = 1 cases, (kernel - FLOOR) / port, on the
# same H100: K max 8.9 (S = 127, var), L2 6.0, per-element 2.3 (S = 256, var); K_COARSE max 14.4, L2 18.6, per-element 25 (d_rays_o);
# K_F16 max 2.7, L2 1.9, per-element 1.4 -- each equal to the default mode's, as the forward and the ray gradients are bit-identical.
K = {"max": 14.0, "l2": 10.0, "pe_max": 6.0, "pe_999": 6.0}
K_COARSE = {"max": 22.0, "l2": 28.0, "pe_max": 38.0, "pe_999": 38.0}
K_F16 = {"max": 4.0, "l2": 3.0, "pe_max": 2.2, "pe_999": 2.2}
#  * every decoder optimised (FP32-FMA backward), middle / fine / colour stages: max 6.8, L2 6.3, per-element 8.1 (init grids).
#    Deterministic mode (kDet weight-gradient kernels, test_gpu_wgrad_all / test_gpu_mapper_settings): max 7.3 (colour stage N = 31,
#    d_fine.fc_c.0.bias), L2 7.6 (fine + colour N = 64, d_fine.fc_c.4.bias), per-element 10.1 (fine stage x30, d_middle.fc_c.0.bias).
K_FP32_PASS = {"max": 10.0, "l2": 10.0, "pe_max": 12.0, "pe_999": 12.0}
FLOOR = {"max": 1e-7, "l2": 1e-7, "pe_max": 1e-6, "pe_999": 1e-6}
BIAS_BAR = 8e-7     # measured fwd_f16 scale bias: occupancy -2.1e-7, colour -5.0e-7 (float32 port: 1.7e-8, 2.0e-9)
TAU = 1e-5          # measured worst flip: |u| = 3.6e-6 x the layer's largest |u|
TAU_OWN = 4e-6      # knife edge of a kernel without saved ReLU words: just above that worst flip


def _option(name, value):
    from nice_slam_b200 import _lib
    assert _lib.lib().nsb_set_option(name.encode(), int(value)) == 0


class options:
    """Library options for the duration of a block, restored afterwards to the values they had on entry (nsb_get_option)."""

    def __init__(self, **kw):
        self.kw = kw

    def __enter__(self):
        from nice_slam_b200 import _lib
        self.saved = {k: _lib.get_option(k) for k in self.kw}
        for k, v in self.kw.items():
            _option(k, v)

    def __exit__(self, *exc):
        for k, v in self.saved.items():
            _option(k, v)


def cotangents(n, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(n, dtype=torch.float64, generator=g), torch.randn(n, dtype=torch.float64, generator=g),
            torch.randn(n, 3, generator=g))


def kernel_run(renderer, c, dec, ro, rd, gd, stage, cot, grad_grids, grad_decoders):
    r1, r2 = ro.to(DEV).requires_grad_(True), rd.to(DEV).requires_grad_(True)
    for k in c:
        c[k] = c[k].detach().requires_grad_(k in grad_grids)
    for n, p in dec.named_parameters():
        p.grad = None
        p.requires_grad_(n.split("_decoder.")[0] in grad_decoders)
    aux = {}
    d, u, col = renderer.render_batch_ray(c, dec, r2, r1, DEV, stage, gt_depth=gd.to(DEV) if gd is not None else None, aux=aux)
    ((d * cot[0].to(DEV)).sum() + (u * cot[1].to(DEV)).sum() + (col * cot[2].to(DEV)).sum()).backward()
    torch.cuda.synchronize()
    out = dict(depth=d.detach().cpu(), var=u.detach().cpu(), rgb=col.detach().cpu(), raw=aux["raw"].cpu(), z_vals=aux["z_vals"].cpu(),
               masks=fr.unpack_masks(aux["masks"].cpu(), len(fr.STAGE_DECODERS[stage])), d_rays_o=r1.grad.cpu(), d_rays_d=r2.grad.cpu())
    for k in grad_grids:
        out["d_" + k] = c[k].grad.cpu()
    out["d_dec"] = {lvl: {k: v.grad.cpu() for k, v in getattr(dec, lvl + "_decoder").named_parameters()} for lvl in grad_decoders}
    return out


def tensors(run, inb, stage):
    """(name, tensor) pairs of one run that are compared."""
    occ = run["raw"][..., 3][inb]
    yield "depth", run["depth"]
    yield "var", run["var"]
    yield "occ", occ
    if stage == "color":
        yield "rgb", run["rgb"]
        yield "raw_rgb", run["raw"][..., :3]
    for k in ("d_rays_o", "d_rays_d"):
        yield k, run[k]
    for k in sorted(run):
        if k.startswith("d_grid_"):
            yield k, run[k]
    for lvl in sorted(run["d_dec"]):
        for k in sorted(run["d_dec"][lvl]):
            yield "d_%s.%s" % (lvl, k), run["d_dec"][lvl][k]


def yardstick(label, kern, tk, port, tpt, stage, k_bar=K):
    """Compare kernel-vs-truth with port-vs-truth for every tensor; returns the list of failures."""
    failures = []
    inb_k = tk["fixed"]["inb"].reshape(tk["raw"].shape[:2])
    inb_p = tpt["fixed"]["inb"].reshape(tpt["raw"].shape[:2])
    truth_k, truth_p = dict(tensors(tk, inb_k, stage)), dict(tensors(tpt, inb_p, stage))
    mine, ports = dict(tensors(kern, inb_k, stage)), dict(tensors(port, inb_p, stage))
    for name, t in truth_k.items():
        ek, ep = fr.errors(mine[name], t), fr.errors(ports[name], truth_p[name])
        print("f64 %-28s %-26s kernel %s port %s" % (label, name, " ".join("%.1e" % ek[m] for m in METRICS),
                                                     " ".join("%.1e" % ep[m] for m in METRICS)))
        for m in METRICS:
            if not ek[m] <= k_bar[m] * ep[m] + FLOOR[m]:
                failures.append("%s %s %s: kernel %.2e > %.1f x port %.2e + %.0e" % (label, name, m, ek[m], k_bar[m], ep[m], FLOOR[m]))
    return failures


def check_masks(label, kern_masks, pre, inb, tau=TAU):
    """Kernel ReLU bits against the sign of the float64 pre-activation (computed on the kernel's own earlier-layer decisions), at the
    in-bound points: outside the bound the embedding argument |p B| reaches 1e3, where float32 sin is itself only good to ~1e-4, and the
    occupancy is replaced by 100 anyway.  Returns a list of failures."""
    pre, flip = pre[inb], kern_masks[inb] != (pre[inb] > 0)
    n = int(flip.sum())
    worst = 0.0
    if n:
        scale = pre.abs().amax(0, keepdim=True).expand_as(pre)
        worst = float((pre[flip].abs() / scale[flip]).max())
    print("f64 %-28s mask flips %d of %d, worst |u|/scale %.1e" % (label, n, flip.numel(), worst))
    limit = 8 + 4e-6 * flip.numel()
    return ["%s: mask flip at |u|/scale = %.1e > %.0e" % (label, worst, tau)] * (worst > tau) + \
           ["%s: %d mask flips > %d" % (label, n, limit)] * (n > limit)


def without_knife_edge_rays(label, grids, dec_state, ro, rd, stage, gd, bound, cot, n_samples, n_surface, coarse_enlarge):
    """The cotangents with those of the rays zeroed that have an in-bound sample at a ReLU knife edge (|u| <= TAU_OWN x the unit's largest
    |u|).  A kernel that saves no ReLU words decides every unit on its own float32 pre-activation, which the float64 truth cannot follow; at
    a knife edge the two may decide differently, and that sample's gradient then differs by the unit's whole share (one such sample set a
    ray's d_rays_o 7e-2 off, per element, at N = 100, middle stage).  With a zero cotangent such a ray adds nothing to any gradient; its
    forward outputs are still compared."""
    t = fr.run(grids, dec_state, ro, rd, stage, gd, bound, *cot, n_samples=n_samples, n_surface=n_surface, coarse_enlarge=coarse_enlarge)
    pre, inb = t["pre"], t["fixed"]["inb"]
    scale = pre[inb].abs().amax(0, keepdim=True)
    knife = ((pre.abs() <= TAU_OWN * scale).flatten(1).any(1) & inb).reshape(ro.shape[0], -1).any(1)
    print("f64 %-28s %d of %d rays at a knife edge get no cotangent" % (label, int(knife.sum()), knife.numel()))
    return tuple(torch.where(knife.reshape((-1,) + (1,) * (x.dim() - 1)), torch.zeros_like(x), x) for x in cot)


def check_case(label, sc, grids, dec_state, stage, ro, rd, gd, grad_grids=(), grad_decoders=(), n_samples=None, n_surface=None, seed=0,
               k_bar=None, tau=TAU, opts=None, truth_on_saved_masks=True, saved_masks=True, channels_last=True):
    """saved_masks = False: the forward saves no ReLU words (the FP32-FMA kernels), so the truth is taken on its own signs, the rays with
    a sample at a knife edge get no cotangent (without_knife_edge_rays) and there are no mask bits to check."""
    k_bar = k_bar or (K_COARSE if stage == "coarse" else K)
    n_samples = sc["rendering"]["N_samples"] if n_samples is None else n_samples
    n_surface = sc["rendering"]["N_surface"] if n_surface is None else n_surface
    bound = su.scene_bound(sc)
    cot = cotangents(ro.shape[0], seed)
    if not saved_masks:
        cot = without_knife_edge_rays(label, grids, dec_state, ro, rd, stage, gd if stage != "coarse" else None, bound, cot, n_samples,
                                      n_surface, sc["coarse_bound_enlarge"])
    renderer, c, dec = make_renderer(sc, grids, dec_state, DEV, channels_last=channels_last, n_samples=n_samples, n_surface=n_surface)
    with options(**(opts or {})):
        kern = kernel_run(renderer, c, dec, ro, rd, gd, stage, cot, grad_grids, grad_decoders)
    truth_on_saved_masks = truth_on_saved_masks and saved_masks
    gdp = gd if stage != "coarse" else None
    args = (grids, dec_state, ro, rd, stage, gdp, bound) + cot
    kw = dict(grad_grids=grad_grids, grad_decoders=grad_decoders, n_samples=n_samples, n_surface=n_surface)
    port = fr.port_run(*args, **kw)
    tk = fr.run(*args, **kw, coarse_enlarge=sc["coarse_bound_enlarge"], masks=kern["masks"] if truth_on_saved_masks else None)
    tpt = fr.run(*args, **kw, coarse_enlarge=sc["coarse_bound_enlarge"], masks=port["masks"])
    assert torch.equal(kern["z_vals"], tk["z_vals"])
    assert bool((kern["raw"][..., 3][~tk["fixed"]["inb"].reshape(kern["raw"].shape[:2])] == 100).all())
    failures = yardstick(label, kern, tk, port, tpt, stage, k_bar)
    if saved_masks:
        failures += check_masks(label, kern["masks"], tk["pre"], tk["fixed"]["inb"], tau)
    assert not failures, "\n".join(failures)


def scene(name="room0", variant="soft", scale=1.0):
    sc = su.load_scenes()[name]
    grids = su.make_grids(sc, variant)
    if scale != 1.0:
        grids = {k: v * scale for k, v in grids.items()}
    return sc, grids, su.load_decoders(variant)


GRIDS = {"coarse": ("grid_coarse",), "middle": ("grid_middle",), "fine": ("grid_fine", "grid_middle"),
         "color": ("grid_fine", "grid_color", "grid_middle")}


# ------------------------------------------------------------------------------------ tile residues, samples per ray, stages
# Axes shared by the cases below: det = option deterministic (the kDet tile backward and the ordered sums of nsb_det.cu), held to the default
# mode's bars -- both modes add the same float32 products, in another order; channels_last = False keeps the reference's NCDHW grids (the
# strided gathers: gather_tile_strided, gather_tile_kt's strided branch, grid_load4's scalar loads in the scatter).
LAYOUT = {True: "", False: " ncdhw"}


def modes(cases, ncdhw=(), layout=True):
    """pytest.param list over (case..., [channels_last,] det): every case in the default mode on channels-last grids under its own id, and in
    deterministic mode ('-det'); the cases in `ncdhw` also on NCDHW grids ('-ncdhw', '-ncdhw-det')."""
    def one(c, cl, det, suffix):
        c = c if isinstance(c, tuple) else (c,)
        return pytest.param(*(c + ((cl,) if layout else ()) + (det,)), id="-".join(str(v) for v in c) + suffix)
    return [one(c, True, d, "-det" * d) for c in cases for d in (0, 1)] + \
           [one(c, False, d, "-ncdhw" + "-det" * d) for c in ncdhw for d in (0, 1)]


@pytest.mark.parametrize("n_rays,channels_last,det", modes([128, 97, 95, 64, 33, 31, 1], ncdhw=[97]))
def test_tile_residues_against_f64(n_rays, channels_last, det):
    """S = 33 (17 + 16): N * S mod 128 = 0, 1, 63, 64, 65, 127 and one ray alone; rays and every stage grid through the tile backward."""
    sc, grids, dec = scene()
    ro, rd, gd, _ = su.make_rays(sc, n_rays, seed=300 + n_rays)
    check_case("residue N=%d det=%d%s" % (n_rays, det, LAYOUT[channels_last]), sc, grids, dec, "color", ro, rd, gd, GRIDS["color"], n_samples=17,
               n_surface=16, seed=n_rays, opts=dict(deterministic=det), channels_last=channels_last)


@pytest.mark.parametrize("n_samples,n_surface,n_rays,channels_last,det",
                         modes([(8, 0, 40), (5, 4, 40), (111, 16, 20), (112, 16, 20), (113, 16, 20), (240, 16, 9)], ncdhw=[(240, 16, 9)]))
def test_samples_per_ray_against_f64(n_samples, n_surface, n_rays, channels_last, det):
    """S from kMinSamples (8: 16 rays per tile) to NSB_MAX_SAMPLES (256: a ray over two tiles), 127 / 128 / 129 at the tile size."""
    sc, grids, dec = scene()
    ro, rd, gd, _ = su.make_rays(sc, n_rays, seed=400 + n_samples)
    check_case("S=%d det=%d%s" % (n_samples + n_surface, det, LAYOUT[channels_last]), sc, grids, dec, "color", ro, rd, gd, GRIDS["color"],
               n_samples=n_samples, n_surface=n_surface, seed=n_samples, opts=dict(deterministic=det), channels_last=channels_last)


@pytest.mark.parametrize("stage,channels_last,det", modes(["coarse", "middle", "fine"], ncdhw=["coarse"]))
def test_stages_against_f64(stage, channels_last, det):
    """The occupancy stages through the tile kernels (coarse: MLP_no_xyz, no embedding -- the GEMMs alone set the error; on NCDHW grids the
    strided gather at the enlarged coarse bound)."""
    sc, grids, dec = scene()
    ro, rd, gd, _ = su.make_rays(sc, 100, seed=500)
    check_case("stage %s det=%d%s" % (stage, det, LAYOUT[channels_last]), sc, grids, dec, stage, ro, rd, gd, GRIDS[stage], seed=5,
               opts=dict(deterministic=det), channels_last=channels_last)


@pytest.mark.parametrize("wgrad_tc,channels_last,det", [p for p in modes([1, 0], ncdhw=[1]) if p.id != "0-det"])
def test_colour_decoder_weight_gradients_against_f64(wgrad_tc, channels_last, det):
    """Mapping form of the colour stage: colour-decoder weight gradients on the tensor cores (render_bwd_wg_tile_kernel; deterministic mode:
    render_bwd_wg_tile_det_kernel and the ordered tile sum; NCDHW grids: gather_tile_kt's strided branch) and through the FP32-FMA pass
    (wgrad_tc = 0, which deterministic mode refuses); the ragged last tile at N * S = 97 * 48 (mod 128 = 48)."""
    from nice_slam_b200 import _lib
    if not wgrad_tc:
        with options(wgrad_tc=0, deterministic=0):
            assert _lib.lib().nsb_set_option(b"deterministic", 1) != 0
            assert _lib.get_option("deterministic") == 0
    sc, grids, dec = scene()
    ro, rd, gd, _ = su.make_rays(sc, 97, seed=600)
    check_case("wgrad_tc=%d det=%d%s" % (wgrad_tc, det, LAYOUT[channels_last]), sc, grids, dec, "color", ro, rd, gd, GRIDS["color"], ("color",),
               seed=6, opts=dict(wgrad_tc=wgrad_tc, deterministic=det), channels_last=channels_last)


@pytest.mark.parametrize("split_model,det", modes([1, 0], layout=False))
def test_item_split_forms_against_f64(split_model, det):
    """1408 rays x 48 = 528 tiles: with split_model = 1 tile_ws_plan takes one item per tile (all decoders in one CTA, full waves on 132
    SMs), with 0 one item per (tile, decoder)."""
    sc, grids, dec = scene()
    ro, rd, gd, _ = su.make_rays(sc, 1408, seed=700)
    check_case("split_model=%d det=%d" % (split_model, det), sc, grids, dec, "color", ro, rd, gd, GRIDS["color"] if det else (), seed=7,
               opts=dict(split_model=split_model, deterministic=det))


# ------------------------------------------------------------------------------------ value ranges
@pytest.mark.parametrize("variant,scale,det", modes([("init", 1.0), ("soft", 1e-3), ("soft", 30.0)], layout=False))
def test_value_ranges_against_f64(variant, scale, det):
    """Saturated scene (init grids: alpha = 1 at the first sample), tiny features (x 1e-3) and large ones (x 30)."""
    sc, grids, dec = scene(variant=variant, scale=scale)
    ro, rd, gd, _ = su.make_rays(sc, 100, seed=800)
    check_case("%s x%g det=%d" % (variant, scale, det), sc, grids, dec, "color", ro, rd, gd, GRIDS["color"], seed=8, opts=dict(deterministic=det))


def test_out_of_bound_and_zero_depth_rays_against_f64(det=0):
    """A batch mixing rays that start outside the bound (every sample occupancy 100), rays without a sensor depth and ordinary rays."""
    sc, grids, dec = scene()
    ro, rd, gd, _ = su.make_rays(sc, 90, seed=900)
    ro = ro.clone(); gd = gd.clone()
    ro[::3] += 100.0
    gd[1::4] = 0.0
    check_case("oob + zero depth det=%d" % det, sc, grids, dec, "color", ro, rd, gd, GRIDS["color"], seed=9, opts=dict(deterministic=det))


def test_out_of_bound_and_zero_depth_rays_in_deterministic_mode_against_f64():
    """The same batch through the kDet tile backward and the ordered sums."""
    test_out_of_bound_and_zero_depth_rays_against_f64(det=1)


@pytest.mark.parametrize("stage,variant", [("middle", "soft"), ("fine", "soft"), ("color", "soft"), ("color", "init")])
def test_all_decoder_gradients_against_f64(stage, variant):
    """Every decoder of the stage optimised, as the render fixtures request: the backward is then the FP32-FMA pass (render_bwd_kernel),
    which recomputes the forward and takes its ReLU decisions from that float32 recomputation, not from the tile forward's saved bits.  Its
    truth is therefore the float64 reference on its own signs (evaluated on the saved bits instead, one unit the two forwards decide
    differently at |u| ~ 1e-8 of the layer scale moved the middle decoder's layer-0 bias gradient by 7e-3 of its largest element).  Covers the
    middle / fine weight gradients, and the saturated scene that needs TOL_SATURATED against the float32 reference (there the kernel's fine
    decoder gradients are 1.2e-3 from float64, the float32 port's 2.0e-3).  The coarse stage in this form is left to the fixture test: against
    the own-sign truth one layer-4 bias element of the coarse decoder sat 1.3e-3 (per element) off while the port's own decisions gave 8.7e-6,
    a spread this test cannot attribute without the FP32 pass's decisions."""
    sc, grids, dec = scene(variant=variant)
    ro, rd, gd, _ = su.make_rays(sc, 96, seed=1000)
    check_case("all dec %s %s" % (stage, variant), sc, grids, dec, stage, ro, rd, gd, GRIDS[stage], fr.STAGE_DECODERS[stage], seed=10,
               k_bar=K_FP32_PASS, truth_on_saved_masks=False)


# ------------------------------------------------------------------------------------ option fwd_f16
@pytest.mark.parametrize("variant,scale,det", modes([("soft", 1.0), ("init", 1.0), ("soft", 30.0)], layout=False))
def test_fp16_split_forward_against_f64(variant, scale, det):
    """Option fwd_f16 (FP16 hi | lo forward, DESIGN §4.4): 22 significant bits for operands in [2^-3, 65504], absolute 2^-25 below.  The
    init fine grid (sigma = 1e-4) is the absolute regime; soft x 30 drives activations into the tens."""
    sc, grids, dec = scene(variant=variant, scale=scale)
    ro, rd, gd, _ = su.make_rays(sc, 100, seed=1100)
    check_case("f16 %s x%g det=%d" % (variant, scale, det), sc, grids, dec, "color", ro, rd, gd, GRIDS["color"], seed=11, k_bar=K_F16, tau=1e-4,
               opts=dict(fwd_f16=1, deterministic=det))


def test_fp16_split_forward_has_no_scale_bias():
    """fwd_f16 splits every activation operand as hi = fp16(x), lo = fp16(x - hi), both rounded to nearest, so the split is unbiased: over
    many points the kernel's decoder outputs carry no systematic scale error.  Scale bias b = sum((x - t) t) / sum(t^2) over 65 536 in-bound
    points (points mode, colour stage) against the float64 truth, beside the float32 port's; a split that shrinks operands (lo rounded toward
    zero) would show here long before a max-norm metric moves.  The kernel does carry a small bias of its own (-5e-7 on the colour outputs;
    the float32 port's is 2e-9), which the bar holds in place."""
    sc, grids, dec_state = scene()
    renderer, c, dec = make_renderer(sc, grids, dec_state, DEV)
    bound = su.scene_bound(sc)
    g = torch.Generator().manual_seed(65536)
    lo, hi = bound[:, 0], bound[:, 1]
    p = lo + (hi - lo) * (0.02 + 0.96 * torch.rand(65536, 3, generator=g, dtype=torch.float64))
    with options(fwd_f16=1):
        got = renderer.eval_points(p.to(DEV), dec, c, "color", DEV).cpu().double()
    port = tp.eval_points(p, grids, dec_state, "color", bound).double()
    t = fr.eval_points(p, grids, dec_state, "color", bound, sc["coarse_bound_enlarge"])
    bias = lambda x, ch: float(((x[:, ch] - t[:, ch]) * t[:, ch]).sum() / (t[:, ch] ** 2).sum())
    failures = []
    for name, ch in (("occ", 3), ("rgb", slice(0, 3))):
        bk, bp = bias(got, ch), bias(port, ch)
        print("f64 f16 scale bias %-4s kernel %.2e port %.2e" % (name, bk, bp))
        if not abs(bk) <= BIAS_BAR:
            failures.append("%s: kernel scale bias %.2e (port %.2e)" % (name, bk, bp))
    assert not failures, failures


# ------------------------------------------------------------------------------------ points mode
def check_points(label, n_points, k_bar=K, k_bar_coarse=K_COARSE, opts=None, channels_last=True):
    """FusedRenderer.eval_points at n_points points in and around the bound (seeded by n_points), coarse and colour stages, against
    fr.eval_points beside the float32 port."""
    sc, grids, dec_state = scene()
    renderer, c, dec = make_renderer(sc, grids, dec_state, DEV, channels_last=channels_last)
    bound = su.scene_bound(sc)
    g = torch.Generator().manual_seed(n_points)
    lo, hi = bound[:, 0] - 0.2, bound[:, 1] + 0.2
    p = lo + (hi - lo) * torch.rand(n_points, 3, generator=g, dtype=torch.float64)
    failures = []
    for stage in ("coarse", "color"):
        with options(**(opts or {})):
            got = renderer.eval_points(p.to(DEV), dec, c, stage, DEV).cpu()
        port = tp.eval_points(p, grids, dec_state, stage, bound)
        t = fr.eval_points(p, grids, dec_state, stage, bound, sc["coarse_bound_enlarge"])
        inb = tp.in_bound_mask(p, bound)
        assert torch.equal(got[:, 3] == 100, ~inb)
        for name, sel in (("occ", (inb, 3)), ("rgb", (slice(None), slice(0, 3)))):
            if stage == "coarse" and name == "rgb":
                continue
            ek, ep = fr.errors(got[sel], t[sel]), fr.errors(port[sel], t[sel])
            print("f64 %-28s %-26s kernel %s port %s" % ("%s n=%d %s" % (label, n_points, stage), name, " ".join("%.1e" % ek[m] for m in METRICS),
                                                         " ".join("%.1e" % ep[m] for m in METRICS)))
            kb = k_bar_coarse if stage == "coarse" else k_bar
            failures += ["%s %s %s %s" % (stage, name, m, ek[m]) for m in METRICS if not ek[m] <= kb[m] * ep[m] + FLOOR[m]]
    assert not failures, failures


@pytest.mark.parametrize("n_points,channels_last,det", [p for p in modes([256, 129, 191, 192, 193, 255], ncdhw=[129]) if p.id == "129-ncdhw-det" or "det" not in p.id])
def test_eval_points_against_f64(n_points, channels_last, det):
    """FusedRenderer.eval_points (points mode, one sample per 'ray'): point counts with residues 0, 1, 63, 64, 65, 127 mod 128; NCDHW grids
    through the strided gather, in both modes."""
    check_points("points%s det=%d" % (LAYOUT[channels_last], det), n_points, opts=dict(deterministic=det), channels_last=channels_last)


# ------------------------------------------------------------------------------------ option pdl
def test_pdl_launch_gives_identical_bits():
    """Option pdl launches the tracking iteration's backward as a programmatic dependent of the forward: the same kernels in another launch
    order, so loss, ray gradients and pose gradient are bit-identical with the plain stream order."""
    from nice_slam_b200.steps import IterationContext
    sc, grids, dec_state = scene()
    renderer, c, dec = make_renderer(sc, grids, dec_state, DEV)
    n = 200
    ro, rd, gd, gc = su.make_rays(sc, n, seed=1200)
    dirs = torch.randn(n, 3, generator=torch.Generator().manual_seed(12)).to(DEV)
    out = {}
    for pdl in (1, 0):
        with options(pdl=pdl):
            ctx = IterationContext(renderer, n, "color", DEV, kind="track")
            ctx.run(c, dec, ro.to(DEV), rd.to(DEV), gd.to(DEV), gc.double().to(DEV), dirs=dirs)
            torch.cuda.synchronize()
            out[pdl] = (ctx.loss.clone(), ctx.depth.clone(), ctx.rgb.clone(), ctx.d_rays_o.clone(), ctx.d_rays_d.clone(), ctx.d_c2w.clone())
    assert float(out[0][3].abs().max()) > 0
    for a, b in zip(out[1], out[0]):
        assert torch.equal(a, b)
