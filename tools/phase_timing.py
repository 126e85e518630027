#!/usr/bin/env python
"""Cycle breakdown of one CTA of the tensor-core kernels (instrumented build: make -C nice_slam_b200/csrc ../libnsb_timing.so).
   NSB_LIB=nice_slam_b200/libnsb_timing.so python tools/phase_timing.py [n_rays]"""
import ctypes as C
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))

TILE_NAMES = {40: "fwd: launch -> depth max done", 41: "fwd: ray table (bbox far, near)", 43: "fwd: sample z + rank sort", 44: "fwd: point geometry + syncs",
              1: "fwd: gather (per grid)", 5: "fwd: publish + wait all warps' gather", 11: "fwd: wait fc_c weight units (TMA)",
              2: "fwd: issue + complete fc_c MMAs", 6: "fwd: wait free buffer (E block)",
              3: "fwd: embed block compute", 10: "fwd: publish + wait all warps' E block", 4: "fwd: issue layer-0 block (+ retire block 0)",
              7: "fwd: wait MMAs of the layer (layer 0: its whole chain)", 8: "fwd: layer epilogue (relu, masks, H write)", 9: "fwd: publish + issue hidden layer", 12: "fwd: output layer + syncs",
              14: "fwd: dealloc + sync", 15: "fwd: parts store + ray completion", 16: "fwd: compositing of completed rays",
              20: "bwd: launch -> ray prologue (weights, dL/docc)", 21: "bwd: point geometry + sync", 22: "bwd: layer epilogue (G/DU write)", 23: "bwd: issue + wait layer MMAs", 24: "bwd: weight-gradient groups (WG)",
              27: "bwd: dc rows + cos chain", 29: "bwd: scatter + dp", 30: "bwd: per-ray partial sums", 31: "bwd: ray completion", 32: "bwd: final ray reduce"}
NAMES = {0: "fwd: tail sync of previous decoder", 1: "fwd: gather", 2: "fwd: fc_c publish + issue", 3: "fwd: E block 0", 4: "fwd: E block 1",
         5: "fwd: E block 2", 6: "fwd: wait fc_c / layer-0 MMAs", 7: "fwd: layer step 0", 8: "fwd: layer step 1", 9: "fwd: layer step 2",
         10: "fwd: layer step 3", 11: "fwd: layer 4 epilogue", 12: "fwd: output layer", 13: "fwd: sampling prologue", 14: "fwd: tmem dealloc",
         15: "fwd: compositing + store", 20: "bwd: tail sync / scatter of previous decoder", 21: "bwd: header wait + g init", 22: "bwd: layer 4",
         23: "bwd: layer 3", 24: "bwd: layer 2", 25: "bwd: layer 1", 26: "bwd: layer 0", 27: "bwd: dc rows + embedding chain", 28: "bwd: sync",
         29: "bwd: scatter", 30: "bwd: ray reduce"}


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 200
    os.environ.setdefault("NSB_LIB", os.path.join(ROOT, "nice_slam_b200", "libnsb_timing.so"))       # before nice_slam_b200._lib loads
    import torch
    import scene_util as su
    from gpu_util import make_renderer
    from nice_slam_b200 import _lib
    from nice_slam_b200.steps import IterationContext
    dev = torch.device("cuda")
    sc = su.load_scenes()["room0"]
    renderer, c, dec = make_renderer(sc, su.make_grids(sc, "soft"), su.load_decoders("soft"), dev)
    ro, rd, gd, gc = [t.to(dev) for t in su.make_rays(sc, n, seed=3)]
    ctx = IterationContext(renderer, n, "color", dev, kind="track")
    _lib.lib()
    fn = C.CDLL(os.environ["NSB_LIB"]).nsb_debug_phases
    fn.argtypes = [C.c_void_p, C.c_int]
    buf = (C.c_longlong * 64)()
    iters = 50
    for it in range(3 + iters):
        if it == 3:
            torch.cuda.synchronize(); fn(buf, 1)
        ctx.run(c, dec, ro, rd, gd, gc.double())
    torch.cuda.synchronize()
    fn(buf, 0)
    tot_f = sum(buf[i] for i in range(0, 20)); tot_b = sum(buf[i] for i in range(20, 40))
    print("cycles per launch of CTA 0 (avg of %d iterations, %d rays): forward %.0f, backward %.0f" % (iters, n, tot_f / iters, tot_b / iters))
    for i in range(64):
        if buf[i]:
            tot = tot_f if i < 20 else tot_b
            print("  %2d %-46s %9.0f  %5.1f %%" % (i, (TILE_NAMES if os.environ.get("NSB_MLP_BACKEND", "0") in ("0", "3") else NAMES).get(i, "?"), buf[i] / iters, 100.0 * buf[i] / tot))


if __name__ == "__main__":
    main()
