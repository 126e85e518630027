#!/usr/bin/env python
"""Where the tile kernels' items run and how long each takes (instrumented build: make -C nice_slam_b200/csrc ../libnsb_items.so).

    NSB_LIB=nice_slam_b200/libnsb_items.so python tools/item_timing.py [--iters K] [--out DIR]

Thread 0 of every tile CTA records its SM (%smid), its item (tile, decoder) and %globaltimer at start, at the end of its decoder chain and
at exit.  The tool runs bench.py's tracking iteration at 64 and 200 rays and the 996-ray mapping iteration (BASELINE configs[1]), each one
iteration at a time with L2 flushed in between, and reports per launch:
  * per decoder kind, the item latency (start -> exit, and start -> end of chain) alone on an SM and while another item shares it;
  * which kinds share SMs (pairs of items whose [start, exit) overlap on one SM);
  * the order in which blocks reach SMs: whether the first round puts one block on every SM, and whether block m + j (m = SM count)
    lands on the SM of block j;
  * which SM finishes last (last exit, last chain end) and what runs on it.
DIR/item_timing.json holds the figures, DIR/report.txt the same as text, DIR/<workload>_<launch>.npy the raw records."""
import argparse
import ctypes as C
import json
import os
import statistics
import sys
from collections import Counter, defaultdict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from measure import Flush  # noqa: E402

LAUNCHES = ("forward", "backward", "weight-gradient backward")
LEVEL_NAMES = {-1: "all", 0: "coarse", 1: "middle", 2: "fine", 3: "color"}
RECORD = np.dtype([("sm", "<i4"), ("tile", "<i4"), ("my", "<i4"), ("level", "<i4"), ("t", "<u8", (3,))])
MAX_BLOCKS = 4096


def read_records(fn, launch):
    buf = np.zeros(MAX_BLOCKS, dtype=RECORD)
    if fn(launch, buf.ctypes.data_as(C.c_void_p), MAX_BLOCKS, 0) != 0:
        raise RuntimeError("nsb_debug_items failed")
    n = int(np.count_nonzero(buf["t"][:, 0]))
    assert np.all(buf["t"][:n, 0] != 0) and np.all(buf["t"][n:, 0] == 0), "records of one launch are not blocks 0..n-1"
    return buf[:n].copy()


def latency_stats(v):
    """count, mean, median, min and max of a list of microsecond figures, which may be empty"""
    return {"n": len(v), "mean_us": statistics.mean(v), "median_us": statistics.median(v), "min_us": min(v), "max_us": max(v)} if v else {"n": 0}


def analyse(runs, sms):
    """runs: list of record arrays of one launch (one per iteration)."""
    lat = defaultdict(lambda: {"alone": [], "shared": []})
    chain = defaultdict(lambda: {"alone": [], "shared": []})
    pairs, last_exit, last_chain, spans = Counter(), Counter(), Counter(), []
    first_round_distinct, second_round_same, second_round_n, start_spread = [], 0, 0, []
    for rec in runs:
        n = len(rec)
        t0 = rec["t"][:, 0].astype(np.int64); t1 = rec["t"][:, 1].astype(np.int64); t2 = rec["t"][:, 2].astype(np.int64)
        base = t0.min()
        spans.append((t2.max() - base) / 1e3)
        kinds = [LEVEL_NAMES.get(int(l), str(l)) for l in rec["level"]]
        by_sm = defaultdict(list)
        for b in range(n):
            by_sm[int(rec["sm"][b])].append(b)
        partners = defaultdict(list)
        for blocks in by_sm.values():
            for i in range(len(blocks)):
                for j in range(i + 1, len(blocks)):
                    a, b = blocks[i], blocks[j]
                    if t0[a] < t2[b] and t0[b] < t2[a]:
                        partners[a].append(b); partners[b].append(a)
                        pairs["+".join(sorted((kinds[a], kinds[b])))] += 1
        for b in range(n):
            key = "shared" if partners[b] else "alone"
            lat[kinds[b]][key].append((t2[b] - t0[b]) / 1e3)
            chain[kinds[b]][key].append((t1[b] - t0[b]) / 1e3)
        m = min(n, sms)
        first_round_distinct.append(len(set(int(s) for s in rec["sm"][:m])) == m)
        for j in range(n - sms if n > sms else 0):
            if j + sms < n:
                second_round_n += 1
                second_round_same += int(rec["sm"][j + sms] == rec["sm"][j])
        start_spread.append((t0[:m].max() - t0[:m].min()) / 1e3)

        def on_sm(b):
            return "+".join(sorted(kinds[x] for x in by_sm[int(rec["sm"][b])]))
        last_exit[on_sm(int(np.argmax(t2)))] += 1
        last_chain[on_sm(int(np.argmax(t1)))] += 1
    return {"blocks": len(runs[0]), "iterations": len(runs), "launch_span_us": latency_stats(spans),
            "item_latency_us": {k: {s: latency_stats(v[s]) for s in v} for k, v in sorted(lat.items())},
            "chain_latency_us": {k: {s: latency_stats(v[s]) for s in v} for k, v in sorted(chain.items())},
            "sharing_pairs_per_launch": {k: v / len(runs) for k, v in pairs.most_common()},
            "dispatch": {"first_round_one_block_per_sm": sum(first_round_distinct) / len(runs),
                         "block_m_plus_j_on_sm_of_block_j": (second_round_same / second_round_n) if second_round_n else None,
                         "first_round_start_spread_us": latency_stats(start_spread),
                         "first_round_sm_order_of_one_launch": [int(s) for s in runs[-1]["sm"][:min(len(runs[-1]), sms)]]},
            "last_sm_by_exit": dict(last_exit.most_common()), "last_sm_by_chain_end": dict(last_chain.most_common())}


def report_lines(name, launch, a):
    out = ["%s, %s launch: %d blocks, span %.1f us (median %.1f)" % (name, launch, a["blocks"], a["launch_span_us"]["mean_us"], a["launch_span_us"]["median_us"])]
    for k, v in a["item_latency_us"].items():
        ch = a["chain_latency_us"][k]
        out.append("  %-6s item (chain) us: alone %s   shared %s" % (k, fmt(v["alone"], ch["alone"]), fmt(v["shared"], ch["shared"])))
    out.append("  sharing pairs per launch: %s" % ", ".join("%s %.1f" % kv for kv in a["sharing_pairs_per_launch"].items()))
    d = a["dispatch"]
    out.append("  dispatch: first round one block per SM in %.0f %% of launches; block m+j on block j's SM: %s; first-round start spread %.2f us"
               % (100 * d["first_round_one_block_per_sm"], "n/a" if d["block_m_plus_j_on_sm_of_block_j"] is None else
                  "%.0f %%" % (100 * d["block_m_plus_j_on_sm_of_block_j"]), d["first_round_start_spread_us"]["mean_us"]))
    out.append("  last SM to exit runs: %s" % a["last_sm_by_exit"])
    out.append("  last SM to end a chain runs: %s" % a["last_sm_by_chain_end"])
    return out


def fmt(v, ch):
    return "n=%d %.1f (%.1f)" % (v["n"], v["mean_us"], ch["mean_us"]) if v["n"] else "n=0"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--out", default="item_timing")
    args = ap.parse_args()
    os.environ.setdefault("NSB_LIB", os.path.join(ROOT, "nice_slam_b200", "libnsb_items.so"))       # before nice_slam_b200._lib loads
    import bench
    from nice_slam_b200 import _lib
    from nice_slam_b200.steps import IterationContext
    dev = torch.device("cuda")
    sc, renderer, c, dec = bench.build_scene(dev)
    _lib.lib()
    fn = C.CDLL(os.environ["NSB_LIB"]).nsb_debug_items
    fn.argtypes = [C.c_int, C.c_void_p, C.c_int, C.c_int]
    props = torch.cuda.get_device_properties(dev)
    sms = props.multi_processor_count
    flush = Flush(dev)
    os.makedirs(args.out, exist_ok=True)
    result = {"device": props.name, "sms": sms, "workloads": {}}
    lines = ["%s, %d SMs; %d iterations per workload, L2 flushed before each" % (props.name, sms, args.iters)]
    for name, n, kind in (("tracking_64", 64, "track"), ("tracking_200", 200, "track"), ("mapping_996", 996, "map")):
        ro, rd, dirs, gd, gc = [t.to(dev) for t in bench.make_batch(sc, n, 101 if kind == "map" else 0)]
        if kind == "map":
            ctx = IterationContext(renderer, n, "color", dev, kind="map", grad_grids=("grid_middle", "grid_fine", "grid_color"), grad_decoders=("color",))
            step = lambda: ctx.run(c, dec, ro, rd, gd, gc.float())          # noqa: E731
        else:
            ctx = IterationContext(renderer, n, "color", dev, kind="track")
            step = lambda: ctx.run(c, dec, ro, rd, gd, gc, dirs=dirs)       # noqa: E731
        for _ in range(5):
            step()
        torch.cuda.synchronize()
        runs = defaultdict(list)
        for _ in range(args.iters):
            fn(0, None, 0, 1)
            flush.flush()
            step()
            torch.cuda.synchronize()
            for launch in range(3):
                rec = read_records(fn, launch)
                if len(rec):
                    runs[launch].append(rec)
        result["workloads"][name] = {}
        for launch, rr in sorted(runs.items()):
            a = analyse(rr, sms)
            result["workloads"][name][LAUNCHES[launch]] = a
            lines += report_lines(name, LAUNCHES[launch], a)
            np.save(os.path.join(args.out, "%s_%s.npy" % (name, LAUNCHES[launch].replace(" ", "_"))), np.stack(rr))
        del ctx
    with open(os.path.join(args.out, "item_timing.json"), "w") as f:
        json.dump(result, f, indent=1)
    with open(os.path.join(args.out, "report.txt"), "w") as f:
        f.write("\n".join(lines) + "\n")
    print("\n".join(lines))


if __name__ == "__main__":
    main()
