"""Runs bench.extra_workloads alone (development aid: validates the `extra` section without the headline loops)."""
import json, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch
import bench


def main():
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    sc, renderer, c, dec = bench.build_scene(dev)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)        # bench.py's own flush buffer, as bench.main passes it
    out = bench.extra_workloads(sc, renderer, c, dec, dev, flush, bench.peaks()[0])
    print(json.dumps(out))


if __name__ == "__main__":
    main()
