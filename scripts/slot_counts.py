#!/usr/bin/env python
"""(source group, hub) pairs and slots of the source-blocked split on one rank, and the device memory the graph holds.

    python scripts/slot_counts.py [scale [steps]]   # RMAT-<scale>, edge factor 16, seed 27 (bench.py's graph); default 22

The library's verbose line reports, per group kind (tier-0 blocks, tier blocks, cold segments), how many (group, hub)
pairs there are and how many have at least one edge: only those get a slot of the partial array (panel.cuh).  The
JSON line adds the device memory in use after init() (cudaMemGetInfo before and after) and the split's statistics.
With steps, that many runs of 10 PageRank iterations follow (with LUXB_PHASE_TIMING=1 the library prints where their
time went when the graph is closed)."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.dont_write_bytecode = True


def main():
    import torch
    import lux_b200 as L
    scale = int(sys.argv[1]) if len(sys.argv) > 1 else 22
    steps = int(sys.argv[2]) if len(sys.argv) > 2 else 0
    nv, ne = 1 << scale, 16 << scale
    torch.cuda.init()
    free0, _ = torch.cuda.mem_get_info()
    g = L.LuxGraph.from_rmat(scale, nv, ne, 27, verbose=True)
    g.init()
    torch.cuda.synchronize()
    free1, _ = torch.cuda.mem_get_info()
    st = g.stats()
    sys.stdout.flush()
    keys = ["panel_hubs", "panel_blocks", "panel_edges", "tier_blocks", "tier_slots", "tier_edges", "cold_hub_edges", "cold_hub_segments"]
    print(json.dumps({"scale": scale, "device_bytes_after_init": free0 - free1, **{k: st[k] for k in keys if k in st}}))
    for _ in range(steps):
        g.iterate(10)
    torch.cuda.synchronize()
    sys.stdout.flush()
    g.close()


if __name__ == "__main__":
    main()
