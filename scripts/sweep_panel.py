"""Dev tool: sweep the source-blocked sweep's parameters (panel.cuh) on one GPU at RMAT-<scale>.
usage: sweep_panel.py [scale] ["PANEL_SHAPE:BLOCKS:MIN_INDEG[:BS[:MAIN_SHAPE[:MAIN_CTAS]]],..."]
       PANEL_SHAPE = off -> flagged stream without the split (then MAIN_SHAPE / MAIN_CTAS are fields 4 / 5); merge -> pull.cuh tiles
Prints per configuration: panel coverage, ms/iteration, the per-phase device times (LUXB_PHASE_TIMING) and a one-step
parity check against the oracle on pseudo-random destination blocks."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
os.environ["LUXB_PHASE_TIMING"] = "1"
import lux_b200 as L  # noqa: E402
import oracle as O  # noqa: E402

scale = int(sys.argv[1]) if len(sys.argv) > 1 else 27
cfgs = sys.argv[2].split(",") if len(sys.argv) > 2 else ["merge", "off", "off::::1", "off::::3:2", "0:48:64", "1:48:64", "2:48:64", "1:64:32", "1:32:64"]
nv, ne = 1 << scale, 16 << scale
blk = None
extra_keys = set()
for c in cfgs:
    c, _, extra = c.partition("@")          # "...@ENV=VAL;ENV=VAL": extra environment for this configuration
    for k in extra_keys:
        os.environ.pop(k, None)
    for kv in filter(None, extra.split(";")):
        k, _, v = kv.partition("=")
        os.environ[k] = v
        extra_keys.add(k)
    c_label = c + ("@" + extra if extra else "")
    f = c.split(":")
    for k in ("LUXB_SEG_PANEL_SHAPE", "LUXB_SB_BLOCKS", "LUXB_SB_MIN_INDEG", "LUXB_SB_BS", "LUXB_SEG_MAIN_SHAPE", "LUXB_PULL_CTAS", "LUXB_SWEEP"):
        os.environ.pop(k, None)
    if f[0] == "merge":
        os.environ["LUXB_SWEEP"] = "merge"
    elif f[0] == "off":
        os.environ["LUXB_SB"] = "0"
    else:
        os.environ["LUXB_SB"] = "1"
        os.environ["LUXB_SEG_PANEL_SHAPE"], os.environ["LUXB_SB_BLOCKS"], os.environ["LUXB_SB_MIN_INDEG"] = f[0], f[1], f[2]
        if len(f) > 3 and f[3]:
            os.environ["LUXB_SB_BS"] = f[3]
    if len(f) > 4 and f[4]:
        os.environ["LUXB_SEG_MAIN_SHAPE"] = f[4]
    if len(f) > 5 and f[5]:
        os.environ["LUXB_PULL_CTAS"] = f[5]
    with L.LuxGraph.from_rmat(scale, nv, ne, 27) as g:
        g.init()
        st = g.stats()
        g.iterate(5)
        x5 = g.values()
        g.iterate(1)
        x6 = g.values()
        g.enable_kernel_timing(True)
        s0 = g.stats()
        g.iterate(20)
        s1 = g.stats()
        if blk is None:
            bs = min(14, scale - 6)
            sel = (np.random.default_rng(5).integers(0, 64, nv >> bs) == 0).astype(np.uint8)
            sel[0] = 1
            blk = O.rmat_blocks(scale, nv, ne, 27, bs, sel, want_deg=True)
        ref = O.pagerank_iter_compact(nv, blk, blk["deg"], x5)
        err = (np.abs(x6[blk["vid"]].astype(np.float64) - ref) / np.abs(ref.astype(np.float64))).max()
        k = (s1["dominant_kernel_seconds"] - s0["dominant_kernel_seconds"]) / 20
        t = (s1["loop_seconds"] - s0["loop_seconds"]) / 20
        print("cfg %-40s panel %.1f%% of edges, %d hubs x %d blocks, tiers %d blocks %d slots %.1f%% of edges | sweep %.3f ms, iter %.3f ms, %.1f GTEPS, frac %.3f | parity %.2e %s" % (
            c_label, 100.0 * st["panel_edges"] / ne, st["panel_hubs"], st["panel_blocks"], st["tier_blocks"], st["tier_slots"],
            100.0 * st["tier_edges"] / ne, k * 1e3, t * 1e3, ne / t / 1e9,
            (8 * ne + 16 * nv) / k / 1e9 / 6486.8, err, "OK" if err <= 1e-6 else "FAIL"), flush=True)
