"""CLI drivers with the reference's flags and stdout lines (SURVEY §8 f2):

  python apps/lux_cli.py pagerank   -ng 1 -ni 10 -file g.lux [-verbose]            # pagerank/pagerank.cc:121-148
  python apps/lux_cli.py components -ng 2 -file g.lux [-check] [-verbose]          # components/components.cc:145-175
  python apps/lux_cli.py sssp       -ng 1 -file g.lux -start 0 [-check]            # sssp/sssp.cc
  python apps/lux_cli.py sssp       -weighted -file w.lux -start 0 [-check]        # weighted SSSP (i32 weight trailer; ours)
  python apps/lux_cli.py colfilter  -ng 1 -ni 10 -file ratings.lux                 # col_filter/colfilter.cc:85-107
  python apps/lux_cli.py bc         -ng 1 -file g.lux [-start v | -nsrc K -seed S] [-out scores.npy] [-verbose]
                                                                                   # betweenness centrality (ours)
  python apps/lux_cli.py bc         -weighted -file w.lux [-start v | -nsrc K -seed S] [-out scores.npy]
                                                                                   # weighted BC (i32 trailer, w >= 1; ours)
  python apps/lux_cli.py tc         -ng 1 -file g.lux [-out t.npy]                  # triangle counting (ours)
  python apps/lux_cli.py kcore      -ng 1 -file g.lux [-check] [-out core.npy]      # k-core decomposition (ours)
  python apps/lux_cli.py truss      -ng 1 -file g.lux [-check] [-out truss.npz]     # k-truss decomposition (ours)
  python apps/lux_cli.py converter  -nv N -ne M -input edges.txt -output g.lux     # tools/converter.cc:13-39 (host only)

`-ll:gpu N` is accepted as a synonym of `-ng N` (README.md:47); -ll:fsize / -ll:zsize are accepted and ignored (HBM is
managed by the library).  With -ng > 1 the driver re-launches itself under torch.distributed.run, one rank per GPU.
Prints the reference's lines: "[Memory Setting] Set ll:fsize >= %zuMB and ll:zsize >= %zuMB" (pagerank.cc:84-85,
components.cc:87-88), "ELAPSED TIME = %7.7f s" (pagerank.cc:118), "[PASS]/[FAIL] Check task: rowLeft(%u)
numMistakes(%u)" (components_gpu.cu:831-836).  `-out file.npy` additionally saves the vertex values (the reference never writes its results anywhere, SURVEY §5).

`bc` (no reference counterpart) sums Brandes' dependencies over a list of sources into f64 scores, not normalised.  The
sources: `-start v` alone is the single source v; `-nsrc K` takes K distinct vertices
numpy.random.default_rng(S).choice(nv, K, replace=False) with `-seed S` (default 0); neither flag means every vertex
(exact BC).  It prints "ELAPSED TIME" (device time of the BC run) and no "[Memory Setting]" line: the reference has no
formula for BC.  `bc -weighted` reads the .lux i32 weight trailer and runs weighted BC (shortest paths by weighted
distance, every weight >= 1) with the same source flags.

`tc` (no reference counterpart) counts the triangles of the graph read as undirected and simple (self-loops, parallel
edges and both directions of an edge collapse; weights are ignored).  It prints "ELAPSED TIME" (device time of the count)
and "TRIANGLES = T" on rank 0, and no "[Memory Setting]" line; `-out` saves the u64 triangle count of every vertex.

`kcore` (no reference counterpart) computes the core number of every vertex of the same undirected simple graph.  It
prints "ELAPSED TIME" (device time of the peel) and "DEGENERACY = K" (the largest core number) on rank 0, and no
"[Memory Setting]" line; `-check` prints the check line above per rank (vertices that are not a fixpoint of the h-index
operator); `-out` saves the u32 core numbers.

`truss` (no reference counterpart) computes the support and truss number of every edge of the same undirected simple
graph.  It prints "ELAPSED TIME" (device time of the support count and the peel) and "KMAX = K" (the largest truss
number) on rank 0, and no "[Memory Setting]" line; `-check` prints the check line above per rank (this rank's edges that
fail the truss check); `-out` saves an .npz with the u32 arrays lo, hi (the edges, ascending), support, truss and vertex
(the largest truss number at each vertex).
"""
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

APPS = {"pagerank": 0, "components": 1, "sssp": 2, "colfilter": 3, "bc": 5, "tc": 7, "kcore": 8, "truss": 9}


def parse(argv):
    opt = dict(ng=1, ni=10, file=None, start=0, verbose=False, check=False, out=None, weighted=False, start_set=False, nsrc=None,
               seed=0)
    i = 0
    while i < len(argv):
        a = argv[i]
        if a in ("-ng", "-ll:gpu"):
            opt["ng"] = int(argv[i + 1]); i += 1
        elif a == "-ni":
            opt["ni"] = int(argv[i + 1]); i += 1
        elif a == "-file":
            opt["file"] = argv[i + 1]; i += 1
        elif a == "-start":
            opt["start"] = int(argv[i + 1]); opt["start_set"] = True; i += 1
        elif a == "-nsrc":
            opt["nsrc"] = int(argv[i + 1]); i += 1
        elif a == "-seed":
            opt["seed"] = int(argv[i + 1]); i += 1
        elif a == "-out":
            opt["out"] = argv[i + 1]; i += 1
        elif a in ("-verbose", "-v"):
            opt["verbose"] = True
        elif a in ("-check", "-c"):
            opt["check"] = True
        elif a == "-weighted":
            opt["weighted"] = True
        elif a in ("-ll:fsize", "-ll:zsize", "-ll:cpu", "-ll:util"):
            i += 1  # Legion/Realm memory flags: accepted, not needed
        i += 1
    return opt


def memory_setting(app, nv, ne, bounds, frontier_bytes, weighted=False):
    """The reference's advice formulas, verbatim in sizes: pagerank.cc:61-85, components.cc:57-88.  `sssp -weighted`
    (no reference counterpart) adds 4 B per edge for the i32 weights to both figures."""
    W = 4 if weighted else 0
    V, E, VTX = 4, 8, (80 if app == "colfilter" else 4)
    max_fb, max_edges = 0, 0
    P = len(bounds["row_left"])
    for p in range(P):
        nodes = int(bounds["row_right"][p]) - int(bounds["row_left"][p]) + 1
        nodes = max(nodes, 0) if nodes < (1 << 31) else 0
        nxt = int(bounds["col_left"][p + 1]) if p + 1 < P else ne
        edges = max(nxt - int(bounds["col_left"][p]), 0)
        if app in ("pagerank", "colfilter"):
            edge_struct, node_struct = (12 if app == "colfilter" else 8), 16
            fb = edges * edge_struct + nodes * node_struct + nodes * V + nodes * VTX + nv * VTX
        else:
            fb = edges * 8 + edges * 4 + nodes * 8 + nv * 8 + nodes * 2 * VTX + nv * VTX + frontier_bytes * 2 + edges * W
        max_fb, max_edges = max(max_fb, fb), max(max_edges, edges)
    if app in ("pagerank", "colfilter"):
        zc = ne * V + nv * E + nv * V + nv * 2 * VTX
    else:
        zc = ne * V + nv * E + nv * 2 * VTX + frontier_bytes * 2 + nv * 8 + max_edges * 4 + ne * W
    return max_fb // 1024 // 1024 + 1, zc // 1024 // 1024 + 1


def bc_sources(opt, nv):
    """The sources of `bc`: -nsrc K -> numpy.random.default_rng(seed).choice(nv, K, replace=False); -start v -> [v];
    otherwise every vertex."""
    if opt["nsrc"] is not None:
        return np.random.default_rng(opt["seed"]).choice(nv, opt["nsrc"], replace=False).astype(np.uint32)
    if opt["start_set"]:
        return np.array([opt["start"]], np.uint32)
    return np.arange(nv, dtype=np.uint32)


def converter(argv):
    """tools/converter.cc: same flags, same first stdout line; the conversion itself is luxb_convert_edgelist."""
    nv, ne, inp, out = 0, 0, "", ""
    i = 0
    while i < len(argv):
        if argv[i] == "-nv":
            nv = int(argv[i + 1]); i += 1
        elif argv[i] == "-ne":
            ne = int(argv[i + 1]); i += 1
        elif argv[i] == "-input":
            inp = argv[i + 1]; i += 1
        elif argv[i] == "-output":
            out = argv[i + 1]; i += 1
        i += 1
    print("nv = %d ne = %d input = %s output = %s" % (nv, ne, inp, out), flush=True)  # converter.cc:80
    import lux_b200 as L
    try:
        L.convert_edgelist(inp, out, nv, ne)
    except L.LuxError as e:
        print("converter: %s" % e, file=sys.stderr)
        return 1
    return 0


def main():
    if len(sys.argv) >= 2 and sys.argv[1] == "converter":
        return converter(sys.argv[2:])
    if len(sys.argv) < 2 or sys.argv[1] not in APPS:
        print(__doc__)
        return 2
    app = sys.argv[1]
    opt = parse(sys.argv[2:])
    if not opt["file"]:
        print("Missing -file (graph in .lux format, see tools/converter.cc)")
        return 2
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if opt["ng"] > 1 and world == 1:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(opt["ng"]),
               "--master-addr", "127.0.0.1", "--master-port", os.environ.get("LUX_PORT", "29611")] + sys.argv
        return subprocess.call(cmd)
    rank, local = int(os.environ.get("RANK", "0")), int(os.environ.get("LOCAL_RANK", "0"))
    import lux_b200 as L
    if world > 1:
        import torch
        import torch.distributed as dist
        torch.cuda.set_device(local)
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    weighted = opt["weighted"] and app in ("sssp", "bc")  # weighted SSSP / BC over the .lux i32 weight trailer
    weighted_app = {"sssp": L.APP_SSSP_WEIGHTED, "bc": L.APP_BC_WEIGHTED}
    g = L.LuxGraph.from_file(opt["file"], app=weighted_app[app] if weighted else APPS[app], rank=rank, nranks=world, device=local,
                             start=opt["start"], verbose=opt["verbose"])
    b = g.bounds()
    if rank == 0 and app not in ("bc", "tc", "kcore", "truss"):
        fb, zc = memory_setting(app, g.nv, g.ne, b, int(b["fq_right"][-1]) + 1, weighted)
        print("[Memory Setting] Set ll:fsize >= %dMB and ll:zsize >= %dMB" % (fb, zc), flush=True)
    g.comm_init_torch()
    g.init()
    if app in ("pagerank", "colfilter"):
        g.iterate(opt["ni"])
    elif app == "bc":
        g.bc_run(bc_sources(opt, g.nv))
    elif app == "tc":
        total = g.tc_run()
    elif app == "kcore":
        degeneracy = g.kcore_run()
    elif app == "truss":
        kmax = g.truss_run()
    else:
        g.run_to_convergence()
    if rank == 0:
        print("ELAPSED TIME = %7.7f s" % g.stats()["loop_seconds"], flush=True)
        if app == "tc":
            print("TRIANGLES = %d" % total, flush=True)
        if app == "kcore":
            print("DEGENERACY = %d" % degeneracy, flush=True)
        if app == "truss":
            print("KMAX = %d" % kmax, flush=True)
    if opt["check"] and app in ("components", "sssp", "kcore", "truss"):
        bad = g.check()
        print("[%s] Check task: rowLeft(%u) numMistakes(%u)" % ("PASS" if bad == 0 else "FAIL", int(b["row_left"][rank]), bad),
              flush=True)
    if opt["out"]:
        vals = g.values()
        if rank == 0 and app == "truss":
            lo, hi, support, truss = g.truss_edges()
            np.savez(opt["out"], lo=lo, hi=hi, support=support, truss=truss, vertex=vals)
        elif rank == 0:
            np.save(opt["out"], vals)
    g.close()
    if world > 1:
        import torch.distributed as dist
        dist.barrier()
        dist.destroy_process_group()
    return 0


if __name__ == "__main__":
    sys.exit(main())
