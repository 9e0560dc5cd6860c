"""Betweenness centrality on the C4 graph (device-generated RMAT-24, edge factor 16, seed 24) from K sources: vertex 0
and K - 1 seeded vertices with out-degree > 0 (numpy.random.default_rng(--seed) draws from them), on 1 GPU or on N GPUs
(re-launches itself under torch.distributed.run).  Prints ONE JSON line:

  card name and power limit (read in the same call); ms per source (median and min over --reps runs of all K sources),
  split into BFS (levels and level lists included), sigma and delta with LUXB_PHASE_TIMING=2; BFS levels per source;
  edges touched (luxb_stats edges_processed: BFS scans + sigma edges + delta edges, summed over ranks); MTEPS = ne * K / t;
  a parity flag against the CPU oracle (tests/bc_oracle.c) with its CPU time and core count; and, in the same call,
  unweighted SSSP from vertex 0 (scripts/bench_sssp.py's BFS) for the BFS part.

  python scripts/bench_bc.py [--gpus N] [--scale 24] [--k 8] [--reps 3] [--seed 1] [--no-oracle] [--weighted]

--weighted runs weighted BC instead, over the generator's [1, 255] weights (luxb_open_rmat), with the same sources: the
SSSP part is then weighted SSSP, "levels" are distance classes (from the weighted oracle, tests/bc_weighted_oracle.c,
which also gives the parity flag) and the reference SSSP run is weighted SSSP from vertex 0.  Both modes report the
kernel launches per source (luxb_stats kernel_launches), which bound the per-level / per-class overhead.

Algorithmic bound: each of the sigma and delta sweeps reads an id and a level per reached edge, 8 bytes, so
8 * ne bytes per sweep at most; the JSON line states each sweep's time against that volume at the data-sheet 3.35 TB/s."""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))  # the BC oracle lives with the tests
DATASHEET_TBPS = 3.35  # H100 SXM5 80 GB HBM3


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        name, power = [s.strip() for s in out[0].split(",")]
        return name, power
    except Exception:  # noqa: BLE001
        import torch
        return torch.cuda.get_device_name(0), "unknown"


class StderrCapture:
    """The library prints its phase means on fd 2: catch them in a temporary file."""

    def __enter__(self):
        self.f = tempfile.TemporaryFile(mode="w+b")
        sys.stderr.flush()
        self.saved = os.dup(2)
        os.dup2(self.f.fileno(), 2)
        return self

    def __exit__(self, *exc):
        os.dup2(self.saved, 2)
        os.close(self.saved)
        self.f.seek(0)
        self.text = self.f.read().decode(errors="replace")
        self.f.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--scale", type=int, default=24)
    ap.add_argument("--k", type=int, default=8)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--no-oracle", action="store_true")
    ap.add_argument("--weighted", action="store_true")
    args = ap.parse_args()
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if args.gpus > 1 and world == 1:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(args.gpus), "--master-addr",
               "127.0.0.1", "--master-port", os.environ.get("LUX_PORT", "29641")] + sys.argv
        return subprocess.call(cmd)
    rank, local = int(os.environ.get("RANK", "0")), int(os.environ.get("LOCAL_RANK", "0"))
    import torch
    import lux_b200 as L
    if world > 1:
        import torch.distributed as dist
        torch.cuda.set_device(local)
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    scale, seed = args.scale, 24
    nv, ne = 1 << scale, 16 << scale
    name, power = card()
    bc_app, sssp_app = (L.APP_BC_WEIGHTED, L.APP_SSSP_WEIGHTED) if args.weighted else (L.APP_BC, L.APP_SSSP)
    result = dict(bench="bc_weighted" if args.weighted else "bc", graph="RMAT-%d ef16 seed %d" % (scale, seed), nv=nv, ne=ne, gpus=world, card=name, power_limit=power,
                  k=args.k)
    exchange = L.EXCHANGE_P2P if world > 1 else L.EXCHANGE_NCCL

    def open_graph(app):
        g = L.LuxGraph.from_rmat(scale, nv, ne, seed, app=app, rank=rank, nranks=world, device=local, start=0, exchange=exchange)
        g.comm_init_torch()
        g.init()
        if world > 1:
            g.p2p_connect_torch()
        return g

    def reduce_max_sum(t, n):
        if world == 1:
            return t, n
        v = torch.tensor([t, float(n)], dtype=torch.float64, device="cuda")
        tmax = v[:1].clone()
        dist.all_reduce(tmax, op=dist.ReduceOp.MAX)
        dist.all_reduce(v[1:], op=dist.ReduceOp.SUM)
        return float(tmax), int(v[1])

    # the BFS (weighted: the weighted SSSP) alone, from vertex 0
    sssp_t = []
    for _ in range(max(args.reps, 1)):
        g = open_graph(sssp_app)
        it = g.run_to_convergence()
        sssp_t.append(reduce_max_sum(g.stats()["loop_seconds"], 0)[0])
        g.close()
    result["sssp_from_0"] = dict(iterations=it, ms_median=1e3 * float(np.median(sssp_t)), ms_min=1e3 * min(sssp_t))

    g = open_graph(bc_app)
    row_end, src, weight = g.local_csc(weighted=True) if args.weighted else (g.local_csc() + (None,))
    outdeg = np.bincount(src, minlength=nv).astype(np.int64)
    if world > 1:
        t = torch.from_numpy(outdeg).cuda()
        dist.all_reduce(t)
        outdeg = t.cpu().numpy()
    cand = np.nonzero(outdeg > 0)[0]
    cand = cand[cand != 0]
    sources = np.concatenate([[0], np.random.default_rng(args.seed).choice(cand, args.k - 1, replace=False)]).astype(np.uint32)
    result["sources"] = sources.tolist()
    os.environ["LUXB_PHASE_TIMING"] = "2"  # one line of phase means per luxb_bc_run call
    per_source = {"total": [], "sigma": [], "delta": []}
    edges = 0
    k0 = g.stats()["kernel_launches"]
    for rep in range(max(args.reps, 1)):
        e0 = g.stats()["edges_processed"]
        t0 = g.stats()["loop_seconds"]
        sig = dl = 0.0
        for s in sources:
            with StderrCapture() as cap:
                g.bc_run([s])
            m = re.search(r"bc_sigma ([0-9.]+) ms; bc_delta ([0-9.]+) ms", cap.text)
            if m:
                sig += float(m.group(1))
                dl += float(m.group(2))
        t, e = reduce_max_sum(g.stats()["loop_seconds"] - t0, g.stats()["edges_processed"] - e0)
        per_source["total"].append(1e3 * t / len(sources))
        per_source["sigma"].append(sig / len(sources))
        per_source["delta"].append(dl / len(sources))
        edges = e
    os.environ.pop("LUXB_PHASE_TIMING")
    launches = (g.stats()["kernel_launches"] - k0) / (len(sources) * max(args.reps, 1))
    bc = g.values()
    g.close()
    med = {k: float(np.median(v)) for k, v in per_source.items()}
    bound_ms = 8.0 * ne / (DATASHEET_TBPS * 1e12) * 1e3
    result["ms_per_source"] = dict(median=med["total"], min=min(per_source["total"]), sigma_median=med["sigma"], delta_median=med["delta"],
                                   bfs_and_levels_median=med["total"] - med["sigma"] - med["delta"], reps=len(per_source["total"]))
    result["edges_touched_per_run"] = edges
    result["kernel_launches_per_source"] = launches
    result["mteps"] = ne * len(sources) / (med["total"] * 1e-3 * len(sources)) / 1e6
    result["sweep_bound_ms_at_datasheet"] = bound_ms
    result["sigma_fraction_of_datasheet"] = bound_ms / med["sigma"] if med["sigma"] else None
    result["delta_fraction_of_datasheet"] = bound_ms / med["delta"] if med["delta"] else None
    if rank == 0 and not args.no_oracle:
        import bc_oracle as B
        import bc_weighted_oracle as BW
        import weighted_oracle as WO
        import oracle as O
        if world > 1:
            row_end, src = O.gen_rmat_csc(scale, nv, ne, seed)
            weight = WO.rmat_weights(seed, row_end, src) if args.weighted else None
        t0 = time.perf_counter()
        if args.weighted:
            ref = BW.run(row_end, src, weight, sources)
            result["classes_per_source"] = ref["classes"].tolist()
        else:
            ref = B.run(row_end, src, sources)
            result["levels_per_source"] = ref["levels"].tolist()
        result["oracle_cpu_s"] = time.perf_counter() - t0
        reps = max(args.reps, 1)
        want = ref["scores"] * reps  # every rep added the same K sources
        result["parity"] = bool(np.array_equal(bc == 0, want == 0) and np.allclose(bc, want, rtol=1e-10, atol=0))
        result["oracle_threads"] = O.num_threads()
        result["host_cpus"] = os.cpu_count()
    if rank == 0:
        print(json.dumps(result), flush=True)
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()
    return 0


if __name__ == "__main__":
    sys.exit(main())
